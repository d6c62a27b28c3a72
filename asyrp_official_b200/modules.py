"""Drop-in nn.Module mirrors of the reference's UNet classes, backed by the CUDA engine.

Same constructors, state-dict keys, `setattr_layers`, `layer_i` attributes and forward signature / return tuple as
  models/ddpm/diffusion.py          DDPM            (:327-580)
  models/improved_ddpm/unet.py      UNetModel       (:438-773)   + script_util.i_DDPM (:102-109)
  models/guided_diffusion/unet.py   UNetModel       (:437-776)   + script_util.guided_Diffusion (:173-178)

The modules hold parameters only (so `load_state_dict`, `.to(device)`, `state_dict()` and the Δh checkpoint format
work unchanged); `forward` runs the hand-written sm_90a kernels through UNetEngine — there is no PyTorch compute
path, and calling forward without a CUDA device raises.
"""
import math
import weakref

import torch
import torch.nn as nn

from . import arch as A
from .engine import UNetEngine
from ._lib import AsyrpError


class _Node(nn.Module):
    """anonymous container so that parameter paths equal the reference's dotted names"""


def _register(root, name, tensor):
    parts = name.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Node())
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


def _default_init(name, shape, shapes, zero=False):
    """torch's default Conv/Linear/GroupNorm initialisation (kaiming_uniform(a=sqrt(5)) => U(+-1/sqrt(fan_in)))"""
    base = name.rsplit(".", 1)[0]
    wshape = shapes.get(base + ".weight")
    if zero:
        return torch.zeros(shape)
    if wshape is not None and len(wshape) >= 2:
        bound = 1.0 / math.sqrt(math.prod(wshape[1:]))
        return (torch.rand(shape) * 2 - 1) * bound
    return torch.ones(shape) if name.endswith(".weight") else torch.zeros(shape)


class _EngineUNet(nn.Module):
    """shared machinery: parameter tree, weight versioning, engine dispatch"""

    def __init__(self, arch: A.Arch):
        super().__init__()
        object.__setattr__(self, "arch", arch)
        self._n_delta = 0
        self._version = 0
        self._engine = None
        self._engine_version = -1
        shapes = A.param_shapes(arch, 0)
        for name, shp in shapes.items():
            _register(self, name, _default_init(name, shp, shapes, zero=self._zero_init(name)))
        self._hook_tree(self)

    def _zero_init(self, name):
        return False

    def _hook_tree(self, mod):
        ref = weakref.ref(self)

        def bump(module, incompatible_keys):
            s = ref()
            if s is not None:
                s._version += 1

        for m in mod.modules():
            m.register_load_state_dict_post_hook(bump)

    # reference API ------------------------------------------------------------------------------
    def setattr_layers(self, nums):
        """create layer_0 .. layer_{nums-1} DeltaBlocks (ddpm/diffusion.py:433-444, improved_ddpm/unet.py:756-773)"""
        dev = next(self.parameters()).device
        shapes = A.delta_block_shapes(self.arch, nums)
        for i in range(nums):
            node = _Node()
            pref = f"layer_{i}."
            for name, shp in shapes.items():
                if name.startswith(pref):
                    _register(node, name[len(pref):], _default_init(name, shp, shapes).to(dev))
            setattr(self, f"layer_{i}", node)
            self._hook_tree(node)
        self._n_delta = nums
        self._version += 1

    def refresh_weights(self):
        """re-pack device weights after parameters were modified in place"""
        self._version += 1

    @property
    def engine(self) -> UNetEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise AsyrpError("asyrp_official_b200 models run on a CUDA device only: call model.to('cuda') "
                             "(there is no CPU / PyTorch fallback path)")
        if self._engine is None or self._engine_version != self._version or self._engine.device != dev:
            self._engine = UNetEngine(self.arch, self.state_dict(), dev, n_delta=self._n_delta)
            self._engine_version = self._version
        return self._engine

    def _forward(self, x, t, index, t_edit, hs_coeff, delta_h, ignore_timestep, use_mask):
        eng = self.engine
        if not isinstance(hs_coeff, (tuple, list)):
            hs_coeff = (hs_coeff,)
        return eng.forward(x.to(eng.device), t.to(eng.device), index=index, t_edit=t_edit, hs_coeff=hs_coeff,
                           ignore_timestep=ignore_timestep, delta_h=delta_h, use_mask=use_mask)


class DDPM(_EngineUNet):
    """DDPM(config): config.model.{ch,out_ch,ch_mult,num_res_blocks,attn_resolutions,dropout,in_channels,
    resamp_with_conv}, config.data.image_size  (models/ddpm/diffusion.py:327-337)"""

    def __init__(self, config):
        m = config.model
        if not getattr(m, "resamp_with_conv", True):
            raise NotImplementedError("resamp_with_conv=False is not used by any config of the reference")
        super().__init__(A.ddpm_arch(ch=m.ch, out_ch=m.out_ch, ch_mult=tuple(m.ch_mult),
                                     num_res_blocks=m.num_res_blocks, attn_resolutions=tuple(m.attn_resolutions),
                                     in_channels=m.in_channels, image_size=config.data.image_size))
        self.config = config
        self.ch, self.temb_ch = m.ch, m.ch * 4
        self.num_resolutions, self.num_res_blocks = len(m.ch_mult), m.num_res_blocks
        self.resolution, self.in_channels = config.data.image_size, m.in_channels

    def forward(self, x, t, index=None, t_edit=400, hs_coeff=(1.0, 1.0), delta_h=None, ignore_timestep=False,
                use_mask=False):
        assert x.shape[2] == x.shape[3] == self.resolution
        return self._forward(x, t, index, t_edit, hs_coeff, delta_h, ignore_timestep, use_mask)


class UNetModel(_EngineUNet):
    """ADM / iDDPM UNet with the hyper-parameter surface the reference uses (resblock_updown, scale-shift norm,
    64-channel heads)."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None,
                 use_checkpoint=False, use_fp16=False, num_heads=1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, resblock_updown=False, use_new_attention_order=False):
        if not (use_scale_shift_norm and resblock_updown and num_head_channels == 64 and dims == 2
                and not use_new_attention_order and not use_fp16):
            raise NotImplementedError("only the configuration instantiated by the reference's script_util dicts "
                                      "(resblock_updown, use_scale_shift_norm, num_head_channels=64) is built")
        # attention_resolutions here are downsample rates, as UNetModel receives them (script_util.py:76-78)
        res = tuple(image_size // int(ds) for ds in attention_resolutions)
        super().__init__(A.adm_arch(image_size=image_size, model_channels=model_channels,
                                    num_res_blocks=num_res_blocks, attention_resolutions=res,
                                    channel_mult=tuple(channel_mult), num_head_channels=num_head_channels,
                                    out_channels=out_channels, in_channels=in_channels))
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks, self.channel_mult = out_channels, num_res_blocks, tuple(channel_mult)
        self.num_classes = num_classes
        self.dtype = torch.float32

    def _zero_init(self, name):
        # zero_module(): ResBlock out conv, attention proj_out, final conv (improved_ddpm/unet.py:252-254,336,657)
        return (".out_layers.3." in name or ".proj_out." in name or name.startswith("out.2."))

    def forward(self, x, timesteps, y=None, index=None, t_edit=400, hs_coeff=(1.0, 1.0), delta_h=None,
                ignore_timestep=False, use_mask=False):
        return self._forward(x, timesteps, index, t_edit, hs_coeff, delta_h, ignore_timestep, use_mask)


def _create_adm(hp):
    ds = tuple(hp["image_size"] // r for r in hp["attention_resolutions"])
    return UNetModel(image_size=hp["image_size"], in_channels=3, model_channels=hp["model_channels"],
                     out_channels=hp["out_channels"], num_res_blocks=hp["num_res_blocks"], attention_resolutions=ds,
                     channel_mult=hp["channel_mult"], num_head_channels=hp["num_head_channels"],
                     use_scale_shift_norm=True, resblock_updown=True)


def i_DDPM(dataset_name='AFHQ'):
    """models/improved_ddpm/script_util.py:102-109"""
    if dataset_name in ['AFHQ', 'FFHQ']:
        return _create_adm(A.AFHQ_HP)
    if dataset_name == 'IMAGENET':
        return _create_adm(A.IMAGENET_HP)
    raise ValueError(f"i_DDPM: dataset {dataset_name!r} not implemented")


def guided_Diffusion(dataset_name='MetFACE'):
    """models/guided_diffusion/script_util.py:173-178"""
    if dataset_name in ['MetFACE']:
        return _create_adm(A.METFACE_HP)
    if dataset_name in ['CelebA_HQ_P2']:
        return _create_adm(A.CELEBA_HQ_P2_HP)
    raise ValueError(f"guided_Diffusion: dataset {dataset_name!r} not implemented")
