"""CPU emulation of the ENGINE'S numerics on the DDPM family — TEST / ANALYSIS INFRASTRUCTURE ONLY.

The same network as oracle/ddpm.py (which restates models/ddpm/diffusion.py), evaluated in fp32 on the CPU but with
the roundings the CUDA engine performs, each behind a switch, so that the engine-vs-reference error of a trajectory
can be attributed to its sources without GPU time (scripts/attribute_error.py):

  w16      conv weights rounded to fp16                         (asyrp_official_b200/ops.py pack_conv_weight)
  in16     conv operands act(GN(x)) rounded to fp16             (in-kernel transform, csrc/conv_gemm.cu transform_fast)
  store16  conv outputs stored as fp16 NHWC                     (conv epilogue)
  stats32  GroupNorm statistics taken from the pre-rounding fp32 values of the producer's accumulator while the
           consumer normalises the fp16-rounded tensor          (epilogue partial sums)
  p16      attention probabilities rounded to fp16              (csrc/attention.cu softmax_rows)
  x16      UNet input x_t rounded to fp16                       (pack_input)
  tanh11   SiLU of the fused operands as h + h*tanh(h), h = x/2, with an 11-bit tanh (tanh.approx.f32: max relative error
           2^-11; csrc/ptx.cuh silu_tanh_half), modelled as a uniform relative perturbation.  The engine's default since
           round 2; not part of ALL so that the earlier attribution tables stay reproducible (pass {**ALL, "tanh11": True})

All switches on = the engine (up to summation order); all off = oracle/ddpm.py.
"""
import torch
import torch.nn.functional as F

from . import ddpm as od

ALL = dict(w16=True, in16=True, store16=True, stats32=True, p16=True, x16=True)
_G = torch.Generator().manual_seed(99)


def _act(x, fl):
    """SiLU of a conv operand (GroupNorm output) as the transform computes it"""
    if not fl.get("tanh11"):
        return od.swish(x)
    h = 0.5 * x
    t = torch.tanh(h) * (1.0 + (torch.rand(x.shape, generator=_G) * 2 - 1) * 2.0 ** -11)
    return h + h * t

NONE = {k: False for k in ALL}


def r16(x):
    return x.to(torch.float16).to(torch.float32)


class T:
    """activation as the engine holds it: `v` the stored value, `pre` the fp32 accumulator value it was rounded from"""
    __slots__ = ("v", "pre")

    def __init__(self, pre, fl):
        self.pre = pre
        self.v = r16(pre) if fl["store16"] else pre


def _gn(sd, p, ts, fl, eps=1e-6):
    """GroupNorm(32) over the channel concat of `ts` -> normalised tensor (affine applied), fp32"""
    v = torch.cat([t.v for t in ts], 1)
    s = torch.cat([t.pre for t in ts], 1) if fl["stats32"] else v
    n, c = v.shape[:2]
    g = s.reshape(n, 32, -1).double()
    mean = g.mean(-1)
    var = (g * g).mean(-1) - mean * mean
    rstd = (var + eps).rsqrt()
    a = rstd.repeat_interleave(c // 32, 1).float() * sd[p + ".weight"][None]
    b = sd[p + ".bias"][None] - mean.repeat_interleave(c // 32, 1).float() * a
    return v * a[:, :, None, None] + b[:, :, None, None]


def _conv(sd, p, x, fl, **kw):
    w = sd[p + ".weight"]
    return F.conv2d(r16(x) if fl["in16"] else x, r16(w) if fl["w16"] else w, sd[p + ".bias"], **kw)


def _res(sd, p, ts, temb, fl):
    x = torch.cat([t.v for t in ts], 1)
    h = _conv(sd, p + ".conv1", _act(_gn(sd, p + ".norm1", ts, fl), fl), fl, padding=1)
    h = T(h + F.linear(od.swish(temb), sd[p + ".temb_proj.weight"], sd[p + ".temb_proj.bias"])[:, :, None, None], fl)
    o = _conv(sd, p + ".conv2", _act(_gn(sd, p + ".norm2", [h], fl), fl), fl, padding=1)
    if (p + ".nin_shortcut.weight") in sd:
        x = _conv(sd, p + ".nin_shortcut", x, fl)
    return T(x + o, fl)


def _attn(sd, p, t, fl):
    hn = _gn(sd, p + ".norm", [t], fl)
    q, k, v = (T(_conv(sd, p + "." + n, hn, fl), fl).v for n in ("q", "k", "v"))
    b, c, hh, ww = q.shape
    s = torch.bmm(q.reshape(b, c, -1).permute(0, 2, 1), k.reshape(b, c, -1)) * (int(c) ** (-0.5))
    w_ = torch.softmax(s, dim=2)
    if fl["p16"]:
        w_ = r16(w_)
    o = T(torch.bmm(v.reshape(b, c, -1), w_.permute(0, 2, 1)).reshape(b, c, hh, ww), fl)
    return T(t.v + _conv(sd, p + ".proj_out", o.v, fl), fl)


def _decoder(sd, cfg, h, hs, temb, fl):
    nres = len(cfg["ch_mult"])
    idx = -1
    for lvl in reversed(range(nres)):
        for blk in range(cfg["num_res_blocks"] + 1):
            h = _res(sd, f"up.{lvl}.block.{blk}", [h, hs[idx]], temb, fl)
            idx -= 1
            if f"up.{lvl}.attn.{blk}.norm.weight" in sd:
                h = _attn(sd, f"up.{lvl}.attn.{blk}", h, fl)
        if lvl != 0:
            h = T(_conv(sd, f"up.{lvl}.upsample.conv", F.interpolate(h.v, scale_factor=2.0, mode="nearest"), fl,
                        padding=1), fl)
    return _conv(sd, "conv_out", _act(_gn(sd, "norm_out", [h], fl), fl), fl, padding=1)  # fp32 output


@torch.no_grad()
def ddpm_forward(sd, cfg, x, t, index=None, t_edit=400, hs_coeff=(1.0, 1.0), flags=ALL, **_):
    fl = flags
    temb = od.temb_mlp(sd, t, cfg["ch"])
    nres = len(cfg["ch_mult"])
    hs = [T(_conv(sd, "conv_in", r16(x) if fl["x16"] else x, fl, padding=1), fl)]
    for lvl in range(nres):
        for blk in range(cfg["num_res_blocks"]):
            h = _res(sd, f"down.{lvl}.block.{blk}", [hs[-1]], temb, fl)
            if f"down.{lvl}.attn.{blk}.norm.weight" in sd:
                h = _attn(sd, f"down.{lvl}.attn.{blk}", h, fl)
            hs.append(h)
        if lvl != nres - 1:
            hs.append(T(_conv(sd, f"down.{lvl}.downsample.conv", F.pad(hs[-1].v, (0, 1, 0, 1)), fl, stride=2), fl))
    h = _res(sd, "mid.block_1", [hs[-1]], temb, fl)
    h = _attn(sd, "mid.attn_1", h, fl)
    h = _res(sd, "mid.block_2", [h], temb, fl)
    et_mod, dh = None, None
    if index is not None:
        if t[0] >= t_edit:
            acc = None
            for i in range(index + 1):
                p = f"layer_{i}"
                d1 = T(_conv(sd, p + ".conv1", h.v, fl) + F.linear(od.swish(temb), sd[p + ".temb_proj.weight"],
                                                                   sd[p + ".temb_proj.bias"])[:, :, None, None], fl)
                dh = _conv(sd, p + ".conv2", _act(_gn(sd, p + ".norm2", [d1], fl), fl), fl)
                base = h.v * hs_coeff[0] if acc is None else acc.v
                acc = T(base + dh * hs_coeff[i + 1], fl)
            et_mod = _decoder(sd, cfg, acc, hs, temb, fl)
    et = _decoder(sd, cfg, h, hs, temb, fl)
    if index is not None and et_mod is None:
        et_mod = et
    return et, et_mod, dh, h.v
