"""ArcFace IR-SE50 on the engine's kernels, and the identity similarity of the reference's IDLoss (losses/id_loss.py),
the quantity `--id_similarity` reports for each edit.

    extract_feats  IDLoss.extract_feats: crop x[:, :, 35:223, 32:220], AdaptiveAvgPool2d((112, 112)), facenet =
                   Backbone(112, 50, 'ir_se') in eval mode (models/insight_face/model_irse.py, helpers.py):
                     input_layer   conv 3x3 (3 -> 64), BN, PReLU
                     body          24 bottleneck_IR_SE blocks at 112 -> 56 -> 28 -> 14 -> 7 (stride 2 in blocks 0, 3, 7,
                                   21): res = BN0, conv 3x3, PReLU, conv 3x3 / stride, BN4, SE(reduction 16); shortcut =
                                   MaxPool2d(1, stride) when in == depth, else conv 1x1 / stride + BN; out = res + shortcut
                     output_layer  BN2d, Dropout (identity in eval), flatten NCHW, Linear(25088, 512), BN1d
                   then l2_norm (no epsilon).
    id_similarity  1 - IDLoss(src, edited) per row: the dot product of the two unit features.

Load-time folding (exact algebra, fp64 on the host): the BN after every conv (input_layer.1, res_layer.4,
shortcut_layer.1) scales the conv's output channels and becomes its bias; output_layer.0 and output_layer.4 fold into
the linear layer, whose columns are also permuted from NCHW's c*49 + h*7 + w to the NHWC activations' (h*7 + w)*512
+ c.  The pre-conv BN (res_layer.0) cannot fold into its conv, which zero-pads BN0(x), not x: BN0(x) is written as a
second output of the previous block's last kernel (of an affine kernel for block 0).

Weights: the reference's pretrained/model_ir_se50.pth, a torch.save of Backbone(112, 50, 'ir_se').state_dict()
(INTEGRATION.md lists the keys).  Every arithmetic operation is a kernel of libasyrp_b200.so (csrc/arcface.cu, the
TF32 implicit GEMM of csrc/tf32_gemm.cuh): fp32 activations, TF32 conv and linear operands.
"""
import torch

from . import _lib, ops

# (in_channel, depth, stride) of the 24 bottlenecks: models/insight_face/helpers.py get_blocks(50)
BLOCKS = tuple([(64, 64, 2)] + [(64, 64, 1)] * 2 + [(64, 128, 2)] + [(128, 128, 1)] * 3 + [(128, 256, 2)] +
               [(256, 256, 1)] * 13 + [(256, 512, 2)] + [(512, 512, 1)] * 2)
BN_EPS = 1e-5
FEATURE_DIM = 512
CROP = (35, 223, 32, 220)  # IDLoss.extract_feats: x[:, :, 35:223, 32:220]
MIN_H, MIN_W = CROP[1], CROP[3]
POOL = 112
BN_STATS = ("weight", "bias", "running_mean", "running_var")


def _bn_prefixes():
    out = ["input_layer.1", "output_layer.0", "output_layer.4"]
    for i, (cin, depth, _) in enumerate(BLOCKS):
        out += [f"body.{i}.res_layer.0", f"body.{i}.res_layer.4"]
        if cin != depth:
            out.append(f"body.{i}.shortcut_layer.1")
    return out


def state_dict_shapes():
    """name -> shape of every tensor of Backbone(112, 50, 'ir_se').state_dict() except the BNs' num_batches_tracked"""
    shapes = {"input_layer.0.weight": (64, 3, 3, 3), "input_layer.2.weight": (64,),
              "output_layer.3.weight": (FEATURE_DIM, 512 * 7 * 7), "output_layer.3.bias": (FEATURE_DIM,)}
    width = {"input_layer.1": 64, "output_layer.0": 512, "output_layer.4": FEATURE_DIM}
    for i, (cin, depth, _) in enumerate(BLOCKS):
        p = f"body.{i}."
        if cin != depth:
            shapes[p + "shortcut_layer.0.weight"] = (depth, cin, 1, 1)
            width[p + "shortcut_layer.1"] = depth
        width[p + "res_layer.0"] = cin
        shapes[p + "res_layer.1.weight"] = (depth, cin, 3, 3)
        shapes[p + "res_layer.2.weight"] = (depth,)
        shapes[p + "res_layer.3.weight"] = (depth, depth, 3, 3)
        width[p + "res_layer.4"] = depth
        shapes[p + "res_layer.5.fc1.weight"] = (depth // 16, depth, 1, 1)
        shapes[p + "res_layer.5.fc2.weight"] = (depth, depth // 16, 1, 1)
    for prefix in _bn_prefixes():
        for s in BN_STATS:
            shapes[f"{prefix}.{s}"] = (width[prefix],)
    return shapes


def load_state_dict(sd_or_path):
    """Validate a Backbone(112, 50, 'ir_se') state dict (or the path of its torch.save) and return its tensors as fp32
    on the host, keyed as in the state dict.  The BNs' num_batches_tracked entries are accepted and ignored.  Raises
    ValueError on a missing, mis-shaped or unknown key, and on a file that is not a state dict."""
    sd = sd_or_path
    if not isinstance(sd, dict):
        try:
            sd = torch.load(sd_or_path, map_location="cpu", weights_only=True)
        except Exception as e:  # a truncated file, another format, ...
            raise ValueError(f"ArcFace weights {sd_or_path!r}: cannot be read as a torch.save'd state dict ({e})") \
                from None
        if not isinstance(sd, dict):
            raise ValueError(f"ArcFace weights {sd_or_path!r}: not a state dict (got {type(sd).__name__})")
    expected = state_dict_shapes()
    tracked = {f"{p}.num_batches_tracked" for p in _bn_prefixes()}
    unknown = sorted(k for k in sd if k not in expected and k not in tracked)
    if unknown:
        raise ValueError(f"ArcFace state dict: unexpected keys {unknown[:8]}{' ...' if len(unknown) > 8 else ''} "
                         "(expected the layout of Backbone(112, 50, 'ir_se'))")
    out = {}
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f"ArcFace state dict: missing key {k!r}")
        t = torch.as_tensor(sd[k])
        if tuple(t.shape) != shape:
            raise ValueError(f"ArcFace state dict: {k!r} has shape {tuple(t.shape)}, expected {shape}")
        out[k] = t.detach().float().cpu().contiguous()
    return out


def _bn(sd, prefix):
    """(scale, shift) of an eval-mode BatchNorm, fp64: y = x * scale + shift"""
    g = {s: sd[f"{prefix}.{s}"].double() for s in BN_STATS}
    scale = g["weight"] / torch.sqrt(g["running_var"] + BN_EPS)
    return scale, g["bias"] - g["running_mean"] * scale


def fold(sd):
    """the folded parameters of a load_state_dict() result, fp32 on the host: 'input' (weight [64][3][3][3], bias,
    prelu), per block 'body.i' {bn0 (scale, shift), w1, prelu, w2, b2, fc1 [C/16][C], fc2 [C][C/16], sc_w / sc_b or
    None}, and 'head' (weight [512][25088] in NHWC column order, bias [512])"""
    f = lambda t: t.float().contiguous()  # noqa: E731
    out = {}
    s, t = _bn(sd, "input_layer.1")
    out["input"] = dict(weight=f(sd["input_layer.0.weight"].double() * s[:, None, None, None]), bias=f(t),
                        prelu=f(sd["input_layer.2.weight"]))
    for i, (cin, depth, _) in enumerate(BLOCKS):
        p = f"body.{i}."
        s0, t0 = _bn(sd, p + "res_layer.0")
        s4, t4 = _bn(sd, p + "res_layer.4")
        blk = dict(bn0=(f(s0), f(t0)), w1=sd[p + "res_layer.1.weight"], prelu=sd[p + "res_layer.2.weight"],
                   w2=f(sd[p + "res_layer.3.weight"].double() * s4[:, None, None, None]), b2=f(t4),
                   fc1=f(sd[p + "res_layer.5.fc1.weight"].reshape(depth // 16, depth)),
                   fc2=f(sd[p + "res_layer.5.fc2.weight"].reshape(depth, depth // 16)), sc_w=None, sc_b=None)
        if cin != depth:
            ss, ts = _bn(sd, p + "shortcut_layer.1")
            blk["sc_w"] = f(sd[p + "shortcut_layer.0.weight"].double() * ss[:, None, None, None])
            blk["sc_b"] = f(ts)
        out[f"body.{i}"] = blk
    a, b = _bn(sd, "output_layer.0")                                        # BN2d over the 512 channels
    w = sd["output_layer.3.weight"].double().reshape(FEATURE_DIM, 512, 49)  # [out][c][h*7 + w]
    bias = sd["output_layer.3.bias"].double() + (w * b[None, :, None]).sum((1, 2))
    w = w * a[None, :, None]
    k, m = _bn(sd, "output_layer.4")                                        # BN1d over the 512 features
    w, bias = w * k[:, None, None], bias * k + m
    out["head"] = dict(weight=f(w.permute(0, 2, 1).reshape(FEATURE_DIM, 49 * 512)), bias=f(bias))
    return out


def check_image_size(H, W):
    if H < MIN_H or W < MIN_W:
        raise ValueError(f"ArcFace's crop x[:, :, 35:223, 32:220] needs images of at least {MIN_H} x {MIN_W} "
                         f"(H x W), got {H} x {W}")


class ArcFace:
    """ArcFace(weights).extract_feats(x) -> fp32 [B][512] unit vectors on the device, for x [B][3][H][W] (any scale,
    H >= 223, W >= 220).  Every operation is a kernel of libasyrp_b200.so; an image's features are bit-identical
    whatever batch it is in."""

    def __init__(self, state_dict_or_path, device=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("ArcFace needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        folded = fold(load_state_dict(state_dict_or_path))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        dev = self.device
        with torch.cuda.device(dev):
            fi = folded["input"]
            self.input = (ops.pack_lpips_conv_weight(fi["weight"], cin_pad=4).to(dev), fi["bias"].to(dev),
                          fi["prelu"].to(dev))
            self.blocks = []
            for i in range(len(BLOCKS)):
                b = folded[f"body.{i}"]
                self.blocks.append(dict(
                    bn0=tuple(t.to(dev) for t in b["bn0"]), w1=ops.pack_lpips_conv_weight(b["w1"]).to(dev),
                    prelu=b["prelu"].to(dev), w2=ops.pack_lpips_conv_weight(b["w2"]).to(dev), b2=b["b2"].to(dev),
                    fc1=b["fc1"].to(dev), fc2=b["fc2"].to(dev),
                    sc_w=None if b["sc_w"] is None else ops.pack_lpips_conv_weight(b["sc_w"]).to(dev),
                    sc_b=None if b["sc_b"] is None else b["sc_b"].to(dev)))
            self.head = (folded["head"]["weight"].to(dev), folded["head"]["bias"].to(dev))

    @torch.no_grad()
    def extract_feats(self, x):
        """x [B][3][H][W] -> fp32 [B][512] unit features on the device (IDLoss.extract_feats)"""
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] == 0:
            raise ValueError(f"images must be [B][3][H][W], got {tuple(x.shape)}")
        check_image_size(x.shape[2], x.shape[3])
        B = x.shape[0]
        f32 = dict(dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            x = x.to(**f32).contiguous()
            x112 = torch.empty(B, POOL, POOL, 4, **f32)
            ops.arcface_preprocess(x, x112)
            w, bias, prelu = self.input
            h = torch.empty(B, POOL, POOL, 64, **f32)
            ops.arcface_conv(x112, w, bias, h, 3, 1, 1, prelu=prelu)
            hb = torch.empty_like(h)
            ops.arcface_affine(h, *self.blocks[0]["bn0"], hb)
            for i, (cin, depth, stride) in enumerate(BLOCKS):
                blk = self.blocks[i]
                H, W = h.shape[1:3]
                t = torch.empty(B, H, W, depth, **f32)
                ops.arcface_conv(hb, blk["w1"], None, t, 3, 1, 1, prelu=blk["prelu"])
                Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
                r = torch.empty(B, Ho, Wo, depth, **f32)
                ops.arcface_conv(t, blk["w2"], blk["b2"], r, 3, stride, 1)
                if blk["sc_w"] is not None:
                    sc, sc_stride = torch.empty(B, Ho, Wo, depth, **f32), 1
                    ops.arcface_conv(h, blk["sc_w"], blk["sc_b"], sc, 1, stride, 0)
                else:
                    sc, sc_stride = h, stride
                gate = torch.empty(B, depth, **f32)
                ops.arcface_se_scale(r, blk["fc1"], blk["fc2"], gate)
                out = torch.empty_like(r)
                nxt = self.blocks[i + 1]["bn0"] if i + 1 < len(BLOCKS) else None
                out2 = torch.empty_like(r) if nxt is not None else None
                ops.arcface_se_apply(r, gate, sc, out, sc_stride, bn=nxt, out2=out2)
                h, hb = out, out2
            raw = torch.empty(B, FEATURE_DIM, **f32)
            ops.clip_linear(h.reshape(B, -1), self.head[0], self.head[1], raw)
            feats = torch.empty_like(raw)
            ops.arcface_l2norm(raw, feats)
        return feats

    @torch.no_grad()
    def id_similarity(self, src, edited):
        """1 - IDLoss(src, edited) per row: fp32 [len(edited)] on the host.  edited may hold k * B rows for B source
        images: row j is paired with source row j % B, so a batch edited at several strengths encodes its sources
        once."""
        src, edited = torch.as_tensor(src), torch.as_tensor(edited)
        B, N = src.shape[0], edited.shape[0]
        if B == 0 or N % B:
            raise ValueError(f"edited images ({N}) must be a whole multiple of the source images ({B})")
        feats = self.extract_feats(torch.cat([src.to(self.device), edited.to(self.device)]))
        out = torch.empty(N, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ops.arcface_dot(feats[:B], feats[B:], out)
        return out.cpu()
