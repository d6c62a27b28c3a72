"""Face-parsing BiSeNet on the engine's kernels, and the segmentation consistency (SC) that `--seg_consistency` reports
for each edit.

The reference has no segmentation network and no SC code: the network and the metric here are this project's
definition.  The network is the public face-parsing BiSeNet(n_classes=19) in eval mode, whose usual checkpoint is
79999_iter.pth (a torch.save of its state dict); only the main head is evaluated.

    input      clamp the [-1, 1] image (the image its PNG shows), map to [0, 1], bilinear resize to 512 x 512
               (align_corners=False), normalise with ImageNet's mean and std
    cp.resnet  ResNet-18: conv1 7x7 / 2 pad 3, bn1, ReLU, max-pool 3x3 / 2 pad 1, layer1..4 of two BasicBlocks (64,
               128, 256, 512 channels, strides 1, 2, 2, 2; layer{2,3,4}.0 have a 1x1 downsample + BN) -> feat8 (64^2 x
               128), feat16 (32^2 x 256), feat32 (16^2 x 512)
    cp         avg = conv_avg(mean_hw(feat32)); s32 = arm32(feat32) + avg; up32 = conv_head32(nearest2x(s32));
               s16 = arm16(feat16) + up32; up16 = conv_head16(nearest2x(s16)); ARM(x) = f * sigmoid(bn_atten(
               conv_atten(mean_hw(f)))), f = ConvBNReLU3x3(x)
    ffm        f = convblk(cat[feat8, up16]); out = f * sigmoid(conv2(relu(conv1(mean_hw(f))))) + f
    conv_out   ConvBNReLU3x3, 1x1 to n_classes -> logits at 64^2; bilinear align_corners=True to 512^2; argmax (the
               first class wins a tie)
    SC         edited row j against source row j % B: the fraction of the 512^2 pixels whose labels are equal

ConvBNReLU(k) is conv (no bias) -> BN (eps 1e-5) -> ReLU.  Load-time folding (exact algebra, fp64 on the host): every
BN that follows a conv scales the conv's output channels and becomes its bias; bn_atten folds into conv_atten.  The
1x1 convblk over cat[feat8, up16] runs as two GEMMs over the two inputs, the second adding the first before the ReLU,
so the concatenation is never materialised; the head's Cout is zero-padded to the GEMM's 64.  Every arithmetic
operation is a kernel of libasyrp_b200.so (csrc/face_parsing.cu, the TF32 implicit GEMM of csrc/tf32_gemm.cuh): fp32
activations, TF32 conv operands.  No real 79999_iter.pth has been loaded by this project's tests: the key list below
follows the public model definition, and the loader refuses any other layout by name.
"""
import torch

from . import _lib, ops

BN_EPS = 1e-5
SIZE = 512                 # input and label-map size
LOGIT_SIZE = SIZE // 8     # the head's resolution
LOGIT_LD = 64              # the head's Cout padded to the GEMM's multiple: n_classes <= 64
LAYERS = ((64, 1), (128, 2), (256, 2), (512, 2))  # (channels, stride of block 0) of layer1..4
BN_STATS = ("weight", "bias", "running_mean", "running_var")
AUX_HEADS = ("conv_out16", "conv_out32")  # BiSeNetOutput(128, 64, n_classes): training-only heads, ignored
# fp32 bytes of the activations live at once per image at the peak (the stem: packed input, conv1's output and the
# max-pool's): rows are scored in chunks of ACTIVATION_BUDGET // ROW_BYTES images
ROW_BYTES = 4 * (SIZE * SIZE * 4 + (SIZE // 2) ** 2 * 64 + (SIZE // 4) ** 2 * 64)
ACTIVATION_BUDGET = 1 << 30


def _conv_bn(shapes, prefix, cout, cin, k):
    shapes[f"{prefix}.conv.weight"] = (cout, cin, k, k)
    for s in BN_STATS:
        shapes[f"{prefix}.bn.{s}"] = (cout,)


def _bn_prefixes(shapes):
    return sorted({k.rsplit(".", 1)[0] for k in shapes if k.endswith(".running_var")})


def state_dict_shapes(n_classes=19):
    """name -> shape of every tensor BiSeNet(n_classes) evaluates, without num_batches_tracked and the two auxiliary
    heads (aux_head_shapes)"""
    shapes = {"cp.resnet.conv1.weight": (64, 3, 7, 7)}
    for s in BN_STATS:
        shapes[f"cp.resnet.bn1.{s}"] = (64,)
    cin = 64
    for li, (c, stride) in enumerate(LAYERS):
        for b in range(2):
            p = f"cp.resnet.layer{li + 1}.{b}"
            bin_ = cin if b == 0 else c
            shapes[f"{p}.conv1.weight"] = (c, bin_, 3, 3)
            shapes[f"{p}.conv2.weight"] = (c, c, 3, 3)
            for s in BN_STATS:
                shapes[f"{p}.bn1.{s}"] = (c,)
                shapes[f"{p}.bn2.{s}"] = (c,)
            if b == 0 and (stride != 1 or bin_ != c):
                shapes[f"{p}.downsample.0.weight"] = (c, bin_, 1, 1)
                for s in BN_STATS:
                    shapes[f"{p}.downsample.1.{s}"] = (c,)
        cin = c
    for name, c in (("arm16", 256), ("arm32", 512)):
        _conv_bn(shapes, f"cp.{name}.conv", 128, c, 3)
        shapes[f"cp.{name}.conv_atten.weight"] = (128, 128, 1, 1)
        for s in BN_STATS:
            shapes[f"cp.{name}.bn_atten.{s}"] = (128,)
    _conv_bn(shapes, "cp.conv_head32", 128, 128, 3)
    _conv_bn(shapes, "cp.conv_head16", 128, 128, 3)
    _conv_bn(shapes, "cp.conv_avg", 128, 512, 1)
    _conv_bn(shapes, "ffm.convblk", 256, 256, 1)
    shapes["ffm.conv1.weight"] = (64, 256, 1, 1)
    shapes["ffm.conv2.weight"] = (256, 64, 1, 1)
    _conv_bn(shapes, "conv_out.conv", 256, 256, 3)
    shapes["conv_out.conv_out.weight"] = (n_classes, 256, 1, 1)
    return shapes


def aux_head_shapes(n_classes=19):
    """the auxiliary heads conv_out16 / conv_out32 (BiSeNetOutput(128, 64, n_classes)), accepted and ignored"""
    shapes = {}
    for h in AUX_HEADS:
        _conv_bn(shapes, f"{h}.conv", 64, 128, 3)
        shapes[f"{h}.conv_out.weight"] = (n_classes, 64, 1, 1)
    return shapes


def load_state_dict(sd_or_path):
    """Validate a BiSeNet state dict (or the path of its torch.save) and return the tensors the main head evaluates as
    fp32 on the host, keyed as in the state dict.  n_classes (1 .. 64) is read from conv_out.conv_out.weight.  The
    auxiliary heads and every BN's num_batches_tracked are accepted, checked and ignored.  Raises ValueError naming the
    key on a missing, mis-shaped or unknown key, and on a file that is not a state dict."""
    sd = sd_or_path
    if not isinstance(sd, dict):
        try:
            sd = torch.load(sd_or_path, map_location="cpu", weights_only=True)
        except Exception as e:  # a truncated file, another format, ...
            raise ValueError(f"face-parsing weights {sd_or_path!r}: cannot be read as a torch.save'd state dict "
                             f"({e})") from None
        if not isinstance(sd, dict):
            raise ValueError(f"face-parsing weights {sd_or_path!r}: not a state dict (got {type(sd).__name__})")
    head = "conv_out.conv_out.weight"
    if head not in sd:
        raise ValueError(f"face-parsing state dict: missing key {head!r}")
    n_classes = int(torch.as_tensor(sd[head]).shape[0]) if torch.as_tensor(sd[head]).dim() == 4 else 0
    if not 1 <= n_classes <= LOGIT_LD:
        raise ValueError(f"face-parsing state dict: {head!r} has shape {tuple(torch.as_tensor(sd[head]).shape)}, "
                         f"expected (n_classes, 256, 1, 1) with 1 <= n_classes <= {LOGIT_LD}")
    expected = state_dict_shapes(n_classes)
    aux = aux_head_shapes(n_classes)
    tracked = {f"{p}.num_batches_tracked" for p in _bn_prefixes({**expected, **aux})}
    unknown = sorted(k for k in sd if k not in expected and k not in aux and k not in tracked)
    if unknown:
        raise ValueError(f"face-parsing state dict: unexpected keys {unknown[:8]}{' ...' if len(unknown) > 8 else ''} "
                         f"(expected the layout of BiSeNet(n_classes={n_classes}))")
    for k, shape in aux.items():
        if k in sd and tuple(torch.as_tensor(sd[k]).shape) != shape:
            raise ValueError(f"face-parsing state dict: {k!r} has shape {tuple(torch.as_tensor(sd[k]).shape)}, "
                             f"expected {shape}")
    out = {}
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f"face-parsing state dict: missing key {k!r}")
        t = torch.as_tensor(sd[k])
        if tuple(t.shape) != shape:
            raise ValueError(f"face-parsing state dict: {k!r} has shape {tuple(t.shape)}, expected {shape}")
        out[k] = t.detach().float().cpu().contiguous()
    return out


def _bn(sd, prefix):
    """(scale, shift) of an eval-mode BatchNorm, fp64: y = x * scale + shift"""
    g = {s: sd[f"{prefix}.{s}"].double() for s in BN_STATS}
    scale = g["weight"] / torch.sqrt(g["running_var"] + BN_EPS)
    return scale, g["bias"] - g["running_mean"] * scale


def _fold_conv(sd, wkey, bnp):
    """(weight, bias) of a conv followed by a BatchNorm, fp32 (folded in fp64)"""
    s, t = _bn(sd, bnp)
    return (sd[wkey].double() * s[:, None, None, None]).float().contiguous(), t.float().contiguous()


def fold(sd):
    """the folded parameters of a load_state_dict() result, fp32 on the host, torch Conv2d layouts:
    'stem' (w, b); 'layer{l}.{b}' {conv1, conv2, downsample (or None)} as (w, b); 'arm16' / 'arm32' {conv (w, b),
    atten (w [128][128], b)}; 'conv_head32', 'conv_head16', 'conv_out' (w, b); 'conv_avg' (w [128][512], b);
    'ffm' {convblk_a (w over feat8's 128 channels, b), convblk_b (w over up16's), conv1 [64][256], conv2 [256][64]};
    'classes' (w [n_classes][256][1][1])"""
    out = {"stem": _fold_conv(sd, "cp.resnet.conv1.weight", "cp.resnet.bn1")}
    for li, (c, _) in enumerate(LAYERS):
        for b in range(2):
            p = f"cp.resnet.layer{li + 1}.{b}"
            out[f"layer{li + 1}.{b}"] = dict(
                conv1=_fold_conv(sd, f"{p}.conv1.weight", f"{p}.bn1"),
                conv2=_fold_conv(sd, f"{p}.conv2.weight", f"{p}.bn2"),
                downsample=(_fold_conv(sd, f"{p}.downsample.0.weight", f"{p}.downsample.1")
                            if f"{p}.downsample.0.weight" in sd else None))
    for name in ("arm16", "arm32"):
        w, b = _fold_conv(sd, f"cp.{name}.conv_atten.weight", f"cp.{name}.bn_atten")
        out[name] = dict(conv=_fold_conv(sd, f"cp.{name}.conv.conv.weight", f"cp.{name}.conv.bn"),
                         atten=(w.reshape(128, 128).contiguous(), b))
    for name in ("conv_head32", "conv_head16"):
        out[name] = _fold_conv(sd, f"cp.{name}.conv.weight", f"cp.{name}.bn")
    w, b = _fold_conv(sd, "cp.conv_avg.conv.weight", "cp.conv_avg.bn")
    out["conv_avg"] = (w.reshape(128, 512).contiguous(), b)
    w, b = _fold_conv(sd, "ffm.convblk.conv.weight", "ffm.convblk.bn")
    out["ffm"] = dict(convblk_a=(w[:, :128].contiguous(), b), convblk_b=(w[:, 128:].contiguous(), None),
                      conv1=sd["ffm.conv1.weight"].reshape(64, 256).contiguous(),
                      conv2=sd["ffm.conv2.weight"].reshape(256, 64).contiguous())
    out["conv_out"] = _fold_conv(sd, "conv_out.conv.conv.weight", "conv_out.conv.bn")
    out["classes"] = sd["conv_out.conv_out.weight"].contiguous()
    return out


class FaceParser:
    """FaceParser(weights, device): logits(x), labels(x) and seg_consistency(src, edited) of images x [B][3][H][W] in
    [-1, 1] (any size; resized to 512 x 512).  Every operation is a kernel of libasyrp_b200.so; an image's logits and
    labels are bit-identical whatever batch it is in.  Rows run in chunks of max_rows images (default: ACTIVATION_BUDGET
    // ROW_BYTES), which bounds the activations at max_rows * ROW_BYTES bytes."""

    def __init__(self, state_dict_or_path, device=None, max_rows=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("FaceParser needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        sd = load_state_dict(state_dict_or_path)
        self.n_classes = sd["conv_out.conv_out.weight"].shape[0]
        folded = fold(sd)
        self.max_rows = max(1, int(max_rows) if max_rows is not None else ACTIVATION_BUDGET // ROW_BYTES)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        dev = self.device

        def conv(wb, cin_pad=None):
            w, b = wb
            return ops.pack_lpips_conv_weight(w, cin_pad=cin_pad).to(dev), None if b is None else b.to(dev)

        with torch.cuda.device(dev):
            self.stem = conv(folded["stem"], cin_pad=4)
            self.blocks = []
            for li, (c, stride) in enumerate(LAYERS):
                for b in range(2):
                    blk = folded[f"layer{li + 1}.{b}"]
                    self.blocks.append(dict(conv1=conv(blk["conv1"]), conv2=conv(blk["conv2"]), c=c,
                                            stride=stride if b == 0 else 1,
                                            downsample=None if blk["downsample"] is None else conv(blk["downsample"])))
            self.arm = {k: dict(conv=conv(folded[k]["conv"]), atten=tuple(t.to(dev) for t in folded[k]["atten"]))
                        for k in ("arm16", "arm32")}
            self.head32, self.head16 = conv(folded["conv_head32"]), conv(folded["conv_head16"])
            self.conv_avg = tuple(t.to(dev) for t in folded["conv_avg"])
            f = folded["ffm"]
            self.ffm = dict(a=conv(f["convblk_a"]), b=conv(f["convblk_b"]),
                            conv1=f["conv1"].to(dev), conv2=f["conv2"].to(dev))
            self.conv_out = conv(folded["conv_out"])
            cls = torch.zeros(LOGIT_LD, 256, 1, 1)
            cls[:self.n_classes] = folded["classes"]
            self.classes = conv((cls, None))

    def _chunk_logits(self, x):
        """padded NHWC logits [B][64][64][LOGIT_LD] (classes past n_classes zero) of one chunk of images"""
        B = x.shape[0]
        f32 = dict(dtype=torch.float32, device=self.device)
        x = x.to(**f32).contiguous()
        h = torch.empty(B, SIZE, SIZE, 4, **f32)
        ops.faceparse_pack(x, h)
        c1 = torch.empty(B, SIZE // 2, SIZE // 2, 64, **f32)
        ops.faceparse_conv(h, *self.stem, c1, 7, 2, 3, relu=True)
        h = torch.empty(B, SIZE // 4, SIZE // 4, 64, **f32)
        ops.faceparse_maxpool(c1, h)
        del c1
        feats = []
        for i, blk in enumerate(self.blocks):
            s, c = blk["stride"], blk["c"]
            Ho = (h.shape[1] - 1) // s + 1
            t = torch.empty(B, Ho, Ho, c, **f32)
            ops.faceparse_conv(h, *blk["conv1"], t, 3, s, 1, relu=True)
            sc = h
            if blk["downsample"] is not None:
                sc = torch.empty(B, Ho, Ho, c, **f32)
                ops.faceparse_conv(h, *blk["downsample"], sc, 1, s, 0)
            h = torch.empty(B, Ho, Ho, c, **f32)
            ops.faceparse_conv(t, *blk["conv2"], h, 3, 1, 1, residual=sc)
            if i % 2 == 1 and i >= 3:
                feats.append(h)
        feat8, feat16, feat32 = feats
        avg = torch.empty(B, 128, **f32)
        ops.faceparse_gate(feat32, *self.conv_avg, ops.FP_ACT_RELU, avg)
        up = None
        for name, feat, add, head in (("arm32", feat32, avg, self.head32), ("arm16", feat16, None, self.head16)):
            arm = self.arm[name]
            H = feat.shape[1]
            f = torch.empty(B, H, H, 128, **f32)
            ops.faceparse_conv(feat, *arm["conv"], f, 3, 1, 1, relu=True)
            g = torch.empty(B, 128, **f32)
            ops.faceparse_gate(f, *arm["atten"], ops.FP_ACT_SIGMOID, g)
            s = torch.empty(B, 2 * H, 2 * H, 128, **f32)
            ops.faceparse_apply(f, g, add if add is not None else up, s, up=2)
            up = torch.empty(B, 2 * H, 2 * H, 128, **f32)
            ops.faceparse_conv(s, *head, up, 3, 1, 1, relu=True)
        L = LOGIT_SIZE
        fa = torch.empty(B, L, L, 256, **f32)
        ops.faceparse_conv(feat8, *self.ffm["a"], fa, 1, 1, 0)
        f = torch.empty(B, L, L, 256, **f32)
        ops.faceparse_conv(up, *self.ffm["b"], f, 1, 1, 0, residual=fa)
        a = torch.empty(B, 256, **f32)
        ops.faceparse_gate(f, self.ffm["conv1"], None, ops.FP_ACT_RELU, a, w2=self.ffm["conv2"],
                           act2=ops.FP_ACT_SIGMOID)
        ff = torch.empty_like(f)
        ops.faceparse_apply(f, a, f, ff)
        h = torch.empty_like(f)
        ops.faceparse_conv(ff, *self.conv_out, h, 3, 1, 1, relu=True)
        lg = torch.empty(B, L, L, LOGIT_LD, **f32)
        ops.faceparse_conv(h, *self.classes, lg, 1, 1, 0)
        return lg

    def _logits_nhwc(self, x):
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] == 0:
            raise ValueError(f"images must be [B][3][H][W], got {tuple(x.shape)}")
        with torch.cuda.device(self.device):
            return torch.cat([self._chunk_logits(x[i:i + self.max_rows])
                              for i in range(0, x.shape[0], self.max_rows)])

    @torch.no_grad()
    def logits(self, x):
        """the main head's logits, fp32 [B][n_classes][64][64] on the device (a view of the NHWC result)"""
        return self._logits_nhwc(x)[..., :self.n_classes].permute(0, 3, 1, 2)

    @torch.no_grad()
    def labels(self, x):
        """uint8 [B][512][512] label maps on the device: argmax of the bilinear align-corners upsampled logits"""
        lg = self._logits_nhwc(x)
        out = torch.empty(lg.shape[0], SIZE, SIZE, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            ops.faceparse_labels(lg, self.n_classes, out)
        return out

    @torch.no_grad()
    def seg_consistency(self, src, edited):
        """SC per edited row: fp64 [len(edited)] on the host, the fraction of the 512^2 pixels whose label equals the
        label of source row j % B.  edited may hold k * B rows for B source images; the sources are parsed once and the
        label maps never reach device memory."""
        src, edited = torch.as_tensor(src), torch.as_tensor(edited)
        B, N = src.shape[0], edited.shape[0]
        if B == 0 or N % B:
            raise ValueError(f"edited images ({N}) must be a whole multiple of the source images ({B})")
        src_lg = self._logits_nhwc(src)
        agree = torch.empty(N, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            for i in range(0, N, self.max_rows):
                lg = self._chunk_logits(edited[i:i + self.max_rows])
                ops.faceparse_agreement(src_lg, lg, self.n_classes, (SIZE, SIZE), agree[i:i + lg.shape[0]], row0=i)
        return agree.cpu().double() / (SIZE * SIZE)
