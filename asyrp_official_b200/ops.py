"""Python handles over the C-ABI entry points (include/asyrp_b200.h), operating on torch CUDA tensors.

torch is used for device memory and streams only; every computation below is a kernel of
libasyrp_b200.so.  Layout conventions: activations NHWC fp16, weights [Cout][taps*Cin] fp16 (tap-major),
statistics / affine tables / embeddings / sampler state fp32.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import AsyrpConvDesc, check

MODE_1x1, MODE_3x3, MODE_3x3_S2 = 0, 1, 2
RESAMPLE_NONE, RESAMPLE_AVGPOOL2, RESAMPLE_UP2 = 0, 1, 2


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.AsyrpError("asyrp_official_b200 ops need CUDA tensors (there is no CPU path)")


def pack_conv_weight(w):
    """[O][I][kh][kw] (torch Conv2d) or [O][I] / [O][I][1] -> [O][kh*kw*I] fp16, tap-major / channel-minor."""
    if w.dim() == 2:
        w = w[:, :, None, None]
    if w.dim() == 3:
        w = w[:, :, :, None]
    o = w.shape[0]
    return w.permute(0, 2, 3, 1).reshape(o, -1).to(torch.float16).contiguous()


def pack_upconv_weight(w):
    """Upsample.conv weights [O][I][3][3] -> sub-pixel form fp16 [4*O][4*I]: row (a*2+b)*O + o is the 2x2 kernel of
    output phase (2i+a, 2j+b); column (dy*2+dx)*I + i multiplies source pixel (i-1+a+dy, j-1+b+dx).  The 3x3 taps that
    land on the same source pixel under nearest-x2 upsampling are summed in fp32 before the fp16 rounding."""
    w = w.float()
    o, i = w.shape[:2]
    groups = {0: ([0], [1, 2]), 1: ([0, 1], [2])}  # phase -> original tap indices per dy (dx)
    rows = []
    for a in (0, 1):
        for b in (0, 1):
            taps = []
            for dy in (0, 1):
                for dx in (0, 1):
                    acc = torch.zeros(o, i, dtype=torch.float32, device=w.device)
                    for ky in groups[a][dy]:
                        for kx in groups[b][dx]:
                            acc = acc + w[:, :, ky, kx]
                    taps.append(acc)
            rows.append(torch.stack(taps, 1).reshape(o, 4 * i))  # [O][4][I] -> tap-major, channel-minor
    return torch.cat(rows, 0).to(torch.float16).contiguous()


def conv_stats_tiles(H, W, C, has_3x3):
    return _lib.load().asyrp_conv_stats_tiles(H, W, C, int(has_3x3))


def conv_tile_config(H, W, C, has_3x3):
    """(BN, MT) of the tile the library uses for this output geometry: BN output channels x MT * 128 pixels"""
    v = _lib.load().asyrp_conv_tile_config(H, W, C, int(has_3x3))
    return v // 16, v % 16


def conv_stats_tiles_up2(H, W, C):
    """slots per sample of the statistics an up2 conv over an H x W source writes (0: geometry unsupported)"""
    return _lib.load().asyrp_conv_stats_tiles_up2(H, W, C)


def new_stats(N, H, W, C, device, has_3x3):
    """Partial GroupNorm sums written by a conv epilogue: [N][tiles][C/2][2] fp32.  The tile geometry depends on
    whether the producing conv has a 3x3 stride-1 segment."""
    return torch.zeros(N, conv_stats_tiles(H, W, C, has_3x3), C // 2, 2, dtype=torch.float32, device=device)


STAT_SCALE = 262144.0  # 2^18: fixed-point scale of the int64 (sum, sum of squares) accumulators (csrc kStatScale)


def new_sums(N, C, device):
    """[N][C/2][2] int64 accumulators a conv epilogue adds its output statistics to (zero them before the producer runs)"""
    return torch.zeros(N, C // 2, 2, dtype=torch.int64, device=device)


class GNSpec:
    """A GroupNorm(32 groups) that the CONSUMING conv finalises inside its kernel (AsyrpConvSeg.gn_*) instead of reading
    an affine table written by asyrp_gn_finalize: `sums` are the int64 accumulators (ConvOp(sums_out=...)) of the one
    or two producers of the (virtually concatenated) input, `C` their channel counts."""
    __slots__ = ("sums", "C", "gamma", "beta", "eps", "hw", "ss", "ss_stride")

    def __init__(self, sums, C, gamma, beta, eps, hw, ss=None, ss_stride=0):
        self.sums, self.C, self.gamma, self.beta, self.eps, self.hw = list(sums), list(C), gamma, beta, float(eps), int(hw)
        self.ss, self.ss_stride = ss, int(ss_stride)
        for t, c in zip(self.sums, self.C):
            assert t.dtype == torch.int64 and t.is_contiguous() and t.shape[1:] == (c // 2, 2), (t.shape, c)
        assert gamma.dtype == torch.float32 and gamma.numel() == sum(self.C) == beta.numel()


class ConvOp:
    """One implicit-GEMM convolution launch (asyrp_conv_create / asyrp_conv_launch).

    segs: list of (src NHWC fp16 tensor, mode) or (src, mode, affine, affine_offset_channels, act): with an affine
    table ([N][Ctot][2] fp32, GroupNorm finalise output) the operand becomes act(a*x + b), applied in shared memory
    inside the kernel (the activated tensor is never materialised).  The output is [N][H][W][Cout]; for MODE_3x3_S2
    the source is [N][2H][2W][C].  weight: packed fp16 [Cout][K] ([N][Cout][K] when weight_batched).
    """

    def __init__(self, segs, weight, out=None, ebias=None, ebias_stride=0, residual=None, res_scale=1.0,
                 acc_scale=1.0, stats=None, out_planar=None, out_shape=None, weight_batched=False, a_heads=1,
                 b_heads=1, out_heads=1, up2=False, scales=None, res_mode=0, sums_out=None):
        lib = _lib.load()
        segs = [tuple(sg) + (None, 0, 0) * (len(sg) == 2) for sg in segs]
        srcs = [sg[0] for sg in segs]
        affs = [sg[2] for sg in segs]
        _need_cuda(*srcs, *[a for a in affs if not isinstance(a, GNSpec)], weight, out, ebias, residual, stats,
                   out_planar, sums_out)
        if out is not None:
            N, H, W, Cout = out.shape
            if out_heads > 1:  # out [n][H][W][heads*Cout] receives batch entries (n, head)
                N, Cout = N * out_heads, Cout // out_heads
        else:
            N, H, W, Cout = out_shape
        if up2:  # descriptor geometry = the source image; out is [N][2H][2W][Cout]
            assert H % 2 == 0 and W % 2 == 0 and len(segs) == 1 and segs[0][1] == MODE_3x3
            H, W = H // 2, W // 2
        d = AsyrpConvDesc()
        d.up2 = int(up2)
        d.N, d.H, d.W, d.Cout = N, H, W, Cout
        d.nseg = len(segs)
        ktot = 0
        for i, (src, mode, aff, aff_off, act) in enumerate(segs):
            # dense NHWC, or a channel slice of a dense NHWC tensor (pixel pitch ld = stride of the W axis)
            n_, h_, w_, c_ = src.shape
            ld = src.stride(2)
            assert src.dtype == torch.float16 and src.stride(3) == 1 and src.stride(1) == w_ * ld \
                and (n_ == 1 or src.stride(0) == h_ * w_ * ld), src.stride()
            d.seg[i].src = src.data_ptr()
            d.seg[i].C = src.shape[-1]
            d.seg[i].mode = mode
            d.seg[i].ld = ld
            if isinstance(aff, GNSpec):  # GroupNorm finalised in the kernel; aff_off = first channel on the concat axis
                d.seg[i].gn_sums_a, d.seg[i].gn_Ca = aff.sums[0].data_ptr(), aff.C[0]
                if len(aff.sums) > 1:
                    d.seg[i].gn_sums_b, d.seg[i].gn_Cb = aff.sums[1].data_ptr(), aff.C[1]
                d.seg[i].gn_gamma, d.seg[i].gn_beta = aff.gamma.data_ptr(), aff.beta.data_ptr()
                if aff.ss is not None:
                    d.seg[i].gn_scale_shift, d.seg[i].gn_ss_stride = aff.ss.data_ptr(), aff.ss_stride
                d.seg[i].gn_eps, d.seg[i].gn_hw, d.seg[i].gn_off = aff.eps, aff.hw, aff_off
                d.seg[i].act = int(act)
            elif aff is not None:
                assert aff.dtype == torch.float32 and aff.is_contiguous() and aff.shape[-1] == 2
                d.seg[i].affine = aff.data_ptr() + aff_off * 2 * 4
                d.seg[i].affine_stride = aff.shape[1] * 2
                d.seg[i].act = int(act)
            ktot += (1 if mode == MODE_1x1 else (4 if up2 else 9)) * src.shape[-1]
        assert weight.dtype == torch.float16 and weight.stride(-1) == 1 and weight.shape[-1] == ktot, \
            (weight.shape, weight.stride(), ktot)
        assert weight.shape[-2] == Cout * (4 if up2 else 1)
        d.weight = weight.data_ptr()
        d.weight_batched = int(weight_batched)
        d.weight_ld = weight.stride(-2)
        d.weight_batch_stride = weight.stride(0) if (weight_batched and weight.dim() == 3) else 0
        d.a_heads, d.b_heads, d.out_heads = a_heads, b_heads, out_heads
        d.out_f32 = int(out is not None and out.dtype == torch.float32)
        d.ebias = ebias.data_ptr() if ebias is not None else None
        d.ebias_stride = ebias_stride
        d.residual = residual.data_ptr() if residual is not None else None
        d.res_scale, d.acc_scale = res_scale, acc_scale
        d.res_mode = int(res_mode)  # 1: residual is [N][H/2][W/2][Cout] (nearest-x2); 2: [N][2H][2W][Cout] (avg-pool)
        if scales is not None:  # device-side (acc_scale, res_scale): overrides the two values above at run time
            assert scales.dtype == torch.float32 and scales.is_cuda and scales.numel() >= 2 and scales.is_contiguous()
            d.scales = scales.data_ptr()
        d.out = out.data_ptr() if out is not None else None
        d.stats = stats.data_ptr() if stats is not None else None
        if sums_out is not None:
            assert sums_out.dtype == torch.int64 and sums_out.is_contiguous() and stats is not None
            d.sums_out = sums_out.data_ptr()
        if out_planar is not None:
            assert out_planar.dtype == torch.float32
            d.out_planar = out_planar.data_ptr()
            d.planar_c = out_planar.shape[1]
        self._keep = (srcs, affs, weight, out, ebias, residual, stats, out_planar, scales, sums_out)
        h = C.c_void_p()
        check(lib.asyrp_conv_create(C.byref(d), C.byref(h)), "asyrp_conv_create")
        self._h = h
        self._lib = lib

    def launch(self):
        check(self._lib.asyrp_conv_launch(self._h, _stream()), "asyrp_conv_launch")

    __call__ = launch

    def set_scales(self, acc_scale, res_scale):
        check(self._lib.asyrp_conv_set_scales(self._h, acc_scale, res_scale), "asyrp_conv_set_scales")

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.asyrp_conv_destroy(self._h)
            self._h = None


def gn_finalize(stats_a, Ca, stats_b, Cb, gamma, beta, eps, N, HW, affine, scale_shift=None, ss_stride=0):
    lib = _lib.load()
    Ta = stats_a.shape[1]
    Tb = stats_b.shape[1] if stats_b is not None else 0
    check(lib.asyrp_gn_finalize(_ptr(stats_a), Ca, Ta, _ptr(stats_b), Cb, Tb, _ptr(gamma), _ptr(beta), eps, N, HW,
                                _ptr(scale_shift), ss_stride, _ptr(affine), _stream()), "asyrp_gn_finalize")


def apply(src_a, src_b, affine, out, act, resample=RESAMPLE_NONE, affine_offset=0):
    """out = resample(act(a*x+b)); affine [N][Ctot][2] may cover more channels than the sources: the sources' first
    channel is `affine_offset` within it"""
    lib = _lib.load()
    N, Hi, Wi, Ca = src_a.shape
    Cb = src_b.shape[-1] if src_b is not None else 0
    aptr, astride = None, 0
    if affine is not None:
        aptr = C.c_void_p(affine.data_ptr() + affine_offset * 2 * 4)
        astride = affine.shape[1] * 2
    check(lib.asyrp_apply(_ptr(src_a), Ca, _ptr(src_b), Cb, aptr, astride, _ptr(out), N, Hi, Wi, int(act),
                          resample, _stream()), "asyrp_apply")


def pack_input(x, out):
    lib = _lib.load()
    N, Cin, H, W = x.shape
    check(lib.asyrp_pack_input(_ptr(x), _ptr(out), N, Cin, H, W, _stream()), "asyrp_pack_input")


def timestep_embedding(t, out, variant):
    lib = _lib.load()
    N, dim = out.shape
    check(lib.asyrp_timestep_embedding(_ptr(t), _ptr(out), N, dim, variant, _stream()), "asyrp_timestep_embedding")


def linear(inp, weight, bias, out, act_in=False, act_out=False):
    lib = _lib.load()
    N, I = inp.shape
    O = weight.shape[0]
    assert weight.shape[1] == I and out.shape[1] >= O
    check(lib.asyrp_linear(_ptr(inp), inp.stride(0), _ptr(weight), _ptr(bias), _ptr(out), out.stride(0), N, I, O,
                           int(act_in), int(act_out), _stream()), "asyrp_linear")


def ddim_update(x, et, em, z, x_next, x0_out, at, an, c1, c2):
    lib = _lib.load()
    N, Cx, H, W = x.shape
    Ce = et.shape[1]
    check(lib.asyrp_ddim_update(_ptr(x), _ptr(et), _ptr(em), _ptr(z), _ptr(x_next), _ptr(x0_out), N, Cx, Ce, H * W,
                                at, an, c1, c2, _stream()), "asyrp_ddim_update")


def attention(qkv, out, heads, head_dim, scale):
    lib = _lib.load()
    N, T, _ = qkv.shape
    check(lib.asyrp_attention(_ptr(qkv), _ptr(out), N, T, heads, head_dim, scale, _stream()), "asyrp_attention")


def axpby(a, b, out, alpha, beta):
    lib = _lib.load()
    check(lib.asyrp_axpby(_ptr(a), _ptr(b), _ptr(out), alpha, beta, a.numel(), _stream()), "asyrp_axpby")


def unpack_nchw(inp, out):
    """NHWC fp16 -> NCHW fp32"""
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    check(lib.asyrp_unpack_nchw(_ptr(inp), _ptr(out), N, Cc, H * W, _stream()), "asyrp_unpack_nchw")


def slerp_h(h, dh, h2, stats, t, use_mask=False):
    """h2 = slerp(t, h, |h|*dh/|dh|): h, h2 NHWC fp16; dh fp32 [C][H][W] (shared) or [N][C][H][W]; stats [N][T][C/2][2]"""
    lib = _lib.load()
    N, H, W, Cc = h.shape
    stride = dh.stride(0) if dh.dim() == 4 else 0
    check(lib.asyrp_slerp_h(_ptr(h), _ptr(dh), stride, _ptr(h2), _ptr(stats), stats.shape[1], N, Cc, H, W, float(t),
                            int(use_mask), _stream()), "asyrp_slerp_h")


def transpose_tc(inp, out):
    """inp [N][T][C] (may be a channel slice: last-dim stride 1, row stride ld) -> out [N][C][T] fp16"""
    lib = _lib.load()
    N, T, Cc = inp.shape
    check(lib.asyrp_transpose_tc(_ptr(inp), _ptr(out), N, T, Cc, inp.stride(1), _stream()), "asyrp_transpose_tc")


def softmax_rows(S, P, scale):
    lib = _lib.load()
    T = S.shape[-1]
    check(lib.asyrp_softmax_rows(_ptr(S), _ptr(P), S.numel() // T, T, float(scale), _stream()), "asyrp_softmax_rows")


def ddpm_update(x, et, z, x_next, at, bt, logvar, learned_sigma, mask):
    lib = _lib.load()
    N, Cx, H, W = x.shape
    check(lib.asyrp_ddpm_update(_ptr(x), _ptr(et), _ptr(z), _ptr(x_next), N, Cx, et.shape[1], H * W, at, bt, logvar,
                                int(learned_sigma), mask, _stream()), "asyrp_ddpm_update")
