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
    scales: device (acc_scale, res_scale) read at run time; with scales_stride > 0 it is sample 0's pair of a per-sample
    table, sample n's pair scales_stride floats after sample n-1's.
    """

    def __init__(self, segs, weight, out=None, ebias=None, ebias_stride=0, residual=None, res_scale=1.0,
                 acc_scale=1.0, stats=None, out_planar=None, out_shape=None, weight_batched=False, a_heads=1,
                 b_heads=1, out_heads=1, up2=False, scales=None, res_mode=0, sums_out=None, scales_stride=0):
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
            # scales_stride > 0: `scales` is sample 0's pair of a table whose row n starts scales_stride floats further
            if scales_stride > 0:
                need = (scales.storage_offset() + (N - 1) * scales_stride + 2) * 4
                assert need <= scales.untyped_storage().nbytes(), "scales table shorter than the batch"
        d.scales_stride = int(scales_stride)
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

    @property
    def drain_at(self):
        """K-schedule entries of tile i+1 the kernel readies before it runs the epilogue of tile i"""
        return self._lib.asyrp_conv_drain_at(self._h)

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


def ddim_update_rows(x, et, em, z, x_next, x0_out, at, an, c12):
    """ddim_update with one (c1, c2) pair per sample: c12 fp32 [N][2] on the device (row n gives the bits of
    ddim_update with scalars c12[n]; z is read only by rows with c1 != 0)"""
    lib = _lib.load()
    N, Cx, H, W = x.shape
    Ce = et.shape[1]
    if not (c12.is_cuda and c12.dtype == torch.float32 and tuple(c12.shape) == (N, 2) and c12.is_contiguous()):
        raise _lib.AsyrpError(f"ddim_update_rows: c12 must be a contiguous fp32 [{N}][2] device tensor, got "
                              f"{c12.dtype} {tuple(c12.shape)} on {c12.device}")
    check(lib.asyrp_ddim_update_rows(_ptr(x), _ptr(et), _ptr(em), _ptr(z), _ptr(x_next), _ptr(x0_out), N, Cx, Ce,
                                     H * W, at, an, _ptr(c12), _stream()), "asyrp_ddim_update_rows")


def ddim_update_anchored(x, et, em, x_next, x0_out, a_cur, a_next, e_cur, at, an, c2=0.0, c12=None):
    """the DDIM update anchored to a recorded inversion (exact inversion): row n with image b = n % B becomes
    A_next[b] + (y - yr), y = ddim_update's result without noise, yr the same operations on (A_cur[b], E_cur[b],
    E_cur[b]).  x, x_next, x0_out fp32 [N][Cx][H][W] (x_next may be x, x0_out None); et, em fp32 [N][Ce][H][W], Ce >= Cx;
    a_cur, a_next, e_cur fp32 [B][Cx][H][W], N a multiple of B.  c12 fp32 [N][2] on the device gives row n its c2 from
    column 1 (column 0, c1, is not read); without it every row takes c2."""
    lib = _lib.load()
    _need_cuda(x, et, em, x_next, x0_out, a_cur, a_next, e_cur, c12)
    req = (("x", x), ("et", et), ("em", em), ("x_next", x_next), ("A_cur", a_cur), ("A_next", a_next),
           ("E_cur", e_cur)) + ((("x0_out", x0_out),) if x0_out is not None else ())
    for name, t in req:
        if not (t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4):
            raise _lib.AsyrpError(f"ddim_update_anchored: {name} must be a contiguous fp32 [rows][C][H][W] tensor, got "
                                  f"{t.dtype} {tuple(t.shape)}")
    N, Cx, H, W = x.shape
    B, Ce = a_cur.shape[0], et.shape[1]
    if tuple(x_next.shape) != (N, Cx, H, W) or (x0_out is not None and tuple(x0_out.shape) != (N, Cx, H, W)):
        raise _lib.AsyrpError(f"ddim_update_anchored: x_next and x0_out must be [{N}][{Cx}][{H}][{W}]")
    if tuple(et.shape) != (N, Ce, H, W) or tuple(em.shape) != (N, Ce, H, W) or Ce < Cx:
        raise _lib.AsyrpError(f"ddim_update_anchored: et and em must be [{N}][Ce >= {Cx}][{H}][{W}], got "
                              f"{tuple(et.shape)} and {tuple(em.shape)}")
    for name, t in (("A_cur", a_cur), ("A_next", a_next), ("E_cur", e_cur)):
        if tuple(t.shape) != (B, Cx, H, W) or B == 0 or N % B:
            raise _lib.AsyrpError(f"ddim_update_anchored: {name} must be [B][{Cx}][{H}][{W}] with N = {N} a multiple "
                                  f"of B = {B}, got {tuple(t.shape)}")
    if c12 is not None and not (c12.dtype == torch.float32 and tuple(c12.shape) == (N, 2) and c12.is_contiguous()):
        raise _lib.AsyrpError(f"ddim_update_anchored: c12 must be a contiguous fp32 [{N}][2] device tensor, got "
                              f"{c12.dtype} {tuple(c12.shape)}")
    if len({t.device for _, t in req} | ({c12.device} if c12 is not None else set())) != 1:
        raise _lib.AsyrpError("ddim_update_anchored: every tensor must live on one device")
    check(lib.asyrp_ddim_update_anchored(_ptr(x), _ptr(et), _ptr(em), _ptr(a_cur), _ptr(a_next), _ptr(e_cur),
                                         _ptr(x_next), _ptr(x0_out), N, B, Cx, Ce, H * W, at, an, c2, _ptr(c12),
                                         _stream()), "asyrp_ddim_update_anchored")


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
    assert dh.is_contiguous() or (dh.dim() == 4 and dh[0].is_contiguous()), "dh must be dense [C][H][W] per sample"
    stride = dh.stride(0) if dh.dim() == 4 else 0
    check(lib.asyrp_slerp_h(_ptr(h), _ptr(dh), stride, _ptr(h2), _ptr(stats), stats.shape[1], N, Cc, H, W, float(t),
                            int(use_mask), _stream()), "asyrp_slerp_h")


def slerp_h_rows(h, dh, h2, stats, t_rows, use_mask=False):
    """slerp_h with sample n's weight read from t_rows[n]: t_rows fp32 [N] on the device (row n gives the bits of
    slerp_h with t = t_rows[n])"""
    lib = _lib.load()
    N, H, W, Cc = h.shape
    assert dh.is_contiguous() or (dh.dim() == 4 and dh[0].is_contiguous()), "dh must be dense [C][H][W] per sample"
    if not (t_rows.is_cuda and t_rows.dtype == torch.float32 and tuple(t_rows.shape) == (N,) and t_rows.is_contiguous()):
        raise _lib.AsyrpError(f"slerp_h_rows: t_rows must be a contiguous fp32 [{N}] device tensor, got "
                              f"{t_rows.dtype} {tuple(t_rows.shape)} on {t_rows.device}")
    stride = dh.stride(0) if dh.dim() == 4 else 0
    check(lib.asyrp_slerp_h_rows(_ptr(h), _ptr(dh), stride, _ptr(h2), _ptr(stats), stats.shape[1], N, Cc, H, W,
                                 _ptr(t_rows), int(use_mask), _stream()), "asyrp_slerp_h_rows")


def add_h_rows(h, direction, h2, stats, coef):
    """h2[n] = c0_n * h[n] + α_n * direction, each element fmaf(α_n, direction, c0_n * h) in fp32, stored as fp16:
    h, h2 NHWC fp16 [N][H][W][C]; direction fp32 [C][H][W] (shared); stats [N][T][C/2][2] (slot 0 the sums of the fp32
    values, the others zeroed); coef fp32 [N][2] = (c0_n, α_n) on the device (a graph input)"""
    lib = _lib.load()
    N, H, W, Cc = h.shape
    _need_cuda(h, direction, h2, stats, coef)
    if not (h.dtype == h2.dtype == torch.float16 and h.is_contiguous() and h2.is_contiguous()
            and tuple(h2.shape) == tuple(h.shape)):
        raise _lib.AsyrpError(f"add_h_rows: h and h2 must be contiguous fp16 NHWC tensors of one shape, got "
                              f"{h.dtype} {tuple(h.shape)} / {h2.dtype} {tuple(h2.shape)}")
    if not (direction.dtype == torch.float32 and direction.is_contiguous() and tuple(direction.shape) == (Cc, H, W)):
        raise _lib.AsyrpError(f"add_h_rows: direction must be a contiguous fp32 [{Cc}][{H}][{W}] tensor, got "
                              f"{direction.dtype} {tuple(direction.shape)}")
    if not (coef.dtype == torch.float32 and coef.is_contiguous() and tuple(coef.shape) == (N, 2)):
        raise _lib.AsyrpError(f"add_h_rows: coef must be a contiguous fp32 [{N}][2] device tensor, got "
                              f"{coef.dtype} {tuple(coef.shape)}")
    if not (stats.dtype == torch.float32 and stats.is_contiguous() and stats.dim() == 4
            and tuple(stats.shape[:1]) + tuple(stats.shape[2:]) == (N, Cc // 2, 2)):
        raise _lib.AsyrpError(f"add_h_rows: stats must be a contiguous fp32 [{N}][T][{Cc // 2}][2] tensor, got "
                              f"{stats.dtype} {tuple(stats.shape)}")
    check(lib.asyrp_add_h_rows(_ptr(h), _ptr(direction), _ptr(h2), _ptr(stats), stats.shape[1], N, Cc, H, W,
                               _ptr(coef), _stream()), "asyrp_add_h_rows")


def h_gram(x, mu):
    """G fp64 [n][n] on the device: G[i][j] = sum_k (x[i][k] - mu[k]) (x[j][k] - mu[k]), the centred sample Gram of
    x fp32 [n][d] with mu fp64 [d], each sum in feature order with fp64 fma"""
    lib = _lib.load()
    _need_cuda(x, mu)
    if not (x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()):
        raise _lib.AsyrpError(f"h_gram: x must be a contiguous fp32 [n][d] tensor, got {x.dtype} {tuple(x.shape)}")
    n, d = x.shape
    if not (mu.dtype == torch.float64 and mu.is_contiguous() and tuple(mu.shape) == (d,)):
        raise _lib.AsyrpError(f"h_gram: mu must be a contiguous fp64 [{d}] tensor, got {mu.dtype} {tuple(mu.shape)}")
    G = torch.empty(max(n, 0), max(n, 0), dtype=torch.float64, device=x.device)
    check(lib.asyrp_h_gram(_ptr(x), _ptr(mu), _ptr(G), n, d, _stream()), "asyrp_h_gram")
    return G


def h_combine(x, w, mu=None):
    """out fp64 [K][d] on the device: out[k][j] = sum_r w[k][r] (x[r][j] - mu[j]) (mu None: 0), the rows r in order
    with fp64 fma; x fp32 [n][d], w fp64 [K][n], mu fp64 [d]"""
    lib = _lib.load()
    _need_cuda(x, w, mu)
    if not (x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()):
        raise _lib.AsyrpError(f"h_combine: x must be a contiguous fp32 [n][d] tensor, got {x.dtype} {tuple(x.shape)}")
    n, d = x.shape
    if not (w.dtype == torch.float64 and w.dim() == 2 and w.is_contiguous() and w.shape[1] == n):
        raise _lib.AsyrpError(f"h_combine: w must be a contiguous fp64 [K][{n}] tensor, got {w.dtype} "
                              f"{tuple(w.shape)}")
    if mu is not None and not (mu.dtype == torch.float64 and mu.is_contiguous() and tuple(mu.shape) == (d,)):
        raise _lib.AsyrpError(f"h_combine: mu must be a contiguous fp64 [{d}] tensor, got {mu.dtype} "
                              f"{tuple(mu.shape)}")
    out = torch.empty(w.shape[0], d, dtype=torch.float64, device=x.device)
    check(lib.asyrp_h_combine(_ptr(x), _ptr(w), _ptr(mu), _ptr(out), n, d, w.shape[0], _stream()), "asyrp_h_combine")
    return out


def blend_rows(x, ref, mask):
    """in place, x[n] = m * x[n] + (1 - m) * ref[n % B] per pixel with m = mask[n % B], each element
    fmaf(m, x, (1 - m) * r) in fp32: x fp32 [N][C][H][W], ref fp32 [B][C][H][W], mask fp32 [B][H][W], N a multiple of B"""
    lib = _lib.load()
    _need_cuda(x, ref, mask)
    if not (x.dtype == ref.dtype == mask.dtype == torch.float32 and x.is_contiguous() and ref.is_contiguous()
            and mask.is_contiguous()):
        raise _lib.AsyrpError(f"blend_rows: x, ref and mask must be contiguous fp32 tensors, got {x.dtype}, {ref.dtype} "
                              f"and {mask.dtype}")
    if x.dim() != 4 or ref.dim() != 4 or mask.dim() != 3:
        raise _lib.AsyrpError(f"blend_rows: x [N][C][H][W], ref [B][C][H][W] and mask [B][H][W], got "
                              f"{tuple(x.shape)}, {tuple(ref.shape)} and {tuple(mask.shape)}")
    N, Cc, H, W = x.shape
    B = ref.shape[0]
    if tuple(ref.shape[1:]) != (Cc, H, W) or tuple(mask.shape) != (B, H, W) or B == 0 or N % B:
        raise _lib.AsyrpError(f"blend_rows: ref must be [B][{Cc}][{H}][{W}] and mask [B][{H}][{W}] with N = {N} a "
                              f"multiple of B, got {tuple(ref.shape)} and {tuple(mask.shape)}")
    if len({x.device, ref.device, mask.device}) != 1:
        raise _lib.AsyrpError(f"blend_rows: x, ref and mask live on {x.device}, {ref.device} and {mask.device}")
    check(lib.asyrp_blend_rows(_ptr(x), _ptr(ref), _ptr(mask), N, B, Cc, H * W, _stream()), "asyrp_blend_rows")


def compose_rows(x, ref, masks):
    """in place, the K attribute rows of every image replaced by their per-pixel composite against ref: x fp32
    [K B][C][H][W] attribute-major (row k B + j), ref fp32 [B][C][H][W], masks fp32 [K][B][H][W], 1 <= K <= 8.  Weights
    w_k = M_k, w_0 = 1 - sum M (or M_k / sum M and 0 where the masks sum above 1); every row of image j becomes
    w_0 r + sum_k w_k x[k B + j], each step rounded in fp32 in that order (asyrp_compose_rows)"""
    lib = _lib.load()
    _need_cuda(x, ref, masks)
    if not (x.dtype == ref.dtype == masks.dtype == torch.float32 and x.is_contiguous() and ref.is_contiguous()
            and masks.is_contiguous()):
        raise _lib.AsyrpError(f"compose_rows: x, ref and masks must be contiguous fp32 tensors, got {x.dtype}, "
                              f"{ref.dtype} and {masks.dtype}")
    if x.dim() != 4 or ref.dim() != 4 or masks.dim() != 4:
        raise _lib.AsyrpError(f"compose_rows: x [K B][C][H][W], ref [B][C][H][W] and masks [K][B][H][W], got "
                              f"{tuple(x.shape)}, {tuple(ref.shape)} and {tuple(masks.shape)}")
    N, Cc, H, W = x.shape
    K, B = masks.shape[0], ref.shape[0]
    if tuple(ref.shape[1:]) != (Cc, H, W) or tuple(masks.shape) != (K, B, H, W) or N != K * B:
        raise _lib.AsyrpError(f"compose_rows: ref must be [B][{Cc}][{H}][{W}] and masks [K][B][{H}][{W}] with N = {N} "
                              f"= K B, got {tuple(ref.shape)} and {tuple(masks.shape)}")
    if len({x.device, ref.device, masks.device}) != 1:
        raise _lib.AsyrpError(f"compose_rows: x, ref and masks live on {x.device}, {ref.device} and {masks.device}")
    check(lib.asyrp_compose_rows(_ptr(x), _ptr(ref), _ptr(masks), K, B, Cc, H * W, _stream()), "asyrp_compose_rows")


def _mask_pair(name, inp, out):
    _need_cuda(inp, out)
    if not (inp.dtype == out.dtype == torch.float32 and inp.is_contiguous() and out.is_contiguous()
            and inp.dim() == 3 and inp.shape[1] == inp.shape[2] and tuple(out.shape) == tuple(inp.shape)):
        raise _lib.AsyrpError(f"{name}: in and out must be contiguous fp32 [N][S][S] tensors of one shape, got "
                              f"{inp.dtype} {tuple(inp.shape)} / {out.dtype} {tuple(out.shape)}")
    if inp.device != out.device or inp.data_ptr() == out.data_ptr():
        raise _lib.AsyrpError(f"{name}: in and out must be distinct tensors on one device")
    return inp.shape[0], inp.shape[1]


def region_mask(labels, class_bits, mask):
    """mask fp32 [N][S][S] = 1 where a label of the pixel's footprint in labels u8 [N][512][512] has its bit in
    class_bits, else 0 (S <= 512)"""
    lib = _lib.load()
    _need_cuda(labels, mask)
    if not (labels.dtype == torch.uint8 and labels.is_contiguous() and labels.dim() == 3
            and tuple(labels.shape[1:]) == (512, 512)):
        raise _lib.AsyrpError(f"region_mask: labels must be a contiguous u8 [N][512][512] tensor, got {labels.dtype} "
                              f"{tuple(labels.shape)}")
    if not (mask.dtype == torch.float32 and mask.is_contiguous() and mask.dim() == 3
            and mask.shape[0] == labels.shape[0] and mask.shape[1] == mask.shape[2]):
        raise _lib.AsyrpError(f"region_mask: mask must be a contiguous fp32 [{labels.shape[0]}][S][S] tensor, got "
                              f"{mask.dtype} {tuple(mask.shape)}")
    if labels.device != mask.device:
        raise _lib.AsyrpError(f"region_mask: labels on {labels.device}, mask on {mask.device}")
    if not 0 <= int(class_bits) < (1 << 32):
        raise _lib.AsyrpError(f"region_mask: class_bits {class_bits} is not a 32-bit mask")
    check(lib.asyrp_region_mask(_ptr(labels), C.c_uint(int(class_bits)), _ptr(mask), mask.shape[0], mask.shape[1],
                                _stream()), "asyrp_region_mask")


def mask_dilate(inp, out, r, axis):
    """out = the max of inp over [i - r, i + r] along axis (0: x, 1: y) of fp32 [N][S][S], indices outside the image
    left out"""
    lib = _lib.load()
    N, S = _mask_pair("mask_dilate", inp, out)
    check(lib.asyrp_mask_dilate(_ptr(inp), _ptr(out), N, S, int(r), int(axis), _stream()), "asyrp_mask_dilate")


def mask_blur(inp, taps, out, axis):
    """out = sum_k taps[k + R] inp[clamp(i + k)] along axis (0: x, 1: y) of fp32 [N][S][S] in tap order; flat windows
    return their value.  taps fp32 [2R + 1] on the device"""
    lib = _lib.load()
    N, S = _mask_pair("mask_blur", inp, out)
    _need_cuda(taps)
    if not (taps.dtype == torch.float32 and taps.is_contiguous() and taps.dim() == 1 and taps.numel() % 2 == 1
            and taps.device == inp.device):
        raise _lib.AsyrpError(f"mask_blur: taps must be a contiguous fp32 [2R + 1] tensor on {inp.device}, got "
                              f"{taps.dtype} {tuple(taps.shape)} on {taps.device}")
    check(lib.asyrp_mask_blur(_ptr(inp), _ptr(taps), _ptr(out), N, S, taps.numel() // 2, int(axis), _stream()),
          "asyrp_mask_blur")


def transpose_tc(inp, out):
    """inp [N][T][C] (may be a channel slice: last-dim stride 1, row stride ld) -> out [N][C][T] fp16"""
    lib = _lib.load()
    N, T, Cc = inp.shape
    check(lib.asyrp_transpose_tc(_ptr(inp), _ptr(out), N, T, Cc, inp.stride(1), _stream()), "asyrp_transpose_tc")


def softmax_rows(S, P, scale):
    lib = _lib.load()
    T = S.shape[-1]
    check(lib.asyrp_softmax_rows(_ptr(S), _ptr(P), S.numel() // T, T, float(scale), _stream()), "asyrp_softmax_rows")


def lpips_conv_kpad(cin, kh, kw):
    """columns of a packed LPIPS conv weight: kh*kw*cin rounded up to the kernel's K slice"""
    return _lib.load().asyrp_lpips_conv_kpad(cin, kh, kw)


def pack_lpips_conv_weight(w, cin_pad=None):
    """torch Conv2d weight [O][I][kh][kw] -> fp32 [O][Kpad], tap-major / channel-minor, input channels zero-padded to
    cin_pad (conv1 reads the 4-channel packed image), zero columns past kh*kw*cin_pad"""
    o, i, kh, kw = w.shape
    cin = cin_pad or i
    wp = torch.zeros(o, cin, kh, kw, dtype=torch.float32, device=w.device)
    wp[:, :i] = w.float()
    out = torch.zeros(o, lpips_conv_kpad(cin, kh, kw), dtype=torch.float32, device=w.device)
    out[:, :kh * kw * cin] = wp.permute(0, 2, 3, 1).reshape(o, -1)
    return out.contiguous()


def lpips_pack(x, shift_scale, out):
    """x fp32 NCHW [N][3][H][W] -> (x - shift)/scale, fp32 NHWC [N][H][W][4]"""
    lib = _lib.load()
    N, _, H, W = x.shape
    _need_cuda(x, shift_scale, out)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[1] == 3 and tuple(out.shape) == (N, H, W, 4)
    check(lib.asyrp_lpips_pack(_ptr(x), _ptr(shift_scale), _ptr(out), N, H, W, _stream()), "asyrp_lpips_pack")


def lpips_conv(inp, weight, bias, out, kh, kw, stride, pad):
    """out = relu(conv(inp) + bias), fp32 NHWC, TF32 tensor cores; weight from pack_lpips_conv_weight"""
    lib = _lib.load()
    N, H, W, cin = inp.shape
    cout = out.shape[-1]
    _need_cuda(inp, weight, bias, out)
    assert inp.is_contiguous() and out.is_contiguous() and weight.is_contiguous()
    assert tuple(weight.shape) == (cout, lpips_conv_kpad(cin, kh, kw)) and weight.dtype == torch.float32
    assert tuple(out.shape) == (N, (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1, cout)
    check(lib.asyrp_lpips_conv(_ptr(inp), _ptr(weight), _ptr(bias), _ptr(out), N, H, W, cin, cout, kh, kw, stride, pad,
                               _stream()), "asyrp_lpips_conv")


def lpips_maxpool(inp, out):
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    _need_cuda(inp, out)
    assert tuple(out.shape) == (N, (H - 3) // 2 + 1, (W - 3) // 2 + 1, Cc)
    check(lib.asyrp_lpips_maxpool(_ptr(inp), _ptr(out), N, H, W, Cc, _stream()), "asyrp_lpips_maxpool")


def lpips_distance_chunks(hw):
    return _lib.load().asyrp_lpips_distance_chunks(hw)


def lpips_distance(probe, ref, lin_w, partial, counters, d, accumulate):
    """d[n] (+)= mean over pixels of sum_c lin_w[c] * (probe[n]/|probe[n]| - ref[n % B]/|ref[n % B]|)^2, per pixel;
    probe [N][H][W][C], ref [B][H][W][C] fp32; partial / counters: scratch (lpips_distance_chunks(H*W) floats and one
    int per row, zero-initialised, left zero)"""
    lib = _lib.load()
    N, H, W, Cc = probe.shape
    B = ref.shape[0]
    _need_cuda(probe, ref, lin_w, partial, counters, d)
    assert ref.shape[1:] == probe.shape[1:] and lin_w.numel() == Cc and d.numel() >= N and counters.numel() >= N
    assert partial.numel() >= N * lpips_distance_chunks(H * W) and counters.dtype == torch.int32 and d.is_contiguous()
    check(lib.asyrp_lpips_distance(_ptr(probe), _ptr(ref), N, B, H * W, Cc, _ptr(lin_w), _ptr(partial),
                                   _ptr(counters), _ptr(d), int(accumulate), _stream()), "asyrp_lpips_distance")


CLIP_EPI_BIAS, CLIP_EPI_QUICK_GELU, CLIP_EPI_RESIDUAL = 1, 2, 3


def clip_embed(ids, token_embedding, positional_embedding, out):
    """out [P][T][w] = token_embedding[ids] + positional_embedding; ids int32 [P][T]"""
    lib = _lib.load()
    P, T = ids.shape
    w = token_embedding.shape[1]
    _need_cuda(ids, token_embedding, positional_embedding, out)
    assert ids.dtype == torch.int32 and ids.is_contiguous() and tuple(positional_embedding.shape) == (T, w)
    assert tuple(out.shape) == (P, T, w) and out.dtype == torch.float32
    check(lib.asyrp_clip_embed(_ptr(ids), _ptr(token_embedding), _ptr(positional_embedding), _ptr(out), P, T, w,
                               _stream()), "asyrp_clip_embed")


def clip_layernorm(x, gamma, beta, out):
    """LayerNorm(eps 1e-5) over the last dim of fp32 x; out may be x"""
    lib = _lib.load()
    w = x.shape[-1]
    _need_cuda(x, gamma, beta, out)
    assert x.is_contiguous() and out.shape == x.shape and gamma.numel() == w and beta.numel() == w
    check(lib.asyrp_clip_layernorm(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), x.numel() // w, w, _stream()),
          "asyrp_clip_layernorm")


def clip_linear(x, weight, bias, out, epilogue=CLIP_EPI_BIAS, residual=None):
    """out = epilogue(x @ weight.T + bias) over the last dim, TF32 tensor cores (the LPIPS conv's GEMM); weight fp32
    [N][K] (nn.Linear layout), bias [N] or None; CLIP_EPI_RESIDUAL adds residual (which may be out)"""
    lib = _lib.load()
    K = x.shape[-1]
    N = weight.shape[0]
    M = x.numel() // K
    _need_cuda(x, weight, bias, out, residual)
    assert x.is_contiguous() and weight.is_contiguous() and tuple(weight.shape) == (N, K)
    assert out.is_contiguous() and out.numel() == M * N and out.shape[-1] == N
    assert residual is None or (residual.is_contiguous() and residual.shape == out.shape)
    check(lib.asyrp_clip_linear(_ptr(x), _ptr(weight), _ptr(bias), _ptr(residual), _ptr(out), M, K, N, int(epilogue),
                                _stream()), "asyrp_clip_linear")


def clip_attention(qkv, out, heads, causal=True):
    """multi-head attention (head size 64): qkv [P][T][3w] (q | k | v), out [P][T][w]; causal (the text tower,
    T <= 128) or full (the image tower, T <= 257)"""
    lib = _lib.load()
    P, T, w3 = qkv.shape
    _need_cuda(qkv, out)
    assert qkv.is_contiguous() and w3 == 3 * 64 * heads and tuple(out.shape) == (P, T, 64 * heads)
    if causal:
        check(lib.asyrp_clip_attention(_ptr(qkv), _ptr(out), P, T, heads, _stream()), "asyrp_clip_attention")
    else:
        check(lib.asyrp_clip_attention_full(_ptr(qkv), _ptr(out), P, T, heads, _stream()),
              "asyrp_clip_attention_full")


def clip_layernorm_rows(x, gamma, beta, out):
    """out [B][w] = LayerNorm(eps 1e-5)(x[:, 0]) of x [B][T][w]: ln_post of the class token, read in place"""
    lib = _lib.load()
    B, T, w = x.shape
    _need_cuda(x, gamma, beta, out)
    assert x.is_contiguous() and tuple(out.shape) == (B, w) and out.is_contiguous()
    assert gamma.numel() == w and beta.numel() == w
    check(lib.asyrp_clip_layernorm_rows(_ptr(x), T * w, _ptr(gamma), _ptr(beta), _ptr(out), B, w, _stream()),
          "asyrp_clip_layernorm_rows")


def clip_image_kpad(patch):
    """columns of the patch matrix: 3 * patch^2 rounded up to the GEMM's K multiple (32)"""
    return -(-3 * patch * patch // 32) * 32


def clip_image_patches(x, out, grid, patch):
    """CLIPLoss.preprocess + patchify: x fp32 [B][3][S][S] in [-1, 1] -> out [B*grid^2][clip_image_kpad(patch)]
    (asyrp_b200.h gives the resize, normalisation and layout)"""
    lib = _lib.load()
    B, C, S, S2 = x.shape
    _need_cuda(x, out)
    kpad = clip_image_kpad(patch)
    assert C == 3 and S == S2 and x.dtype == torch.float32 and x.is_contiguous()
    assert tuple(out.shape) == (B * grid * grid, kpad) and out.is_contiguous()
    check(lib.asyrp_clip_image_patches(_ptr(x), _ptr(out), B, S, grid, patch, kpad, _stream()),
          "asyrp_clip_image_patches")


def clip_image_tokens(patch_emb, class_embedding, positional_embedding, out):
    """out [B][T][w]: row 0 = class_embedding + pos[0], row 1+p = patch_emb[b*(T-1) + p] + pos[1+p]"""
    lib = _lib.load()
    B, T, w = out.shape
    _need_cuda(patch_emb, class_embedding, positional_embedding, out)
    assert patch_emb.is_contiguous() and patch_emb.numel() == B * (T - 1) * w and class_embedding.numel() == w
    assert tuple(positional_embedding.shape) == (T, w) and out.is_contiguous()
    check(lib.asyrp_clip_image_tokens(_ptr(patch_emb), _ptr(class_embedding), _ptr(positional_embedding), _ptr(out), B,
                                      T, w, _stream()), "asyrp_clip_image_tokens")


def clip_direction(src, trg, out, group_rows, add_eps):
    """out[g] = d / (|d| + add_eps), d = mean over the group's rows i of trg_i/|trg_i| - src_i/|src_i|; src, trg fp32
    [groups * group_rows][dim], out [groups][dim]"""
    lib = _lib.load()
    n, dim = src.shape
    _need_cuda(src, trg, out)
    assert src.is_contiguous() and trg.is_contiguous() and trg.shape == src.shape and n % group_rows == 0
    assert tuple(out.shape) == (n // group_rows, dim) and out.is_contiguous()
    check(lib.asyrp_clip_direction(_ptr(src), _ptr(trg), _ptr(out), n // group_rows, group_rows, dim, float(add_eps),
                                   _stream()), "asyrp_clip_direction")


def clip_pool(x, ids, gamma, beta, out):
    """out [P][w] = LayerNorm(x[p][first argmax of ids[p]]); x [P][T][w], ids int32 [P][T]"""
    lib = _lib.load()
    P, T, w = x.shape
    _need_cuda(x, ids, gamma, beta, out)
    assert ids.dtype == torch.int32 and tuple(ids.shape) == (P, T) and tuple(out.shape) == (P, w)
    check(lib.asyrp_clip_pool(_ptr(x), _ptr(ids), _ptr(gamma), _ptr(beta), _ptr(out), P, T, w, _stream()),
          "asyrp_clip_pool")


def clip_cosine(a, b, out, eps=1e-6):
    """out[n] = torch.nn.CosineSimilarity(dim=1, eps)(a, b)[n]; a, b fp32 [n][dim]"""
    lib = _lib.load()
    n, dim = a.shape
    _need_cuda(a, b, out)
    assert a.is_contiguous() and b.is_contiguous() and b.shape == a.shape and out.numel() == n
    check(lib.asyrp_clip_cosine(_ptr(a), _ptr(b), _ptr(out), n, dim, float(eps), _stream()), "asyrp_clip_cosine")


CLIP_EPI_GELU = 7  # asyrp_clip_linear's exact-GELU epilogue (DINO's MLP)
DINO_LN_EPS = 1e-6  # DINO's LayerNorm eps


def _dino_f32(name, *ts):
    for t in ts:
        if t.dtype != torch.float32:
            raise _lib.AsyrpError(f"{name}: fp32 tensors expected, got {t.dtype}")
    if len({t.device for t in ts}) != 1:
        raise _lib.AsyrpError(f"{name}: tensors live on {sorted(str(t.device) for t in ts)}")


def dino_pack(x, out, grid, patch):
    """DINO's input transform and patch matrix: x fp32 [B][3][S][S] in [-1, 1] -> (x+1)/2, antialiased bilinear resize
    to grid*patch, ImageNet Normalize -> out [B*grid^2][clip_image_kpad(patch)] in (c, ky, kx) column order"""
    lib = _lib.load()
    _need_cuda(x, out)
    _dino_f32("dino_pack", x, out)
    if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != x.shape[3] or not x.is_contiguous():
        raise _lib.AsyrpError(f"dino_pack: x must be contiguous [B][3][S][S], got {tuple(x.shape)}")
    B, S = x.shape[0], x.shape[2]
    kpad = clip_image_kpad(patch)
    if tuple(out.shape) != (B * grid * grid, kpad) or not out.is_contiguous():
        raise _lib.AsyrpError(f"dino_pack: out must be contiguous [{B * grid * grid}][{kpad}], got {tuple(out.shape)}")
    check(lib.asyrp_dino_pack(_ptr(x), _ptr(out), B, S, grid, patch, kpad, _stream()), "asyrp_dino_pack")


def dino_layernorm(x, gamma, beta, out, eps=DINO_LN_EPS):
    """out [rows][w] = LayerNorm(eps)(rows of x): x a 2-D view [rows][w] whose rows may be strided (x.stride(0) >= w,
    x.stride(1) == 1) or a contiguous tensor [..][w]; out dense, which may be x only when x is dense"""
    lib = _lib.load()
    _need_cuda(x, gamma, beta, out)
    _dino_f32("dino_layernorm", x, gamma, beta, out)
    w = x.shape[-1]
    if x.dim() != 2:
        if not x.is_contiguous():
            raise _lib.AsyrpError("dino_layernorm: an x of other than 2 dims must be contiguous")
        x = x.view(-1, w)
    rows, ld = x.shape[0], x.stride(0)
    if x.stride(1) != 1 or out.numel() != rows * w or out.shape[-1] != w or not out.is_contiguous():
        raise _lib.AsyrpError(f"dino_layernorm: x rows of unit column stride and a dense out [{rows}][{w}], got x "
                              f"strides {x.stride()} and out {tuple(out.shape)}")
    if gamma.numel() != w or beta.numel() != w:
        raise _lib.AsyrpError(f"dino_layernorm: gamma and beta must have {w} elements")
    check(lib.asyrp_dino_layernorm(_ptr(x), ld, _ptr(gamma), _ptr(beta), _ptr(out), rows, w, float(eps), _stream()),
          "asyrp_dino_layernorm")


def dino_attention(qkv, out, heads):
    """non-causal multi-head attention (head size 64, T <= 1025): qkv fp32 [B][T][3D] (q | k | v), out [B][T][D]"""
    lib = _lib.load()
    _need_cuda(qkv, out)
    _dino_f32("dino_attention", qkv, out)
    if qkv.dim() != 3 or not qkv.is_contiguous() or not out.is_contiguous():
        raise _lib.AsyrpError(f"dino_attention: contiguous qkv [B][T][3D] and out [B][T][D], got {tuple(qkv.shape)}")
    B, T, w3 = qkv.shape
    if w3 != 3 * 64 * heads or tuple(out.shape) != (B, T, 64 * heads):
        raise _lib.AsyrpError(f"dino_attention: qkv [B][T][{3 * 64 * heads}] and out [B][T][{64 * heads}] for {heads} "
                              f"heads, got {tuple(qkv.shape)} and {tuple(out.shape)}")
    check(lib.asyrp_dino_attention(_ptr(qkv), _ptr(out), B, T, heads, _stream()), "asyrp_dino_attention")


def dino_selfsim_distance(keys, ia, ib, T, out, eps=1e-8):
    """out fp64 [P]: the structure distance (1/T^2) sum_ij (Sa_ij - Sb_ij)^2 of each pair p, S the cosine
    self-similarity of the T key rows starting at row ia[p] (image a) and ib[p] (image b) of keys, a 2-D fp32 view
    [rows][D] of unit column stride whose rows may be strided (the key columns of a qkv buffer); ia, ib int64 [P] on
    the device"""
    lib = _lib.load()
    _need_cuda(keys, ia, ib, out)
    _dino_f32("dino_selfsim_distance", keys)
    if keys.dim() != 2 or keys.stride(1) != 1 or keys.stride(0) < keys.shape[1]:
        raise _lib.AsyrpError(f"dino_selfsim_distance: keys must be a 2-D view [rows][D] of unit column stride, got "
                              f"shape {tuple(keys.shape)} strides {keys.stride()}")
    if ia.dtype != torch.int64 or ib.dtype != torch.int64 or ia.dim() != 1 or ib.shape != ia.shape:
        raise _lib.AsyrpError("dino_selfsim_distance: ia and ib must be int64 [P]")
    if not (ia.is_contiguous() and ib.is_contiguous() and out.is_contiguous()) or out.dtype != torch.float64 or \
            out.shape != ia.shape:
        raise _lib.AsyrpError("dino_selfsim_distance: out must be a contiguous fp64 [P]")
    P, D = ia.shape[0], keys.shape[1]
    ntp = lib.asyrp_dino_selfsim_partials(int(T))
    if ntp < 0:
        raise _lib.AsyrpError(f"dino_selfsim_distance: T={T} outside 1..1025")
    if P and (int(ia.min()) < 0 or int(ib.min()) < 0 or max(int(ia.max()), int(ib.max())) + T > keys.shape[0]):
        raise _lib.AsyrpError(f"dino_selfsim_distance: the rows ia[p] .. ia[p] + {T} and ib[p] .. ib[p] + {T} must lie "
                              f"in the {keys.shape[0]} key rows")
    partial = torch.empty(max(P, 1) * ntp, dtype=torch.float64, device=out.device)
    check(lib.asyrp_dino_selfsim_distance(_ptr(keys), keys.stride(0), _ptr(ia), _ptr(ib), P, int(T), D, float(eps),
                                          _ptr(partial), _ptr(out), _stream()), "asyrp_dino_selfsim_distance")


def arcface_preprocess(x, out):
    """IDLoss's crop x[:, :, 35:223, 32:220] and AdaptiveAvgPool2d(112): x fp32 [B][3][H][W] -> out fp32 NHWC
    [B][112][112][4], channel 3 zero"""
    lib = _lib.load()
    B, C, H, W = x.shape
    _need_cuda(x, out)
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous() and tuple(out.shape) == (B, 112, 112, 4)
    check(lib.asyrp_arcface_preprocess(_ptr(x), _ptr(out), B, H, W, _stream()), "asyrp_arcface_preprocess")


def arcface_conv(inp, weight, bias, out, k, stride, pad, prelu=None):
    """out = conv(inp) + bias (bias may be None), then PReLU with per-channel slopes when prelu is given; fp32 NHWC,
    TF32 tensor cores; weight from pack_lpips_conv_weight"""
    lib = _lib.load()
    N, H, W, cin = inp.shape
    cout = out.shape[-1]
    _need_cuda(inp, weight, bias, out, prelu)
    assert inp.is_contiguous() and out.is_contiguous() and weight.is_contiguous()
    assert tuple(weight.shape) == (cout, lpips_conv_kpad(cin, k, k)) and weight.dtype == torch.float32
    assert tuple(out.shape) == (N, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, cout)
    check(lib.asyrp_arcface_conv(_ptr(inp), _ptr(weight), _ptr(bias), _ptr(prelu), _ptr(out), N, H, W, cin, cout, k,
                                 stride, pad, _stream()), "asyrp_arcface_conv")


def arcface_affine(inp, scale, shift, out):
    """out = inp * scale[c] + shift[c] over the last dim of fp32 inp"""
    lib = _lib.load()
    C = inp.shape[-1]
    _need_cuda(inp, scale, shift, out)
    assert inp.is_contiguous() and out.is_contiguous() and out.shape == inp.shape
    assert scale.numel() == C and shift.numel() == C
    check(lib.asyrp_arcface_affine(_ptr(inp), _ptr(scale), _ptr(shift), _ptr(out), inp.numel() // C, C, _stream()),
          "asyrp_arcface_affine")


def arcface_se_scale(res, fc1, fc2, scale):
    """SEModule's gate: scale [N][C] = sigmoid(fc2 relu(fc1 mean_hw(res))) of res [N][H][W][C]; fc1 [C/16][C],
    fc2 [C][C/16]"""
    lib = _lib.load()
    N, H, W, C = res.shape
    _need_cuda(res, fc1, fc2, scale)
    assert res.is_contiguous() and tuple(fc1.shape) == (C // 16, C) and tuple(fc2.shape) == (C, C // 16)
    assert fc1.is_contiguous() and fc2.is_contiguous() and tuple(scale.shape) == (N, C)
    check(lib.asyrp_arcface_se_scale(_ptr(res), _ptr(fc1), _ptr(fc2), _ptr(scale), N, H * W, C, _stream()),
          "asyrp_arcface_se_scale")


def arcface_se_apply(res, scale, shortcut, out, stride=1, bn=None, out2=None):
    """out = res * scale[n][c] + shortcut[:, ::stride, ::stride]; with bn = (scale, shift) also out2 = out * bn_scale +
    bn_shift (the next block's pre-conv BatchNorm)"""
    lib = _lib.load()
    N, Ho, Wo, C = res.shape
    _, Hs, Ws, Cs = shortcut.shape
    bs, bt = bn if bn is not None else (None, None)
    _need_cuda(res, scale, shortcut, out, bs, bt, out2)
    assert Cs == C and shortcut.shape[0] == N and res.is_contiguous() and shortcut.is_contiguous()
    assert out.shape == res.shape and out.is_contiguous() and tuple(scale.shape) == (N, C)
    assert (bn is None) == (out2 is None) and (out2 is None or (out2.shape == res.shape and out2.is_contiguous()))
    check(lib.asyrp_arcface_se_apply(_ptr(res), _ptr(scale), _ptr(shortcut), _ptr(out), _ptr(bs), _ptr(bt), _ptr(out2),
                                     N, Ho, Wo, C, Hs, Ws, stride, _stream()), "asyrp_arcface_se_apply")


def arcface_l2norm(x, out):
    """out = x / |x| per row of fp32 [rows][dim] (no epsilon); out must not be x"""
    lib = _lib.load()
    rows, dim = x.shape
    _need_cuda(x, out)
    assert x.is_contiguous() and out.is_contiguous() and out.shape == x.shape and out.data_ptr() != x.data_ptr()
    check(lib.asyrp_arcface_l2norm(_ptr(x), _ptr(out), rows, dim, _stream()), "asyrp_arcface_l2norm")


def arcface_dot(src, edited, out):
    """out[j] = edited[j] . src[j % B]; src [B][dim], edited [n][dim] fp32"""
    lib = _lib.load()
    B, dim = src.shape
    n = edited.shape[0]
    _need_cuda(src, edited, out)
    assert src.is_contiguous() and edited.is_contiguous() and edited.shape[1] == dim and out.numel() >= n
    check(lib.asyrp_arcface_dot(_ptr(src), _ptr(edited), _ptr(out), n, B, dim, _stream()), "asyrp_arcface_dot")


FP_ACT_NONE, FP_ACT_RELU, FP_ACT_SIGMOID = 0, 1, 2


def faceparse_pack(x, out):
    """x fp32 [B][3][H][W] in [-1, 1] -> out fp32 NHWC [B][S][S][4]: clamp, map to [0, 1], bilinear resize to S x S
    (align_corners=False), ImageNet normalisation; channel 3 zero"""
    lib = _lib.load()
    B, C, H, W = x.shape
    S = out.shape[1]
    _need_cuda(x, out)
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous() and tuple(out.shape) == (B, S, S, 4)
    assert out.dtype == torch.float32 and out.is_contiguous()
    check(lib.asyrp_faceparse_pack(_ptr(x), _ptr(out), B, H, W, S, _stream()), "asyrp_faceparse_pack")


def faceparse_conv(inp, weight, bias, out, k, stride, pad, relu=False, residual=None):
    """out = conv(inp) + bias (bias may be None), then max(., 0) with relu, or max(residual + ., 0) with residual (the
    BasicBlock end); fp32 NHWC, TF32 tensor cores; weight from pack_lpips_conv_weight"""
    lib = _lib.load()
    N, H, W, cin = inp.shape
    cout = out.shape[-1]
    _need_cuda(inp, weight, bias, out, residual)
    assert inp.is_contiguous() and out.is_contiguous() and weight.is_contiguous()
    assert tuple(weight.shape) == (cout, lpips_conv_kpad(cin, k, k)) and weight.dtype == torch.float32
    assert tuple(out.shape) == (N, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, cout)
    assert residual is None or (residual.shape == out.shape and residual.is_contiguous())
    check(lib.asyrp_faceparse_conv(_ptr(inp), _ptr(weight), _ptr(bias), _ptr(residual), _ptr(out), N, H, W, cin, cout,
                                   k, stride, pad, int(relu or residual is not None), _stream()),
          "asyrp_faceparse_conv")


def faceparse_maxpool(inp, out):
    """MaxPool2d(3, 2, padding 1) over fp32 NHWC"""
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    _need_cuda(inp, out)
    assert inp.is_contiguous() and out.is_contiguous() and tuple(out.shape) == (N, (H - 1) // 2 + 1, (W - 1) // 2 + 1,
                                                                               Cc)
    check(lib.asyrp_faceparse_maxpool(_ptr(inp), _ptr(out), N, H, W, Cc, _stream()), "asyrp_faceparse_maxpool")


def faceparse_gate(inp, w1, b1, act1, out, w2=None, b2=None, act2=FP_ACT_NONE):
    """per sample n of inp [N][H][W][C]: h = act1(w1 mean_hw(inp[n]) + b1), out[n] = act2(w2 h + b2), or h without w2;
    w1 [C1][C], w2 [C2][C1], biases may be None"""
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    C1 = w1.shape[0]
    C2 = w2.shape[0] if w2 is not None else 0
    _need_cuda(inp, w1, b1, w2, b2, out)
    assert inp.is_contiguous() and w1.is_contiguous() and tuple(w1.shape) == (C1, Cc)
    assert w2 is None or (w2.is_contiguous() and tuple(w2.shape) == (C2, C1))
    assert (b1 is None or b1.numel() == C1) and (b2 is None or b2.numel() == C2)
    assert out.is_contiguous() and tuple(out.shape) == (N, C2 if w2 is not None else C1)
    check(lib.asyrp_faceparse_gate(_ptr(inp), _ptr(w1), _ptr(b1), C1, int(act1), _ptr(w2), _ptr(b2), C2, int(act2),
                                   _ptr(out), N, H * W, Cc, _stream()), "asyrp_faceparse_gate")


def faceparse_apply(f, gate, add, out, up=1):
    """out[n][y][x][c] = f[n][y/up][x/up][c] * gate[n][c] + add, add [N][C] (broadcast) or the size of f"""
    lib = _lib.load()
    N, H, W, Cc = f.shape
    _need_cuda(f, gate, add, out)
    add_map = add.dim() == 4
    assert f.is_contiguous() and gate.is_contiguous() and add.is_contiguous() and out.is_contiguous()
    assert tuple(gate.shape) == (N, Cc) and (add.shape == f.shape if add_map else tuple(add.shape) == (N, Cc))
    assert tuple(out.shape) == (N, H * up, W * up, Cc)
    check(lib.asyrp_faceparse_apply(_ptr(f), _ptr(gate), _ptr(add), int(add_map), _ptr(out), N, H, W, Cc, up,
                                    _stream()), "asyrp_faceparse_apply")


def faceparse_labels(logits, ncls, labels):
    """labels uint8 [N][Ho][Wo] = argmax over classes 0..ncls-1 (the first wins a tie) of the bilinear align-corners
    upsampling of logits fp32 NHWC [N][Hi][Wi][ld]"""
    lib = _lib.load()
    N, Hi, Wi, ld = logits.shape
    _, Ho, Wo = labels.shape
    _need_cuda(logits, labels)
    assert logits.is_contiguous() and labels.is_contiguous() and labels.dtype == torch.uint8 and labels.shape[0] == N
    check(lib.asyrp_faceparse_labels(_ptr(logits), _ptr(labels), N, Hi, Wi, ld, ncls, Ho, Wo, _stream()),
          "asyrp_faceparse_labels")


def faceparse_agreement(src_logits, edited_logits, ncls, out_hw, agree, row0=0):
    """agree int32 [n]: pixels where the labels (faceparse_labels at out_hw) of edited row j equal those of source row
    (row0 + j) % B; src_logits [B][Hi][Wi][ld], edited_logits [n][Hi][Wi][ld]"""
    lib = _lib.load()
    B, Hi, Wi, ld = src_logits.shape
    n = edited_logits.shape[0]
    _need_cuda(src_logits, edited_logits, agree)
    assert src_logits.is_contiguous() and edited_logits.is_contiguous() and edited_logits.shape[1:] == src_logits.shape[1:]
    assert agree.dtype == torch.int32 and agree.is_contiguous() and agree.numel() == n
    check(lib.asyrp_faceparse_agreement(_ptr(src_logits), _ptr(edited_logits), _ptr(agree), n, B, int(row0), Hi, Wi, ld, ncls,
                                        out_hw[0], out_hw[1], _stream()), "asyrp_faceparse_agreement")


FID_POOL_MAX3S2, FID_POOL_AVG3S1, FID_POOL_MAX3S1 = 0, 1, 2


def fid_pack(x, out):
    """x fp32 [B][3][H][W] in [-1, 1] -> out fp32 NHWC [B][S][S][4]: the u8 save_image writes, / 255, bilinear resize to
    S x S (align_corners=False), 2 v - 1; channel 3 zero"""
    lib = _lib.load()
    B, C, H, W = x.shape
    S = out.shape[1]
    _need_cuda(x, out)
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous() and tuple(out.shape) == (B, S, S, 4)
    assert out.dtype == torch.float32 and out.is_contiguous()
    check(lib.asyrp_fid_pack(_ptr(x), _ptr(out), B, H, W, S, _stream()), "asyrp_fid_pack")


def fid_pack_u8(x, out):
    """x u8 [B][H][W][3] (decoded image files) -> out fp32 NHWC [B][S][S][4]: u8 / 255, bilinear resize to S x S
    (align_corners=False), 2 v - 1; channel 3 zero.  The same bits as fid_pack(x / 127.5 - 1)"""
    lib = _lib.load()
    B, H, W, C = x.shape
    S = out.shape[1]
    _need_cuda(x, out)
    assert C == 3 and x.dtype == torch.uint8 and x.is_contiguous() and tuple(out.shape) == (B, S, S, 4)
    assert out.dtype == torch.float32 and out.is_contiguous()
    check(lib.asyrp_fid_pack_u8(_ptr(x), _ptr(out), B, H, W, S, _stream()), "asyrp_fid_pack_u8")


def fid_conv(inp, weight, bias, out, kh, kw, stride=1, pad=(0, 0), cstore=None):
    """out[..., :cstore] = max(conv(inp) + bias, 0), fp32 NHWC, TF32 tensor cores, zero padding pad = (rows, columns);
    weight [Cout][Kpad] from pack_lpips_conv_weight and bias [Cout] with Cout a multiple of 64 (zero rows past cstore);
    out may be a channel slice out_full[..., c0:c0 + cstore] of a contiguous tensor (its row pitch is kept)"""
    lib = _lib.load()
    N, H, W, cin = inp.shape
    cout = weight.shape[0]
    cstore = out.shape[-1] if cstore is None else cstore
    _need_cuda(inp, weight, bias, out)
    assert inp.is_contiguous() and weight.is_contiguous() and bias.is_contiguous() and out.dtype == torch.float32
    assert tuple(weight.shape) == (cout, lpips_conv_kpad(cin, kh, kw)) and weight.dtype == torch.float32
    assert bias.numel() == cout
    Ho, Wo = (H + 2 * pad[0] - kh) // stride + 1, (W + 2 * pad[1] - kw) // stride + 1
    assert tuple(out.shape) == (N, Ho, Wo, cstore) and out.stride(3) == 1
    ldo = out.stride(2)
    assert out.stride(1) == Wo * ldo and out.stride(0) == Ho * Wo * ldo
    check(lib.asyrp_fid_conv(_ptr(inp), _ptr(weight), _ptr(bias), _ptr(out), N, H, W, cin, cout, kh, kw, stride,
                             pad[0], pad[1], ldo, cstore, _stream()), "asyrp_fid_conv")


def fid_pool(inp, out, mode):
    """3 x 3 pooling of fp32 NHWC inp into out, which may be a channel slice of a contiguous tensor: FID_POOL_MAX3S2
    (stride 2, no padding), FID_POOL_AVG3S1 (stride 1, pad 1, count_include_pad=False), FID_POOL_MAX3S1 (stride 1,
    pad 1)"""
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    _need_cuda(inp, out)
    Ho, Wo = ((H - 3) // 2 + 1, (W - 3) // 2 + 1) if mode == FID_POOL_MAX3S2 else (H, W)
    assert inp.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == (N, Ho, Wo, Cc)
    ldo = out.stride(2)
    assert out.stride(3) == 1 and out.stride(1) == Wo * ldo and out.stride(0) == Ho * Wo * ldo
    check(lib.asyrp_fid_pool(_ptr(inp), _ptr(out), N, H, W, Cc, int(mode), ldo, _stream()), "asyrp_fid_pool")


def fid_mean(inp, out):
    """out [N][C] = mean of fp32 NHWC inp over its pixels, summed in pixel order"""
    lib = _lib.load()
    N, H, W, Cc = inp.shape
    _need_cuda(inp, out)
    assert inp.is_contiguous() and out.is_contiguous() and tuple(out.shape) == (N, Cc)
    check(lib.asyrp_fid_mean(_ptr(inp), _ptr(out), N, H * W, Cc, _stream()), "asyrp_fid_mean")


def fid_moments(x):
    """(mu [d], sigma [d][d]) fp64 on the device: the column means and the n - 1 normalised centred covariance of
    x fp32 [n][d] (n >= 2, d a multiple of 64)"""
    lib = _lib.load()
    n, d = x.shape
    _need_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    mu = torch.empty(d, dtype=torch.float64, device=x.device)
    sigma = torch.empty(d, d, dtype=torch.float64, device=x.device)
    check(lib.asyrp_fid_moments(_ptr(x), _ptr(mu), _ptr(sigma), n, d, _stream()), "asyrp_fid_moments")
    return mu, sigma


def fid_kernel_sum(x, y, exclude_diag=False):
    """sum over the rows x_i of x [n][d] and y_j of y [m][d] (fp32) of (x_i . y_j / d + 1)^3, fp64, without the pairs
    i == j with exclude_diag: a 0-d fp64 tensor on the device"""
    lib = _lib.load()
    (n, d), m = x.shape, y.shape[0]
    _need_cuda(x, y)
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    assert y.shape[1] == d
    part = torch.empty(max(1, lib.asyrp_fid_kernel_sum_partials(n, m)), dtype=torch.float64, device=x.device)
    out = torch.empty((), dtype=torch.float64, device=x.device)
    check(lib.asyrp_fid_kernel_sum(_ptr(x), _ptr(y), _ptr(part), _ptr(out), n, m, d, int(bool(exclude_diag)),
                                   _stream()), "asyrp_fid_kernel_sum")
    return out


def fid_kernel_sum_subsets(x, y, idx_x, idx_y, exclude_diag=False):
    """out[z] = fid_kernel_sum(x[idx_x[z]], y[idx_y[z]], exclude_diag) for every subset z, the same bits, all subsets in
    one launch: x [n][d], y [m][d] fp32, idx_x / idx_y int32 [subsets][s] on the device.  The indices are checked here
    (the kernel reads them unchecked).  fp64 [subsets] on the device"""
    lib = _lib.load()
    (n, d), m = x.shape, y.shape[0]
    _need_cuda(x, y, idx_x, idx_y)
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    assert y.shape[1] == d
    if idx_x.dtype != torch.int32 or idx_y.dtype != torch.int32 or idx_x.dim() != 2 or idx_x.shape != idx_y.shape:
        raise _lib.AsyrpError(f"fid_kernel_sum_subsets: idx_x / idx_y must be int32 [subsets][s] of one shape, got "
                              f"{idx_x.dtype} {tuple(idx_x.shape)} / {idx_y.dtype} {tuple(idx_y.shape)}")
    idx_x, idx_y = idx_x.contiguous(), idx_y.contiguous()
    subsets, s = idx_x.shape
    for name, idx, rows in (("idx_x", idx_x, n), ("idx_y", idx_y, m)):
        if idx.numel():
            lo, hi = (int(v) for v in torch.aminmax(idx))
            if lo < 0 or hi >= rows:
                raise _lib.AsyrpError(f"fid_kernel_sum_subsets: {name} holds rows in [{lo}, {hi}], outside [0, {rows})")
    count = lib.asyrp_fid_kernel_sum_subsets_partials(s, subsets)
    part = torch.empty(max(1, count), dtype=torch.float64, device=x.device)
    out = torch.empty(max(0, subsets), dtype=torch.float64, device=x.device)
    check(lib.asyrp_fid_kernel_sum_subsets(_ptr(x), _ptr(y), _ptr(idx_x), _ptr(idx_y), _ptr(part), _ptr(out), n, m,
                                           s, subsets, d, int(bool(exclude_diag)), _stream()),
          "asyrp_fid_kernel_sum_subsets")
    return out


def fid_knn_radii(x, k):
    """fp64 [n] on the device: the (k + 1)-th smallest D(x_i, x_j) = sum_c (x_ic - x_jc)^2 (fp64) over every row j of
    x fp32 [n][d], j = i included, i.e. the squared distance to the k-th nearest other row (1 <= k <= 32, n > k)"""
    lib = _lib.load()
    n, d = x.shape
    _need_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    size = lib.asyrp_fid_knn_radii_workspace(n, int(k))
    work = torch.empty(max(1, size), dtype=torch.float64, device=x.device)
    radii = torch.empty(n, dtype=torch.float64, device=x.device)
    check(lib.asyrp_fid_knn_radii(_ptr(x), _ptr(radii), _ptr(work), n, d, int(k), _stream()), "asyrp_fid_knn_radii")
    return radii


def fid_knn_counts(a, ra, b, rb, out=None):
    """(b_in_a [m], a_in_b [n], a_covered [n]) int32 on the device for a fp32 [n][d], b fp32 [m][d] and their radii
    ra fp64 [n], rb fp64 [m]: b_in_a[j] = #{i : D(a_i, b_j) < ra[i]}, a_in_b[i] = #{j : D < rb[j]},
    a_covered[i] = #{j : D < ra[i]}, D the squared distance in fp64.  out: three int32 tensors to overwrite"""
    lib = _lib.load()
    (n, d), m = a.shape, b.shape[0]
    _need_cuda(a, ra, b, rb)
    assert a.dtype == torch.float32 and b.dtype == torch.float32 and a.is_contiguous() and b.is_contiguous()
    assert b.shape[1] == d
    assert ra.dtype == torch.float64 and rb.dtype == torch.float64 and ra.is_contiguous() and rb.is_contiguous()
    assert ra.numel() == n and rb.numel() == m
    if out is None:
        out = tuple(torch.empty(s, dtype=torch.int32, device=a.device) for s in (m, n, n))
    b_in_a, a_in_b, a_covered = out
    for t, s in zip(out, (m, n, n)):
        assert t.dtype == torch.int32 and t.is_contiguous() and t.numel() == s and t.is_cuda
    check(lib.asyrp_fid_knn_counts(_ptr(a), _ptr(ra), n, _ptr(b), _ptr(rb), m, d, _ptr(b_in_a), _ptr(a_in_b),
                                   _ptr(a_covered), _stream()), "asyrp_fid_knn_counts")
    return b_in_a, a_in_b, a_covered


def png_quantize(x, q, lvl0=None, xq=None):
    """x fp32 [B][3][H][W] -> q u8 [B][3][H][W], the value save_image writes; lvl0 fp64 q / 255 and xq fp32
    (2 q - 255) / 255 of the same shape, each written when given"""
    lib = _lib.load()
    B, C, H, W = x.shape
    _need_cuda(x, q, lvl0, xq)
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous()
    assert q.dtype == torch.uint8 and q.is_contiguous() and q.shape == x.shape
    assert lvl0 is None or (lvl0.dtype == torch.float64 and lvl0.is_contiguous() and lvl0.shape == x.shape)
    assert xq is None or (xq.dtype == torch.float32 and xq.is_contiguous() and xq.shape == x.shape)
    check(lib.asyrp_png_quantize(_ptr(x), _ptr(q), _ptr(lvl0), _ptr(xq), B, H, W, _stream()), "asyrp_png_quantize")


def preserve_sse(src, edited, sse):
    """sse int64 [n]: sum of (edited[j] - src[j % B])^2 over the u8 values of each row; src [B][...], edited [n][...]"""
    lib = _lib.load()
    B, n = src.shape[0], edited.shape[0]
    _need_cuda(src, edited, sse)
    assert src.dtype == torch.uint8 and edited.dtype == torch.uint8 and src.is_contiguous() and edited.is_contiguous()
    assert src.shape[1:] == edited.shape[1:] and sse.dtype == torch.int64 and sse.is_contiguous() and sse.numel() == n
    check(lib.asyrp_preserve_sse(_ptr(src), _ptr(edited), _ptr(sse), n, B, src[0].numel(), _stream()),
          "asyrp_preserve_sse")


def ssim_level(src, edited, stats):
    """stats fp64 [n][3][2]: per channel of edited row j against source row j % B, the means of the SSIM and cs maps
    over the valid pixels (11-tap Gaussian, sigma 1.5, no padding); src fp64 [B][3][H][W], edited fp64 [n][3][H][W]"""
    lib = _lib.load()
    B, C, H, W = src.shape
    n = edited.shape[0]
    _need_cuda(src, edited, stats)
    assert C == 3 and src.dtype == torch.float64 and edited.dtype == torch.float64 and edited.shape[1:] == src.shape[1:]
    assert src.is_contiguous() and edited.is_contiguous()
    assert stats.dtype == torch.float64 and stats.is_contiguous() and tuple(stats.shape) == (n, 3, 2)
    check(lib.asyrp_ssim_level(_ptr(src), _ptr(edited), _ptr(stats), n, B, H, W, _stream()), "asyrp_ssim_level")


def ssim_pool2(inp, out):
    """out = avg_pool2d(inp, 2, stride 2, padding (H mod 2, W mod 2)) of fp64 [rows][3][H][W], count_include_pad"""
    lib = _lib.load()
    rows, C, H, W = inp.shape
    _need_cuda(inp, out)
    assert C == 3 and inp.dtype == torch.float64 and out.dtype == torch.float64
    assert inp.is_contiguous() and out.is_contiguous() and tuple(out.shape) == (rows, 3, (H + 1) // 2, (W + 1) // 2)
    check(lib.asyrp_ssim_pool2(_ptr(inp), _ptr(out), rows, H, W, _stream()), "asyrp_ssim_pool2")


def ddpm_update(x, et, z, x_next, at, bt, logvar, learned_sigma, mask):
    lib = _lib.load()
    N, Cx, H, W = x.shape
    check(lib.asyrp_ddpm_update(_ptr(x), _ptr(et), _ptr(z), _ptr(x_next), N, Cx, et.shape[1], H * W, at, bt, logvar,
                                int(learned_sigma), mask, _stream()), "asyrp_ddpm_update")
