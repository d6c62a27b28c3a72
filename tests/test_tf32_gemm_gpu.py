"""The TF32 implicit GEMM of csrc/tf32_gemm.cuh through its three entry points (asyrp_lpips_conv: ReLU;
asyrp_clip_linear: bias, QuickGELU, residual; asyrp_arcface_conv: bias, PReLU) at the edges of the shapes they admit.

Reference: both operands rounded to TF32 as cvt.rna does (to nearest, ties away from zero), the product summed in
fp64 and the epilogue applied in fp64.  What is left is the kernel's fp32 accumulation, one m16n8k8 MMA per 8 columns
of the zero-padded K, plus the epilogue's own fp32 roundings:

    |out - ref| <= gain * C_ACC * (Kpad/8 + 2) * 2^-24 * (|a_t| @ |b_t|) + C_EPI * 2^-24 * (|v| + |bias| + |res| + |ref|)

C_ACC = 1: one rounding of the accumulator per MMA (Kpad/8 of them, +2 for the bias add and slack).  Measured on an
H100 SXM (80 GB HBM3, 700 W power limit) the largest error of the cases below is 0.26 of this bound, so the hardware
needs no larger constant.  gain is 1.1 for QuickGELU (its largest slope) and max(1, |slope|) for PReLU.  C_EPI = 4, 8
for QuickGELU (expf, the reciprocal and two products).  On all-positive operands, where truncation errors add up, the
bound is at least 10x tighter than 2^-11 * (|a| @ |b|), the error of operands truncated to TF32 rather than rounded
(a build with cvt.rz in place of cvt.rna fails these cases by 150x and more, and every bit-exact case).

Exactness: with one non-zero weight per output channel every output is one product of two TF32 values, exact in
fp32, so the reference rounds the operands (low 13 bits 0x1000 included: ties away from zero, not to even), multiplies,
and applies the epilogue in fp32 in the kernel's order, and the kernel must match it bit for bit (QuickGELU: within 4
ulps, its expf is not torch's).

Every input, weight, bias and output sits at the front of a buffer with a NaN tail (one extra sample or weight row):
the output tail must still be NaN and the output finite.  A second launch gives the same bits, and a sample's conv
output is the same bits alone and at every position of a batch.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, ops

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C_ACC, C_EPI, C_EPI_GELU = 1.0, 4.0, 8.0
NAN = float("nan")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _tf32(x):
    """cvt.rna.tf32.f32 of fp32 x, as fp32: round the low 13 bits to nearest, ties away from zero"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _ties(x, g):
    """x with the low 13 bits of every other element set to exactly 0x1000: a tie of the TF32 rounding"""
    b = x.float().clone().view(torch.int32)
    sel = torch.rand(x.shape, generator=g) < 0.5
    b[sel] = (b[sel] & ~0x1FFF) | 0x1000
    return b.view(torch.float32)


def _guarded(t, dev):
    """t copied to the front of a device buffer with one more NaN row; returns (buffer, view of t)"""
    buf = torch.full((t.shape[0] + 1, *t.shape[1:]), NAN, dtype=torch.float32, device=dev)
    buf[:t.shape[0]] = t.to(dev)
    return buf, buf[:t.shape[0]]


def _empty_guarded(shape, dev):
    buf = torch.full((shape[0] + 1, *shape[1:]), NAN, dtype=torch.float32, device=dev)
    return buf, buf[:shape[0]]


def _check_tail(buf, n):
    assert torch.isnan(buf[n:]).all(), "a store past the output"
    assert torch.isfinite(buf[:n]).all(), "an output element was not written, or read past an operand"


def _conv_geometry(H, W, kh, kw, s, p):
    return (H + 2 * p - kh) // s + 1, (W + 2 * p - kw) // s + 1


def _pack(w):
    """[O][I][kh][kw] -> fp32 [O][Kpad], tap-major / channel-minor, zero columns past K"""
    o, i, kh, kw = w.shape
    out = torch.zeros(o, ops.lpips_conv_kpad(i, kh, kw))
    out[:, :kh * kw * i] = w.float().permute(0, 2, 3, 1).reshape(o, -1)
    return out


def _run_conv(entry, x, w, bias, slope, stride, pad, dev):
    """run the conv entry point on guarded buffers; returns the output (CPU, NCHW fp32) after checking the guards and a
    second launch"""
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = w.shape
    Ho, Wo = _conv_geometry(H, W, kh, kw, stride, pad)
    _, xin = _guarded(x.permute(0, 2, 3, 1).contiguous(), dev)
    _, wp = _guarded(_pack(w), dev)
    b = None if bias is None else _guarded(bias, dev)[1]
    sl = None if slope is None else _guarded(slope, dev)[1]
    obuf, out = _empty_guarded((N, Ho, Wo, Cout), dev)

    def launch():
        if entry == "lpips":
            ops.lpips_conv(xin, wp, b, out, kh, kw, stride, pad)
        else:
            assert kh == kw
            ops.arcface_conv(xin, wp, b, out, kh, stride, pad, prelu=sl)

    launch()
    first = out.clone()
    _check_tail(obuf, N)
    launch()
    assert torch.equal(out, first), "a second launch changed the bits"
    return first.permute(0, 3, 1, 2).cpu()


def _run_linear(x, w, bias, epi, res, dev, in_place=False):
    """clip_linear on guarded buffers; res is written to the output first when in_place"""
    M, _ = x.shape
    N = w.shape[0]
    _, xin = _guarded(x, dev)
    _, wd = _guarded(w, dev)
    b = None if bias is None else _guarded(bias, dev)[1]
    obuf, out = _empty_guarded((M, N), dev)
    if res is not None and in_place:
        r = out
    elif res is not None:
        r = _guarded(res, dev)[1]
    else:
        r = None

    def launch():
        if in_place:
            out.copy_(res.to(dev))
        ops.clip_linear(xin, wd, b, out, epi, residual=r)

    launch()
    first = out.clone()
    _check_tail(obuf, M)
    launch()
    assert torch.equal(out, first), "a second launch changed the bits"
    return first.cpu()


def _epilogue64(z, epi, bias, slope, res):
    """fp64 epilogue on z = a_t @ b_t (channels on dim 1): (pre-activation v, output)"""
    shape = [1, -1] + [1] * (z.dim() - 2)
    v = z if bias is None else z + bias.double().view(shape)
    if epi == "relu":
        return v, v.clamp_min(0)
    if epi == "prelu":
        return v, torch.where(v > 0, v, slope.double().view(shape) * v)
    if epi == "gelu":
        return v, v * torch.sigmoid(1.702 * v)
    if epi == "residual":
        return v, res.double() + v
    return v, v


def _check_bound(out, z, S, kpad, epi, bias=None, slope=None, res=None):
    v, ref = _epilogue64(z, epi, bias, slope, res)
    shape = [1, -1] + [1] * (z.dim() - 2)
    gain = 1.0
    if epi == "gelu":
        gain = 1.1
    elif epi == "prelu":
        gain = slope.double().abs().clamp_min(1).view(shape)
    babs = 0.0 if bias is None else bias.double().abs().view(shape)
    rabs = 0.0 if res is None else res.double().abs()
    bound = gain * C_ACC * (kpad / 8 + 2) * U * S + \
        (C_EPI_GELU if epi == "gelu" else C_EPI) * U * (v.abs() + babs + rabs + ref.abs())
    err = (out.double() - ref).abs()
    ratio = (err / bound).max().item()
    assert (err <= bound).all(), f"{epi}: error {ratio:.3g}x the bound"
    return ratio


# --------------------------------------------------------------------------------------------------------------------
# conv entry points: (entry, N, H, W, Cin, Cout, kh, kw, stride, pad)
CONV_CASES = [
    ("lpips", 1, 11, 11, 4, 64, 11, 11, 4, 0),     # M = 1; nk = 16, Kpad > K
    ("lpips", 2, 64, 64, 4, 64, 11, 11, 4, 2),     # LPIPS conv1 at 64^2: (64 + 4 - 11) % 4 = 1
    ("lpips", 3, 67, 61, 4, 64, 11, 11, 4, 2),     # conv1 at an odd size, tiles across samples
    ("lpips", 3, 9, 13, 4, 192, 3, 5, 2, 2),       # kh != kw, pad = kh - 1, 3 channel tiles
    ("lpips", 2, 10, 11, 8, 64, 1, 7, 1, 3),       # 1 x 7, pad = kw // 2
    ("lpips", 2, 7, 6, 32, 64, 1, 1, 1, 1),        # pad > k: the border sees only padding; nk = 1, K % 32 == 0
    ("arcface", 1, 3, 3, 4, 64, 3, 3, 1, 0),       # M = 1, nk = 2
    ("arcface", 1, 127, 1, 4, 64, 3, 3, 1, 1),     # M = 127
    ("arcface", 2, 16, 16, 8, 192, 3, 3, 2, 1),    # M = 128 exactly, nk = 3, (16 + 2 - 3) % 2 = 1
    ("arcface", 3, 1, 43, 32, 64, 1, 1, 1, 0),     # M = 129: one pixel in the second tile, nk = 1
    ("arcface", 2, 13, 11, 4, 64, 5, 5, 1, 4),     # k = 5, pad = k - 1, nk = 4
    ("arcface", 2, 23, 21, 4, 64, 7, 7, 4, 3),     # k = 7, stride 4, ragged rows
    ("arcface", 2, 6, 7, 4, 64, 3, 3, 2, 3),       # pad = k: corner pixels see only padding
    ("arcface", 2, 9, 8, 4, 64, 1, 1, 4, 0),       # 1x1 stride 4, nk = 1 with K = 4
    ("arcface", 2, 7, 7, 512, 512, 3, 3, 1, 1),    # K = 3*3*512, 8 channel tiles
]


def _conv_ref(x, w, stride, pad):
    xt, wt = _tf32(x).double(), _tf32(w).double()
    return F.conv2d(xt, wt, stride=stride, padding=pad), F.conv2d(xt.abs(), wt.abs(), stride=stride, padding=pad)


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "-".join(map(str, c)))
def test_conv_against_tf32_fp64(cuda_device, case):
    entry, N, H, W, Cin, Cout, kh, kw, s, p = case
    g = _g(sum(case[1:]))
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, kh, kw, generator=g) / math.sqrt(Cin * kh * kw)
    bias = torch.randn(Cout, generator=g) * 0.5
    kpad = ops.lpips_conv_kpad(Cin, kh, kw)
    z, S = _conv_ref(x, w, s, p)
    if entry == "lpips":
        _check_bound(_run_conv("lpips", x, w, bias, None, s, p, cuda_device), z, S, kpad, "relu", bias=bias)
        return
    # slopes of both signs, zero among them
    slope = torch.randn(Cout, generator=g)
    slope[::7] = 0
    _check_bound(_run_conv("arcface", x, w, bias, None, s, p, cuda_device), z, S, kpad, "bias", bias=bias)
    _check_bound(_run_conv("arcface", x, w, None, None, s, p, cuda_device), z, S, kpad, "bias")
    _check_bound(_run_conv("arcface", x, w, bias, slope, s, p, cuda_device), z, S, kpad, "prelu", bias=bias,
                 slope=slope)
    _check_bound(_run_conv("arcface", x, w, None, slope, s, p, cuda_device), z, S, kpad, "prelu", slope=slope)


# clip_linear: (M, K, N)
LINEAR_CASES = [(1, 32, 64), (127, 64, 192), (128, 96, 64), (129, 128, 512), (77, 4608, 64),
                (3 * 132 * 128 + 77, 64, 128)]  # the last: 794 CTAs, more than one wave, a partial last tile


@pytest.mark.parametrize("M,K,N", LINEAR_CASES)
def test_linear_against_tf32_fp64(cuda_device, M, K, N):
    g = _g(M + K + N)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    bias = torch.randn(N, generator=g) * 0.5
    res = torch.randn(M, N, generator=g)
    xt, wt = _tf32(x).double(), _tf32(w).double()
    z, S = xt @ wt.t(), xt.abs() @ wt.abs().t()
    _check_bound(_run_linear(x, w, bias, ops.CLIP_EPI_BIAS, None, cuda_device), z, S, K, "bias", bias=bias)
    _check_bound(_run_linear(x, w, None, ops.CLIP_EPI_BIAS, None, cuda_device), z, S, K, "bias")
    # QuickGELU out to |z| ~ 100, where expf(-1.702 z) overflows or underflows
    xs = x * torch.linspace(0.1, 30, M).view(M, 1)
    zs = _tf32(xs).double() @ wt.t()
    Ss = _tf32(xs).double().abs() @ wt.abs().t()
    _check_bound(_run_linear(xs, w, bias, ops.CLIP_EPI_QUICK_GELU, None, cuda_device), zs, Ss, K, "gelu", bias=bias)
    sep = _run_linear(x, w, bias, ops.CLIP_EPI_RESIDUAL, res, cuda_device)
    _check_bound(sep, z, S, K, "residual", bias=bias, res=res)
    assert torch.equal(_run_linear(x, w, bias, ops.CLIP_EPI_RESIDUAL, res, cuda_device, in_place=True), sep)


def _assert_positive_bound_is_tight(kpad):
    assert C_ACC * (kpad / 8 + 2) * U <= 2.0 ** -11 / 10


def test_positive_operands_linear(cuda_device):
    """post-ReLU activations times positive weights: every rounding error has the same sign, none cancel"""
    g = _g(31)
    M, K, N = 129, 288, 128
    _assert_positive_bound_is_tight(K)
    x = torch.rand(M, K, generator=g)
    w = torch.rand(N, K, generator=g) / K
    bias = torch.rand(N, generator=g)
    xt, wt = _tf32(x).double(), _tf32(w).double()
    z = xt @ wt.t()
    _check_bound(_run_linear(x, w, bias, ops.CLIP_EPI_BIAS, None, cuda_device), z, z, K, "bias", bias=bias)


def test_positive_operands_conv(cuda_device):
    g = _g(32)
    N, Cin, H, W, Cout = 2, 64, 9, 10, 64
    kpad = ops.lpips_conv_kpad(Cin, 3, 3)
    _assert_positive_bound_is_tight(kpad)
    x = torch.rand(N, Cin, H, W, generator=g)
    w = torch.rand(Cout, Cin, 3, 3, generator=g) / (9 * Cin)
    bias = torch.rand(Cout, generator=g)
    z, S = _conv_ref(x, w, 1, 1)
    _check_bound(_run_conv("lpips", x, w, bias, None, 1, 1, cuda_device), z, S, kpad, "relu", bias=bias)


# --------------------------------------------------------------------------------------------------------------------
def _one_hot_weight(Cout, Cin, kh, kw, g):
    """one non-zero weight per output channel, at a random (tap, channel), half of them TF32 ties"""
    w = torch.zeros(Cout, Cin * kh * kw)
    col = torch.randint(0, Cin * kh * kw, (Cout,), generator=g)
    w[torch.arange(Cout), col] = _ties(torch.randn(Cout, generator=g), g)
    return w.view(Cout, Cin, kh, kw)


def _exact_product(x, w, stride=1, pad=0):
    """the one product per output, rna(x) * rna(w), exact in fp32 (fp64 sums it with exact zeros)"""
    return F.conv2d(_tf32(x).double(), _tf32(w).double(), stride=stride, padding=pad).float()


def _ulps(a, b):
    """distance in fp32 ulps (same-sign values; +0 and -0 are one value)"""
    ia = a.contiguous().view(torch.int32).long()
    ib = b.contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return (ia - ib).abs()


@pytest.mark.parametrize("entry,N,H,W,Cin,Cout,k,s,p", [("lpips", 3, 13, 11, 4, 64, 3, 2, 2),
                                                     ("lpips", 2, 9, 9, 8, 192, 5, 1, 4),
                                                     ("arcface", 3, 10, 9, 12, 128, 3, 1, 1),
                                                     ("arcface", 2, 15, 14, 4, 64, 11, 4, 2)])
def test_conv_exact_single_term(cuda_device, entry, N, H, W, Cin, Cout, k, s, p):
    """ReLU, bias and PReLU epilogues bit for bit, TF32 ties rounded away from zero"""
    g = _g(H * W + Cin)
    x = _ties(torch.randn(N, Cin, H, W, generator=g) * 4, g)
    x[:, :, ::5, ::3] = 0  # v exactly 0 (as are the outputs whose one tap lies in the padding)
    w = _one_hot_weight(Cout, Cin, k, k, g)
    bias = torch.randn(Cout, generator=g)
    prod = _exact_product(x, w, s, p)
    v = prod + bias.view(1, -1, 1, 1)  # one fp32 rounding, as the kernel's acc + bias
    if entry == "lpips":
        assert torch.equal(_run_conv("lpips", x, w, bias, None, s, p, cuda_device), v.clamp_min(0))
        return
    slope = torch.randn(Cout, generator=g)
    slope[::5] = 0
    sv = slope.view(1, -1, 1, 1)
    assert torch.equal(_run_conv("arcface", x, w, bias, None, s, p, cuda_device), v)
    assert torch.equal(_run_conv("arcface", x, w, None, None, s, p, cuda_device), prod)
    assert torch.equal(_run_conv("arcface", x, w, bias, slope, s, p, cuda_device), torch.where(v > 0, v, sv * v))
    assert (prod == 0).any()
    assert torch.equal(_run_conv("arcface", x, w, None, slope, s, p, cuda_device),
                       torch.where(prod > 0, prod, sv * prod))


def test_linear_exact_single_term(cuda_device):
    """bias and residual epilogues bit for bit; QuickGELU within 4 ulps over |z| up to 100"""
    g = _g(77)
    M, K, N = 133, 96, 128
    x = _ties(torch.randn(M, K, generator=g) * 8, g)
    w = _one_hot_weight(N, K, 1, 1, g).view(N, K)
    bias = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    prod = (_tf32(x).double() @ _tf32(w).double().t()).float()
    v = prod + bias
    assert torch.equal(_run_linear(x, w, bias, ops.CLIP_EPI_BIAS, None, cuda_device), v)
    assert torch.equal(_run_linear(x, w, None, ops.CLIP_EPI_BIAS, None, cuda_device), prod)
    want = res + v
    assert torch.equal(_run_linear(x, w, bias, ops.CLIP_EPI_RESIDUAL, res, cuda_device), want)
    assert torch.equal(_run_linear(x, w, bias, ops.CLIP_EPI_RESIDUAL, res, cuda_device, in_place=True), want)
    # QuickGELU: z * (1 / (1 + expf(-(1.702 z)))) in fp32; |v| reaches ~100
    xs = _ties(torch.linspace(-12.5, 12.5, M).view(M, 1) * torch.ones(M, K), g)
    ws = w.clone()
    ws[ws != 0] = _ties(torch.linspace(-8, 8, N), g)
    vs = (_tf32(xs).double() @ _tf32(ws).double().t()).float() + bias
    assert vs.abs().max().item() > 90
    got = _run_linear(xs, ws, bias, ops.CLIP_EPI_QUICK_GELU, None, cuda_device)
    want = vs * (1.0 / (1.0 + torch.exp(-(1.702 * vs))))
    assert _ulps(got, want).max().item() <= 4


# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry,H,W,Cin,k,s,p", [("lpips", 19, 17, 4, 11, 4, 2), ("arcface", 11, 13, 8, 3, 2, 1)])
def test_conv_output_does_not_depend_on_the_batch(cuda_device, entry, H, W, Cin, k, s, p):
    """a sample's output is the same bits alone and at every position of a batch of four (Ho*Wo is not a multiple of
    128, so its pixels share tiles with different neighbours at each position)"""
    g = _g(H + k)
    N, Cout = 4, 64
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k)
    bias = torch.randn(Cout, generator=g)
    Ho, Wo = _conv_geometry(H, W, k, k, s, p)
    assert (Ho * Wo) % 128 != 0
    alone = [_run_conv(entry, x[n:n + 1], w, bias, None, s, p, cuda_device) for n in range(N)]
    for shift in range(N):
        perm = [(i + shift) % N for i in range(N)]
        out = _run_conv(entry, x[perm], w, bias, None, s, p, cuda_device)
        for pos, n in enumerate(perm):
            assert torch.equal(out[pos:pos + 1], alone[n]), (n, pos)


# --------------------------------------------------------------------------------------------------------------------
def test_lpips_conv_rejects_a_null_bias_and_aliasing(cuda_device):
    x = torch.zeros(1, 8, 8, 4, device=cuda_device)
    w = torch.zeros(64, ops.lpips_conv_kpad(4, 3, 3), device=cuda_device)
    out = torch.zeros(1, 8, 8, 64, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="bias"):
        ops.lpips_conv(x, w, None, out, 3, 3, 1, 1)
    lib = _lib.load()
    stream = ops._stream()
    bias = torch.zeros(64, device=cuda_device)
    # in == out (the wrapper's shapes cannot express it: call the entry point)
    rc = lib.asyrp_lpips_conv(ops._ptr(out), ops._ptr(w), ops._ptr(bias), ops._ptr(out), 1, 8, 8, 64, 64, 1, 1, 1, 0,
                              stream)
    assert rc == -1 and b"alias" in lib.asyrp_last_error()


def test_conv_wrappers_require_contiguous_tensors(cuda_device):
    x = torch.zeros(1, 4, 8, 8, device=cuda_device).permute(0, 2, 3, 1)  # NHWC view of NCHW memory
    w = torch.zeros(64, ops.lpips_conv_kpad(4, 3, 3), device=cuda_device)
    bias = torch.zeros(64, device=cuda_device)
    out = torch.zeros(1, 8, 8, 64, device=cuda_device)
    with pytest.raises(AssertionError):
        ops.lpips_conv(x, w, bias, out, 3, 3, 1, 1)
    with pytest.raises(AssertionError):
        ops.lpips_conv(x.contiguous(), w, bias, torch.zeros(1, 64, 8, 8, device=cuda_device).permute(0, 2, 3, 1),
                       3, 3, 1, 1)
