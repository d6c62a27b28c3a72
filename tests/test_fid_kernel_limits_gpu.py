"""The FID / KID kernels (csrc/fid.cu, and the TF32 conv launcher of csrc/tf32_gemm.cuh) at the limits their entry
points admit.

  * Every ASYRP_REQUIRE clause of the asyrp_fid_* entry points of fid.cu has a row in REFUSALS: the refused call (made
    through the C ABI, since the ops wrappers assert shapes first) returns ASYRP_ERR_INVALID with a message naming the
    entry point (or "tf32 conv" for the shared launcher), leaves a NaN-filled output (a sentinel-filled one for counts)
    untouched, and its nearest accepted neighbour launches and is checked.  Calls whose shapes describe more memory
    than exists get buffers of 64 elements: each refusal comes before any read.  The rows:
      pack / pack_u8: B, H, W, S = 0, out at +4 bytes (float4 stores).
      conv: Cin = 6 and 0, Cout = 96 and 0, each clause of the geometry (N, H, W, kh, kw, stride = 0, padh, padw = -1,
      H + 2 padh = kh - 1 and the same in W), a padded extent past 2^31 - 1 (pads 2^30 and 2^30 - 1 at H = 2 or
      W = 2, and pad 2^31 - 1 at H = 8, whose 32-bit extent wrapped to 6 and was accepted), K = kh kw Cin = 2^32
      (32768 x 32768 taps of 4 channels, which wrapped to K = 0: the call was accepted and wrote max(bias, 0)),
      cstore = 3, 0 and 66 > Cout, ldo = 65 and ldo < cstore, a null bias, out at +4 bytes, in == out, N Ho Wo = 2^31
      and 2^90 (which wrapped in 64 bits), and through the launcher Cout = 65536 * 64 (grid y), in or weight at
      +4 bytes (16-byte cp.async).
      pool: N, H, W, C = 0, C = 6, ldo < C, ldo % 4 = 2, mode 3 and -1, max 3x3 / 2 at H = 2 and W = 2, in or out at
      +4 bytes, in == out.  mean: N, HW, C = 0.
      moments: n = 1, d = 0, 32 and 65536 * 64, n d = 2^40, n = 2^31 - 15 (the gram kernel steps through the rows
      16 at a time in int).
      kernel sum: n, m, d = 0, d = 8, exclude_diag = 2, n = 65535 * 64 + 1 and 2^31 - 1 (whose tile count wrapped),
      65535 x 32769 tiles (the partial count wrapped to a negative int: a one-double workspace and 2.1e9 partials
      written past it) and 131 x 16393003 = 2^31 - 255 tiles (fid_sum_kernel's strided int loop would wrap).
      kernel sum subsets: n, m, s, subsets, d = 0, d = 8, subsets = 65536, exclude_diag = 2, exclude_diag at s = 1,
      182 x 182 x 65535 tiles, a null idx_x or idx_y.  knn_counts: n = 2^31 - 1.
      The launcher's rows through asyrp_lpips_conv, asyrp_arcface_conv and asyrp_faceparse_conv: Cout = 65536 * 64,
      in at +4 bytes, and out at +4 bytes through asyrp_lpips_conv.
    Without an accepted neighbour, because it cannot be allocated: K = 2^32 (a 512 GiB weight at the largest admitted
    Kpad), N Ho Wo = 2^31 (its neighbour 2^31 - 1 is test_conv_largest_m), moments d = 65536 * 64 (a 128 TiB sigma),
    n d = 2^40 (4 TiB) and n = 2^31 - 15 (512 GiB), kernel sum past 2^31 - 256 tiles (test_kernel_sum_partial_counts
    checks the count at the bound; launching 2.1e9 CTAs would take hours), subsets past the count (likewise).
  * The edges of each kernel against references: the conv with small-integer operands (exact in TF32, every partial
    sum below 2^24) bit for bit against fp64, at one-sided 7x1 / 1x7 / 3x1 / 1x3 padding on 1 x 1 and 2 x 2 images,
    stride 2 with padw != padh at edge tiles, channel slices inside a wider ldo with NaN on both sides, Kpad > K, the
    largest M = 2^31 - 1 (16 GiB of output) and an input past 2^31 elements; pack within the first-order error of
    its fp32 source position, at S = 1 and 2, past the grid cap, an output past 2^31 elements and an input past 2^31
    elements for each reader (each sampled image the bits of the same image packed alone); the pools exactly against
    torch; the mean bit for bit against a numpy fp32 restatement (sequential sum, one divide); moments and kernel
    sums bit for bit against numpy on integer features (exact integers, exact dyadics), including rows past 2^31
    elements, and within 1e-12 relative on random features.

u = 2^-24.  Large cases check free device memory first and skip, naming the amount they need, when it is short.
The whole file takes 23-27 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit (15-17 s of it in the tests, the rest
collection), with a peak of 16.50 GiB of device memory (torch.cuda.max_memory_allocated).  The file's wall time, peak
memory and worst error / bound per kernel (0 for the bit-exact ones) are printed at the end (pytest -s).
"""
import ctypes as C
import re
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, ops
from oracle import fid as ofid

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
NAN = float("nan")
GiB = float(1 << 30)
TAIL = 64
INT_MAX = 2 ** 31 - 1
BIG_COUT = 65536 * 64  # one channel tile past the largest grid y dimension
WORST = {}  # kernel -> worst err / bound seen, printed at the end of the file (pytest -s)
ERR_INVALID = -1


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _p(t, off=0):
    """device pointer of t, off elements of t past its start (off = 1 of a float buffer: +4 bytes)"""
    return None if t is None else C.c_void_p(t.data_ptr() + off * t.element_size())


def _st():
    return ops._stream()


def _lib_():
    return _lib.load()


def _need_memory(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + GiB // 2:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")


def _nan(n, dev, dtype=torch.float32):
    return torch.full((n,), NAN, dtype=dtype, device=dev)


def _untouched(t):
    if t.is_floating_point():
        return bool(torch.isnan(t).all())
    return bool((t == -1).all())


def _record(kernel, ratio):
    WORST[kernel] = max(WORST.get(kernel, 0.0), ratio)


def _exact(kernel, got, want, what=""):
    bad = got != want
    if bad.any():
        at = [tuple(i) for i in np.argwhere(np.asarray(bad.cpu() if torch.is_tensor(bad) else bad))[:4].tolist()]
        pairs = [(i, float(got[i]), float(want[i])) for i in at]
        raise AssertionError(f"{kernel} {what}: {int(bad.sum())} elements differ; (index, got, want): {pairs}")
    _record(kernel, 0.0)


def _within(kernel, err, bound, what=""):
    ratio = (err / bound).max().item()
    _record(kernel, ratio)
    assert (err <= bound).all(), f"{kernel} {what}: error {ratio:.3g}x the bound"


def _samples(N, k):
    return sorted({0, N - 1, *range(k, N - 1, k)})


def _release():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def _conv_ref(x, w, b, stride, padh, padw, relu=True):
    """x [N][H][W][Cin], w [Cout][Cin][kh][kw], b [Cout] -> fp64 NHWC conv + bias (then ReLU), tap by tap: the padding
    is never materialised, so pads near 2^30 cost nothing"""
    N, H, W, _ = x.shape
    Cout, _, kh, kw = w.shape
    Ho, Wo = (H + 2 * padh - kh) // stride + 1, (W + 2 * padw - kw) // stride + 1
    x, w = x.double(), w.double()
    acc = torch.zeros(N, Ho, Wo, Cout, dtype=torch.float64)
    oy, ox = torch.arange(Ho) * stride - padh, torch.arange(Wo) * stride - padw
    for ky in range(kh):
        iy = oy + ky
        vy = (iy >= 0) & (iy < H)
        if not vy.any():
            continue
        for kx in range(kw):
            ix = ox + kx
            vx = (ix >= 0) & (ix < W)
            if not vx.any():
                continue
            g = x[:, iy.clamp(0, H - 1)][:, :, ix.clamp(0, W - 1)]
            g = g * (vy.view(1, -1, 1, 1) & vx.view(1, 1, -1, 1))
            acc += g @ w[:, :, ky, kx].t()
    v = acc + b.double()
    return v.clamp_min(0) if relu else v


def _pack_ref(x, S, u8):
    """fp64 bilinear (align_corners=False) of the fp32 pixel values q / 255 the kernel reads, then 2 v - 1, NHWC"""
    q = x.cpu().permute(0, 3, 1, 2).float() if u8 else ofid.quantise(x.cpu()).float()
    v = F.interpolate((q / 255).double(), (S, S), mode="bilinear", align_corners=False)
    return (2 * v - 1).permute(0, 2, 3, 1)


def _pack_bound(H, W):
    """the source coordinate (Y + 1/2) H / S - 1/2 is off by at most 1.5 u H, which moves the blend of values in
    [0, 1] by at most that; a few roundings of the blends and of 2 v - 1; twice that"""
    return (6 * (H + W) + 24) * U


def _mean_ref(x):
    """x fp32 [N][HW][C] -> the kernel's arithmetic in numpy fp32: a sequential sum in pixel order from 0, then one
    divide"""
    a = x.numpy()
    s = np.zeros((a.shape[0], a.shape[2]), np.float32)
    for k in range(a.shape[1]):
        s += a[:, k]
    return torch.from_numpy(s / np.float32(a.shape[1]))


def _int_rows(n, d, g, lo=-8, hi=8):
    """integer features [n][d] whose column sums are multiples of n: mu is an exact integer"""
    x = torch.randint(lo, hi + 1, (n, d), generator=g, dtype=torch.int64)
    x[-1] -= x.sum(0) % n
    return x


def _ksum_ref(x, y, excl):
    """sum_ij ((x_i . y_j) / d + 1)^3 for integer x, y and d a power of two: every term is (dot + d)^3 / d^3, summed in
    int64 and divided once (exact below 2^53)"""
    d = x.shape[-1]
    dots = x.long() @ y.long().transpose(-1, -2)
    num = (dots + d) ** 3
    if excl:
        k = min(x.shape[-2], y.shape[-2])
        num[..., torch.arange(k), torch.arange(k)] = 0
    tot = num.sum((-1, -2))
    assert (tot.abs() < 2 ** 53).all()
    return tot.double() / d ** 3


# ------------------------------------------------------------------------------------------------------------------
# makers: each returns (call, outputs that must stay untouched when refused, check of the accepted call)
# ------------------------------------------------------------------------------------------------------------------
def _pack(dev, B=2, H=3, W=5, S=4, u8=False, off=0):
    Bp, Hp, Wp, Sp = max(B, 1), max(H, 1), max(W, 1), max(S, 1)
    g = _g(B * 7 + H * 5 + W * 3 + S)
    if u8:
        x = torch.randint(0, 256, (Bp, Hp, Wp, 3), generator=g, dtype=torch.uint8)
    else:
        x = torch.rand(Bp, 3, Hp, Wp, generator=g) * 2.4 - 1.2
    xd = x.to(dev)
    n = Bp * Sp * Sp * 4
    full = _nan(n + TAIL + off, dev)
    entry = "asyrp_fid_pack_u8" if u8 else "asyrp_fid_pack"

    def check():
        assert _untouched(full[n:]), "written past the output"
        out = full[:n].view(B, S, S, 4)
        ref = _pack_ref(x, S, u8)
        _within("pack", (out[..., :3].double().cpu() - ref).abs(), _pack_bound(H, W), f"{B}x{H}x{W} -> {S}")
        assert (out[..., 3] == 0).all()
    return lambda: getattr(_lib_(), entry)(_p(xd), _p(full, off), B, H, W, S, _st()), [full], check


def _fconv(dev, N=2, H=5, W=6, Cin=4, Cout=64, kh=3, kw=3, stride=1, padh=1, padw=1, cstore=None, ldo=None, c0=0,
           bias=True, in_off=0, w_off=0, alias=False, tiny=False):
    """asyrp_fid_conv through the C ABI on small-integer operands (exact in TF32); out is the channel offset c0 of rows
    of pitch ldo.  tiny: buffers of 64 floats (the call must refuse before any read)"""
    cstore = Cout if cstore is None else cstore
    ldo = c0 + cstore if ldo is None else ldo

    def call_with(xb, wb, bb, ob):
        return lambda: _lib_().asyrp_fid_conv(_p(xb, in_off), _p(wb, w_off), _p(bb) if bias else None, _p(ob, c0), N, H,
                                              W, Cin, Cout, kh, kw, stride, padh, padw, ldo, cstore, _st())
    if tiny:
        xb, wb, bb = (torch.zeros(64, device=dev) for _ in range(3))
        ob = xb.fill_(NAN) if alias else _nan(64, dev)
        return call_with(xb, wb, bb, ob), [ob], None
    g = _g(N + 3 * H + 5 * W + 7 * Cin + 11 * kh + 13 * kw + (padh + padw) % 1000 + 17 * cstore + c0)
    cin, rows = max(-(-Cin // 4) * 4, 4), max(-(-Cout // 64) * 64, 64)
    Nn, Hh, Ww, kkh, kkw, s = max(N, 1), max(H, 1), max(W, 1), max(kh, 1), max(kw, 1), max(stride, 1)
    x = torch.randint(-3, 4, (Nn, Hh, Ww, cin), generator=g).float()
    w = torch.randint(-2, 3, (rows, cin, kkh, kkw), generator=g).float()
    b = torch.randint(-6, 7, (rows,), generator=g).float()
    xb = torch.cat([torch.zeros(in_off), x.view(-1)]).to(dev)
    wb = torch.cat([torch.zeros(w_off), ops.pack_lpips_conv_weight(w).view(-1)]).to(dev)
    bb = b.to(dev)
    Ho = max((Hh + 2 * max(padh, 0) - kkh) // s + 1, 1)
    Wo = max((Ww + 2 * max(padw, 0) - kkw) // s + 1, 1)
    n = Nn * Ho * Wo * max(ldo, 1)
    ob = xb.fill_(NAN) if alias else _nan(n + TAIL, dev)

    def check():
        out = ob[:n].view(N, Ho, Wo, ldo)
        ref = _conv_ref(x, w[:Cout], b[:Cout], stride, padh, padw)[..., :cstore]
        if cstore >= 8:
            assert (ref != b[:cstore].double().clamp_min(0)).any(), "no output pixel saw the input"
        what = f"{N}x{H}x{W} {kh}x{kw}/{stride} pad {padh},{padw}"
        _exact("conv", out[..., c0:c0 + cstore].double().cpu(), ref, what)
        assert _untouched(out[..., :c0]) and _untouched(out[..., c0 + cstore:]), "written outside the channel slice"
        assert _untouched(ob[n:]), "written past the output"
    return call_with(xb, wb, bb, ob), [ob], check


def _tconv(dev, entry, Cout=64, in_off=0, out_off=0, tiny=False):
    """a conv of asyrp_lpips_conv (ReLU), asyrp_arcface_conv or asyrp_faceparse_conv (bias alone), the launcher's other
    callers: 3 x 3 pad 1 on a 3 x 3 image of 4 channels, or 1 x 1 on a 1 x 1 image for the widest Cout"""
    wide = Cout > 4096
    N, H, W, Cin, k, pad = (1, 1, 1, 4, 1, 0) if wide or tiny else (1, 3, 3, 4, 3, 1)

    def call_with(xb, wb, bb, ob):
        lib = _lib_()
        if entry == "asyrp_lpips_conv":
            return lambda: lib.asyrp_lpips_conv(_p(xb, in_off), _p(wb), _p(bb), _p(ob, out_off), N, H, W, Cin, Cout,
                                                k, k, 1, pad, _st())
        if entry == "asyrp_arcface_conv":
            return lambda: lib.asyrp_arcface_conv(_p(xb, in_off), _p(wb), _p(bb), None, _p(ob, out_off), N, H, W, Cin,
                                                  Cout, k, 1, pad, _st())
        return lambda: lib.asyrp_faceparse_conv(_p(xb, in_off), _p(wb), _p(bb), None, _p(ob, out_off), N, H, W, Cin,
                                                Cout, k, 1, pad, 0, _st())
    if tiny:
        xb, wb, bb = (torch.zeros(64, device=dev) for _ in range(3))
        ob = _nan(64, dev)
        return call_with(xb, wb, bb, ob), [ob], None
    relu = entry == "asyrp_lpips_conv"
    g = _g(Cout + len(entry))
    x = torch.randint(-3, 4, (N, H, W, Cin), generator=g).float()
    xb = torch.cat([torch.zeros(in_off), x.view(-1)]).to(dev)
    n = N * H * W * Cout
    ob = _nan(n + TAIL, dev)
    if wide:  # one weight row per channel past the first two is zero: v = bias there
        wb = torch.zeros(Cout, 32, device=dev)
        w2 = torch.randint(-2, 3, (2, Cin), generator=g).float()
        wb[:2, :Cin] = w2.to(dev)
        bb = (torch.arange(Cout, device=dev) % 13 - 6).float()
        want = bb.clone()
        want[:2] += (w2 @ x.view(Cin)).to(dev)
        want = want.clamp_min(0) if relu else want
    else:
        w = torch.randint(-2, 3, (Cout, Cin, k, k), generator=g).float()
        b = torch.randint(-6, 7, (Cout,), generator=g).float()
        wb, bb = ops.pack_lpips_conv_weight(w).to(dev), b.to(dev)
        want = _conv_ref(x, w, b, 1, pad, pad, relu).view(-1).float().to(dev)

    def check():
        _exact("conv", ob[:n], want, entry)
        assert _untouched(ob[n:]), "written past the output"
    return call_with(xb, wb, bb, ob), [ob], check


def _pool(dev, N=2, H=5, W=6, C=8, mode=1, ldo=None, c0=0, in_off=0, alias=False):
    ldo = c0 + C if ldo is None else ldo
    Nn, Hh, Ww, Cc = max(N, 1), max(H, 1), max(W, 1), max(-(-C // 4) * 4, 4)
    x = torch.randn(Nn, Cc, Hh, Ww, generator=_g(N + H * 3 + W * 5 + C)).to(dev)
    xb = torch.cat([torch.zeros(in_off, device=dev), x.permute(0, 2, 3, 1).reshape(-1)])
    Ho, Wo = ((Hh - 3) // 2 + 1, (Ww - 3) // 2 + 1) if mode == 0 and min(Hh, Ww) >= 3 else (Hh, Ww)
    n = Nn * Ho * Wo * max(ldo, 1)
    ob = xb.fill_(NAN) if alias else _nan(n + TAIL, dev)

    def check():
        out = ob[:n].view(N, Ho, Wo, ldo)
        _exact("pool", out[..., c0:c0 + C], _pool_ref(x, mode).permute(0, 2, 3, 1), f"mode {mode} {H}x{W}")
        assert _untouched(out[..., :c0]) and _untouched(out[..., c0 + C:]), "written outside the channel slice"
        assert _untouched(ob[n:]), "written past the output"
    return (lambda: _lib_().asyrp_fid_pool(_p(xb, in_off), _p(ob, c0), N, H, W, C, mode, ldo, _st()), [ob], check)


def _pool_ref(x, mode):
    """torch's pools of NCHW x (on the device, as the kernel's: the same sums, in the same order)"""
    if mode == 0:
        return F.max_pool2d(x, 3, 2)
    if mode == 1:
        return F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
    return F.max_pool2d(x, 3, 1, 1)


def _mean(dev, N=2, HW=5, C=8):
    x = torch.randn(max(N, 1), max(HW, 1), max(C, 1), generator=_g(N + HW + C))
    xd = x.to(dev)
    n = max(N, 1) * max(C, 1)
    ob = _nan(n + TAIL, dev)

    def check():
        _exact("mean", ob[:n].view(N, C).cpu(), _mean_ref(x), f"N={N} HW={HW} C={C}")
        assert _untouched(ob[n:]), "written past the output"
    return lambda: _lib_().asyrp_fid_mean(_p(xd), _p(ob), N, HW, C, _st()), [ob], check


def _moments(dev, n=3, d=64, tiny=False):
    if tiny:
        xb = torch.zeros(64, device=dev)
        mu, sigma = _nan(64, dev, torch.float64), _nan(64, dev, torch.float64)
        return (lambda: _lib_().asyrp_fid_moments(_p(xb), _p(mu), _p(sigma), n, d, _st()), [mu, sigma], None)
    x = _int_rows(max(n, 2), max(d, 1), _g(n * 7 + d))
    xd = x.float().to(dev)
    mu, sigma = _nan(d + TAIL, dev, torch.float64), _nan(d * d + TAIL, dev, torch.float64)

    def check():
        _check_moments(x, mu, sigma)
    return lambda: _lib_().asyrp_fid_moments(_p(xd), _p(mu), _p(sigma), n, d, _st()), [mu, sigma], check


def _check_moments(x, mu, sigma):
    """x int64 [n][d] with integer column means: every centred product and sum is an exact integer, so sigma must be
    numpy's S / (n - 1) bit for bit"""
    n, d = x.shape
    rmu = x.sum(0) // n
    xc = (x - rmu).double().numpy()
    assert (np.abs(xc).T @ np.abs(xc)).max() < 2 ** 53  # every partial sum an exact integer, in any order
    S = xc.T @ xc
    _exact("moments", mu[:d].cpu(), rmu.double(), "mu")
    _exact("moments", sigma[:d * d].view(d, d).cpu().numpy(), S.astype(np.float64) / (n - 1), f"sigma n={n} d={d}")
    assert _untouched(mu[d:]) and _untouched(sigma[d * d:]), "written past the output"


def _ksum(dev, n=5, m=7, d=16, excl=0, tiny=False):
    if tiny:
        xb = torch.zeros(64, device=dev)
        part, out = _nan(64, dev, torch.float64), _nan(64, dev, torch.float64)
        return (lambda: _lib_().asyrp_fid_kernel_sum(_p(xb), _p(xb), _p(part), _p(out), n, m, d, excl, _st()),
                [part, out], None)
    g = _g(n + 3 * m + d)
    x, y = (torch.randint(-1, 2, (max(k, 1), max(d, 1)), generator=g) for k in (n, m))
    xd, yd = x.float().to(dev), y.float().to(dev)
    count = max(_lib_().asyrp_fid_kernel_sum_partials(n, m), 1)
    part, out = _nan(count + TAIL, dev, torch.float64), _nan(1 + TAIL, dev, torch.float64)

    def check():
        _exact("kernel_sum", out[:1].cpu(), _ksum_ref(x, y, excl).view(1), f"n={n} m={m} d={d} excl={excl}")
        assert not torch.isnan(part[:count]).any() and _untouched(part[count:]) and _untouched(out[1:])
    return (lambda: _lib_().asyrp_fid_kernel_sum(_p(xd), _p(yd), _p(part), _p(out), n, m, d, excl, _st()),
            [part, out], check)


def _subsets(dev, n=9, m=7, s=3, subsets=4, d=16, excl=0, null=None, tiny=False):
    lib = _lib_()
    if tiny:
        xb, ib = torch.zeros(64, device=dev), torch.zeros(64, dtype=torch.int32, device=dev)
        part, out = _nan(64, dev, torch.float64), _nan(64, dev, torch.float64)
        return (lambda: lib.asyrp_fid_kernel_sum_subsets(_p(xb), _p(xb), _p(ib), _p(ib), _p(part), _p(out), n, m, s,
                                                         subsets, d, excl, _st()), [part, out], None)
    g = _g(n + m * 3 + s * 5 + subsets + d)
    Z, S = max(subsets, 1), max(s, 1)
    x, y = (torch.randint(-1, 2, (max(k, 1), max(d, 1)), generator=g) for k in (n, m))
    ix = torch.randint(0, max(n, 1), (Z, S), generator=g, dtype=torch.int32)
    iy = torch.randint(0, max(m, 1), (Z, S), generator=g, dtype=torch.int32)
    xd, yd, ixd, iyd = x.float().to(dev), y.float().to(dev), ix.to(dev), iy.to(dev)
    count = max(lib.asyrp_fid_kernel_sum_subsets_partials(s, subsets), 1)
    part, out = _nan(count + TAIL, dev, torch.float64), _nan(Z + TAIL, dev, torch.float64)

    def check():
        want = _ksum_ref(x[ix.long()], y[iy.long()], excl)
        _exact("kernel_sum_subsets", out[:Z].cpu(), want, f"s={s} subsets={subsets} excl={excl}")
        assert _untouched(part[count:]) and _untouched(out[Z:]), "written past the output"
    return (lambda: lib.asyrp_fid_kernel_sum_subsets(_p(xd), _p(yd), None if null == "x" else _p(ixd),
                                                     None if null == "y" else _p(iyd), _p(part), _p(out), n, m, s,
                                                     subsets, d, excl, _st()), [part, out], check)


def _knn(dev, n=5, m=4, d=1, tiny=False):
    lib = _lib_()

    def call_with(a, ra, b, rb, outs):
        return lambda: lib.asyrp_fid_knn_counts(_p(a), _p(ra), n, _p(b), _p(rb), m, d, *(_p(o) for o in outs), _st())
    if tiny:
        a, ra = torch.zeros(64, device=dev), torch.zeros(64, dtype=torch.float64, device=dev)
        outs = [torch.full((64,), -1, dtype=torch.int32, device=dev) for _ in range(3)]
        return call_with(a, ra, a, ra, outs), outs, None
    a = torch.randint(-20, 21, (n, d), generator=_g(n)).float().to(dev)
    b = torch.randint(-20, 21, (m, d), generator=_g(m + 1)).float().to(dev)
    ra = torch.randint(0, 50, (n,), generator=_g(2)).double().to(dev)
    rb = torch.randint(0, 50, (m,), generator=_g(3)).double().to(dev)
    outs = [torch.full((k + TAIL,), -1, dtype=torch.int32, device=dev) for k in (m, n, n)]

    def check():
        D = ((a.double()[:, None, :] - b.double()[None, :, :]) ** 2).sum(-1)  # [n][m]
        want = [(D < ra[:, None]).sum(0), (D < rb[None, :]).sum(1), (D < ra[:, None]).sum(1)]
        for o, w, k in zip(outs, want, (m, n, n)):
            _exact("knn_counts", o[:k].long(), w)
            assert _untouched(o[k:]), "written past the output"
    return call_with(a, ra, b, rb, outs), outs, check


# ------------------------------------------------------------------------------------------------------------------
# refusals: one row per ASYRP_REQUIRE clause
# ------------------------------------------------------------------------------------------------------------------
def R(row, entry, pattern, maker, bad, good):
    """(row id, entry point, regex the library's message must match, refused call, accepted call or None)"""
    return (row, entry, pattern, lambda d: maker(d, **bad), None if good is None else lambda d: maker(d, **good))


T = dict(tiny=True)
FP, FPU, FC, FPOOL, FM = "asyrp_fid_pack", "asyrp_fid_pack_u8", "asyrp_fid_conv", "asyrp_fid_pool", "asyrp_fid_mean"
FMOM, FKS, FKSS = "asyrp_fid_moments", "asyrp_fid_kernel_sum", "asyrp_fid_kernel_sum_subsets"
KNN = "asyrp_fid_knn_counts"
GEOM = FC + r": bad geometry"
TF32 = "tf32 conv: "
# the pad rows' accepted neighbour: H = 1 gives H + 2 padh = 2^31 - 1 exactly; with stride 32767, output row
# 32769 sits at 32769 * 32767 - (2^30 - 1) = 0, the only one that sees the image, and the last row at 2^31 - 2
PAD_OK = dict(N=1, H=1, W=3, Cin=4, kh=1, kw=1, stride=32767, padh=2 ** 30 - 1, padw=0)
PADW_OK = dict(N=1, H=3, W=1, Cin=4, kh=1, kw=1, stride=32767, padh=0, padw=2 ** 30 - 1)
assert 32769 * 32767 == 2 ** 30 - 1 and (2 ** 31 - 2) % 32767 == 0
WIDE = dict(N=1, H=1, W=1, kh=1, kw=1, padh=0, padw=0, cstore=2, ldo=2)
KS_OK = dict(n=65535 * 64, m=1, d=16)

REFUSALS = [
    *(R(f"pack{'_u8' if u8 else ''}_{k.lower()}_0", FPU if u8 else FP, f"{FPU if u8 else FP}: bad shape .*{k}=0",
        _pack, {k: 0, "u8": u8}, {k: 1, "u8": u8}) for u8 in (False, True) for k in "BHWS"),
    *(R(f"pack{'_u8' if u8 else ''}_out_plus_4", FPU if u8 else FP, f"{FPU if u8 else FP}: out must be 16-byte aligned",
        _pack, {"off": 1, "u8": u8}, {"u8": u8}) for u8 in (False, True)),
    R("conv_cin_6", FC, FC + ": Cin=6", _fconv, dict(Cin=6), dict(Cin=8)),
    R("conv_cin_0", FC, FC + ": Cin=0", _fconv, dict(Cin=0), dict(Cin=4)),
    R("conv_cout_96", FC, FC + ": Cout=96", _fconv, dict(Cout=96), dict(Cout=128)),
    R("conv_cout_0", FC, FC + ": Cout=0", _fconv, dict(Cout=0), dict(Cout=64)),
    R("conv_n_0", FC, GEOM + " N=0", _fconv, dict(N=0), dict(N=1)),
    R("conv_h_0", FC, GEOM + " N=2 H=0", _fconv, dict(H=0, kh=1, padh=0), dict(H=1, kh=1, padh=0)),
    R("conv_w_0", FC, GEOM + " .* W=0", _fconv, dict(W=0, kw=1, padw=0), dict(W=1, kw=1, padw=0)),
    R("conv_kh_0", FC, GEOM + " .* kh=0", _fconv, dict(kh=0), dict(kh=1)),
    R("conv_kw_0", FC, GEOM + " .* kw=0", _fconv, dict(kw=0), dict(kw=1)),
    R("conv_stride_0", FC, GEOM + " .* stride=0", _fconv, dict(stride=0), dict(stride=1)),
    R("conv_padh_neg", FC, GEOM + " .* padh=-1", _fconv, dict(padh=-1), dict(padh=0)),
    R("conv_padw_neg", FC, GEOM + " .* padw=-1", _fconv, dict(padw=-1), dict(padw=0)),
    R("conv_h_below_kh", FC, GEOM + " .* H=4 .* kh=7", _fconv, dict(H=4, kh=7, kw=1, padh=1, padw=0),
      dict(H=5, kh=7, kw=1, padh=1, padw=0)),
    R("conv_w_below_kw", FC, GEOM + " .* W=4 kh=1 kw=7", _fconv, dict(W=4, kh=1, kw=7, padh=0, padw=1),
      dict(W=5, kh=1, kw=7, padh=0, padw=1)),
    R("conv_padh_2_to_the_30", FC, FC + ": padded extent H \\+ 2 padh=2147483650", _fconv,
      dict(N=1, H=2, W=3, kh=1, kw=1, stride=32767, padh=2 ** 30, padw=0, tiny=True), PAD_OK),
    R("conv_padh_2_to_the_30_minus_1", FC, FC + ": padded extent H \\+ 2 padh=2147483648", _fconv,
      dict(N=1, H=2, W=3, kh=1, kw=1, stride=32767, padh=2 ** 30 - 1, padw=0, tiny=True), PAD_OK),
    R("conv_padw_2_to_the_30", FC, FC + ": padded extent .* W \\+ 2 padw=2147483650", _fconv,
      dict(N=1, H=3, W=2, kh=1, kw=1, stride=32767, padh=0, padw=2 ** 30, tiny=True), PADW_OK),
    R("conv_padw_2_to_the_30_minus_1", FC, FC + ": padded extent .* W \\+ 2 padw=2147483648", _fconv,
      dict(N=1, H=3, W=2, kh=1, kw=1, stride=32767, padh=0, padw=2 ** 30 - 1, tiny=True), PADW_OK),
    R("conv_pad_int_max", FC, FC + ": padded extent", _fconv,
      dict(N=1, H=8, W=8, kh=1, kw=1, padh=INT_MAX, padw=INT_MAX, tiny=True), PAD_OK),
    R("conv_k_wraps", FC, FC + ": K = kh \\* kw \\* Cin = 32768 \\* 32768 \\* 4", _fconv,
      dict(N=1, H=1, W=1, kh=32768, kw=32768, padh=16384, padw=16384, tiny=True), None),
    R("conv_cstore_odd", FC, FC + ": cstore=3", _fconv, dict(cstore=3, ldo=4), dict(cstore=2, ldo=4)),
    R("conv_cstore_0", FC, FC + ": cstore=0", _fconv, dict(cstore=0, ldo=4), dict(cstore=2, ldo=4)),
    R("conv_cstore_above_cout", FC, FC + ": cstore=66", _fconv, dict(cstore=66), dict(cstore=64, ldo=66)),
    R("conv_ldo_odd", FC, FC + ": .*ldo=65", _fconv, dict(ldo=65), dict(ldo=66)),
    R("conv_ldo_below_cstore", FC, FC + ": .*ldo=62", _fconv, dict(ldo=62), dict(ldo=64)),
    R("conv_null_bias", FC, FC + ": needs a bias", _fconv, dict(bias=False), dict()),
    R("conv_out_plus_4", FC, FC + ": needs a bias and an 8-byte aligned out", _fconv, dict(c0=1, ldo=68),
      dict(c0=2, ldo=68)),
    R("conv_in_is_out", FC, FC + ": out must not alias in", _fconv, dict(alias=True, tiny=True), dict()),
    R("conv_m_2_to_the_31", FC, FC + ": too many output pixels", _fconv,
      dict(N=2, H=1, W=2, kh=1, kw=1, padh=0, padw=2 ** 29 - 1, cstore=2, tiny=True), None),
    R("conv_m_2_to_the_90", FC, FC + ": too many output pixels", _fconv,
      dict(N=2 ** 30, H=2 ** 30, W=2 ** 30, kh=1, kw=1, padh=0, padw=0, tiny=True), None),
    R("conv_cout_65536_tiles", FC, TF32 + f"Cout={BIG_COUT}", _fconv, dict(Cout=BIG_COUT, tiny=True, **WIDE),
      dict(Cout=BIG_COUT - 64, **WIDE)),
    R("conv_in_plus_4", FC, TF32 + "in and weight must be 16-byte aligned", _fconv, dict(in_off=1), dict()),
    R("conv_weight_plus_4", FC, TF32 + "in and weight must be 16-byte aligned", _fconv, dict(w_off=1), dict()),
    *(R(f"{e[6:]}_cout_65536_tiles", e, TF32 + f"Cout={BIG_COUT}", _tconv, dict(entry=e, Cout=BIG_COUT, tiny=True),
        dict(entry=e, Cout=BIG_COUT - 64))
      for e in ("asyrp_lpips_conv", "asyrp_arcface_conv", "asyrp_faceparse_conv")),
    *(R(f"{e[6:]}_in_plus_4", e, TF32 + "in and weight must be 16-byte aligned", _tconv, dict(entry=e, in_off=1),
        dict(entry=e)) for e in ("asyrp_lpips_conv", "asyrp_arcface_conv", "asyrp_faceparse_conv")),
    R("lpips_conv_out_plus_4", "asyrp_lpips_conv", TF32 + "out and residual must be 8-byte aligned", _tconv,
      dict(entry="asyrp_lpips_conv", out_off=1), dict(entry="asyrp_lpips_conv")),
    *(R(f"pool_{k.lower()}_0", FPOOL, FPOOL + f": bad shape .*{k}=0", _pool, {k: 0}, {k: 1} if k != "C" else {k: 4})
      for k in ("N", "H", "W", "C")),
    R("pool_c_6", FPOOL, FPOOL + ": bad shape .*C=6", _pool, dict(C=6), dict(C=8)),
    R("pool_ldo_below_c", FPOOL, FPOOL + ": bad shape .*ldo=4", _pool, dict(ldo=4), dict(ldo=8)),
    R("pool_ldo_mod_4", FPOOL, FPOOL + ": bad shape .*ldo=10", _pool, dict(ldo=10), dict(ldo=12)),
    R("pool_mode_3", FPOOL, FPOOL + ": mode=3", _pool, dict(mode=3), dict(mode=2)),
    R("pool_mode_neg", FPOOL, FPOOL + ": mode=-1", _pool, dict(mode=-1), dict(mode=0)),
    R("pool_max3s2_h_2", FPOOL, FPOOL + ": H=2 W=6 below", _pool, dict(mode=0, H=2), dict(mode=0, H=3)),
    R("pool_max3s2_w_2", FPOOL, FPOOL + ": H=5 W=2 below", _pool, dict(mode=0, W=2), dict(mode=0, W=3)),
    R("pool_in_plus_4", FPOOL, FPOOL + ": in and out must be 16-byte aligned", _pool, dict(in_off=1), dict()),
    R("pool_out_plus_4", FPOOL, FPOOL + ": in and out must be 16-byte aligned", _pool, dict(c0=1, ldo=12),
      dict(c0=4, ldo=12)),
    R("pool_in_is_out", FPOOL, FPOOL + ": out must not alias in", _pool, dict(alias=True), dict()),
    *(R(f"mean_{k.lower()}_0", FM, FM + f": bad shape .*{k}=0", _mean, {k: 0}, {k: 1}) for k in ("N", "HW", "C")),
    R("moments_n_1", FMOM, FMOM + ": bad shape n=1", _moments, dict(n=1), dict(n=2)),
    R("moments_d_0", FMOM, FMOM + ": bad shape .*d=0", _moments, dict(d=0), dict(d=64)),
    R("moments_d_32", FMOM, FMOM + ": bad shape .*d=32", _moments, dict(d=32), dict(d=64)),
    R("moments_d_65536_tiles", FMOM, FMOM + f": bad shape .*d={BIG_COUT}", _moments, dict(d=BIG_COUT, tiny=True),
      None),
    R("moments_nd_2_to_the_40", FMOM, FMOM + ": n \\* d too large", _moments, dict(n=2 ** 24, d=2 ** 16, tiny=True),
      None),
    R("moments_n_int_max_minus_14", FMOM, FMOM + f": n={INT_MAX - 14} above {INT_MAX - 15} rows", _moments,
      dict(n=INT_MAX - 14, d=64, tiny=True), None),
    *(R(f"kernel_sum_{k}_0", FKS, FKS + f": bad shape .*{k}=0", _ksum, {k: 0}, {k: 1 if k != "d" else 16})
      for k in ("n", "m", "d")),
    R("kernel_sum_d_8", FKS, FKS + ": bad shape .*d=8", _ksum, dict(d=8), dict(d=16)),
    R("kernel_sum_exclude_diag_2", FKS, FKS + ": exclude_diag=2", _ksum, dict(excl=2), dict(excl=1)),
    R("kernel_sum_n_65535_tiles_plus_1", FKS, FKS + f": n={65535 * 64 + 1} too large", _ksum,
      dict(n=65535 * 64 + 1, m=1, d=16, tiny=True), KS_OK),
    R("kernel_sum_n_int_max", FKS, FKS + f": n={INT_MAX} too large", _ksum, dict(n=INT_MAX, m=1, d=16, tiny=True),
      KS_OK),
    R("kernel_sum_partials_wrap", FKS, FKS + f": n={65535 * 64} x m={32769 * 64} too large", _ksum,
      dict(n=65535 * 64, m=32769 * 64, d=16, tiny=True), None),
    R("kernel_sum_partials_2_to_the_31_minus_255", FKS, FKS + f": n={131 * 64} x m={16393003 * 64} too large", _ksum,
      dict(n=131 * 64, m=16393003 * 64, d=16, tiny=True), None),
    *(R(f"subsets_{k}_0", FKSS, FKSS + f": bad shape .*{k}=0", _subsets, {k: 0}, {k: 1 if k != "d" else 16})
      for k in ("n", "m", "s", "subsets", "d")),
    R("subsets_d_8", FKSS, FKSS + ": d=8", _subsets, dict(d=8), dict(d=16)),
    R("subsets_65536", FKSS, FKSS + ": subsets=65536", _subsets, dict(subsets=65536, s=1, tiny=True),
      dict(subsets=65535, s=2)),
    R("subsets_exclude_diag_2", FKSS, FKSS + ": exclude_diag=2", _subsets, dict(excl=2), dict(excl=1)),
    R("subsets_exclude_diag_s_1", FKSS, FKSS + ": exclude_diag needs s >= 2", _subsets, dict(excl=1, s=1),
      dict(excl=1, s=2)),
    R("subsets_count_too_large", FKSS, FKSS + f": s={182 * 64} x subsets=65535 too large", _subsets,
      dict(s=182 * 64, subsets=65535, tiny=True), None),
    R("subsets_null_idx_x", FKSS, FKSS + ": needs idx_x and idx_y", _subsets, dict(null="x"), dict()),
    R("subsets_null_idx_y", FKSS, FKSS + ": needs idx_x and idx_y", _subsets, dict(null="y"), dict()),
    R("knn_counts_n_int_max", KNN, KNN + f": n={INT_MAX} above", _knn, dict(n=INT_MAX, tiny=True),
      dict(n=65535 * 64, m=1, d=1)),
]


@pytest.mark.parametrize("row", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_entry_point_refusals(cuda_device, row):
    name, entry, pattern, bad, good = row
    lib = _lib_()
    call, outs, _ = bad(cuda_device)
    torch.cuda.synchronize()
    rc = call()
    msg = lib.asyrp_last_error().decode(errors="replace")
    assert rc == ERR_INVALID, f"{name}: rc={rc} ({msg})"
    assert re.match(pattern, msg), f"{name}: {msg!r} does not match {pattern!r}"
    torch.cuda.synchronize()
    for o in outs:
        assert _untouched(o), f"{name}: the refused call wrote its output"
    del call, outs
    if good is None:
        return
    call, outs, check = good(cuda_device)
    _lib.check(call(), entry)
    torch.cuda.synchronize()
    check()
    del call, outs, check
    _release()


def test_kernel_sum_partial_counts():
    """one partial per 64 x 64 tile, -1 where the call refuses: n or m not positive, or more than 2^31 - 256 tiles
    (fid_sum_kernel's threads step through the count by 256 in int).  The bound itself, 12032 x 178481 tiles, and
    65535 x 32768 tiles are admitted; 65535 x 32769 (2^31 + 32767) and 131 x 16393003 (2^31 - 255) are not"""
    lib = _lib_()
    f = lib.asyrp_fid_kernel_sum_partials
    assert f(1, 1) == 1 and f(64, 64) == 1 and f(65, 64) == 2 and f(65, 65) == 4
    assert f(0, 1) == -1 and f(1, 0) == -1 and f(-1, 5) == -1
    assert f(1, INT_MAX) == 2 ** 25  # the tile count of m = 2^31 - 1 in 64 bits
    assert f(65535 * 64, 32768 * 64) == 65535 * 32768
    assert f(12032 * 64, 178481 * 64) == 12032 * 178481 == 2 ** 31 - 256
    assert f(65535 * 64, 32769 * 64) == -1
    assert f(131 * 64, 16393003 * 64) == -1 and 131 * 16393003 == 2 ** 31 - 255
    g = lib.asyrp_fid_kernel_sum_subsets_partials
    assert g(181 * 64, 65535) == 181 * 181 * 65535 and g(182 * 64, 65535) == -1
    assert g(INT_MAX, 1) == -1 and g(0, 1) == -1


# ------------------------------------------------------------------------------------------------------------------
# conv: exact at the edges (small-integer operands are exact in TF32 and every partial sum is below 2^24)
# ------------------------------------------------------------------------------------------------------------------
# one-sided padding of the 7x1 / 1x7 / 3x1 / 1x3 convs on 1 x 1 and 2 x 2 images; stride 2 with padw != padh over
# several pixel tiles and channel tiles with partial edge tiles; a 3 x 3 / 2 without padding on an odd size; channel
# slices of width 2 and Cout - 2 inside a wider pitch (NaN on both sides); Kpad > K (K = 4 and 108)
CONV_CASES = {
    "7x1_on_1x1": dict(N=2, H=1, W=1, Cin=8, kh=7, kw=1, padh=3, padw=0),
    "1x7_on_1x1": dict(N=2, H=1, W=1, Cin=8, kh=1, kw=7, padh=0, padw=3),
    "7x1_on_2x2": dict(N=2, H=2, W=2, Cin=4, kh=7, kw=1, padh=3, padw=0),
    "1x7_on_2x2": dict(N=2, H=2, W=2, Cin=4, kh=1, kw=7, padh=0, padw=3),
    "3x1_on_2x2": dict(N=3, H=2, W=2, Cin=4, kh=3, kw=1, padh=1, padw=0),
    "1x3_on_1x1": dict(N=3, H=1, W=1, Cin=4, kh=1, kw=3, padh=0, padw=1),
    "stride2_padw_gt_padh": dict(N=3, H=35, W=33, Cin=12, Cout=128, kh=3, kw=3, stride=2, padh=0, padw=1),
    "stride2_padh_gt_padw": dict(N=2, H=17, W=19, Cin=8, Cout=192, kh=3, kw=5, stride=2, padh=2, padw=0),
    "3x3_s2_no_pad_odd": dict(N=2, H=37, W=37, Cin=4, kh=3, kw=3, stride=2, padh=0, padw=0),
    "cstore_2_in_ldo_8": dict(N=2, H=9, W=7, Cin=8, cstore=2, c0=2, ldo=8),
    "cstore_cout_minus_2": dict(N=2, H=9, W=7, Cin=8, Cout=128, cstore=126, c0=4, ldo=136),
    "kpad_32_k_4": dict(N=2, H=6, W=5, Cin=4, kh=1, kw=1, padh=0, padw=0),
    "kpad_128_k_108": dict(N=2, H=6, W=5, Cin=12, kh=3, kw=3),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_exact_at_the_edges(cuda_device, case):
    call, _, check = _fconv(cuda_device, **CONV_CASES[case])
    _lib.check(call(), "asyrp_fid_conv")
    torch.cuda.synchronize()
    check()


def test_conv_largest_m(cuda_device):
    """M = 2^31 - 1 output pixels (prime: N = 1, Ho = 1, Wo = 2^31 - 1 from W = 1 and padw = 2^30 - 1), cstore = ldo =
    2 (16 GiB): only pixel 2^30 - 1 sees the input, every other one is max(bias, 0); compared in chunks"""
    M = INT_MAX
    _need_memory(8 * M + 1024, "the conv at M = 2^31 - 1")
    dev = cuda_device
    x = torch.tensor([1.0, -2.0, 3.0, 2.0], device=dev)
    w = torch.zeros(64, 32, device=dev)
    w[0, :4] = torch.tensor([1.0, 1.0, 1.0, 1.0])
    w[1, :4] = torch.tensor([2.0, 1.0, 2.0, 1.0])
    b = torch.zeros(64, device=dev)
    b[0], b[1] = 3.0, -2.0
    out = torch.empty(2 * M + TAIL, device=dev)
    out[-TAIL - 2:].fill_(NAN)
    _lib.check(_lib_().asyrp_fid_conv(_p(x), _p(w), _p(b), _p(out), 1, 1, 1, 4, 64, 1, 1, 1, 0, 2 ** 30 - 1, 2, 2,
                                      _st()), "asyrp_fid_conv")
    torch.cuda.synchronize()
    rows = out[:2 * M].view(M, 2)
    hit = 2 ** 30 - 1
    assert rows[hit].tolist() == [3.0 + 4.0, -2.0 + 8.0]
    rest = torch.tensor([3.0, 0.0], device=dev)
    step = 1 << 27
    for a in range(0, M, step):
        chunk = rows[a:min(M, a + step)]
        ok = (chunk == rest).all(1)
        if a <= hit < a + step:
            ok[hit - a] = True
        assert ok.all(), f"pixels {a} .. {a + len(chunk) - 1}: {int((~ok).sum())} differ"
    assert _untouched(out[2 * M:]), "written past the output"
    _record("conv", 0.0)
    del out, rows
    _release()


def test_conv_input_past_2_to_the_31_elements(cuda_device):
    """in [2][8192][8192][20] (2.7e9 floats): a 3 x 3 / 8191 conv with padding 1 reads the windows at the four corners
    of each sample, the last at the last pixel of the last sample; small integers in those windows, zeros elsewhere,
    exact"""
    N, H, Cin = 2, 8192, 20
    n = N * H * H * Cin
    assert n > 2 ** 31
    _need_memory(4 * n + (1 << 20), "the conv input past 2^31 elements")
    dev = cuda_device
    g = _g(31)
    x = torch.zeros(N, H, H, Cin, device=dev)
    corner = torch.randint(-3, 4, (N, 2, 2, 2, 2, Cin), generator=g).float()  # sample, corner y, x, window y, x
    for cy in range(2):
        for cx in range(2):
            ys = slice(0, 2) if cy == 0 else slice(H - 2, H)
            xs = slice(0, 2) if cx == 0 else slice(H - 2, H)
            x[:, ys, xs] = corner[:, cy, cx].to(dev)
    w = torch.randint(-2, 3, (64, Cin, 3, 3), generator=g).float()
    b = torch.randint(-6, 7, (64,), generator=g).float()
    out = _nan(N * 2 * 2 * 64 + TAIL, dev)
    wd, bd = ops.pack_lpips_conv_weight(w).to(dev), b.to(dev)  # held until the launch has run
    _lib.check(_lib_().asyrp_fid_conv(_p(x), _p(wd), _p(bd), _p(out), N, H, H, Cin, 64, 3, 3, H - 1, 1, 1, 64, 64,
                                      _st()), "asyrp_fid_conv")
    torch.cuda.synchronize()
    # the same windows on a small image: the corners of a 4 x 4 image with padding 1 and stride 3
    small = torch.zeros(N, 4, 4, Cin)
    for cy in range(2):
        for cx in range(2):
            small[:, 2 * cy:2 * cy + 2, 2 * cx:2 * cx + 2] = corner[:, cy, cx]
    ref = _conv_ref(small, w, b, 3, 1, 1)
    assert ref.shape == (N, 2, 2, 64)
    got = out[:N * 256].view(N, 2, 2, 64)
    alone = torch.empty(N, 2, 2, 64, device=dev)
    ops.fid_conv(small.to(dev), wd, bd, alone, 3, 3, 3, (1, 1))
    _exact("conv", alone.double().cpu(), ref, "the windows on a 4 x 4 image")
    _exact("conv", got.double().cpu(), ref, "input past 2^31 elements")
    assert _untouched(out[N * 256:])
    del x, out
    _release()


# ------------------------------------------------------------------------------------------------------------------
# pack
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("u8", [False, True], ids=["fp32", "u8"])
@pytest.mark.parametrize("B,H,W,S", [(3, 1, 1, 1), (3, 37, 45, 1), (2, 1000, 3, 2), (2, 3, 1000, 2), (2, 2, 2, 2),
                                     (8, 37, 41, 299)])
def test_pack_sizes(cuda_device, u8, B, H, W, S):
    """S = 1 and 2 (down- and upsampling), and B S^2 = 715,208 above the grid cap (132 SMs x 16 x 256 = 540,672
    threads): the grid-stride loop runs twice.  fp32 and u8 of the same u8 values give the same bits."""
    if B * S * S > 132 * 16 * 256:
        props = torch.cuda.get_device_properties(cuda_device)
        assert B * S * S > props.multi_processor_count * 16 * 256
    call, _, check = _pack(cuda_device, B=B, H=H, W=W, S=S, u8=u8)
    _lib.check(call(), "asyrp_fid_pack")
    torch.cuda.synchronize()
    check()
    if u8:
        x = torch.randint(0, 256, (B, H, W, 3), generator=_g(5), dtype=torch.uint8).to(cuda_device)
        a, b = torch.empty(B, S, S, 4, device=cuda_device), torch.empty(B, S, S, 4, device=cuda_device)
        ops.fid_pack_u8(x, a)
        ops.fid_pack((x.cpu().permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous().to(cuda_device), b)
        assert torch.equal(a, b)


def _pm1(B, dev):
    """the per-sample values +-1 of each channel (clamped by the quantiser to q = 0 or 255: pixel values 0 and 1,
    which the blend keeps exactly)"""
    n, c = torch.arange(B, device=dev).view(B, 1), torch.arange(3, device=dev).view(1, 3)
    return ((n * 5 + c * 3) % 7 < 3).float() * 2 - 1


def test_pack_output_past_2_to_the_31_elements(cuda_device):
    """6007 samples of 299^2 x 4 floats (2^31 + 2.5 M, 8.6 GB) from 4 x 4 images: each sampled image equals the same
    image packed alone"""
    B, S = 6007, 299
    assert B * S * S * 4 > 2 ** 31
    _need_memory(B * S * S * 16, "pack past 2^31 elements")
    dev = cuda_device
    x = (torch.rand(B, 3, 4, 4, generator=_g(9)) * 2.4 - 1.2).to(dev)
    n = B * S * S * 4
    full = torch.empty(n + TAIL, device=dev)
    full[n:].fill_(NAN)
    out = full[:n].view(B, S, S, 4)
    ops.fid_pack(x, out)
    one = torch.empty(1, S, S, 4, device=dev)
    torch.cuda.synchronize()
    for s in _samples(B, 97):
        ops.fid_pack(x[s:s + 1], one)
        assert torch.equal(out[s], one[0]), f"sample {s} of {B}"
    assert _untouched(full[n:]), "written past the output"
    _record("pack", 0.0)
    del full, out
    _release()


@pytest.mark.parametrize("u8", [False, True], ids=["fp32", "u8"])
def test_pack_input_past_2_to_the_31_elements(cuda_device, u8):
    """3 images of 16384^2 (fp32 NCHW: 2.4e9 floats; u8 NHWC: 2.4e9 bytes) to 64 x 64: samples 0 and 1 uniform
    (+-1: exact values), sample 2 random, its last pixels past element 2^31; each sample equals itself packed alone"""
    B, H, S = 3, 16384, 64
    n = B * 3 * H * H
    assert n > 2 ** 31
    _need_memory(n * (1 if u8 else 4) + (1 << 20), "pack input past 2^31 elements")
    dev = cuda_device
    pm = _pm1(B, dev)
    if u8:
        x = torch.empty(B, H, H, 3, dtype=torch.uint8, device=dev)
        for s in range(B - 1):
            x[s] = ((pm[s] + 1) * 127.5).to(torch.uint8)
        x[B - 1].random_(0, 256)
    else:
        x = torch.empty(B, 3, H, H, device=dev)
        for s in range(B - 1):
            x[s] = pm[s].view(3, 1, 1)
        x[B - 1].uniform_(-1.2, 1.2)
    out, one = torch.empty(B, S, S, 4, device=dev), torch.empty(1, S, S, 4, device=dev)
    pack = ops.fid_pack_u8 if u8 else ops.fid_pack
    pack(x, out)
    torch.cuda.synchronize()
    for s in range(B):
        pack(x[s:s + 1], one)
        assert torch.equal(out[s], one[0]), f"sample {s}"
        if s < B - 1:
            want = torch.cat([pm[s], torch.zeros(1, device=dev)])
            assert torch.equal(out[s], want.expand(S, S, 4)), f"sample {s}"
    _record("pack", 0.0)
    del x, out
    _release()


# ------------------------------------------------------------------------------------------------------------------
# pool
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("H", [1, 2, 3, 4])
def test_pool_smallest_maps(cuda_device, mode, H):
    """every W in 1..4 (mode 0 from 3), C = 4 at channel 4 of rows of 12 floats (NaN on both sides)"""
    for W in range(1, 5):
        if mode == 0 and min(H, W) < 3:
            continue
        call, _, check = _pool(cuda_device, N=3, H=H, W=W, C=4, mode=mode, c0=4, ldo=12)
        _lib.check(call(), "asyrp_fid_pool")
        torch.cuda.synchronize()
        check()


def test_pool_input_past_2_to_the_31_elements(cuda_device):
    """129 samples of 128^2 x 1024 floats (2^31 + 16.8 M) through each mode, exact against torch on the first
    sample, the last and every 16th"""
    N, H, C = 129, 128, 1024
    n = N * H * H * C
    assert n > 2 ** 31
    _need_memory(8 * n + (1 << 20), "the pools past 2^31 elements")
    dev = cuda_device
    x = torch.empty(N, H, H, C, device=dev).normal_(generator=torch.Generator(dev).manual_seed(4))
    out = torch.empty(n + TAIL, device=dev)
    for mode in range(3):
        Ho = (H - 3) // 2 + 1 if mode == 0 else H
        m = N * Ho * Ho * C
        out[m:m + TAIL].fill_(NAN)
        ops.fid_pool(x, out[:m].view(N, Ho, Ho, C), mode)
        torch.cuda.synchronize()
        o = out[:m].view(N, Ho, Ho, C)
        for s in _samples(N, 16):
            ref = _pool_ref(x[s:s + 1].permute(0, 3, 1, 2).contiguous(), mode).permute(0, 2, 3, 1)
            _exact("pool", o[s:s + 1], ref, f"mode {mode} sample {s}")
        assert _untouched(out[m:m + TAIL])
    del x, out
    _release()


# ------------------------------------------------------------------------------------------------------------------
# mean
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,HW,C", [(3, 1, 1), (3, 1, 3), (2, 64, 1), (2, 64, 3), (2, 100003, 1), (2, 100003, 3),
                                    (600, 3, 1024)])
def test_mean_bit_for_bit(cuda_device, N, HW, C):
    """against numpy fp32: the sum in pixel order from 0, one divide; N C = 614,400 above the grid cap"""
    call, _, check = _mean(cuda_device, N=N, HW=HW, C=C)
    _lib.check(call(), "asyrp_fid_mean")
    torch.cuda.synchronize()
    check()


def test_mean_input_past_2_to_the_31_elements(cuda_device):
    """[2][2^20 + 1][1024] (2^31 + 2048 floats) of integers in [-7, 7]: every fp32 partial sum is an exact integer
    below 2^24, so each mean is fl(S / HW) of the exact sum"""
    N, HW, C = 2, 2 ** 20 + 1, 1024
    assert N * HW * C > 2 ** 31
    _need_memory(4 * N * HW * C + (1 << 20), "the mean past 2^31 elements")
    dev = cuda_device
    x = torch.empty(N, HW, C, device=dev).random_(0, 15, generator=torch.Generator(dev).manual_seed(6)).sub_(7)
    out = _nan(N * C + TAIL, dev)
    _lib.check(_lib_().asyrp_fid_mean(_p(x), _p(out), N, HW, C, _st()), "asyrp_fid_mean")
    torch.cuda.synchronize()
    for s in range(N):
        S = torch.zeros(C, dtype=torch.float64, device=dev)
        for a in range(0, HW, 1 << 16):
            S += x[s, a:a + (1 << 16)].double().sum(0)
        assert S.abs().max().item() < 2 ** 24
        want = torch.from_numpy(S.float().cpu().numpy() / np.float32(HW))  # one correctly rounded fp32 divide
        _exact("mean", out[s * C:(s + 1) * C].cpu(), want, f"sample {s}")
    assert _untouched(out[N * C:])
    del x
    _release()


# ------------------------------------------------------------------------------------------------------------------
# moments
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,d", [(2, 64), (2, 192), (17, 64), (4097, 128), (1000, 2048)])
def test_moments_exact_on_integer_features(cuda_device, n, d):
    """n = 2, n = 1 (mod 16) and d = 64: integer column means, every centred product and sum an exact integer"""
    call, _, check = _moments(cuda_device, n=n, d=d)
    _lib.check(call(), "asyrp_fid_moments")
    torch.cuda.synchronize()
    check()


@pytest.mark.parametrize("n,d", [(2, 64), (33, 192), (4097, 64)])
def test_moments_within_1e_12(cuda_device, n, d):
    g = np.random.default_rng(n + d)
    f = (g.standard_normal((n, d)) * g.uniform(0.1, 3, d) + g.uniform(0, 2, d)).astype(np.float32)
    mu, sigma = ops.fid_moments(torch.from_numpy(f).to(cuda_device))
    rmu, rs = ofid.moments(f)
    rs = np.atleast_2d(rs)
    _within("moments", np.abs(mu.cpu().numpy() - rmu).max(), 1e-12 * np.abs(rmu).max(), "mu")
    _within("moments", np.abs(sigma.cpu().numpy() - rs).max(), 1e-12 * np.abs(rs).max(), "sigma")


def test_moments_rows_past_2_to_the_31_elements(cuda_device):
    """n = 2^20, d = 2112 (2^31 + 67 M floats): a background of rows +-1 (alternating, column sums 0) with three pairs
    of planted integer rows v, -v (one even and one odd row each, so the sums stay 0), two of them past element 2^31:
    mu = 0 and S = (n - 6) J + sum of the planted rows' outer products, exactly"""
    n, d = 2 ** 20, 2112
    assert n * d > 2 ** 31 and 1016801 * d > 2 ** 31
    _need_memory(4 * n * d + 9 * d * d + (1 << 20), "the moments past 2^31 elements")
    dev = cuda_device
    x = ((torch.arange(n, device=dev) % 2) * 2 - 1).float().view(n, 1).expand(n, d).contiguous()
    g = _g(12)
    pairs = [(4, 1016803), (1016802, n - 1), (n - 2, 7)]
    planted = {}
    for a, b in pairs:
        v = torch.randint(-9, 10, (d,), generator=g)
        planted[a], planted[b] = v, -v
    for r, v in planted.items():
        x[r] = v.float().to(dev)
    mu, sigma = _nan(d + TAIL, dev, torch.float64), _nan(d * d + TAIL, dev, torch.float64)
    _lib.check(_lib_().asyrp_fid_moments(_p(x), _p(mu), _p(sigma), n, d, _st()), "asyrp_fid_moments")
    torch.cuda.synchronize()
    del x
    P = torch.stack(list(planted.values())).double()
    S = (n - len(planted)) + P.t() @ P
    _exact("moments", mu[:d].cpu(), torch.zeros(d, dtype=torch.float64), "mu")
    _exact("moments", sigma[:d * d].view(d, d).cpu(), S / (n - 1), "sigma")
    assert _untouched(mu[d:]) and _untouched(sigma[d * d:])
    _release()


# ------------------------------------------------------------------------------------------------------------------
# kernel sums
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,m,d,excl", [(130, 200, 16, 1), (200, 130, 64, 1), (65, 64, 16, 0), (1, 3, 16, 1),
                                        (65535 * 64, 1, 16, 0), (65535 * 64, 1, 16, 1), (3, 65535 * 64, 16, 1)])
def test_kernel_sum_exact_on_integer_features(cuda_device, n, m, d, excl):
    """features in {-1, 0, 1} and d a power of two: every term is an exact dyadic and every sum exact below 2^53;
    exclude_diag with n != m; n = 65535 * 64, the most rows admitted"""
    call, _, check = _ksum(cuda_device, n=n, m=m, d=d, excl=excl)
    _lib.check(call(), "asyrp_fid_kernel_sum")
    torch.cuda.synchronize()
    check()


@pytest.mark.parametrize("excl", [0, 1])
def test_kernel_sum_rows_past_2_to_the_31_elements(cuda_device, excl):
    """x [2^20 + 1][2048] (2^31 + 2048 floats) of zeros but for 64 planted rows (among them row 0, for the diagonal,
    and the last rows, past element 2^31) with +-16 in 32 features; y [64][2048] of +-16 everywhere: every dot is
    256 c, c an integer, so every term is (8 + c)^3 / 512 and the sum exact"""
    n, m, d = 2 ** 20 + 1, 64, 2048
    assert (n - 1) * d >= 2 ** 31
    _need_memory(4 * n * d + (1 << 24), "the kernel sum past 2^31 elements")
    dev = cuda_device
    g = _g(21 + excl)
    rows = torch.cat([torch.tensor([0, 1, n - 2, n - 1]), torch.randint(2, n - 2, (60,), generator=g)]).unique()
    P = torch.zeros(len(rows), d, dtype=torch.int64)
    for i in range(len(rows)):
        P[i, torch.randperm(d, generator=g)[:32]] = torch.randint(0, 2, (32,), generator=g) * 2 - 1
    Y = torch.randint(0, 2, (m, d), generator=g) * 2 - 1
    x = torch.zeros(n, d, device=dev)
    x[rows.to(dev)] = (16 * P).float().to(dev)
    y = (16 * Y).float().to(dev)
    count = _lib_().asyrp_fid_kernel_sum_partials(n, m)
    part, out = _nan(count + TAIL, dev, torch.float64), _nan(1 + TAIL, dev, torch.float64)
    _lib.check(_lib_().asyrp_fid_kernel_sum(_p(x), _p(y), _p(part), _p(out), n, m, d, excl, _st()),
               "asyrp_fid_kernel_sum")
    torch.cuda.synchronize()
    del x
    c = P @ Y.t()  # [planted][m]: dot / 256
    num = (8 + c) ** 3
    if excl:
        num[rows.view(-1, 1) == torch.arange(m).view(1, -1)] = 0
    # every pair of a zero row has dot 0, term 1 = 512 / 512; the diagonal pairs i == j < m are dropped with excl
    zero_pairs = (n - len(rows)) * m - (excl * (m - int((rows < m).sum())))
    want = (num.sum().item() + 512 * zero_pairs) / 512
    _exact("kernel_sum", out[:1].cpu(), torch.tensor([want], dtype=torch.float64), f"excl={excl}")
    assert _untouched(part[count:]) and _untouched(out[1:])
    _release()


@pytest.mark.parametrize("excl", [0, 1])
def test_kernel_sum_subsets_most_subsets(cuda_device, excl):
    """65535 subsets (the most admitted) of 2 rows, and 3 subsets of 130 rows, exact per subset"""
    for s, subsets in ((2, 65535), (130, 3)):
        call, _, check = _subsets(cuda_device, n=300, m=257, s=s, subsets=subsets, d=32, excl=excl)
        _lib.check(call(), "asyrp_fid_kernel_sum_subsets")
        torch.cuda.synchronize()
        check()


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    """the file's wall time, peak device memory and worst err / bound per kernel, printed at the end (pytest -s)"""
    t0 = time.perf_counter()
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated() / GiB if torch.cuda.is_available() else 0.0
    worst = ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items()))
    print(f"\ntest_fid_kernel_limits_gpu: {time.perf_counter() - t0:.1f} s, peak device memory {peak:.2f} GiB; "
          f"worst err / bound: {worst}")
