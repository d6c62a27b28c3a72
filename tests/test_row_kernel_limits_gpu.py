"""The per-row sampler kernels (asyrp_ddim_update_rows, asyrp_slerp_h_rows in csrc/pointwise.cu) at the limits their
entry points admit.

  * Every ASYRP_REQUIRE has a row in REFUSALS: c12 NULL; C odd, stats_tiles = 0 and t_rows NULL.  The refused call
    (through the C ABI) raises AsyrpError naming the entry point and leaves its NaN-filled outputs untouched; the
    nearest accepted neighbour launches and is checked.  No REQUIRE is untabled.
  * ddim_update_rows with Ce = 6 (the learned-sigma stride of et / em), with and without x0_out, equals an fp32 CPU
    restatement of its explicitly rounded operations bit for bit.  With z == NULL no row adds noise, even a row whose
    c1 is non-zero: the scalar kernel's use_z = 0.  The engine must therefore pass z whenever any row is stochastic.
  * slerp_h_rows at C = 2, at H W C not a multiple of the 256 threads, with 5 GroupNorm tile slots (slots 1-4 zeroed
    from NaN), with a t = 0 row (h2 == h bit for bit, and its statistics equal to an fp32 restatement of the kernel's
    sums), and with use_mask where the mask is a single row (H = 6) or a single column (W = 4).  Where the mask is
    empty (H <= 5 or W <= 3) the kernel keeps h and its statistics, while the reference's slerp of two zero vectors
    would give NaN; that is pinned here, and no shipped model reaches it: every bottleneck is 8 x 8.

Bounds are first order with u = 2^-24: h2 is fp16, so |h2 - v| <= 2^-11 |v| + 2^-25 plus the fp32 error of v, which
is the relative error of the three block sums ((ceil(H W C / 256) + 13) u: thread sums, the butterfly and the 8 warp
partials) carried through acos at |cos| <= 1/2 and the sines (a factor of at most 4 here), plus 16 u for the
elementwise operations, times |s0 a| + |s1 v1|.  The GroupNorm sums of a general row are held to the sum of those
bounds plus (2 H W + 8) u of their magnitudes.  Outputs sit in front of a NaN tail that must stay NaN.  The file takes
about 13 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit, most of it collection; every tensor is under 100 KiB.
"""
import math
import re

import pytest
import torch

from asyrp_official_b200 import _lib, ops

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
NAN = float("nan")
TAIL = 64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _p(t):
    return ops._ptr(t)


def _buf(shape, dev, dtype=torch.float32):
    """(whole buffer, front view of `shape`): the buffer holds TAIL more elements, all NaN"""
    n = math.prod(shape)
    full = torch.full((n + TAIL,), NAN, dtype=dtype, device=dev)
    return full, full[:n].view(shape)


def _tail_ok(full, n):
    assert torch.isnan(full[n:]).all(), "written past the output"
    assert not torch.isnan(full[:n]).any(), "output not written"


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def _ddim_rows_ref(x, et, em, z, at, an, c12):
    """ddim_update_rows_kernel in fp32 on the CPU, one rounding per operation as its __f*_rn intrinsics"""
    f = torch.float32
    at, an = torch.tensor(at, dtype=f), torch.tensor(an, dtype=f)
    sq1, sqa, sqn = torch.sqrt(1 - at), torch.sqrt(at), torch.sqrt(an)
    Cx = x.shape[1]
    e, m = et[:, :Cx].cpu(), em[:, :Cx].cpu()
    x0 = (x.cpu() - m * sq1) / sqa
    c1, c2 = c12[:, 0].cpu().view(-1, 1, 1, 1), c12[:, 1].cpu().view(-1, 1, 1, 1)
    nx = sqn * x0 + c2 * e
    if z is not None:
        nx = torch.where(c1 != 0, nx + c1 * z.cpu(), nx)
    return nx, x0


def _mask(H, W):
    y = torch.arange(H).view(H, 1)
    x = torch.arange(W).view(1, W)
    return (y >= 4) & (y < H - 1) & (x >= 3) & (x < 5)


def _slerp_ref(h, dh, t, use_mask):
    """one sample in fp64: h [H][W][C] (fp16 values), dh [C][H][W] -> (v [H][W][C], error scale |s0 a| + |s1 v1|)"""
    H, W, C = h.shape
    a = h.double().cpu()
    b = dh.double().cpu().permute(1, 2, 0)
    m = _mask(H, W).view(H, W, 1).double() if use_mask else torch.ones(H, W, 1, dtype=torch.float64)
    am, bm = a * m, b * m
    nh, nd = am.norm(), bm.norm()
    cos = (am * bm).sum() / (nh * nd)
    assert abs(cos) <= 0.5, "the bound assumes |cos| <= 1/2"
    th0 = torch.arccos(cos)
    s0, s1 = torch.sin(th0 - th0 * t) / torch.sin(th0), torch.sin(th0 * t) / torch.sin(th0)
    v1 = b * (1.0 if use_mask else nh / nd)
    v = torch.where(m > 0, s0 * a + s1 * v1, a)
    scale = torch.where(m > 0, (s0 * a).abs() + (s1 * v1).abs(), torch.zeros_like(a))
    return v, scale


def _stats_seq(v):
    """the kernel's GroupNorm sums in fp32: per channel pair, pixels in order, the pair's two channels in order"""
    H, W, C = v.shape
    v = v.float().reshape(H * W, C // 2, 2)
    s = torch.zeros(C // 2)
    ss = torch.zeros(C // 2)
    for pix in range(H * W):
        for k in range(2):
            s = s + v[pix, :, k]
            ss = ss + v[pix, :, k] * v[pix, :, k]  # exact for fp16 values: fused or not, one rounding
    return torch.stack([s, ss], -1)


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def _ddim(dev, c12=True, Ce=3):
    g = _g(1)
    x, z = torch.randn(2, 3, 4, 4, generator=g).to(dev), torch.randn(2, 3, 4, 4, generator=g).to(dev)
    et, em = torch.randn(2, Ce, 4, 4, generator=g).to(dev), torch.randn(2, Ce, 4, 4, generator=g).to(dev)
    cc = torch.tensor([[0.0, 0.3], [0.2, 0.5]], device=dev)
    full, out = _buf((2, 3, 4, 4), dev)

    def check():
        _tail_ok(full, out.numel())
        assert torch.equal(out.cpu(), _ddim_rows_ref(x, et, em, z, 0.5, 0.6, cc)[0])
    return (lambda: _lib.load().asyrp_ddim_update_rows(_p(x), _p(et), _p(em), _p(z), _p(out), None, 2, 3, Ce, 16, 0.5,
                                                       0.6, _p(cc) if c12 else None, ops._stream()), [full], check)


def _slerp(dev, C=8, tiles=1, t_rows=True):
    g = _g(2)
    Cp = C + C % 2
    h = torch.randn(2, 4, 4, Cp, generator=g).half().to(dev)
    dh = torch.randn(2, Cp, 4, 4, generator=g).to(dev)
    tr = torch.tensor([0.0, 0.4], device=dev)
    hfull, h2 = _buf((2, 4, 4, Cp), dev, torch.float16)
    sfull, st = _buf((2, max(tiles, 1), Cp // 2, 2), dev)

    def check():
        _tail_ok(hfull, h2.numel())
        _tail_ok(sfull, st.numel())
        assert torch.equal(h2[0], h[0])
        v, scale = _slerp_ref(h[1], dh[1], 0.4, False)
        bound = 2.0 ** -11 * v.abs() + 2.0 ** -25 + 4 * (math.ceil(16 * C / 256) + 29) * U * scale
        assert ((h2[1].double().cpu() - v).abs() <= bound).all()
    return (lambda: _lib.load().asyrp_slerp_h_rows(_p(h), _p(dh), dh.stride(0), _p(h2), _p(st), tiles, 2, C, 4, 4,
                                                   _p(tr) if t_rows else None, 0, ops._stream()), [hfull, sfull],
            check)


# (row, entry point, message fragment, refused call, accepted call)
REFUSALS = [
    ("ddim_rows_c12_null", "asyrp_ddim_update_rows", "c12 is NULL", lambda d: _ddim(d, c12=False),
     lambda d: _ddim(d)),
    ("slerp_rows_odd_c", "asyrp_slerp_h_rows", "bad arguments", lambda d: _slerp(d, C=7), lambda d: _slerp(d, C=8)),
    ("slerp_rows_no_tiles", "asyrp_slerp_h_rows", "bad arguments", lambda d: _slerp(d, tiles=0),
     lambda d: _slerp(d, tiles=1)),
    ("slerp_rows_t_rows_null", "asyrp_slerp_h_rows", "t_rows is NULL", lambda d: _slerp(d, t_rows=False),
     lambda d: _slerp(d)),
]


@pytest.mark.parametrize("row", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_entry_point_refusals(cuda_device, row):
    name, entry, fragment, bad, good = row
    call, outs, _ = bad(cuda_device)
    torch.cuda.synchronize()
    with pytest.raises(_lib.AsyrpError, match=f"{re.escape(entry)}: .*{re.escape(fragment)}") as exc:
        _lib.check(call(), entry)
    assert f"{entry}: " in str(exc.value)
    torch.cuda.synchronize()
    for o in outs:
        assert torch.isnan(o).all(), f"{name}: the refused call wrote its output"
    call, outs, check = good(cuda_device)
    _lib.check(call(), entry)
    torch.cuda.synchronize()
    check()


# ------------------------------------------------------------------------------------------------------------------
# ddim_update_rows
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_x0", [False, True])
def test_ddim_rows_learned_sigma_stride(cuda_device, with_x0):
    """Ce = 6: epsilon is channels 0..2 of a 6-channel et / em; rows with eta = 0 (c1 = 0) and eta = 1, exact"""
    dev = cuda_device
    g = _g(10 + with_x0)
    N, S = 5, 13
    x = torch.randn(N, 3, S, S, generator=g).to(dev)
    et, em = torch.randn(N, 6, S, S, generator=g).to(dev), torch.randn(N, 6, S, S, generator=g).to(dev)
    et[:, 3:] = em[:, 3:] = NAN  # the variance channels are never read
    z = torch.randn(N, 3, S, S, generator=g).to(dev)
    c12 = torch.tensor([[0.0, 0.7], [0.31, 0.52], [0.0, 0.9], [0.05, 0.6], [0.4, 0.1]], device=dev)
    full, out = _buf((N, 3, S, S), dev)
    x0full, x0 = _buf((N, 3, S, S), dev) if with_x0 else (None, None)
    ops.ddim_update_rows(x, et, em, z, out, x0, 0.42, 0.61, c12)
    torch.cuda.synchronize()
    _tail_ok(full, out.numel())
    want, want_x0 = _ddim_rows_ref(x, et, em, z, 0.42, 0.61, c12)
    assert torch.equal(out.cpu(), want)
    if with_x0:
        _tail_ok(x0full, x0.numel())
        assert torch.equal(x0.cpu(), want_x0)


def test_ddim_rows_without_z_add_no_noise(cuda_device):
    """z == NULL: every row is the deterministic update, also where c1 != 0 (the scalar kernel with use_z = 0)"""
    dev = cuda_device
    g = _g(20)
    N, S = 4, 9
    x = torch.randn(N, 3, S, S, generator=g).to(dev)
    et, em = torch.randn(N, 3, S, S, generator=g).to(dev), torch.randn(N, 3, S, S, generator=g).to(dev)
    c12 = torch.tensor([[0.3, 0.5], [0.0, 0.5], [0.7, 0.2], [1.0, 0.0]], device=dev)
    full, out = _buf((N, 3, S, S), dev)
    ops.ddim_update_rows(x, et, em, None, out, None, 0.42, 0.61, c12)
    torch.cuda.synchronize()
    _tail_ok(full, out.numel())
    assert torch.equal(out.cpu(), _ddim_rows_ref(x, et, em, None, 0.42, 0.61, c12)[0])
    one = torch.empty_like(out)
    no_c1 = c12.clone()
    no_c1[:, 0] = 0
    ops.ddim_update_rows(x, et, em, None, one, None, 0.42, 0.61, no_c1)
    assert torch.equal(one, out), "c1 must not matter without z"


# ------------------------------------------------------------------------------------------------------------------
# slerp_h_rows
# ------------------------------------------------------------------------------------------------------------------
# (N, H, W, C, stats tiles, use_mask): C = 2; H W C = 294 and 1890, not multiples of 256; five tile slots; the mask a
# single row (H = 6) and a single column (W = 4); empty masks (H = 5, W = 3)
SLERP_CASES = {
    "c2": (3, 8, 8, 2, 1, False),
    "hwc_294": (3, 7, 7, 6, 1, False),
    "hwc_1890_5_tiles": (3, 9, 7, 30, 5, False),
    "mask_one_row": (3, 6, 8, 16, 2, True),
    "mask_one_column": (3, 8, 4, 16, 1, True),
    "mask_empty_h5": (2, 5, 8, 8, 1, True),
    "mask_empty_w3": (2, 8, 3, 8, 1, True),
}


@pytest.mark.parametrize("case", list(SLERP_CASES))
def test_slerp_rows_edges(cuda_device, case):
    """row 0 has t = 0 (h2 == h and the statistics of h, bit for bit); the other rows against fp64"""
    N, H, W, C, T, use_mask = SLERP_CASES[case]
    dev = cuda_device
    g = _g(H * 100 + W * 10 + C)
    empty = use_mask and not _mask(H, W).any()
    h = (torch.randn(N, H, W, C, generator=g) * 3).half()
    dh = torch.randn(N, C, H, W, generator=g)
    t = torch.tensor([0.0] + [0.1 + 0.8 * i / max(1, N - 1) for i in range(1, N)], dtype=torch.float32)
    hfull, h2 = _buf((N, H, W, C), dev, torch.float16)
    sfull, st = _buf((N, T, C // 2, 2), dev)
    ops.slerp_h_rows(h.to(dev), dh.to(dev), h2, st, t.to(dev), use_mask)
    torch.cuda.synchronize()
    _tail_ok(hfull, h2.numel())
    _tail_ok(sfull, st.numel())
    assert torch.equal(st[:, 1:], torch.zeros_like(st[:, 1:])), "tile slots past 0 not zeroed"
    h2c, stc = h2.cpu(), st.cpu()
    for n in range(N):
        if n == 0 or empty:
            assert torch.equal(h2c[n].view(torch.int16), h[n].view(torch.int16)), f"{case} row {n}: h not kept"
            assert torch.equal(stc[n, 0], _stats_seq(h[n])), f"{case} row {n}: statistics"
            continue
        v, scale = _slerp_ref(h[n], dh[n], float(t[n]), use_mask)
        k = 4 * (math.ceil(H * W * C / 256) + 29) * U
        bound = 2.0 ** -11 * v.abs() + 2.0 ** -25 + k * scale
        err = (h2c[n].double() - v).abs()
        assert (err <= bound).all(), f"{case} row {n}: {(err / bound).max().item():.3g}x the bound"
        if use_mask:
            out_of_mask = ~_mask(H, W)
            assert torch.equal(h2c[n][out_of_mask], h[n][out_of_mask]), "h changed outside the mask"
        vv = v.reshape(H * W, C // 2, 2)
        kv = (k * scale).reshape(H * W, C // 2, 2)
        want = torch.stack([vv.sum((0, 2)), (vv * vv).sum((0, 2))], -1)
        sbound = torch.stack([kv.sum((0, 2)), (2 * vv.abs() * kv + kv * kv).sum((0, 2))], -1) + \
            (2 * H * W + 8) * U * torch.stack([vv.abs().sum((0, 2)), (vv * vv).sum((0, 2))], -1)
        assert ((stc[n, 0].double() - want).abs() <= sbound).all(), f"{case} row {n}: statistics"
