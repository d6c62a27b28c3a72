"""The fp32 scoring kernels of the LPIPS, CLIP and ArcFace paths at the limits their entry points admit: the largest
admitted shape runs and matches fp64, one step past it raises AsyrpError without launching, and the row kernels run at
widths of 1, 33 and 1000 and at row counts that are not a multiple of their 8 rows per CTA.

Bounds are first-order fp32 error bounds of each kernel's summation order, u = 2^-24: a sequential lane sum of m
terms plus a 5-level butterfly costs at most (m + 5) u of the sum of the magnitudes, and each further operation one u.
Outputs sit at the front of buffers with a NaN tail that must stay NaN.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, ops
from oracle import clip_text as oct

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
NAN = float("nan")
WIDTHS = [1, 33, 1000]
ROWS = 13  # not a multiple of the 8 rows (warps) of a CTA


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _out(shape, dev):
    buf = torch.full((shape[0] + 1, *shape[1:]), NAN, device=dev)
    return buf, buf[:shape[0]]


def _tail_ok(buf, n):
    assert torch.isnan(buf[n:]).all() and torch.isfinite(buf[:n]).all()


# ---- CLIP direction -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups,n,dim", [(2, 1, 12286), (3, 4, 12280), (1, 2048, 8192)])
def test_direction_at_the_shared_memory_limit(cuda_device, groups, n, dim):
    """2n + dim = 12288, the documented limit: 48 KB of dynamic shared memory on top of the kernel's static array"""
    assert 2 * n + dim == 12288
    g = _g(n + dim)
    src, trg = torch.randn(groups * n, dim, generator=g), torch.randn(groups * n, dim, generator=g)
    obuf, out = _out((groups, dim), cuda_device)
    eps = 1e-7 if n == 1 else 0.0
    ops.clip_direction(src.to(cuda_device), trg.to(cuda_device), out, n, eps)
    _tail_ok(obuf, groups)
    s, t = src.double(), trg.double()
    th, sh = t / t.norm(dim=1, keepdim=True), s / s.norm(dim=1, keepdim=True)
    d = (th - sh).view(groups, n, dim).mean(1)
    dn = d.norm(dim=1, keepdim=True)
    ref = d / (dn + eps)
    # the column sums over n rows of two rounded quotients each, the row norms over dim / 32 terms per lane, |d| over
    # dim / 256 terms per thread
    mass = (th.abs() + sh.abs()).view(groups, n, dim).sum(1) / (n * dn)
    bound = (n + math.ceil(dim / 32) + 16) * U * (mass + ref.abs())
    err = (out.cpu().double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()


def test_direction_rejects_past_the_limit(cuda_device):
    src = torch.zeros(1, 12287, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="12288"):
        ops.clip_direction(src, src, torch.empty(1, 12287, device=cuda_device), 1, 0.0)


# ---- attention -------------------------------------------------------------------------------------------------------
def test_attention_rejects_past_the_token_limits(cuda_device):
    qkv = torch.zeros(1, 129, 3 * 64, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="T <= 128"):
        ops.clip_attention(qkv, torch.empty(1, 129, 64, device=cuda_device), 1)


def test_softmax_rows_rejects_more_than_1024_columns(cuda_device):
    S = torch.zeros(2, 1025, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="1024"):
        ops.softmax_rows(S, torch.empty(2, 1025, dtype=torch.float16, device=cuda_device), 1.0)


# ---- ArcFace SE gate -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [16, 512])
@pytest.mark.parametrize("HW", [1, 3136])
def test_se_scale_at_its_channel_limits(cuda_device, C, HW):
    g = _g(C + HW)
    N, Cr = 3, C // 16
    r = torch.randn(N, HW, C, generator=g) + torch.randn(1, 1, C, generator=g)
    fc1 = torch.randn(Cr, C, generator=g) / math.sqrt(C)
    fc2 = torch.randn(C, Cr, generator=g) / math.sqrt(Cr)
    gbuf, gate = _out((N, C), cuda_device)
    ops.arcface_se_scale(r.view(N, HW, 1, C).to(cuda_device), fc1.to(cuda_device), fc2.to(cuda_device), gate)
    _tail_ok(gbuf, N)
    rd = r.double()
    ref = torch.sigmoid(torch.relu(rd.mean(1) @ fc1.double().t()) @ fc2.double().t())
    # thread sums of HW / J pixels (J = 512 / C threads per channel), J partials, the fc1 row over C / 32 per lane,
    # the fc2 row over Cr; sigmoid' <= 1/4
    J = 512 // C
    A = (rd.abs().mean(1) @ fc1.double().abs().t()) @ fc2.double().abs().t()
    bound = 0.25 * (math.ceil(HW / J) + J + math.ceil(C / 32) + Cr + 16) * U * A + 4 * U
    err = (gate.cpu().double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()


def test_se_scale_rejects_a_channel_count_that_does_not_divide_512(cuda_device):
    res = torch.zeros(1, 2, 2, 48, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="dividing 512"):
        ops.arcface_se_scale(res, torch.zeros(3, 48, device=cuda_device), torch.zeros(48, 3, device=cuda_device),
                             torch.empty(1, 48, device=cuda_device))


# ---- LayerNorm, cosine, l2norm, dot ------------------------------------------------------------------------------
def _ln_input(rows, w, g):
    """rows of N(0, 1), and every third row offset so that |mean| / std = 1e3"""
    x = torch.randn(rows, w, generator=g)
    x[::3] = 1e3 + x[::3]
    return x


def _ln_bound(x, gamma, beta):
    """two-pass LayerNorm: the mean's error (a lane sum of ceil(w/32) terms and the butterfly) over the normaliser,
    and a few roundings of x_hat * gamma + beta"""
    xd = x.double()
    w = x.shape[-1]
    mean = xd.mean(-1, keepdim=True)
    sd = (xd.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    k = (math.ceil(w / 32) + 10) * U
    return k * ((xd.abs().mean(-1, keepdim=True) / sd + ((xd - mean) / sd).abs() + 1) * gamma.double().abs()
                + beta.double().abs())


@pytest.mark.parametrize("w", WIDTHS)
def test_layernorm_widths_and_a_large_mean(cuda_device, w):
    g = _g(w)
    x = _ln_input(ROWS, w, g)
    gam, bet = 1 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    obuf, out = _out((ROWS, w), cuda_device)
    ops.clip_layernorm(x.to(cuda_device), gam.to(cuda_device), bet.to(cuda_device), out)
    _tail_ok(obuf, ROWS)
    ref = oct.layer_norm(x.double(), gam.double(), bet.double())
    err = (out.cpu().double() - ref).abs()
    bound = _ln_bound(x, gam, bet)
    assert (err <= bound).all(), (err / bound).max().item()
    # rows read at a stride (ln_post of the class token)
    T = 3
    xr = torch.randn(ROWS, T, w, generator=g)
    xr[:, 0] = x
    pbuf, pooled = _out((ROWS, w), cuda_device)
    ops.clip_layernorm_rows(xr.to(cuda_device), gam.to(cuda_device), bet.to(cuda_device), pooled)
    _tail_ok(pbuf, ROWS)
    assert torch.equal(pooled, out)


@pytest.mark.parametrize("dim", WIDTHS)
def test_cosine_l2norm_and_dot_widths(cuda_device, dim):
    g = _g(100 + dim)
    a, b = torch.randn(ROWS, dim, generator=g), torch.randn(ROWS, dim, generator=g)
    b[1] = -2 * a[1]
    k = math.ceil(dim / 32)
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    cbuf, cos = _out((ROWS,), cuda_device)
    ops.clip_cosine(dev(a), dev(b), cos)
    _tail_ok(cbuf, ROWS)
    ref = torch.nn.CosineSimilarity(dim=1, eps=1e-6)(a.double(), b.double())
    assert ((cos.cpu().double() - ref).abs() <= (2 * k + 20) * U).all()
    assert cos[1].item() == pytest.approx(-1, abs=(2 * k + 20) * U)
    nbuf, nrm = _out((ROWS, dim), cuda_device)
    ops.arcface_l2norm(dev(a), nrm)
    _tail_ok(nbuf, ROWS)
    ref = a.double() / a.double().norm(dim=1, keepdim=True)
    assert ((nrm.cpu().double() - ref).abs() <= (k + 8) * U * ref.abs()).all()
    # id[j] = edited[j] . src[j % B] with n = 13 rows against B = 5
    B = 5
    ibuf, ids = _out((ROWS,), cuda_device)
    ops.arcface_dot(dev(a[:B]), dev(b), ids)
    _tail_ok(ibuf, ROWS)
    src = a.double()[torch.arange(ROWS) % B]
    ref = (b.double() * src).sum(1)
    assert ((ids.cpu().double() - ref).abs() <= (k + 6) * U * (b.double().abs() * src.abs()).sum(1)).all()


# ---- LPIPS distance and max pool -------------------------------------------------------------------------------------
def _lpips_term(probe, ref, lin_w):
    """fp64 layer term and its error scale: d[n] = mean_px sum_c w_c (p/(|p| + 1e-10) - r/(|r| + 1e-10))^2"""
    N, B = probe.shape[0], ref.shape[0]
    p = probe.double().flatten(1, 2)
    r = ref.double().flatten(1, 2)[torch.arange(N) % B]
    pn = p / (p.norm(dim=-1, keepdim=True) + 1e-10)
    rn = r / (r.norm(dim=-1, keepdim=True) + 1e-10)
    w = lin_w.double()
    return ((pn - rn) ** 2 * w).sum(-1).mean(-1), ((pn.abs() + rn.abs()) ** 2 * w.abs()).sum(-1).mean(-1)


@pytest.mark.parametrize("H,W", [(1, 1), (3, 11), (7, 151)])  # H*W = 1, 33, 32*33 + 1 (34 chunks)
def test_lpips_distance_chunks_batches_and_accumulation(cuda_device, H, W):
    g = _g(H * W)
    N, B = 7, 3
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    layers = []
    for C in (40, 64):
        probe, ref = torch.randn(N, H, W, C, generator=g), torch.randn(B, H, W, C, generator=g)
        probe[B:2 * B] = ref + 1e-3 * probe[B:2 * B]  # rows close to their reference
        layers.append((probe, ref, torch.rand(C, generator=g)))
    chunks = ops.lpips_distance_chunks(H * W)
    assert chunks == (H * W + 31) // 32
    partial = torch.full((N * chunks,), NAN, device=cuda_device)
    counters = torch.zeros(N + 1, dtype=torch.int32, device=cuda_device)
    dbuf, d = _out((N,), cuda_device)
    want, scale = torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64)
    for i, (probe, ref, lin_w) in enumerate(layers):
        ops.lpips_distance(dev(probe), dev(ref), dev(lin_w), partial, counters[:N], d, accumulate=i > 0)
        t, s = _lpips_term(probe, ref, lin_w)
        want, scale = want + t, scale + s
        # per pixel: the two norms, the lane sums over C / 32 and the butterflies, 4 pixels per warp in a chunk, the
        # 8 warps, the chunk sums over lanes, the mean; the second layer adds one rounding of d
        C = probe.shape[-1]
        bound = (math.ceil(C / 32) + math.ceil(chunks / 32) + 40) * U * scale
        err = (d.cpu().double() - want).abs()
        assert (err <= bound).all(), (i, (err / bound).max().item())
        assert torch.equal(counters.cpu(), torch.zeros(N + 1, dtype=torch.int32)), "counters not left at zero"
    _tail_ok(dbuf, N)


@pytest.mark.parametrize("H", [3, 4, 7])
def test_lpips_maxpool_small_maps(cuda_device, H):
    for W in (3, 4, 7):
        x = torch.randn(2, H, W, 8, generator=_g(H * W))
        Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
        obuf, out = _out((2, Ho, Wo, 8), cuda_device)
        ops.lpips_maxpool(x.to(cuda_device), out)
        _tail_ok(obuf, 2)
        ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
        assert torch.equal(out.cpu(), ref), (H, W)
