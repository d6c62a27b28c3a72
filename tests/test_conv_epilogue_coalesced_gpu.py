"""Exact-arithmetic test of the conv epilogue's indexing (tiles of 64 and 128 channels).

Activations, weights, bias, residual and scales are small integers or dyadic values, so every fp32 accumulator, every
output, every per-tile GroupNorm statistic and `sums_out` is exact in any summation order: the kernel's results are
compared with `==` against a float64 reference.  A wrong lane, row, channel slice, sample or statistics slot changes
a value by at least one unit of its resolution, which a relative tolerance could let through.

Each case asserts the tile instantiation it exercises and at least two waves of tiles (a persistent CTA reuses its
staging tile and statistics scratch across tiles), fills every output with NaN plus one guard sample behind it, and
checks that a second launch gives the same bits.  The convs are 1x1: the epilogue does not depend on how the
accumulators were formed, and the tile geometry (TW x TH pixels of NB samples) is that of a 1x1 conv of the shape.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

CIN = 64
# v = (acc + bias) * acc_scale + res_scale * res: acc and bias integers, scales in {1/4, 1/2, 1}, res integers (res_mode
# 2: their 2x2 average, multiples of 1/4), so v is a multiple of 1/8 with |v| <= 24: fp16 holds it exactly, and a
# tile's sum of squares (<= 256 rows) stays below 2^24 units of 1/64 — exact in fp32.
VMAX = 24.0

CASES = {
    # <128,1>: ragged x (W 40 in 16-wide tiles) and y (H 20 in 8-row tiles), per-sample bias and scales, residual,
    # stats + sums_out; 270 tiles
    "bn128_ragged_res0": dict(inst=(128, 1), N=30, H=20, W=40, Cout=128, ebias="sample", res=0, scales="sample",
                              stats=True, sums=True),
    # <128,1>, two channel tiles, nearest-x2 residual, shared bias, by-value scales; 272 tiles
    "bn128_res1": dict(inst=(128, 1), N=17, H=32, W=32, Cout=256, ebias="shared", res=1, scales="value", stats=True),
    # <64,2>: 2x2-average residual, per-sample bias and scales, stats + sums_out; 272 tiles
    "bn64x2_res2": dict(inst=(64, 2), N=17, H=64, W=64, Cout=64, ebias="sample", res=2, scales="sample", stats=True,
                        sums=True),
    # <64,1>: ragged x and y, residual, one device scale pair for every sample, stats without sums_out; 270 tiles
    "bn64_ragged_res0": dict(inst=(64, 1), N=45, H=20, W=24, Cout=64, ebias="shared", res=0, scales="pair",
                             stats=True),
    # tiles of two samples (8x8), N odd: the last tile's second sample is past N; per-sample bias rows and scales
    "nb2_res0": dict(inst=(64, 1), NB=2, N=265, H=8, W=8, Cout=128, ebias="sample", res=0, scales="sample", stats=True),
    # tiles of eight samples (4x4), N = 8*33+1, 2x2-average residual
    "nb8_res2": dict(inst=(64, 1), NB=8, N=265, H=4, W=4, Cout=512, ebias="shared", res=2, scales="value", stats=True),
    # fp32 output, per-sample bias; 264 tiles
    "bn128_f32": dict(inst=(128, 1), N=33, H=32, W=32, Cout=128, ebias="sample", out="f32"),
    # two heads: batch entry (n, h) writes channels [64h, 64h+64) of sample n; 272 tiles
    "bn64_heads2": dict(inst=(64, 1), N=136, H=16, W=16, Cout=64, heads=2, ebias="sample", scales="sample"),
}


def _tile_shape(H, W):
    """(TW, TH, NB) of a conv without a 3x3 stride-1 segment (csrc/conv_gemm.cu conv_tile_shape)"""
    tw = min(W, 128) if H == 1 else min(W, 16)
    th = 1 if H == 1 else min(128 // tw, 8, H)
    while 128 % (tw * th):
        th -= 1
    return tw, th, 128 // (tw * th)


def _ints(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _run(spec, dev, seed):
    from asyrp_official_b200 import ops
    g = torch.Generator().manual_seed(seed)
    N, H, W, Cout = spec["N"], spec["H"], spec["W"], spec["Cout"]
    heads = spec.get("heads", 1)
    BN, MT = spec["inst"]
    assert ops.conv_tile_config(H, W, Cout, False) == spec["inst"], ops.conv_tile_config(H, W, Cout, False)
    TW, TH, NB = _tile_shape(H, W)
    assert NB == spec.get("NB", 1), (TW, TH, NB)
    THT = TH * MT
    tiles_x, tiles_y = -(-W // TW), -(-H // THT)
    tiles = tiles_x * tiles_y * -(-N // NB) * (Cout // BN)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    assert tiles >= 2 * sms, f"{tiles} tiles on {sms} SMs: fewer than two waves"

    # ---- operands: sparse {-1, 0, 1} weights keep |acc| small
    x = _ints(g, (N, H, W, CIN), -1, 1)
    w = _ints(g, (Cout, CIN), -1, 1) * (torch.rand(Cout, CIN, generator=g) < 0.2).double()
    ref = torch.einsum("nhwc,oc->nhwo", x, w)
    kw = {}
    if spec.get("ebias"):
        rows = N if spec["ebias"] == "sample" else 1
        eb = _ints(g, (rows, Cout), -3, 3)
        ref = ref + eb[:, None, None, :]
        kw.update(ebias=eb.float().to(dev), ebias_stride=Cout if rows > 1 else 0)
    acc_s, res_s = torch.full((N,), 0.5, dtype=torch.float64), torch.full((N,), 1.0, dtype=torch.float64)
    sc = spec.get("scales")
    if sc == "value":
        kw.update(acc_scale=0.5, res_scale=1.0)
    elif sc == "pair":
        acc_s.fill_(0.25)
        res_s.fill_(0.5)
        kw.update(scales=torch.tensor([0.25, 0.5], device=dev))
    elif sc == "sample":  # rows of 3 floats: the pair, then one unused float
        acc_s = torch.tensor([0.25, 0.5, 1.0], dtype=torch.float64)[torch.arange(N) % 3]
        res_s = torch.tensor([1.0, 0.5], dtype=torch.float64)[torch.arange(N) % 2]
        tab = torch.stack([acc_s, res_s, torch.full((N,), 7.0, dtype=torch.float64)], 1).float()
        kw.update(scales=tab.reshape(-1).to(dev), scales_stride=3)
    else:
        acc_s.fill_(1.0)
    ref = ref * acc_s[:, None, None, None]
    rm = spec.get("res")
    if rm is not None:
        if rm == 0:
            res = _ints(g, (N, H, W, Cout), -2, 2)
            up = res
        elif rm == 1:
            res = _ints(g, (N, H // 2, W // 2, Cout), -2, 2)
            up = res.repeat_interleave(2, 1).repeat_interleave(2, 2)
        else:
            res = _ints(g, (N, 2 * H, 2 * W, Cout), -2, 2)
            up = res.reshape(N, H, 2, W, 2, Cout).sum(dim=(2, 4)) * 0.25
        ref = ref + res_s[:, None, None, None] * up
        kw.update(residual=res.half().to(dev), res_mode=rm)
    assert ref.abs().max().item() <= VMAX, ref.abs().max().item()

    # ---- outputs, NaN-filled, with a guard sample behind each
    f32 = spec.get("out") == "f32"
    oshape = (N // heads, H, W, heads * Cout)
    out_full = torch.full((oshape[0] + 1,) + oshape[1:], float("nan"), dtype=torch.float32 if f32 else torch.float16,
                          device=dev)
    stats_full = sums_full = None
    if spec.get("stats"):
        slots = ops.conv_stats_tiles(H, W, Cout, False)
        stats_full = torch.full((N + 1, slots, Cout // 2, 2), float("nan"), dtype=torch.float32, device=dev)
        kw.update(stats=stats_full[:N])
        if spec.get("sums"):
            sums_full = torch.zeros(N + 1, Cout // 2, 2, dtype=torch.int64, device=dev)
            kw.update(sums_out=sums_full[:N])
    op = ops.ConvOp([(x.half().to(dev), ops.MODE_1x1)], w.half().to(dev), out=out_full[:oshape[0]], out_heads=heads,
                    **kw)
    op.launch()
    torch.cuda.synchronize()

    # ---- output: every element exact, nothing written past the end
    want = ref.reshape(N // heads, heads, H, W, Cout).permute(0, 2, 3, 1, 4).reshape(oshape)
    got = out_full[:-1].double().cpu()
    assert torch.isnan(out_full[-1]).all(), "out: the guard sample was written"
    bad = (got != want).sum().item()
    assert bad == 0, f"out: {bad} of {got.numel()} elements differ (first at {(got != want).nonzero()[0].tolist()})"

    # ---- statistics: [N][slots][Cout/2][2] (sum, sum of squares) of channel pairs
    if stats_full is not None:
        r = ref.reshape(N, H, W, Cout // 2, 2)
        ps = torch.stack([r.sum(-1), (r * r).sum(-1)], -1)  # [N][H][W][C/2][2] per pixel
        if NB == 1:  # one slot per pixel tile
            pad = torch.zeros(N, tiles_y * THT, tiles_x * TW, Cout // 2, 2, dtype=torch.float64)
            pad[:, :H, :W] = ps
            st_want = pad.reshape(N, tiles_y, THT, tiles_x, TW, Cout // 2, 2).sum(dim=(2, 4))
            st_want = st_want.reshape(N, tiles_y * tiles_x, Cout // 2, 2)
        else:  # whole images per tile: one slot per 32-row quarter; row = y*TW*NB + (n % NB)*TW + x
            yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
            st_want = torch.zeros(N, 4, Cout // 2, 2, dtype=torch.float64)
            for n in range(N):
                quarter = (yy * TW * NB + (n % NB) * TW + xx) // 32
                st_want[n].index_add_(0, quarter.reshape(-1), ps[n].reshape(H * W, Cout // 2, 2))
        got_st = stats_full[:-1].double().cpu()
        assert torch.isnan(stats_full[-1]).all(), "stats: the guard sample was written"
        bad = (got_st != st_want).sum().item()
        assert bad == 0, f"stats: {bad} of {got_st.numel()} slots differ"
        if sums_full is not None:
            assert not sums_full[-1].any(), "sums_out: the guard sample was written"
            sums_want = (st_want * ops.STAT_SCALE).sum(1).to(torch.int64)
            assert torch.equal(sums_full[:-1].cpu(), sums_want), "sums_out differs"

    # ---- a second launch gives the same bits
    first = [t.clone() for t in (out_full, stats_full) if t is not None]
    if sums_full is not None:
        sums_first = sums_full.clone()
        sums_full.zero_()
    op.launch()
    torch.cuda.synchronize()
    for a, b in zip(first, [t for t in (out_full, stats_full) if t is not None]):
        assert torch.equal(a.view(torch.int16 if a.dtype == torch.float16 else torch.int32),
                           b.view(torch.int16 if b.dtype == torch.float16 else torch.int32)), "second launch differs"
    if sums_full is not None:
        assert torch.equal(sums_first, sums_full), "sums_out: second launch differs"


@pytest.mark.parametrize("case", sorted(CASES))
def test_conv_epilogue_exact(case):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    _run(CASES[case], torch.device("cuda:0"), seed=sorted(CASES).index(case) + 11)
