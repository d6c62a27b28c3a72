"""The UNet kernels at the limits their entry points admit.

  * The conv kernel decodes a tile index into (channel tile, sample group, tile row, tile column) with three divisions
    (tile_coord in csrc/conv_gemm.cu).  Each is a multiply-high by a magic number while (tile count) x divisor < 2^32,
    and a hardware division above that, which batches of about 90 to 256 reach at 256^2.  The host rule is restated
    here; test_magic_numbers_* check it exhaustively in Python integers (no GPU), and test_tile_decode_across_the_switch
    launches convs on both sides of the switch: exact over the whole output, statistics and sums_out, and bit-identical
    to batch-1 launches of the same samples.
  * asyrp_conv_create refuses a tile count of 2^31 or more (the kernel indexes tiles with int), also when the count
    does not fit 32 bits.
  * Every ASYRP_REQUIRE of asyrp_conv_create and of the UNet's other entry points (csrc/pointwise.cu, csrc/attention.cu)
    has a row in CONV_REFUSALS / CALL_REFUSALS: the refused call raises AsyrpError naming the entry point and leaves a
    NaN-filled output untouched, and its nearest accepted neighbour succeeds.  Not tabled, with the reason:
      - "sums_out needs ... BN >= 32": BN < 32 only for Cout = 16, which already requires stats == nullptr;
      - "resampled residual" with up2 or out_f32: both already refuse any residual;
      - "smem %zu too large": the ring depths are chosen to fit the budget, no tileable geometry exceeds it;
      - "tiles exceed the tile-index range": test_tile_index_guard.
  * apply, axpby and a 1x1 conv whose output has more than 2^31 elements (test_past_2_to_the_31_elements).

The magic number mul = floor(2^32 / d) + 1 is exact for every x with x * d < 2^32, the rule's bound, but not beyond it:
over the plans' geometries the 256^2 1x1 conv to 256 channels at batch 128 (65536 pixel tiles, 2 channel tiles) would
decode tile 131071 as channel tile 2 with the multiply-high.  The rule sends it to the hardware division, which
test_the_hardware_division_branch_is_load_bearing pins, and which case 1x1_256_hw128 launches.

Large cases check free device memory first and skip, naming the amount they need, when it is short.  The whole file
takes about 12 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit (6 s of it collection and the host-side
rule checks), with a peak of 12.25 GiB of device memory (torch.cuda.max_memory_allocated), in
test_past_2_to_the_31_elements.
"""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, ops

NAN = float("nan")
GiB = float(1 << 30)
TWO32 = 1 << 32


# ------------------------------------------------------------------------------------------------------------------
# the tile rule of csrc/conv_gemm.cu (conv_tile_shape / conv_config / magic), restated
# ------------------------------------------------------------------------------------------------------------------
def _tile_shape(H, W, halo):
    if halo:
        return 8, 16, 1
    tw = min(W, 128) if H == 1 else min(W, 16)
    th = 1 if H == 1 else min(128 // tw, 8, H)
    while th > 0 and 128 % (tw * th):
        th -= 1
    return tw, th, 128 // (tw * th) if th else 0


def _host_config(H, W, Cout, halo, phases=1):
    TW, TH, NB = _tile_shape(H, W, halo)
    whole2 = NB == 1 and H > 1 and H % (2 * TH) == 0 and W % TW == 0
    if Cout == 16:
        return 16, 2 if whole2 else 1
    tiles_x, tiles_n = -(-W // TW), -(-16 // NB)  # nominal batch of 16
    best, best_tiles = None, -1
    for bn, mt in ((128, 1), (64, 2), (64, 1)):
        if Cout % bn or (mt == 2 and not whole2):
            continue
        tiles = tiles_x * -(-H // (TH * mt)) * tiles_n * (Cout // bn) * phases
        if tiles >= 106:
            return bn, mt
        if tiles > best_tiles:
            best, best_tiles = (bn, mt), tiles
    return best


def _tiling(N, H, W, Cout, has3, up2=False):
    """tile counts of a conv (H, W: the source's for up2) and the three (divisor, magic) pairs of tile_coord"""
    halo = has3 and H % 16 == 0 and W % 8 == 0
    TW, TH, NB = _tile_shape(H, W, halo)
    BN, MT = _host_config(H, W, Cout, halo, 4 if up2 else 1)
    tx, ty, tn = -(-W // TW), -(-H // (TH * MT)), -(-N // NB)
    m, n = tx * ty * tn, Cout // BN * (4 if up2 else 1)
    xmax = m * n
    divs = {"m_tiles": m, "tiles_x": tx, "tiles_xy": tx * ty}
    return dict(TW=TW, TH=TH, NB=NB, BN=BN, MT=MT, tiles_x=tx, tiles_y=ty, m_tiles=m, n_tiles=n, xmax=xmax,
                mul={k: _magic(xmax, d) for k, d in divs.items()}, divs=divs)


def _magic(xmax, d):
    """asyrp_conv_create's magic(): 0 = divide by one, 1 = hardware division, else the multiply-high factor"""
    if d <= 1:
        return 0
    if xmax * d >= TWO32:
        return 1
    return TWO32 // d + 1


def _first_wrong(d):
    """smallest x with (x * mul) >> 32 != x // d for mul = 2^32 // d + 1.  With x = q d + r and mul d = 2^32 + e, the
    multiply-high gives q + floor((q e + r mul) / 2^32): the first failure is at the first q where r = d - 1 can reach
    2^32, and at the least such r (x grows with q because e / mul << 1)."""
    mul = TWO32 // d + 1
    e = mul * d - TWO32
    q = max(0, -(-(TWO32 - (d - 1) * mul) // e))
    r = max(0, -(-(TWO32 - q * e) // mul))
    return q * d + r


def _magic_wrong_below(d, xmax):
    """every x < xmax whose multiply-high quotient is wrong (numpy, exhaustive)"""
    mul = np.uint64(TWO32 // d + 1)
    bad = []
    for x0 in range(0, xmax, 1 << 22):
        x = np.arange(x0, min(xmax, x0 + (1 << 22)), dtype=np.uint64)
        wrong = ((x * mul) >> np.uint64(32)) != x // np.uint64(d)
        bad.extend(x[wrong][:4].tolist())
    return bad


# a superset of every conv geometry the four bench.WORKLOADS plans create: each level resolution with Cout multiples
# of 64 up to 1024 (1x1, 3x3 and the up2 conv of the level), conv_out, and the attention GEMMs (a 1 x T image, Cout = T
# or the head width, batch entries = samples x heads) of the 64-, 256- and 1024-token maps with up to 16 heads
def _plan_geometries():
    geoms = []
    for r in (256, 128, 64, 32, 16, 8):
        for cout in range(64, 1025, 64):
            geoms += [(r, r, cout, False, False, 1), (r, r, cout, True, False, 1)]
            if r % 16 == 0 and r <= 128:
                geoms.append((r, r, cout, True, True, 1))
    geoms.append((256, 256, 16, True, False, 1))
    for T in (64, 256, 1024):
        for cout in sorted({T, 64, 128, 256, 512}):
            for heads in (1, 2, 4, 8, 16):
                geoms.append((1, T, cout, False, False, heads))
    return geoms


PLAN_BATCHES = range(1, 257)


def _plan_pairs():
    """{(xmax, divisor): magic} over the plan geometries at batches 1..256 and the boundary cases of TILE_CASES"""
    pairs = {}
    for H, W, cout, has3, up2, heads in _plan_geometries():
        for N in PLAN_BATCHES:
            t = _tiling(N * heads, H, W, cout, has3, up2)
            for k, d in t["divs"].items():
                pairs[(t["xmax"], d)] = t["mul"][k]
    for case in TILE_CASES.values():
        t = _tiling(case["N"], 256, 256, case["Cout"], case["k"] == 3)
        for k, d in t["divs"].items():
            pairs[(t["xmax"], d)] = t["mul"][k]
    return pairs


# ------------------------------------------------------------------------------------------------------------------
# the tile decode on both sides of the multiply-high / hardware-division switch
# ------------------------------------------------------------------------------------------------------------------
# Cin, Cout, kernel size, N at 256^2; "a": 3x3 halo conv with a per-sample fused affine, bias, residual, statistics and
# sums_out; "b": 1x1 conv with 2 channel tiles, bias, statistics and sums_out; "c": conv_out (Cout 16, planar fp32,
# MT 2)
# edge: the batch is the last one below the switch (-1), the first one above it (+1), or neither (0)
def _case(kind, N, edge):
    return {"a": dict(kind="a", Cin=128, Cout=128, k=3), "b": dict(kind="b", Cin=64, Cout=256, k=1),
            "c": dict(kind="c", Cin=128, Cout=16, k=3)}[kind] | dict(N=N, edge=edge)


TILE_CASES = {"halo128_magic127": _case("a", 127, -1), "halo128_hw128": _case("a", 128, 1),
              "1x1_256_magic90": _case("b", 90, -1), "1x1_256_hw91": _case("b", 91, 1),
              "1x1_256_hw128": _case("b", 128, 0),
              "conv_out_magic255": _case("c", 255, -1), "conv_out_hw256": _case("c", 256, 1)}


def _case_id(name):
    c = TILE_CASES[name]
    t = _tiling(c["N"], 256, 256, c["Cout"], c["k"] == 3)
    side = "hardware" if t["mul"]["m_tiles"] == 1 else "multiply-high"
    return f"{name}-m_tiles{t['m_tiles']}-n_tiles{t['n_tiles']}-d{t['m_tiles']}-{side}"


def _need_memory(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + GiB // 2:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")


def _pattern(out, salt, mod=61):
    """out[n, y, x, c] = ((5 y + 3 x + 7 c + 11 n + salt) mod `mod`) - mod // 2: integers encoding the position"""
    N, H, W, Cc = out.shape
    dev = out.device
    base = (torch.arange(H, device=dev).view(H, 1, 1) * 5 + torch.arange(W, device=dev).view(1, W, 1) * 3
            + torch.arange(Cc, device=dev).view(1, 1, Cc) * 7 + salt)
    for n0 in range(0, N, 8):
        nn = torch.arange(n0, min(N, n0 + 8), device=dev).view(-1, 1, 1, 1)
        out[n0:n0 + 8] = ((base + 11 * nn) % mod - mod // 2).to(out.dtype)


def _randn_(t, gen, scale=1.0, shift=0.0):
    for n0 in range(0, t.shape[0], 8):
        t[n0:n0 + 8] = torch.randn(t[n0:n0 + 8].shape, generator=gen, device=t.device, dtype=t.dtype) * scale + shift


def _bits(t):
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


def _locate(bad, n0, t, what):
    """fail with the first wrong element of samples n0.. and the tile that owns it"""
    n, y, x, o = bad.nonzero()[0].tolist()
    n += n0
    nt, tile_y, tile_x = o // t["BN"], y // (t["TH"] * t["MT"]), x // t["TW"]
    tile = ((nt * t["m_tiles"]) + (n // t["NB"]) * t["tiles_x"] * t["tiles_y"] + tile_y * t["tiles_x"] + tile_x)
    pytest.fail(f"{what}: {int(bad.sum())} elements wrong, first at (n={n}, y={y}, x={x}, o={o}) = tile index {tile} "
                f"(tx={tile_x}, ty={tile_y}, tn={n // t['NB']}, nt={nt})")


class _TileCase:
    """operands, op and reference of one TILE_CASES entry"""

    def __init__(self, spec, dev):
        self.s, self.dev = spec, dev
        N, Cin, Cout, H = spec["N"], spec["Cin"], spec["Cout"], 256
        self.t = _tiling(N, H, H, Cout, spec["k"] == 3)
        assert ops.conv_tile_config(H, H, Cout, spec["k"] == 3) == (self.t["BN"], self.t["MT"])
        self.x = torch.empty(N, H, H, Cin, dtype=torch.float16, device=dev)
        self.planar = spec["kind"] == "c"
        if self.planar:
            self.full = torch.empty(N + 1, 3, H, H, dtype=torch.float32, device=dev)
        else:
            self.full = torch.empty(N + 1, H, H, Cout, dtype=torch.float16, device=dev)
        self.res = torch.empty(N, H, H, Cout, dtype=torch.float16, device=dev) if spec["kind"] == "a" else None
        self.stats_full = self.sums_full = None
        if not self.planar:
            slots = ops.conv_stats_tiles(H, H, Cout, spec["k"] == 3)
            assert slots == self.t["tiles_x"] * self.t["tiles_y"]
            self.stats_full = torch.empty(N + 1, slots, Cout // 2, 2, dtype=torch.float32, device=dev)
            self.sums_full = torch.empty(N + 1, Cout // 2, 2, dtype=torch.int64, device=dev)
        self.aff = torch.empty(N, Cin, 2, dtype=torch.float32, device=dev) if spec["k"] == 3 else None
        self.eb = torch.empty(N, Cout, dtype=torch.float32, device=dev)

    def op(self, w, act, rows=None, bufs=None):
        """the op over samples `rows` (a slice; all by default), writing `bufs` = (out, stats, sums) views"""
        rows = rows if rows is not None else slice(0, self.s["N"])
        seg = (self.x[rows], ops.MODE_3x3 if self.s["k"] == 3 else ops.MODE_1x1)
        if self.aff is not None:
            seg = seg + (self.aff[rows], 0, act)
        out, stats, sums = bufs
        kw = dict(out_planar=out, out_shape=(out.shape[0], 256, 256, 16)) if self.planar else dict(out=out)
        return ops.ConvOp([seg], w, ebias=self.eb[rows], ebias_stride=self.s["Cout"], stats=stats, sums_out=sums,
                          residual=self.res[rows] if self.res is not None else None, res_scale=1.0, **kw)

    def views(self):
        N = self.s["N"]
        return (self.full[:N], None if self.stats_full is None else self.stats_full[:N],
                None if self.sums_full is None else self.sums_full[:N])

    def fill_outputs(self):
        self.full.fill_(NAN)
        if self.stats_full is not None:
            self.stats_full.fill_(NAN)
            self.sums_full.zero_()
            self.sums_full[-1].fill_(-1)

    def check_guards(self):
        assert torch.isnan(self.full[-1]).all(), "the guard sample behind the output was written"
        if self.stats_full is not None:
            assert torch.isnan(self.stats_full[-1]).all(), "the guard sample behind the statistics was written"
            assert (self.sums_full[-1] == -1).all(), "the guard sample behind sums_out was written"


def _one_hot(Cout, Cin, k, perm, dev):
    """weight row o = 1 at the centre tap of input channel perm[o]"""
    w = torch.zeros(Cout, k * k * Cin, dtype=torch.float16)
    w[torch.arange(Cout), (k * k // 2) * Cin + perm] = 1.0
    return w.to(dev)


def _exact_check(case):
    s, t, dev = case.s, case.t, case.dev
    N, Cin, Cout = s["N"], s["Cin"], s["Cout"]
    o = torch.arange(Cout, device=dev)
    perm = (o * 5 + o // Cin + 3) % Cin  # a permutation of the input channels for Cout == Cin
    _pattern(case.x, 0)
    if case.res is not None:
        _pattern(case.res, 17, mod=33)
    nn = torch.arange(N, device=dev).view(N, 1)
    case.eb.copy_(((5 * nn + o) % 17 - 8).float())
    if case.aff is not None:
        c = torch.arange(Cin, device=dev).view(1, Cin)
        a = torch.tensor([1.0, 0.5, -1.0, -0.5], device=dev)[(nn + c) % 4]
        case.aff.copy_(torch.stack([a, ((3 * nn + c) % 7 - 3).float() * 0.5], -1))
    w = _one_hot(Cout, Cin, s["k"], perm.cpu(), dev)
    case.fill_outputs()
    case.op(w, 0, bufs=case.views()).launch()
    torch.cuda.synchronize()
    case.check_guards()
    out, stats, sums = case.views()
    TH, TW = t["TH"] * t["MT"], t["TW"]
    for n0 in range(0, N, 8):
        n1 = min(N, n0 + 8)
        xs = case.x[n0:n1].float()[..., perm]  # [n][H][W][Cout]: the operand channel each output channel reads
        if case.aff is not None:
            af = case.aff[n0:n1][:, perm]  # [n][Cout][2]
            xs = xs * af[:, None, None, :, 0] + af[:, None, None, :, 1]
        ref = xs + case.eb[n0:n1, None, None, :]
        if case.res is not None:
            ref = ref + case.res[n0:n1].float()
        if case.planar:
            got = out[n0:n1].permute(0, 2, 3, 1)
            ref = ref[..., :3]
        else:
            got = out[n0:n1].float()
        bad = got != ref
        if bad.any():
            _locate(bad, n0, t, "output")
        if stats is None:
            continue
        r = ref.double().view(n1 - n0, t["tiles_y"], TH, t["tiles_x"], TW, Cout // 2, 2)
        want = torch.stack([r.sum((2, 4, 6)), (r * r).sum((2, 4, 6))], -1).reshape(n1 - n0, -1, Cout // 2, 2)
        assert torch.equal(stats[n0:n1].double(), want), f"statistics slots of samples {n0}..{n1 - 1}"
        tot = want.sum(1) * ops.STAT_SCALE
        assert torch.equal(sums[n0:n1], tot.long()), f"sums_out of samples {n0}..{n1 - 1}"


def _independence_check(case):
    """samples 0, N/2 and N-1 of the large launch bit-identical to batch-1 launches of the same sample"""
    s, dev = case.s, case.dev
    N, Cin, Cout, k = s["N"], s["Cin"], s["Cout"], s["k"]
    g = torch.Generator(device=dev).manual_seed(N)
    _randn_(case.x, g, 1.5, 0.3)
    if case.res is not None:
        _randn_(case.res, g)
    case.eb.copy_(torch.randn(N, Cout, generator=g, device=dev))
    if case.aff is not None:
        case.aff.copy_(torch.randn(N, Cin, 2, generator=g, device=dev) * 0.5 + 1.0)
    w = (torch.randn(Cout, k * k * Cin, generator=g, device=dev) / math.sqrt(k * k * Cin)).half()
    case.fill_outputs()
    case.op(w, 1, bufs=case.views()).launch()
    torch.cuda.synchronize()
    case.check_guards()
    big = case.views()
    for n in sorted({0, N // 2, N - 1}):
        one = tuple(None if b is None else torch.full_like(b[:1], NAN if b.is_floating_point() else 0) for b in big)
        case.op(w, 1, rows=slice(n, n + 1), bufs=one).launch()
        torch.cuda.synchronize()
        for name, a, b in zip(("output", "statistics", "sums_out"), big, one):
            if a is not None:
                assert torch.isfinite(b.float()).all(), f"{name} of the batch-1 launch of sample {n} not written"
                assert torch.equal(_bits(a[n]), _bits(b[0])), \
                    f"{name} of sample {n} differs between the batch-{N} and the batch-1 launch"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TILE_CASES), ids=_case_id)
def test_tile_decode_across_the_switch(cuda_device, name):
    s = TILE_CASES[name]
    t = _tiling(s["N"], 256, 256, s["Cout"], s["k"] == 3)
    # the case sits where its name says: the m_tiles division switches to hardware at (tile count) * m_tiles >= 2^32
    hw = t["xmax"] * t["m_tiles"] >= TWO32
    assert hw == ("_hw" in name) and (t["mul"]["m_tiles"] == 1) == hw, (t["xmax"], t["m_tiles"])
    if s["edge"]:
        nb = _tiling(s["N"] - s["edge"], 256, 256, s["Cout"], s["k"] == 3)
        assert (nb["mul"]["m_tiles"] == 1) != hw, "the neighbouring batch must be on the other side of the switch"
    assert t["mul"]["tiles_x"] > 1 and t["mul"]["tiles_xy"] > 1
    print(f"\n{name}: N={s['N']} m_tiles={t['m_tiles']} n_tiles={t['n_tiles']} divisor={t['m_tiles']} "
          f"xmax*d={t['xmax'] * t['m_tiles']} {'>=' if hw else '<'} 2^32: {'hardware' if hw else 'multiply-high'}")
    N, px = s["N"], 256 * 256
    need = 2 * N * px * (s["Cin"] + (2 * s["Cout"] if s["kind"] == "a" else s["Cout"] if s["kind"] == "b" else 6))
    need += 8 * px * max(s["Cin"], s["Cout"]) * 4 * 6  # the reference of 8 samples in fp32 / fp64
    _need_memory(need, name)
    case = _TileCase(s, cuda_device)
    try:
        _exact_check(case)
        _independence_check(case)
    finally:
        del case
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# the magic-number rule, exhaustively (no GPU)
# ------------------------------------------------------------------------------------------------------------------
def test_first_wrong_quotient_closed_form():
    """_first_wrong against an exhaustive search, for every divisor up to 2^12 and around the plans' large ones"""
    for d in list(range(2, 1 << 12, 7)) + [46592, 65024, 65536, 65537, 131072]:
        x0 = _first_wrong(d)
        mul = TWO32 // d + 1
        assert (x0 * mul) >> 32 != x0 // d, d
        if x0 <= 1 << 20:
            assert _magic_wrong_below(d, x0 + 1) == [x0], d


def test_magic_numbers_are_exact_wherever_the_rule_uses_them():
    """every (tile count, divisor) pair the plans reach at batches 1..256 and the TILE_CASES boundaries: where the rule
    takes the multiply-high, (x * mul) >> 32 == x // d for EVERY tile index x below the tile count"""
    need = {}
    for (xmax, d), mul in _plan_pairs().items():
        if mul > 1:
            assert mul == TWO32 // d + 1 and xmax * d < TWO32
            need[d] = max(need.get(d, 0), xmax)
    assert len(need) > 1000, len(need)
    for d, xmax in need.items():
        assert not _magic_wrong_below(d, xmax), (d, xmax)
        assert _first_wrong(d) >= xmax, (d, xmax)


def test_the_hardware_division_branch_is_load_bearing():
    """Among the pairs the rule sends to the hardware division, some would be decoded wrongly by the multiply-high:
    there the `return 1u` branch of magic() is what keeps the decode right.  The rule's own bound x * d < 2^32 is
    sufficient, not necessary: near the switch (TILE_CASES' first hardware batches) the magic number is still exact."""
    pairs = _plan_pairs()
    wrong = sorted((xmax, d) for (xmax, d), mul in pairs.items() if _first_wrong(d) < xmax)
    assert wrong, "no plan geometry needs the hardware division"
    for xmax, d in wrong:
        assert pairs[(xmax, d)] == 1, (xmax, d)
    # the smallest such case: the 256^2 1x1 conv to 256 channels at batch 128, tile 131071 -> channel tile 2 of 2
    t = _tiling(128, 256, 256, 256, False)
    d, xmax = t["m_tiles"], t["xmax"]
    assert (d, xmax) == (65536, 131072) and (xmax, d) in wrong and t["mul"]["m_tiles"] == 1
    assert _magic_wrong_below(d, xmax)[0] == _first_wrong(d) == 131071
    assert (131071 * (TWO32 // d + 1)) >> 32 == 2
    for name in ("halo128_hw128", "1x1_256_hw91", "conv_out_hw256"):
        c = TILE_CASES[name]
        t = _tiling(c["N"], 256, 256, c["Cout"], c["k"] == 3)
        assert t["mul"]["m_tiles"] == 1 and _first_wrong(t["m_tiles"]) >= t["xmax"], name


# ------------------------------------------------------------------------------------------------------------------
# refusals, without a launch
# ------------------------------------------------------------------------------------------------------------------
class _Scratch:
    """device buffers the descriptors point at: creation only encodes tensor maps, nothing is read"""

    def __init__(self, dev):
        self.buf = torch.full((1 << 22,), NAN, dtype=torch.float32, device=dev)  # 16 MB, NaN
        self.P = self.buf.data_ptr()


_SEG_FIELDS = {f[0] for f in _lib.AsyrpConvSeg._fields_}


def _desc(P, over):
    """the base descriptor (N 2, 16 x 16, one 1x1 segment of 64 channels -> 64), with overrides: descriptor fields by
    name, segment fields as s<i>_<field>; the value "P" stands for a device pointer"""
    d = _lib.AsyrpConvDesc()
    d.N, d.H, d.W, d.Cout, d.nseg = 2, 16, 16, 64, 1
    for i in range(3):
        d.seg[i].src, d.seg[i].C, d.seg[i].mode = P, 64, 0
    d.weight = d.out = P
    for k, v in over.items():
        v = P if v == "P" else v
        if k[0] == "s" and k[1].isdigit() and k[3:] in _SEG_FIELDS:
            setattr(d.seg[int(k[1])], k[3:], v)
        else:
            assert hasattr(d, k), k
            setattr(d, k, v)
    return d


def _create(d):
    lib = _lib.load()
    h = C.c_void_p()
    rc = lib.asyrp_conv_create(C.byref(d) if d is not None else None, C.byref(h))
    return rc, h, lib.asyrp_last_error().decode()


UP2 = dict(up2=1, s0_mode=1)
GN = dict(s0_mode=1, s0_gn_gamma="P", s0_gn_beta="P", s0_gn_sums_a="P", s0_gn_Ca=64, s0_gn_hw=256)
C16 = dict(Cout=16, out=None, out_planar="P", planar_c=3)
# (row, message fragment, refused overrides, nearest accepted overrides): one row per ASYRP_REQUIRE condition of
# asyrp_conv_create, in source order
CONV_REFUSALS = [
    ("nseg_0", "nseg=0", dict(nseg=0), dict(nseg=1)),
    ("nseg_4", "nseg=4", dict(nseg=4), dict(nseg=3)),
    ("cout_96", "Cout=96", dict(Cout=96), dict(Cout=128)),
    ("cout16_not_planar", "Cout=16", dict(Cout=16), C16),
    ("cout16_stats", "Cout=16", dict(C16, stats="P"), C16),
    ("cout16_residual", "Cout=16", dict(C16, residual="P"), C16),
    ("cout16_up2", "Cout=16", dict(C16, **UP2), dict(C16, s0_mode=1)),
    ("cout16_batched", "Cout=16", dict(C16, weight_batched=1), C16),
    ("empty_N", "empty geometry N=0", dict(N=0), dict(N=1)),
    ("negative_N", "empty geometry N=-1", dict(N=-1), dict(N=1)),
    ("empty_H_halo", "empty geometry", dict(H=0, s0_mode=1), dict(H=16, s0_mode=1)),
    ("negative_H_halo", "empty geometry", dict(H=-16, s0_mode=1), dict(H=16, s0_mode=1)),
    ("empty_W", "empty geometry", dict(W=0), dict(W=1, H=1)),
    ("negative_W_halo", "empty geometry", dict(W=-8, s0_mode=1), dict(W=8, s0_mode=1)),
    ("untileable", "cannot tile H=2 W=12", dict(H=2, W=12), dict(H=2, W=16)),
    ("batched_nb2", "batched weights need NB==1", dict(H=8, W=8, weight_batched=1), dict(weight_batched=1)),
    ("up2_no_halo", "up2 needs", dict(UP2, H=8, W=8), UP2),
    ("up2_two_segments", "up2 needs", dict(UP2, nseg=2), UP2),
    ("up2_batched", "up2 needs", dict(UP2, weight_batched=1), UP2),
    ("up2_out_f32", "up2 needs", dict(UP2, out_f32=1), UP2),
    ("up2_planar", "up2 needs", dict(UP2, out_planar="P", planar_c=3), UP2),
    ("up2_out_heads", "up2 needs", dict(UP2, out_heads=2), UP2),
    ("up2_a_heads", "up2 needs", dict(UP2, a_heads=2), UP2),
    ("up2_residual", "up2 needs", dict(UP2, residual="P"), UP2),
    ("seg_c_32", "segment channels 32", dict(s0_C=32), dict(s0_C=128)),
    ("seg_c_0", "segment channels 0", dict(s0_C=0), dict(s0_C=64)),
    ("seg_mode_3", "bad segment mode 3", dict(s0_mode=3), dict(s0_mode=2)),
    ("seg_mode_neg", "bad segment mode -1", dict(s0_mode=-1), dict(s0_mode=0)),
    ("affine_s2", "no fused affine on stride-2", dict(s0_mode=2, s0_affine="P"), dict(s0_mode=1, s0_affine="P")),
    ("gn_and_affine", "in-kernel GroupNorm needs", dict(GN, s0_affine="P"), GN),
    ("gn_no_sums", "in-kernel GroupNorm needs", dict(GN, s0_gn_sums_a=None), GN),
    ("gn_no_beta", "in-kernel GroupNorm needs", dict(GN, s0_gn_beta=None), GN),
    ("gn_ca_0", "in-kernel GroupNorm needs", dict(GN, s0_gn_Ca=0), GN),
    ("gn_c_not_64", "in-kernel GroupNorm needs", dict(GN, s0_gn_Ca=32), dict(GN, s0_gn_Ca=32, s0_gn_Cb=32,
                                                                               s0_gn_sums_b="P")),
    ("gn_ca_odd", "in-kernel GroupNorm needs", dict(GN, s0_gn_Ca=63, s0_gn_Cb=1, s0_gn_sums_b="P"),
     dict(GN, s0_gn_Ca=62, s0_gn_Cb=2, s0_gn_sums_b="P")),
    ("gn_cb_no_sums", "in-kernel GroupNorm needs", dict(GN, s0_gn_Cb=64), dict(GN, s0_gn_Cb=64, s0_gn_sums_b="P")),
    ("gn_hw_0", "in-kernel GroupNorm needs", dict(GN, s0_gn_hw=0), GN),
    ("gn_s2", "in-kernel GroupNorm needs", dict(GN, s0_mode=2), dict(GN, s0_mode=0)),
    ("gn_nb2", "in-kernel GroupNorm needs", dict(GN, H=8, W=8), GN),
    ("ld_below_c", "segment ld=32", dict(s0_ld=32), dict(s0_ld=64)),
    ("ld_not_8", "segment ld=68", dict(s0_ld=68), dict(s0_ld=72)),
    ("s2_sliced", "stride-2 segments need a dense source", dict(s0_mode=2, s0_ld=128), dict(s0_mode=0, s0_ld=128)),
    ("a_heads_ld", "a_heads needs", dict(a_heads=2), dict(a_heads=2, s0_ld=128)),
    ("a_heads_n", "a_heads needs", dict(a_heads=2, s0_ld=128, N=3), dict(a_heads=3, s0_ld=192, N=3)),
    ("a_heads_3x3", "a_heads needs", dict(a_heads=2, s0_ld=128, s0_mode=1), dict(a_heads=2, s0_ld=128)),
    ("a_heads_nseg", "a_heads needs", dict(a_heads=2, s0_ld=128, nseg=2), dict(a_heads=2, s0_ld=128)),
    ("weight_ld_below_k", "weight_ld / weight_batch_stride", dict(weight_ld=32), dict(weight_ld=64)),
    ("weight_ld_not_8", "weight_ld / weight_batch_stride", dict(weight_ld=68), dict(weight_ld=72)),
    ("weight_bs_not_8", "weight_ld / weight_batch_stride", dict(weight_batched=1, weight_batch_stride=4100),
     dict(weight_batched=1, weight_batch_stride=4104)),
    ("b_heads_ld", "b_heads needs", dict(weight_batched=1, b_heads=2),
     dict(weight_batched=1, b_heads=2, weight_ld=128)),
    ("k_chunks_65", "more than 64 K chunks", dict(nseg=3, s0_C=1408, s1_C=1408, s2_C=1344),
     dict(nseg=3, s0_C=1408, s1_C=1408, s2_C=1280)),
    ("out_f32_residual", "out_f32 excludes", dict(out_f32=1, residual="P"), dict(out_f32=1)),
    ("out_f32_stats", "out_f32 excludes", dict(out_f32=1, stats="P"), dict(out_f32=1)),
    ("out_f32_planar", "out_f32 excludes", dict(out_f32=1, out_planar="P", planar_c=1), dict(out_f32=1)),
    ("out_heads_n", "out_heads needs", dict(out_heads=2, N=3), dict(out_heads=3, N=3)),
    ("out_heads_stats", "out_heads needs", dict(out_heads=2, stats="P"), dict(out_heads=2)),
    ("out_heads_planar", "out_heads needs", dict(out_heads=2, out_planar="P", planar_c=1), dict(out_heads=2)),
    ("planar_c_0", "planar_c=0", dict(out_planar="P", planar_c=0), dict(out_planar="P", planar_c=1)),
    ("planar_c_9", "planar_c=9", dict(out_planar="P", planar_c=9), dict(out_planar="P", planar_c=8)),
    ("scales_stride_neg", "scales_stride=-1", dict(scales="P", scales_stride=-1), dict(scales="P", scales_stride=0)),
    ("scales_stride_no_table", "scales_stride=2 needs", dict(scales_stride=2), dict(scales="P", scales_stride=2)),
    ("res_mode_3", "res_mode 3", dict(residual="P", res_mode=3), dict(residual="P", res_mode=2)),
    ("res_mode_neg", "res_mode -1", dict(residual="P", res_mode=-1), dict(residual="P", res_mode=0)),
    ("resampled_out_heads", "resampled residual", dict(residual="P", res_mode=1, out_heads=2),
     dict(residual="P", res_mode=1)),
    ("resampled_planar", "resampled residual", dict(residual="P", res_mode=1, out_planar="P", planar_c=1),
     dict(residual="P", res_mode=0, out_planar="P", planar_c=1)),
    ("resampled_odd_h", "resampled residual", dict(residual="P", res_mode=1, H=3),
     dict(residual="P", res_mode=2, H=3)),
    ("sums_out_no_stats", "sums_out needs", dict(sums_out="P"), dict(sums_out="P", stats="P")),
    ("sums_out_nb2", "sums_out needs", dict(sums_out="P", stats="P", H=8, W=8), dict(stats="P", H=8, W=8)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", CONV_REFUSALS, ids=[r[0] for r in CONV_REFUSALS])
def test_conv_create_refusals(cuda_device, row):
    name, fragment, bad, good = row
    sc = _Scratch(cuda_device)
    rc, h, err = _create(_desc(sc.P, bad))
    assert rc == -1 and not h.value, (name, rc)
    assert err.startswith("asyrp_conv_create: ") and fragment in err, (name, err)
    rc, h, err = _create(_desc(sc.P, good))
    assert rc == 0 and h.value, (name, err)
    _lib.load().asyrp_conv_destroy(h)
    torch.cuda.synchronize()
    assert torch.isnan(sc.buf).all(), "a descriptor's buffer was written"


@pytest.mark.gpu
def test_conv_create_null_arguments(cuda_device):
    rc, _, err = _create(None)
    assert rc == -1 and err == "asyrp_conv_create: null argument"
    sc = _Scratch(cuda_device)
    lib = _lib.load()
    assert lib.asyrp_conv_create(C.byref(_desc(sc.P, {})), None) == -1
    assert lib.asyrp_last_error().decode() == "asyrp_conv_create: null argument"


@pytest.mark.gpu
def test_tile_index_guard(cuda_device):
    """1 x 128-pixel images: one pixel tile per sample, one channel tile, so the tile count is the batch.  2^31 - 1
    tiles are accepted (not launched), 2^31 are refused, and so is 4 (2^30 + 1) = 2^32 + 4, whose int product wraps to
    4 tiles"""
    sc = _Scratch(cuda_device)
    t = _tiling(2 ** 31 - 1, 1, 128, 64, False)
    assert (t["m_tiles"], t["n_tiles"], t["mul"]["m_tiles"]) == (2 ** 31 - 1, 1, 1)
    rc, h, err = _create(_desc(sc.P, dict(N=2 ** 31 - 1, H=1, W=128)))
    assert rc == 0 and h.value, err
    _lib.load().asyrp_conv_destroy(h)
    for N, W in ((2 ** 30, 256), (2 ** 30 + 1, 512), (2 ** 31 - 1, 256)):
        assert _tiling(N, 1, W, 64, False)["xmax"] >= 2 ** 31
        rc, h, err = _create(_desc(sc.P, dict(N=N, H=1, W=W)))
        assert rc == -1 and not h.value and "exceed the tile-index range" in err, (N, W, rc, err)
    # the same through the channel-tile factor: 2^29 samples x 4 channel tiles of 64
    rc, h, err = _create(_desc(sc.P, dict(N=2 ** 29, H=1, W=128, Cout=256)))
    assert rc == -1 and "exceed the tile-index range" in err, err
    torch.cuda.synchronize()
    assert torch.isnan(sc.buf).all()


def _conv_1x1_exact(dev, N, H, W, Cout=64, planar_c=0, res_mode=-1):
    """launch an accepted neighbour: 1x1 conv of 64 integer channels with weights in {-1, 0, 1}, exact against fp64"""
    g = torch.Generator().manual_seed(N * 1000 + H * 10 + W)
    x = torch.randint(-2, 3, (N, H, W, 64), generator=g).double()
    w = torch.randint(-1, 2, (Cout, 64), generator=g).double()
    ref = torch.einsum("nhwc,oc->nhwo", x, w)
    kw = {}
    if res_mode >= 0:
        rs = {0: (H, W), 1: (H // 2, W // 2), 2: (2 * H, 2 * W)}[res_mode]
        r = torch.randint(-8, 9, (N, *rs, Cout), generator=g).double()
        kw = dict(residual=r.half().to(dev), res_mode=res_mode)
        if res_mode == 2:
            r = r.view(N, H, 2, W, 2, Cout).mean((2, 4))
        elif res_mode == 1:
            r = r.repeat_interleave(2, 1).repeat_interleave(2, 2)
        ref = ref + r
    if planar_c:
        full = torch.full((N + 1, planar_c, H, W), NAN, device=dev)
        kw.update(out_planar=full[:N], out_shape=(N, H, W, Cout))
    else:
        full = torch.full((N + 1, H, W, Cout), NAN, dtype=torch.float16, device=dev)
        kw.update(out=full[:N])
    ops.ConvOp([(x.half().to(dev), ops.MODE_1x1)], w.half().to(dev), **kw).launch()
    torch.cuda.synchronize()
    assert torch.isnan(full[-1]).all()
    got = full[:N].double().cpu()
    if planar_c:
        got, ref = got, ref[..., :planar_c].permute(0, 3, 1, 2)
    assert torch.equal(got, ref)


@pytest.mark.gpu
def test_conv_accepted_neighbours_launch_exactly(cuda_device):
    """the cheap accepted neighbours at the edges of the table, launched: the smallest image (1 x 1, eight samples to a
    tile holding one), all eight planar channels, and the 2x2 average-pooled residual of an odd-height output"""
    _conv_1x1_exact(cuda_device, 1, 1, 1)
    _conv_1x1_exact(cuda_device, 3, 1, 16)
    _conv_1x1_exact(cuda_device, 2, 16, 16, planar_c=8)
    _conv_1x1_exact(cuda_device, 2, 3, 16, res_mode=2)
    _conv_1x1_exact(cuda_device, 2, 4, 16, res_mode=1)


# ---- the UNet's other entry points --------------------------------------------------------------------------------
def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gn(dev, N=2, Ca=64, HW=4):
    """asyrp_gn_finalize over one statistics slot per sample, every channel pair holding (sum 2, sum of squares 6)"""
    st = torch.zeros(N, 1, max(Ca, 2) // 2, 2, device=dev)
    st[..., 0] = 2.0
    st[..., 1] = 6.0
    gamma, beta = torch.full((max(Ca, 1),), 2.0, device=dev), torch.full((max(Ca, 1),), 0.5, device=dev)
    out = torch.full((N, max(Ca, 1), 2), NAN, device=dev)

    def call():
        return _lib.load().asyrp_gn_finalize(_p(st), Ca, 1, None, 0, 0, _p(gamma), _p(beta), 0.0, N, HW, None, 0,
                                             _p(out), _stream())

    def check():
        # per group (one channel pair): count 2 HW, mean 2 / (2 HW), E[x^2] = 6 / (2 HW)
        cnt = 2.0 * HW
        mean, var = 2.0 / cnt, 6.0 / cnt - (2.0 / cnt) ** 2
        a = 2.0 / math.sqrt(var)
        want = torch.tensor([a, 0.5 - mean * a], dtype=torch.float64)
        for n in (0, N - 1):
            assert torch.allclose(out[n].double().cpu(), want.expand(Ca, 2), rtol=1e-5, atol=0), out[n, 0]
    return call, [out], check


def _apply(dev, N=2, Ca=16, Cb=0, H=4, act=0, resample=0):
    C_ = max(Ca + Cb, 8)
    x = ((torch.arange(N * H * H * max(Ca, 8), device=dev) % 13) - 6).half().view(N, H, H, max(Ca, 8))
    aff = torch.stack([torch.full((N, C_), 0.5, device=dev), torch.full((N, C_), -1.5, device=dev)], -1).contiguous()
    out = torch.full((N, 2 * H, 2 * H, C_), NAN, dtype=torch.float16, device=dev)

    def call():
        return _lib.load().asyrp_apply(_p(x), Ca, None, Cb, _p(aff), 2 * C_, _p(out), N, H, H, act, resample, _stream())

    def check():  # act = 0: exact (dyadic a, b); SiLU: within a few fp16 ulps
        want = x[..., :Ca].float() * 0.5 - 1.5
        if resample == 2:
            want = want.repeat_interleave(2, 1).repeat_interleave(2, 2)
        got = out.view(-1)[:want.numel()].view(want.shape).float()
        if act:
            assert (got - want * torch.sigmoid(want)).abs().max() < 1e-2
        else:
            assert torch.equal(got, want)
    return call, [out], check


def _pack(dev, Cin):
    x = torch.randn(1, Cin, 4, 4, device=dev)
    out = torch.full((1, 4, 4, 64), NAN, dtype=torch.float16, device=dev)

    def check():
        assert torch.equal(out[..., :Cin].float(), x.permute(0, 2, 3, 1).half().float())
        assert (out[..., Cin:] == 0).all()
    return lambda: _lib.load().asyrp_pack_input(_p(x), _p(out), 1, Cin, 4, 4, _stream()), [out], check


def _temb(dev, dim):
    t = torch.tensor([3.0, 500.0], device=dev)
    out = torch.full((2, max(dim, 1)), NAN, device=dev)

    def check():
        half = dim // 2
        f = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64) / (half - 1))
        arg = t.double().cpu()[:, None] * f[None]
        want = torch.cat([arg.sin(), arg.cos()], 1)
        assert (out.double().cpu() - want).abs().max() < 1e-3
    return lambda: _lib.load().asyrp_timestep_embedding(_p(t), _p(out), 2, dim, 0, _stream()), [out], check


def _axpby(dev, numel):
    a = (torch.arange(16, device=dev) % 5).half()
    b = (torch.arange(16, device=dev) % 7 - 3).half()
    out = torch.full((16,), NAN, dtype=torch.float16, device=dev)

    def check():
        want = 0.5 * a.float() - 2.0 * b.float()
        assert torch.equal(out[:numel].float(), want[:numel]) and torch.isnan(out[numel:]).all()
    return (lambda: _lib.load().asyrp_axpby(_p(a), _p(b), _p(out), 0.5, -2.0, numel, _stream()), [out], check)


def _slerp(dev, Cc, tiles):
    h = torch.randn(1, 4, 4, 8, device=dev).half()
    dh = torch.randn(1, 8, 4, 4, device=dev)
    out = torch.full((1, 4, 4, 8), NAN, dtype=torch.float16, device=dev)
    stats = torch.full((1, max(tiles, 1), 4, 2), NAN, device=dev)

    def call():
        return _lib.load().asyrp_slerp_h(_p(h), _p(dh), 0, _p(out), _p(stats), tiles, 1, Cc, 4, 4, 0.5, 0, _stream())
    return call, [out, stats], lambda: torch.isfinite(out.float()).all() or pytest.fail("slerp_h output not written")


def _ddpm(dev, z=True, Ce=3):
    x, z_ = torch.zeros(2, 3, 4, 4, device=dev), torch.zeros(2, 3, 4, 4, device=dev)
    et = torch.zeros(2, Ce, 4, 4, device=dev)
    out = torch.full((2, 3, 4, 4), NAN, device=dev)

    def call():
        return _lib.load().asyrp_ddpm_update(_p(x), _p(et), _p(z_) if z else None, _p(out), 2, 3, Ce, 16, 0.5, 0.1,
                                             -2.0, int(Ce == 6 or Ce == 5), 1.0, _stream())
    return call, [out], lambda: torch.isfinite(out).all() or pytest.fail("ddpm_update output not written")


def _transpose(dev, Cc, N=2, T=5):
    x = ((torch.arange(N * T * max(Cc, 32), device=dev) % 251) - 125).half().view(N, T, max(Cc, 32))
    out = torch.full((N, max(Cc, 32), T), NAN, dtype=torch.float16, device=dev)

    def check():
        for n in (0, N - 1):
            assert torch.equal(out[n], x[n].t())
    return (lambda: _lib.load().asyrp_transpose_tc(_p(x), _p(out), N, T, Cc, max(Cc, 32), _stream()), [out], check)


def _softmax(dev, T):
    S = torch.randn(3, max(T, 1), device=dev)
    out = torch.full((3, max(T, 1)), NAN, dtype=torch.float16, device=dev)

    def check():
        want = torch.softmax(S.double().cpu(), -1)
        assert (out.double().cpu() - want).abs().max() <= 2e-3 * want.max()
    return lambda: _lib.load().asyrp_softmax_rows(_p(S), _p(out), 3, T, 1.0, _stream()), [out], check


def _attention(dev, head_dim, N=2, T=16, heads=1):
    d = max(head_dim, 64)
    qkv = (torch.randn(N, T, 3 * heads * d, device=dev) * 0.5).half()
    out = torch.full((N, T, heads * d), NAN, dtype=torch.float16, device=dev)

    def check():
        for n in (0, N - 1):
            q, k, v = qkv[n].double().cpu().view(T, 3, heads, d).unbind(1)
            p = torch.softmax(torch.einsum("thd,shd->hts", q, k) / math.sqrt(d), -1)
            want = torch.einsum("hts,shd->thd", p, v).reshape(T, heads * d)
            assert (out[n].double().cpu() - want).abs().max() < 1e-2
    return (lambda: _lib.load().asyrp_attention(_p(qkv), _p(out), N, T, heads, head_dim, 1 / math.sqrt(d), _stream()),
            [out], check)


BIG = 65536  # one past the largest grid y / z dimension
# (row, entry point, message fragment, refused call, accepted call): one row per ASYRP_REQUIRE condition of the UNet's
# entry points in csrc/pointwise.cu and csrc/attention.cu; each maker returns (call, outputs, check of the result)
CALL_REFUSALS = [
    ("gn_finalize_c", "asyrp_gn_finalize", "C=32", lambda d: _gn(d, Ca=32), lambda d: _gn(d, Ca=64)),
    ("gn_finalize_n_big", "asyrp_gn_finalize", f"N={BIG}", lambda d: _gn(d, N=BIG), lambda d: _gn(d, N=BIG - 1)),
    ("gn_finalize_n_0", "asyrp_gn_finalize", "N=0", lambda d: _gn(d, N=0), lambda d: _gn(d, N=1)),
    ("apply_channels_8", "asyrp_apply", "multiples of 8", lambda d: _apply(d, Ca=12), lambda d: _apply(d, Ca=16)),
    ("apply_no_channels", "asyrp_apply", "channel count 0", lambda d: _apply(d, Ca=0), lambda d: _apply(d, Ca=8)),
    ("apply_2056_channels", "asyrp_apply", "channel count 2056", lambda d: _apply(d, Ca=2056, H=1),
     lambda d: _apply(d, Ca=2048, H=1)),
    ("apply_resample_3", "asyrp_apply", "resample=3", lambda d: _apply(d, resample=3),
     lambda d: _apply(d, resample=2)),
    ("apply_resample_neg", "asyrp_apply", "resample=-1", lambda d: _apply(d, resample=-1),
     lambda d: _apply(d, resample=0)),
    ("apply_act_2", "asyrp_apply", "act=2", lambda d: _apply(d, act=2), lambda d: _apply(d, act=1)),
    ("apply_act_neg", "asyrp_apply", "act=-1", lambda d: _apply(d, act=-1), lambda d: _apply(d, act=0)),
    ("apply_n_big", "asyrp_apply", f"N={BIG}", lambda d: _apply(d, N=BIG, H=1, Ca=8),
     lambda d: _apply(d, N=BIG - 1, H=1, Ca=8)),
    ("apply_n_0", "asyrp_apply", "N=0", lambda d: _apply(d, N=0), lambda d: _apply(d, N=1)),
    ("pack_input_cin", "asyrp_pack_input", "Cin=65", lambda d: _pack(d, 65), lambda d: _pack(d, 64)),
    ("temb_odd_dim", "asyrp_timestep_embedding", "odd dim 127", lambda d: _temb(d, 127), lambda d: _temb(d, 128)),
    ("axpby_numel", "asyrp_axpby", "multiple of 8", lambda d: _axpby(d, 12), lambda d: _axpby(d, 8)),
    ("slerp_odd_c", "asyrp_slerp_h", "bad arguments", lambda d: _slerp(d, 7, 1), lambda d: _slerp(d, 8, 1)),
    ("slerp_no_tiles", "asyrp_slerp_h", "bad arguments", lambda d: _slerp(d, 8, 0), lambda d: _slerp(d, 8, 1)),
    ("ddpm_no_noise", "asyrp_ddpm_update", "noise tensor required", lambda d: _ddpm(d, z=False), lambda d: _ddpm(d)),
    ("ddpm_learned_sigma", "asyrp_ddpm_update", "learned sigma", lambda d: _ddpm(d, Ce=5), lambda d: _ddpm(d, Ce=6)),
    ("transpose_c", "asyrp_transpose_tc", "C=48", lambda d: _transpose(d, 48), lambda d: _transpose(d, 64)),
    ("transpose_n_big", "asyrp_transpose_tc", f"N={BIG}", lambda d: _transpose(d, 32, N=BIG, T=1),
     lambda d: _transpose(d, 32, N=BIG - 1, T=1)),
    ("softmax_t_0", "asyrp_softmax_rows", "T=0", lambda d: _softmax(d, 0), lambda d: _softmax(d, 1)),
    ("softmax_t_1025", "asyrp_softmax_rows", "T=1025", lambda d: _softmax(d, 1025), lambda d: _softmax(d, 1024)),
    ("attention_head_dim", "asyrp_attention", "unsupported head_dim 96", lambda d: _attention(d, 96),
     lambda d: _attention(d, 64)),
    ("attention_n_big", "asyrp_attention", f"N={BIG}", lambda d: _attention(d, 64, N=BIG, T=1),
     lambda d: _attention(d, 64, N=BIG - 1, T=1)),
    ("attention_heads_0", "asyrp_attention", "heads=0", lambda d: _attention(d, 64, heads=0),
     lambda d: _attention(d, 64, heads=1)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row", CALL_REFUSALS, ids=[r[0] for r in CALL_REFUSALS])
def test_entry_point_refusals(cuda_device, row):
    name, entry, fragment, bad, good = row
    call, outs, _ = bad(cuda_device)
    torch.cuda.synchronize()
    with pytest.raises(_lib.AsyrpError, match=f"{entry}: .*{fragment}|{entry}: {fragment}") as exc:
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
# outputs past 2^31 elements
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_past_2_to_the_31_elements(cuda_device):
    """apply, axpby and a 1x1 conv over 257 samples of 256^2 x 128 fp16 (2^31 + 2^23 elements, 4 GiB per tensor; at
    most three live): exact integer operands, the first and last sample and every 16th between compared whole"""
    dev = cuda_device
    N, H, Cc = 257, 256, 128
    assert N * H * H * Cc > 2 ** 31
    per = N * H * H * Cc * 2
    _need_memory(3 * per + GiB, "the 2^31-element test")
    x = torch.empty(N, H, H, Cc, dtype=torch.float16, device=dev)
    _pattern(x, 0)
    samples = sorted({0, N - 1, *range(1, N - 1, 16)})

    def compare(out, want_fn, what):
        for n in samples:
            want = want_fn(n)
            assert torch.equal(out[n].float(), want), f"{what}: sample {n} of {N}"

    nn = torch.arange(N, device=dev).view(N, 1)
    cc = torch.arange(Cc, device=dev).view(1, Cc)
    a = torch.tensor([1.0, 0.5, -1.0, 2.0], device=dev)[(nn + cc) % 4]
    b = ((nn * 3 + cc) % 9 - 4).float()
    aff = torch.stack([a, b], -1).contiguous()
    y = torch.empty_like(x)
    y.view(-1)[-8:].fill_(NAN)
    ops.apply(x, None, aff, y, 0)
    torch.cuda.synchronize()
    compare(y, lambda n: x[n].float() * a[n] + b[n], "apply")
    z = torch.empty_like(x)
    ops.axpby(x, y, z, 0.5, -1.0)
    torch.cuda.synchronize()
    compare(z, lambda n: x[n].float() * 0.5 - y[n].float(), "axpby")
    del y
    o = torch.arange(Cc)
    w = torch.zeros(Cc, Cc, dtype=torch.float16)
    w[o, (o * 5 + 3) % Cc] = 1.0
    z.fill_(NAN)
    eb = ((nn * 5 + cc) % 17 - 8).float()
    ops.ConvOp([(x, ops.MODE_1x1)], w.to(dev), out=z, ebias=eb, ebias_stride=Cc).launch()
    torch.cuda.synchronize()
    perm = ((o * 5 + 3) % Cc).to(dev)
    compare(z, lambda n: x[n].float()[..., perm] + eb[n], "1x1 conv")
    del x, z
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    """the file's wall time and peak device memory, printed at the end (pytest -s)"""
    t0 = time.perf_counter()
    yield
    peak = torch.cuda.max_memory_allocated() / GiB if torch.cuda.is_available() else 0.0
    print(f"\ntest_unet_kernel_limits_gpu: {time.perf_counter() - t0:.1f} s, peak device memory {peak:.2f} GiB")
