"""Exact tests of the conv kernel's operand side: every tap, segment, sample and padding pixel each load path feeds to
the MMAs, and the fused operand transform per element.

test_conv_epilogue_coalesced_gpu.py checks the epilogue exactly on 1x1 convs; everything that forms the accumulators
(the 3x3 halo tile, the three dx-shifted copies, the stride-2 parity view, the up2 sub-pixel phases, concatenated and
sliced segments, the K schedule, batched weights with heads) is otherwise only checked against a tolerance relative to
max|ref|, which one wrong product in a few edge pixels can pass.  Here:

  * dense cases: operands are small integers, weights sparse {-1, 0, 1}, so every partial sum is an integer far below
    2^24 and every output an integer of magnitude <= VMAX: the result does not depend on the summation order, and the
    kernel's output is compared with `==` against an fp64 CPU reference;
  * one-hot cases: weight row o has a single 1, at K column k(o), so output channel o is exactly the operand element the
    MMA read for that column (segment, tap, source channel, shifted by the tap).  A few launches per case sweep k(o)
    over every K column of every segment; taps outside the image must give exactly 0;
  * the fused transform per element, through the one-hot gather: act = 0 with dyadic (a, b) must match bit for bit
    (up to the sign of zero); both SiLU forms are checked against a per-element bound (see _silu_bound); the in-kernel
    GroupNorm against fp64 GroupNorm of the int64 sums the producers wrote (see test_in_kernel_groupnorm_per_element).

Each case asserts the tile instantiation it exercises (ops.conv_tile_config, and conv_stats_tiles_up2 for up2, against
the host rule restated in _host_config) and at least two waves of tiles, fills the output with NaN plus one guard
sample behind it, and checks that a second launch gives the same bits.  A mismatch is reported as (sample, y, x, output
channel) with the tile that owns it: (tx, ty, tn, nt) of the TW x TH x NB tile shape, the sub-tile when MT = 2 and the
sub-pixel phase for up2.

The whole file takes about 25 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit.
"""
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

VMAX = 2048.0  # integers up to 2^11 are exact in fp16
U = 2.0 ** -24  # unit roundoff of fp32
NAN = float("nan")


def _ops():
    from asyrp_official_b200 import ops
    return ops


# ------------------------------------------------------------------------------------------------------------------
# tile geometry: the host rule of csrc/conv_gemm.cu (conv_tile_shape / conv_config), restated
# ------------------------------------------------------------------------------------------------------------------
def _tile_shape(H, W, halo):
    if halo:
        return 8, 16, 1
    tw = min(W, 128) if H == 1 else min(W, 16)
    th = 1 if H == 1 else min(128 // tw, 8, H)
    while 128 % (tw * th):
        th -= 1
    return tw, th, 128 // (tw * th)


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


class _Geom:
    """Tile geometry of a case.  spec: N (batch entries), H, W (the source's for up2), Cout, segs [(mode, C[, ld, off])]
    with mode "3x3" | "1x1" | "s2", inst (BN, MT), optional NB, up2."""

    def __init__(self, spec, dev):
        ops = _ops()
        self.N, self.H, self.W, self.Cout = spec["N"], spec["H"], spec["W"], spec["Cout"]
        self.up2 = spec.get("up2", False)
        has3 = any(sg[0] == "3x3" for sg in spec["segs"])
        halo = has3 and self.H % 16 == 0 and self.W % 8 == 0
        self.TW, self.TH, self.NB = _tile_shape(self.H, self.W, halo)
        assert self.NB == spec.get("NB", 1), (self.TW, self.TH, self.NB)
        self.BN, self.MT = _host_config(self.H, self.W, self.Cout, halo, 4 if self.up2 else 1)
        assert (self.BN, self.MT) == spec["inst"], (self.BN, self.MT)
        self.THT = self.TH * self.MT
        self.tiles_x, self.tiles_y = -(-self.W // self.TW), -(-self.H // self.THT)
        if self.up2:
            slots = ops.conv_stats_tiles_up2(self.H, self.W, self.Cout)
            assert slots == self.tiles_x * self.tiles_y * 4, slots
        else:
            assert ops.conv_tile_config(self.H, self.W, self.Cout, has3) == spec["inst"], \
                ops.conv_tile_config(self.H, self.W, self.Cout, has3)
        self.tiles = self.tiles_x * self.tiles_y * -(-self.N // self.NB) * (self.Cout // self.BN) * (4 if self.up2 else 1)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        assert self.tiles >= 2 * sms, f"{self.tiles} tiles on {sms} SMs: fewer than two waves"
        self.Ho, self.Wo = (2 * self.H, 2 * self.W) if self.up2 else (self.H, self.W)

    def locate(self, n, y, x, o):
        """the tile that writes output element (sample, y, x, channel)"""
        ph = 0
        if self.up2:
            ph, y, x = (y % 2) * 2 + x % 2, y // 2, x // 2
        nt = ph * (self.Cout // self.BN) + o // self.BN
        s = f"tile (tx={x // self.TW}, ty={y // self.THT}, tn={n // self.NB}, nt={nt})"
        if self.MT == 2:
            s += f" sub-tile {(y % self.THT) // self.TH}"
        if self.up2:
            s += f" phase (a={ph // 2}, b={ph % 2})"
        return s


def _report(geom, bad, got, want, what, extra=None):
    """fail with the first mismatching elements, located"""
    nbad = int(bad.sum())
    if nbad == 0:
        return
    lines = []
    for n, y, x, o in bad.nonzero()[:8].tolist():
        line = f"(n={n}, y={y}, x={x}, o={o}) {geom.locate(n, y, x, o)}: got {got[n, y, x, o].item()!r}, " \
               f"want {want[n, y, x, o].item()!r}"
        if extra is not None:
            line += f" ({extra(n, y, x, o)})"
        lines.append(line)
    pytest.fail(f"{what}: {nbad} of {got.numel()} elements wrong; first:\n  " + "\n  ".join(lines))


class _Out:
    """The output of a case, NaN-filled with one guard sample behind it; launch() runs the op and returns the output as
    [N][Ho][Wo][Cout] (planar: [N][H][W][planar channels]) fp64 on the CPU."""

    def __init__(self, geom, dev, planar=None, f32=False):
        self.planar = planar
        if planar:
            self.full = torch.full((geom.N + 1, planar, geom.H, geom.W), NAN, dtype=torch.float32, device=dev)
            self.kw = dict(out_planar=self.full[:-1], out_shape=(geom.N, geom.H, geom.W, geom.Cout))
        else:
            self.full = torch.full((geom.N + 1, geom.Ho, geom.Wo, geom.Cout), NAN,
                                   dtype=torch.float32 if f32 else torch.float16, device=dev)
            self.kw = dict(out=self.full[:-1])

    def launch(self, op, twice=False):
        self.full.fill_(NAN)
        op.launch()
        torch.cuda.synchronize()
        assert torch.isnan(self.full[-1]).all(), "the guard sample behind the output was written"
        got = self.full[:-1].double().cpu()
        if twice:
            bits = torch.int32 if self.full.dtype == torch.float32 else torch.int16
            first = self.full.clone()
            self.full.fill_(NAN)
            op.launch()
            torch.cuda.synchronize()
            assert torch.equal(first.view(bits), self.full.view(bits)), "a second launch gives different bits"
        return got.permute(0, 2, 3, 1) if self.planar else got


def _ints(g, shape, lo, hi, nonzero=False):
    v = torch.randint(lo, hi + 1, shape, generator=g)
    if nonzero:
        v = torch.where(v == 0, torch.full_like(v, hi), v)
    return v.double()


def _source(seg, vals, dev, g):
    """device fp16 source of a segment holding `vals` ([N][Hs][Ws][C] fp64): a channel slice [off, off+C) of a wider
    NHWC tensor of pixel pitch ld when the segment gives (ld, off), else dense"""
    mode, C = seg[0], seg[1]
    ld, off = (seg[2], seg[3]) if len(seg) > 2 else (C, 0)
    full = torch.randn(*vals.shape[:3], ld, generator=g).to(torch.float16)  # channels around the slice: never read
    full[..., off:off + C] = vals.to(torch.float16)
    assert torch.equal(full[..., off:off + C].double(), vals), "operand not exact in fp16"
    return full.to(dev)[..., off:off + C]


def _src_shape(seg, geom):
    return (geom.N, 2 * geom.H, 2 * geom.W, seg[1]) if seg[0] == "s2" else (geom.N, geom.H, geom.W, seg[1])


_MODE = {"3x3": 1, "1x1": 0, "s2": 2}  # ops.MODE_*


# ------------------------------------------------------------------------------------------------------------------
# the gather reference: what the MMA reads for K column k
# ------------------------------------------------------------------------------------------------------------------
def _column(geom, segs, col):
    """K column -> (segment, ky, kx, source channel): tap-major, channel-minor per segment (up2: the 2x2 taps of a
    phase, (dy, dx))"""
    for s, seg in enumerate(segs):
        taps = 1 if seg[0] == "1x1" else (4 if geom.up2 else 9)
        if col < taps * seg[1]:
            tap, c = divmod(col, seg[1])
            kw = 2 if geom.up2 else 3
            return s, tap // kw, tap % kw, c
        col -= taps * seg[1]
    raise AssertionError("column past K")


def _gather(geom, segs, srcs, rows, pad):
    """sum over row r's (column, weight) entries of weight * the element that column reads, [N][Ho][Wo][Cout] fp64.
    srcs: per segment [N][Hs][Ws][C] (the operand after any transform, or its pre-activation); out-of-image taps read
    `pad`.  rows: one list per weight row (up2: 4 * Cout rows, phase-major)"""
    N, H, W = geom.N, geom.H, geom.W
    out = torch.zeros(N, geom.Ho, geom.Wo, geom.Cout, dtype=torch.float64)
    for r, entries in enumerate(rows):
        ph, o = divmod(r, geom.Cout)
        for col, wv in entries:
            s, ky, kx, c = _column(geom, segs, col)
            mode = segs[s][0]
            ch = srcs[s][..., c].double()
            if mode == "3x3":
                ch = F.pad(ch, (1, 1, 1, 1), value=pad)
            elif mode == "s2":
                ch = F.pad(ch, (0, 1, 0, 1), value=pad)
            if geom.up2:
                a, b = divmod(ph, 2)
                out[:, a::2, b::2, o] += wv * ch[:, a + ky:a + ky + H, b + kx:b + kx + W]
            elif mode == "3x3":
                out[..., o] += wv * ch[:, ky:ky + H, kx:kx + W]
            elif mode == "s2":
                out[..., o] += wv * ch[:, ky:ky + 2 * H:2, kx:kx + 2 * W:2]
            else:
                out[..., o] += wv * ch
    return out


def _row(geom, y, x, o):
    """weight row of output element (y, x, o): up2 rows are phase-major"""
    return ((y % 2) * 2 + x % 2) * geom.Cout + o if geom.up2 else o


def _ktot(geom, segs):
    return sum(seg[1] * (1 if seg[0] == "1x1" else (4 if geom.up2 else 9)) for seg in segs)


def _one_hot_sweep(geom, segs, g):
    """launches x rows of column indices: every K column appears at least once, in a random order"""
    K = _ktot(geom, segs)
    nrows = geom.Cout * (4 if geom.up2 else 1)
    rows_per_phase = geom.Cout
    launches = -(-K // rows_per_phase)
    perm = torch.randperm(K, generator=g)
    sweep = []
    for L in range(launches):
        cols = perm[(L * rows_per_phase + torch.arange(rows_per_phase)) % K]
        if geom.up2:  # every phase sees every column; each phase in its own order
            cols = torch.cat([cols.roll(37 * p) for p in range(4)])
        assert cols.numel() == nrows
        sweep.append(cols.tolist())
    return sweep


def _one_hot_weight(cols, K):
    w = torch.zeros(len(cols), K, dtype=torch.float16)
    w[torch.arange(len(cols)), torch.tensor(cols)] = 1.0
    return w


# ------------------------------------------------------------------------------------------------------------------
# 2. dense exact cases
# ------------------------------------------------------------------------------------------------------------------
DENSE = {
    # mode 3: one halo tile per chunk, every edge mask; 384 tiles
    "halo128": dict(inst=(128, 1), N=6, H=64, W=64, Cout=256, segs=[("3x3", 64)]),
    # MT = 2, two heavy segments (a channel concat); 272 tiles
    "halo64x2_concat": dict(inst=(64, 2), N=17, H=64, W=64, Cout=64, segs=[("3x3", 64), ("3x3", 64)]),
    # separate light ring, spread K schedule, three segments; 320 tiles
    "halo_light_rings": dict(inst=(64, 1), N=40, H=16, W=16, Cout=256,
                             segs=[("3x3", 256), ("1x1", 256), ("1x1", 128)]),
    # mode 1 (three dx-shifted copies): partial x tiles (W 40 in 16-wide tiles); 270 tiles
    "copies128_ragged_x": dict(inst=(128, 1), N=30, H=24, W=40, Cout=128, segs=[("3x3", 64)]),
    # ... partial x and y tiles (W 24, H 20 in 16 x 8 tiles); 288 tiles
    "copies64_ragged_xy": dict(inst=(64, 1), N=24, H=20, W=24, Cout=128, segs=[("3x3", 64)]),
    # tiles of two 8x8 samples, N odd: the last tile's second sample is past N; 272 tiles
    "nb2": dict(inst=(64, 1), NB=2, N=67, H=8, W=8, Cout=512, segs=[("3x3", 64)]),
    # tiles of eight 4x4 samples, N = 8*33 + 1; 272 tiles
    "nb8": dict(inst=(64, 1), NB=8, N=265, H=4, W=4, Cout=512, segs=[("3x3", 64)]),
    # mode 2: stride 2, pad (0,1,0,1), parity view of the 64x64 source; 320 tiles
    "s2": dict(inst=(128, 1), N=40, H=32, W=32, Cout=128, segs=[("s2", 64)]),
    # up2: four sub-pixel phases over a 16x16 source; 272 tiles
    "up2": dict(inst=(128, 1), up2=True, N=34, H=16, W=16, Cout=128, segs=[("3x3", 64)]),
    # conv_out: BN = 16, fp32 planar store of 3 / 6 channels; 288 / 320 tiles
    "conv_out16x1": dict(inst=(16, 1), N=48, H=24, W=24, Cout=16, planar=3, segs=[("3x3", 64)]),
    "conv_out16x2": dict(inst=(16, 2), N=20, H=64, W=64, Cout=16, planar=6, segs=[("3x3", 64)]),
    # channel slices of wider NHWC tensors (TMA pixel pitch != C): a halo 3x3 and a 1x1 (light ring); 264 tiles
    "slices_halo": dict(inst=(64, 1), N=66, H=16, W=16, Cout=128, segs=[("3x3", 64, 192, 64), ("1x1", 64, 160, 32)]),
    # ... a dx-copy 3x3 and a 1x1 on a ragged layer; 270 tiles
    "slices_copies": dict(inst=(64, 1), N=45, H=20, W=24, Cout=64, segs=[("3x3", 64, 136, 8), ("1x1", 128, 200, 64)]),
}


@pytest.mark.parametrize("case", list(DENSE))
def test_dense_exact(cuda_device, case):
    ops = _ops()
    dev = cuda_device
    spec = DENSE[case]
    t0 = time.perf_counter()
    geom = _Geom(spec, dev)
    g = torch.Generator().manual_seed(300 + list(DENSE).index(case))
    segs = spec["segs"]
    acc, wparts, conv_segs, l1 = 0.0, [], [], 0.0
    for seg in segs:
        x = _ints(g, _src_shape(seg, geom), -3, 3)  # every sample its own draws
        k = 1 if seg[0] == "1x1" else 3
        w = _ints(g, (geom.Cout, seg[1], k, k), -1, 1) * (torch.rand(geom.Cout, seg[1], k, k, generator=g) < 0.15)
        l1 = l1 + w.abs().sum(dim=(1, 2, 3)).max().item() * 3.0
        conv_segs.append((_source(seg, x, dev, g), _MODE[seg[0]]))
        xn = x.permute(0, 3, 1, 2)
        if geom.up2:
            wparts.append(ops.pack_upconv_weight(w))  # sums of integer taps: still integers
            acc = acc + F.conv2d(F.interpolate(xn, scale_factor=2.0, mode="nearest"), w, padding=1)
        else:
            wparts.append(ops.pack_conv_weight(w))
            if seg[0] == "s2":
                acc = acc + F.conv2d(F.pad(xn, (0, 1, 0, 1)), w, stride=2)
            else:
                acc = acc + F.conv2d(xn, w, padding=k // 2)
    weight = torch.cat(wparts, -1)
    assert torch.equal(weight.double(), weight.double().round()), "packed weights not integer"
    want = acc.permute(0, 2, 3, 1)
    assert l1 < 2 ** 24, l1  # every partial sum is an integer below 2^24: exact in fp32 in any order
    if spec.get("planar"):
        want = want[..., :spec["planar"]]
    assert want.abs().max().item() <= VMAX, want.abs().max().item()

    out = _Out(geom, dev, planar=spec.get("planar"))
    op = ops.ConvOp(conv_segs, weight.to(dev), up2=geom.up2, **out.kw)
    got = out.launch(op, twice=True)
    _report(geom, got != want, got, want, case)
    print(f"{case}: {geom.tiles} tiles, {time.perf_counter() - t0:.2f} s")


def test_attention_gemms_exact(cuda_device):
    """Batched weights: T = 200 rows (a partial 128-row tile) against per-sample weights that are a column slice of a
    wider row (weight_ld = 3C, k as a slice of qkv); T = 384 with two heads (a_heads = b_heads = 2: 64-channel slices
    of one qkv tensor in both TMA maps), fp32 output"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(320)
    # T = 200: out[n][t][o] = sum_k A[n][t][k] * wide[n][o][C + k]
    N, T, C, Cout = 36, 200, 128, 256
    geom = _Geom(dict(inst=(64, 1), N=N, H=1, W=T, Cout=Cout, segs=[("1x1", C)]), dev)
    A = _ints(g, (N, 1, T, C), -3, 3)
    wide = _ints(g, (N, Cout, 3 * C), -1, 1) * (torch.rand(N, Cout, 3 * C, generator=g) < 0.3)
    want = torch.einsum("ntk,nok->nto", A[:, 0], wide[..., C:2 * C])[:, None]
    assert want.abs().max().item() <= VMAX
    out = _Out(geom, dev)
    wd = wide.to(torch.float16).to(dev)
    op = ops.ConvOp([(A.to(torch.float16).to(dev), ops.MODE_1x1)], wd[..., C:2 * C], weight_batched=True, **out.kw)
    got = out.launch(op, twice=True)
    _report(geom, got != want, got, want, "T=200, weight_ld = 3C")

    # T = 384, two heads: S[2n + h][t][s] = q_h[n][t] . k_h[n][s], q_h / k_h channels [64h, 64h+64) of q / k
    N, T, heads, d = 15, 384, 2, 64
    Cq = heads * d
    geom = _Geom(dict(inst=(128, 1), N=N * heads, H=1, W=T, Cout=T, segs=[("1x1", d)]), dev)
    qkv = _ints(g, (N, T, 3 * Cq), -3, 3)
    q = qkv[..., :Cq].reshape(N, T, heads, d).permute(0, 2, 1, 3)
    k = qkv[..., Cq:2 * Cq].reshape(N, T, heads, d).permute(0, 2, 1, 3)
    want = (q @ k.transpose(-1, -2)).reshape(N * heads, 1, T, T)
    out = _Out(geom, dev, f32=True)
    qd = qkv.to(torch.float16).to(dev)
    op = ops.ConvOp([(qd.view(N, 1, T, 3 * Cq)[..., :d], ops.MODE_1x1)], qd[:, :, Cq:Cq + d], weight_batched=True,
                    a_heads=heads, b_heads=heads, **out.kw)
    got = out.launch(op, twice=True)
    _report(geom, got != want, got, want, "T=384, a_heads = b_heads = 2")


def test_k_schedule_limit(cuda_device):
    """64 K-schedule entries (3x3 of 2048 + 1x1 of 2048 channels on 16x16: 32 heavy chunks spread with 32 light ones)
    are the most a conv takes; weight row o has two +-1 entries, in chunk o and chunk o + 17 (mod 64), so every entry
    of the schedule, the last one included, carries a product into two output channels.  65 entries raise."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(321)
    segs = [("3x3", 2048), ("1x1", 2048)]
    geom = _Geom(dict(inst=(64, 1), N=132, H=16, W=16, Cout=64, segs=segs), dev)
    xs = [torch.randint(-3, 4, _src_shape(seg, geom), generator=g, dtype=torch.int8) for seg in segs]
    K = _ktot(geom, segs)

    def col_in_chunk(chunk):  # a random column of 64-channel chunk `chunk` (heavy chunks first), random tap
        if chunk < 32:
            return int(torch.randint(0, 9, (1,), generator=g)) * 2048 + chunk * 64 + int(torch.randint(0, 64, (1,), generator=g))
        return 9 * 2048 + (chunk - 32) * 64 + int(torch.randint(0, 64, (1,), generator=g))

    rows = [[(col_in_chunk(o), 1.0 - 2.0 * (o % 2)), (col_in_chunk((o + 17) % 64), 1.0)] for o in range(64)]
    weight = torch.zeros(64, K, dtype=torch.float16)
    for o, entries in enumerate(rows):
        for col, wv in entries:
            weight[o, col] = wv
    want = _gather(geom, segs, xs, rows, 0.0)
    out = _Out(geom, dev)
    op = ops.ConvOp([(x.to(torch.float16).to(dev), _MODE[seg[0]]) for seg, x in zip(segs, xs)], weight.to(dev),
                    **out.kw)
    got = out.launch(op, twice=True)
    _report(geom, got != want, got, want, "64 K-schedule entries")
    del op
    with pytest.raises(ops._lib.AsyrpError, match="64 K chunks"):
        ops.ConvOp([(torch.zeros(1, 16, 16, 2048, dtype=torch.float16, device=dev), ops.MODE_3x3),
                    (torch.zeros(1, 16, 16, 2112, dtype=torch.float16, device=dev), ops.MODE_1x1)],
                   torch.zeros(64, 9 * 2048 + 2112, dtype=torch.float16, device=dev),
                   out=torch.empty(1, 16, 16, 64, dtype=torch.float16, device=dev))


# ------------------------------------------------------------------------------------------------------------------
# 3. one-hot gather cases and 4. the fused transform per element
# ------------------------------------------------------------------------------------------------------------------
GATHER = {k: DENSE[k] for k in ("halo128", "halo_light_rings", "copies128_ragged_x", "copies64_ragged_xy", "nb2",
                                "nb8", "s2", "up2")}
# transforms per geometry: the halo tiles reach transform_fast (interior tiles unmasked, edge tiles with the h_l / h_r
# / h_t / h_b masks; the 1x1 segments of the light ring with the plain masks), the dx copies transform_pixels, the
# NB > 1 tiles the per-pixel path with each sample's affine row, up2 the halo path with the phase's taps
TRANSFORMS = {"halo128": ("raw", "act0", "tanh", "ex2"), "halo_light_rings": ("raw", "act0"),
              "copies128_ragged_x": ("raw", "act0", "tanh", "ex2"), "copies64_ragged_xy": ("raw", "act0", "tanh"),
              "nb2": ("raw", "act0", "tanh", "ex2"), "nb8": ("raw", "act0", "tanh"), "s2": ("raw",),
              "up2": ("raw", "act0", "tanh")}
WORST = {}  # form -> (worst observed fraction of the per-element bound, case)


def _silu_bound(y, form):
    """(silu(y), per-element bound of |kernel - silu(y)|) in fp64, for the kernel's SiLU of the fp32 y = fma(a, x, b).

    Both forms: y itself is rounded to fp32 (|silu'(y)| * 2^-24 |y|), and the result is rounded to fp16 (2^-11 of its
    magnitude, or 2^-25 absolute below the fp16 normal range).
    tanh form, silu(y) = h + h * tanh.approx(h) with h = y/2 (the 1/2 is exact): ptx.cuh's contract for tanh.approx.f32
    (relative error <= 2^-11, so |h| * 2^-11 |tanh(h)| <= 2^-12 |y|, an error absolute in |y| and not relative to the
    result), plus the fp32 rounding of the fma (2^-24 of its result).  In the negative tail this dominates: at y = -6
    it is 1.5e-3 on silu(-6) = -0.0148.
    ex2 + rcp form, y * rcp.approx(1 + ex2.approx(-y log2 e)): the PTX ISA gives ex2.approx.ftz.f32 and
    rcp.approx.ftz.f32 maximum relative errors of about 2^-22 and 2^-23; the bound takes 2^-22 for each.  The fp32
    argument -y log2 e carries 2^-23 |y log2 e| absolute error, i.e. 2^-23 |y| relative error in e; the sum 1 + e and
    the product y * r add one fp32 rounding each.  sigma = 1/(1 + e) inherits the relative error of e times (1 - sigma)
    <= 1, so the result's relative error is <= 2^-22 + 2^-23 |y| + 2^-22 + 2 * 2^-24 = (5 + |y|) 2^-23; the bound
    takes (6 + |y|) 2^-23.  With ftz, results below 2^-126 flush to zero, inside the 2^-25 term.

    Worst observed |error| / bound on an NVIDIA H100 80GB HBM3 (700 W power limit), over every GATHER case: 0.76 for
    the tanh form, 0.9995 for the ex2 + rcp form (whose bound is almost all fp16 rounding)."""
    sg = torch.sigmoid(y)
    s = y * sg
    e_in = (sg * (1 + y * (1 - sg))).abs() * y.abs() * U
    if form == "tanh":
        e = 2.0 ** -12 * y.abs() + U * (s.abs() + 2.0 ** -12 * y.abs()) + e_in
    else:
        e = (6.0 + y.abs()) * 2.0 ** -23 * s.abs() + e_in
    return s, e + 2.0 ** -11 * (s.abs() + e) + 2.0 ** -25


def _transform_operands(geom, segs, form, g):
    """per segment: the source x ([N][Hs][Ws][C] fp64, exact in fp16), the affine table slice (a, b) [N][C] and the
    pre-activation y = a*x + b in fp64 (exact for act = 0; for SiLU exact before the kernel's fp32 rounding)"""
    xs, affs, ys = [], [], []
    for seg in segs:
        shape = _src_shape(seg, geom)
        N, C = shape[0], shape[-1]
        if form == "raw":
            x = _ints(g, shape, -1000, 1000, nonzero=True)  # a nonzero element is never mistaken for padding
            xs.append(x)
            affs.append(None)
            ys.append(x)
            continue
        if form == "act0":  # |a x + b| <= 244.5: multiples of 1/4 below 256, exact in fp16
            x = _ints(g, shape, -120, 120)
            a = torch.tensor([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0])[torch.randint(0, 6, (N, C), generator=g)]
            b = _ints(g, (N, C), 1, 18) * 0.25 * (1 - 2 * torch.randint(0, 2, (N, C), generator=g))  # b != 0
        else:  # y over about [-30, 30], +-0, and |y| up to about 1e4
            x = (torch.rand(shape, generator=g) * 24 - 12).to(torch.float16).double()
            u = torch.rand(shape, generator=g)
            big = ((torch.rand(shape, generator=g) * 4000 + 1000) * torch.sign(torch.randn(shape, generator=g)))
            x = torch.where(u < 0.02, big.to(torch.float16).double(), x)
            x = torch.where((u >= 0.02) & (u < 0.04), torch.zeros_like(x), x)
            x = torch.where((u >= 0.04) & (u < 0.06), torch.full_like(x, -0.0), x)
            # a, b on coarse grids: a*x + b is exact in fp64, so the fp32 y the kernel forms is one rounding of it
            a = (torch.rand(N, C, generator=g) * 1.5 + 0.5) * torch.sign(torch.randn(N, C, generator=g))
            a = (a * 4096).round() / 4096
            b = ((torch.rand(N, C, generator=g) * 12 - 6) * 65536).round() / 65536
            sel = torch.rand(N, C, generator=g)
            b = torch.where(sel < 0.125, torch.full_like(b, -0.0), torch.where(sel < 0.25, torch.zeros_like(b), b))
        xs.append(x)
        affs.append((a, b))
        ys.append(x * a[:, None, None, :] + b[:, None, None, :])
    return xs, affs, ys


@pytest.mark.parametrize("case", list(GATHER))
def test_one_hot_gather(cuda_device, case):
    """Every K column of every segment, for the raw operand and each fused transform the geometry reaches (see
    TRANSFORMS): act = 0 bit for bit (up to the sign of zero), SiLU within _silu_bound, padding exactly 0"""
    ops = _ops()
    lib = ops._lib.load()
    dev = cuda_device
    spec = GATHER[case]
    t0 = time.perf_counter()
    geom = _Geom(spec, dev)
    segs = spec["segs"]
    K = _ktot(geom, segs)
    g = torch.Generator().manual_seed(400 + list(GATHER).index(case))
    for form in TRANSFORMS[case]:
        xs, affs, ys = _transform_operands(geom, segs, form, g)
        conv_segs, a_off = [], 0
        aff_tab = None
        if form != "raw":
            aff_tab = torch.cat([torch.stack(ab, -1) for ab in affs], 1).float().contiguous().to(dev)
        act = {"raw": 0, "act0": 0, "tanh": 1, "ex2": 1}[form]
        for seg, x in zip(segs, xs):
            src = _source(seg, x, dev, g)
            if form == "raw":
                conv_segs.append((src, _MODE[seg[0]]))
            else:
                conv_segs.append((src, _MODE[seg[0]], aff_tab, a_off, act))
                a_off += seg[1]
        sweep = _one_hot_sweep(geom, segs, g)
        wbuf = torch.empty(len(sweep[0]), K, dtype=torch.float16, device=dev)
        out = _Out(geom, dev)
        if form in ("tanh", "ex2"):
            lib.asyrp_set_silu_tanh(1 if form == "tanh" else 0)
        try:
            op = ops.ConvOp(conv_segs, wbuf, up2=geom.up2, **out.kw)
        finally:
            lib.asyrp_set_silu_tanh(-1)
        worst = 0.0
        for L, cols in enumerate(sweep):
            wbuf.copy_(_one_hot_weight(cols, K))
            got = out.launch(op, twice=(L == 0))
            pre = _gather(geom, segs, ys, [[(c, 1.0)] for c in cols], NAN)  # NaN: the tap is outside the image
            pad = torch.isnan(pre)
            what = f"{case}, {form}, launch {L}"
            if form in ("raw", "act0"):
                want = torch.where(pad, torch.zeros_like(pre), pre)
                assert torch.equal(want.to(torch.float16).double(), want), "operand not exact in fp16"
                _report(geom, got != want, got, want, what, extra=lambda n, y, x, o:
                        f"(segment, ky, kx, channel) of its column: {_column(geom, segs, cols[_row(geom, y, x, o)])}")
                continue
            yv = torch.where(pad, torch.zeros_like(pre), pre)
            s, bound = _silu_bound(yv, form)
            err = (got - s).abs()
            _report(geom, pad & (got != 0), got, torch.zeros_like(got), what + ": padding")
            _report(geom, ~pad & ~(err <= bound), got, s, what, extra=lambda n, y, x, o: f"y = {yv[n, y, x, o].item()!r}, "
                    f"bound {bound[n, y, x, o].item():.3e}")
            # where tanh(y/2) and 1/(1 + e^-y) round to exactly 1 in fp32, both forms return the fp32 y itself: the
            # fp16 conversion must then be the round-to-nearest of the fp32 y
            sat = ~pad & (yv >= 32.0)
            want_sat = yv.float().half().double()
            _report(geom, sat & (got != want_sat), got, want_sat, what + ": saturated SiLU (y >= 32)")
            assert sat.sum() > 1000
            frac = torch.where(pad, torch.zeros_like(err), err / bound)
            worst = max(worst, frac.max().item())
        if form in ("tanh", "ex2"):
            print(f"{case}: {form} SiLU, worst |err| / bound {worst:.3f}")
            if worst > WORST.get(form, (0.0, ""))[0]:
                WORST[form] = (worst, case)
    print(f"{case}: {geom.tiles} tiles, {time.perf_counter() - t0:.2f} s; worst fractions so far {WORST}")


def test_in_kernel_groupnorm_per_element(cuda_device):
    """In-kernel GroupNorm (GNSpec) over the concat of two producers, with scale / shift, act = 0, one-hot weights: the
    output is fp16(a x + b) with (a, b) the kernel's fp32 finalise of the int64 sums.  The reference computes fp64
    GroupNorm from the very sums the producers wrote, read back from the device, so only the kernel's fp32 finalise
    and transform are measured, not the fixed-point quantisation.  H*W * channels per group is a power of two, so the
    kernel's fp32 1/count is exact.

    Bound per element: mean and rstd are rounded to fp32, a = gamma rstd (1 + scale), b = (beta - mean a0)(1 + scale)
    + shift and y = fma(a, x, b) take at most eight further fp32 roundings, each <= 2^-24 of one of |a x|, |mean a|,
    |beta (1 + scale)|, |shift|, |y|: E = 2^-21 (|a x| + |mean a| + |beta (1 + scale)| + |shift| + |y|); then the fp16
    rounding, 2^-11 (|y| + E) + 2^-25.  Group 3 has |mean| / std of about 30: there y = a (x - mean) + beta cancels and
    E, not the fp16 rounding, dominates.

    On an NVIDIA H100 80GB HBM3 (700 W power limit) the worst observed |error| / bound is 0.996, and the largest error
    in group 3 is 1.9e-3."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(500)
    spec = dict(inst=(64, 1), N=33, H=16, W=16, Cout=256, segs=[("3x3", 64), ("3x3", 64)])
    geom = _Geom(spec, dev)
    N, H, W = geom.N, geom.H, geom.W
    Cg, cpg = 128, 4
    assert (H * W * cpg) & (H * W * cpg - 1) == 0
    srcs, sums = [], []
    for i in range(2):
        xin = torch.randn(N, 64, H, W, generator=g)
        w = torch.randn(64, 64, 1, 1, generator=g) * 0.3
        b = torch.randn(64, generator=g)
        if i == 0:
            b[12:16] += 30.0 * 2.4  # group 3 (concat channels 12..15): producer std ~ 0.3 * sqrt(64) = 2.4
        out = torch.empty(N, H, W, 64, dtype=torch.float16, device=dev)
        sm = ops.new_sums(N, 64, dev)
        ops.ConvOp([(xin.permute(0, 2, 3, 1).contiguous().half().to(dev), ops.MODE_1x1)],
                   ops.pack_conv_weight(w).to(dev), out=out, ebias=b.to(dev), stats=ops.new_stats(N, H, W, 64, dev, False),
                   sums_out=sm).launch()
        srcs.append(out)
        sums.append(sm)
    torch.cuda.synchronize()
    gamma = torch.randn(Cg, generator=g) * 0.3 + 1.0
    beta = torch.randn(Cg, generator=g) * 0.3
    wide = torch.randn(N, 2 * Cg + 5, generator=g) * 0.3
    eps = 1e-5
    ssd = wide.to(dev)[:, 3:3 + 2 * Cg]
    gn = ops.GNSpec(sums, [64, 64], gamma.to(dev), beta.to(dev), eps, H * W, ssd, 2 * Cg + 5)

    # fp64 GroupNorm from the device's int64 sums
    st = torch.cat([s.cpu() for s in sums], 1).double() / ops.STAT_SCALE  # [N][64 pairs][2]
    grp = st.reshape(N, 32, cpg // 2, 2).sum(2)
    count = H * W * cpg
    mean = grp[..., 0] / count
    var = (grp[..., 1] / count - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    a0 = gamma.double() * rstd.repeat_interleave(cpg, 1)
    sc = 1.0 + wide[:, 3:3 + Cg].double()
    sh = wide[:, 3 + Cg:3 + 2 * Cg].double()
    meanc = mean.repeat_interleave(cpg, 1)
    a = a0 * sc
    b = (beta.double() - meanc * a0) * sc + sh
    mag_const = (meanc * a).abs() + (beta.double() * sc).abs() + sh.abs()  # [N][Cg]
    xs = [s.double().cpu() for s in srcs]
    ys = [x * a[:, None, None, 64 * i:64 * i + 64] + b[:, None, None, 64 * i:64 * i + 64] for i, x in enumerate(xs)]
    axs = [(x * a[:, None, None, 64 * i:64 * i + 64]).abs() + mag_const[:, None, None, 64 * i:64 * i + 64]
           for i, x in enumerate(xs)]
    print(f"group 3: |mean| / std = {(mean[:, 3].abs() * rstd[:, 3]).min().item():.1f} .. "
          f"{(mean[:, 3].abs() * rstd[:, 3]).max().item():.1f}")

    segs = spec["segs"]
    K = _ktot(geom, segs)
    wbuf = torch.empty(geom.Cout, K, dtype=torch.float16, device=dev)
    out = _Out(geom, dev)
    op = ops.ConvOp([(srcs[0], ops.MODE_3x3, gn, 0, 0), (srcs[1], ops.MODE_3x3, gn, 64, 0)], wbuf, **out.kw)
    worst, worst_g3 = 0.0, 0.0
    for L, cols in enumerate(_one_hot_sweep(geom, segs, g)):
        wbuf.copy_(_one_hot_weight(cols, K))
        got = out.launch(op, twice=(L == 0))
        rows = [[(c, 1.0)] for c in cols]
        pre = _gather(geom, segs, ys, rows, NAN)
        mag = _gather(geom, segs, axs, rows, 0.0)
        pad = torch.isnan(pre)
        y = torch.where(pad, torch.zeros_like(pre), pre)
        e = 2.0 ** -21 * (mag + y.abs())
        bound = e + 2.0 ** -11 * (y.abs() + e) + 2.0 ** -25
        err = (got - y).abs()
        what = f"in-kernel GroupNorm, launch {L}"
        _report(geom, pad & (got != 0), got, torch.zeros_like(got), what + ": padding")
        _report(geom, ~pad & ~(err <= bound), got, y, what,
                extra=lambda n, yy, xx, o: f"bound {bound[n, yy, xx, o].item():.3e}")
        frac = torch.where(pad, torch.zeros_like(err), err / bound)
        worst = max(worst, frac.max().item())
        g3 = torch.tensor([_column(geom, segs, c)[0] == 0 and 12 <= _column(geom, segs, c)[3] < 16 for c in cols])
        if g3.any():
            worst_g3 = max(worst_g3, err[..., g3].max().item())
    print(f"in-kernel GroupNorm: worst |err| / bound {worst:.3f}; worst |err| in group 3 {worst_g3:.3e}")
