"""Exact tests of the conv kernel's epilogue on every tile geometry and output mode the benchmark plans launch.

test_conv_epilogue_coalesced_gpu.py checks the epilogue exactly on 1x1 convs with raw operands, and
test_conv_operands_exact_gpu.py checks the 3x3 halo tiles, up2, stride 2 and the fused transform exactly, but the output
only.  The convs the plans launch most often combine all of it: a fused GroupNorm-apply 3x3 operand whose transform the
epilogue interleaves with (drain_at), a per-sample bias row, a residual (res_mode 0, or 1 / 2 for the ADM up / down
blocks), device scales and per-tile GroupNorm statistics.  Here every case sets every epilogue feature its geometry
allows at once:

  * operands are small integers (a fused operand: act = 0 with dyadic (a, b), or an in-kernel GroupNorm with gamma = 0,
    which makes the operand exactly beta while the per-tile group statistics still run), weights sparse {-1, 0, 1} with
    a few nonzeros per row, bias and residual integers, scales from {1/4, 1/2, 1}.  Every output is then a multiple of
    1/8 of magnitude <= VMAX (exact in fp16), and every statistics slot a sum of multiples of 1/64 whose magnitude
    stays below 2^24 units: exact in fp32 in any summation order.  Each case asserts both from its fp64 reference;
  * the output, every statistics slot (NB = 1: one per pixel tile, per phase for up2; NB > 1: one per 32-row quarter)
    and sums_out (int64, zeroed before each launch) are compared with `==` against fp64;
  * each case asserts the tile instantiation it exercises (ops.conv_tile_config / conv_stats_tiles_up2 against the host
    rule restated in _host_config), at least two waves of tiles, and for a fused operand that drain_at lies inside the
    K schedule, so that the epilogue really runs between the next tile's transforms.  Outputs and statistics are
    NaN-filled with one guard sample behind them, and a second launch must give the same bits.  A mismatch is reported
    as (sample, y, x, channel) or (sample, slot, channel pair) with the tile that owns it: (tx, ty, tn, nt), the
    sub-tile when MT = 2, the sub-pixel phase for up2, the quarter when NB > 1.

test_plans_reach_only_tabled_signatures records every conv the four bench.WORKLOADS plans launch, under the default
engine and under the option plans of test_engine_options_gpu.py, reduces each to its epilogue signature and fails with
a ready-to-paste list of any signature that no case here covers.

The whole file takes about 70 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit, 20 s of it building and running the
plans.
"""
import inspect
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

VMAX = 128.0  # multiples of 1/8 below 2^8 are exact in fp16
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


# ------------------------------------------------------------------------------------------------------------------
# epilogue signatures
# ------------------------------------------------------------------------------------------------------------------
def _signature(H, W, Cout, has3, up2, xf, bias, res, scales, out, stats, sums):
    """(BN, MT, plain, TW, TH, NB, up2, transform, bias, residual mode, scales, output, stats, sums_out) of a conv with
    output geometry H x W (up2: the source's) and Cout channels.  transform: raw | affine | gn; bias: none | shared |
    sample; scales: value | pair | table; output: f16 | f32 | planar<c> | f16x<k>heads"""
    halo = has3 and H % 16 == 0 and W % 8 == 0
    TW, TH, NB = _tile_shape(H, W, halo)
    BN, MT = _host_config(H, W, Cout, halo, 4 if up2 else 1)
    plain = BN >= 64 and NB == 1 and out == "f16"
    return (BN, MT, plain, TW, TH, NB, up2, xf, bias, res, scales, out, stats, sums)


def _signature_of_conv(a):
    """the signature of ops.ConvOp(**a), a: its bound constructor arguments"""
    ops = _ops()
    segs = [tuple(sg) + (None, 0, 0) * (len(sg) == 2) for sg in a["segs"]]
    heads, out, planar = a["out_heads"], a["out"], a["out_planar"]
    if out is not None:
        _, H, W, Cout = out.shape
        Cout //= heads
    else:
        _, H, W, Cout = a["out_shape"]
    if a["up2"]:
        H, W = H // 2, W // 2
    affs = [sg[2] for sg in segs]
    xf = "gn" if any(isinstance(x, ops.GNSpec) for x in affs) else \
        ("affine" if any(x is not None for x in affs) else "raw")
    bias = "none" if a["ebias"] is None else ("sample" if a["ebias_stride"] > 0 else "shared")
    res = None if a["residual"] is None else int(a["res_mode"])
    scales = "value" if a["scales"] is None else ("table" if a["scales_stride"] > 0 else "pair")
    if planar is not None:
        outk = f"planar{planar.shape[1]}"
    else:
        outk = ("f32" if out.dtype == torch.float32 else "f16") + (f"x{heads}heads" if heads > 1 else "")
    has3 = any(sg[1] == ops.MODE_3x3 for sg in segs)
    sig = _signature(H, W, Cout, has3, bool(a["up2"]), xf, bias, res, scales, outk, a["stats"] is not None,
                     a["sums_out"] is not None)
    if a["up2"]:
        assert ops.conv_stats_tiles_up2(H, W, Cout) > 0
    else:
        assert ops.conv_tile_config(H, W, Cout, has3) == sig[:2], (ops.conv_tile_config(H, W, Cout, has3), sig)
    return sig


def _signature_of_case(spec):
    xf = {"raw": "raw", "act0": "affine", "gn0": "gn"}[spec.get("xf", "raw")]
    scales = {"one": "value", "value": "value", "pair": "pair", "table": "table"}[spec.get("scales", "one")]
    return _signature(spec["H"], spec["W"], spec["Cout"], any(sg[0] == "3x3" for sg in spec["segs"]),
                      spec.get("up2", False), xf, spec.get("bias") or "none", spec.get("res"), scales,
                      spec.get("out", "f16"), spec.get("stats", False), spec.get("sums", False))


# ------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------
# spec: inst (BN, MT), N (batch entries), H, W (the source's for up2), Cout, segs [(mode, C)] with mode "3x3" | "1x1" |
# "s2", optional NB, up2; xf: the operand of segment 0 (raw | act0 | gn0; the other segments are raw); bias: None |
# shared | sample; res: None | 0 | 1 | 2; scales: one (by value, 1 and 1) | value (by value, 1/4 and 1/2) | pair (one
# device pair, 1/2 and 1) | table (per-sample rows: acc_scale 1/4, 1/2, 1, res_scale 1, 1/2 in turn); out: f16 | f32 |
# planar<c> | f16x<k>heads (k heads: batch entry n writes channels [(n % k) Cout, ...) of sample n // k); stats,
# sums.  edge: not a signature the plans launch (kept for the kernel's other paths)
# geometries: 8x16 halo tiles of 128 / 64 channels, up2 over a 16x16 source, 16x8 pixel tiles (1x1 and stride 2) of 128
# / 64 channels, two 8x8 samples per tile (NB = 2) of 64 / 128 channels, rows of 128 pixels (H = 1: the attention GEMMs,
# fp16, fp32 and heads), conv_out's 16-channel tiles; each 270..320 tiles, 8 to 16 tiles per sample
HALO128 = dict(inst=(128, 1), N=40, H=32, W=32, Cout=128)
HALO64 = dict(inst=(64, 1), N=40, H=16, W=16, Cout=256)
UP2 = dict(inst=(128, 1), up2=True, N=40, H=16, W=16, Cout=128)
PX128 = dict(inst=(128, 1), N=40, H=32, W=32, Cout=128)
PX64 = dict(inst=(64, 1), N=40, H=16, W=16, Cout=256)
NB2 = dict(inst=(64, 1), NB=2, N=79, H=8, W=8, Cout=512)  # N odd: the last tile's second sample is past N
NB2_128 = dict(inst=(128, 1), NB=2, N=39, H=8, W=8, Cout=1792)
ROW128 = dict(inst=(128, 1), N=40, H=1, W=256, Cout=512)
ROW64 = dict(inst=(64, 1), N=40, H=1, W=256, Cout=256)
HEADS = dict(inst=(64, 1), N=160, H=1, W=256, Cout=64)
OUT16 = dict(inst=(16, 2), N=20, H=64, W=64, Cout=16)
# a fused segment needs more K-schedule entries than drain_at, so that the epilogue runs between the next tile's stages
X3, X3L, X1 = [("3x3", 256)], [("3x3", 256), ("1x1", 64)], [("1x1", 256)]
R3, R1, RS2 = [("3x3", 64)], [("1x1", 64)], [("s2", 64)]

CASES = {
    # ---- <128,1,T> halo: the ResBlock convs of the 32x32 .. 256x256 layers (conv1 with the temb row per sample, conv2
    # with the shortcut as K columns or a residual: res_mode 1 / 2 in the ADM up / down blocks), conv_in
    "halo128_act0_sample": dict(HALO128, segs=X3, xf="act0", bias="sample", stats=True),
    "halo128_act0_sample_sums": dict(HALO128, segs=X3, xf="act0", bias="sample", scales="value", stats=True, sums=True),
    "halo128_act0_res0": dict(HALO128, segs=X3, xf="act0", bias="shared", res=0, scales="value", stats=True),
    "halo128_act0_res1": dict(HALO128, segs=X3, xf="act0", bias="shared", res=1, scales="value", stats=True),
    "halo128_act0_res1_sums": dict(HALO128, segs=X3, xf="act0", bias="shared", res=1, stats=True, sums=True),
    "halo128_act0_res2": dict(HALO128, segs=X3, xf="act0", bias="shared", res=2, scales="value", stats=True),
    "halo128_act0_res2_sums": dict(HALO128, segs=X3, xf="act0", bias="shared", res=2, stats=True, sums=True),
    "halo128_act0": dict(HALO128, segs=X3L, xf="act0", bias="shared", stats=True),
    "halo128_act0_sums": dict(HALO128, segs=X3L, xf="act0", bias="shared", scales="value", stats=True, sums=True),
    "halo128_gn0_sample_sums": dict(HALO128, segs=X3, xf="gn0", bias="sample", stats=True, sums=True),
    "halo128_gn0_res1_sums": dict(HALO128, segs=X3, xf="gn0", bias="shared", res=1, scales="value", stats=True,
                                  sums=True),
    "halo128_gn0_res2_sums": dict(HALO128, segs=X3, xf="gn0", bias="shared", res=2, stats=True, sums=True),
    "halo128_gn0_sums": dict(HALO128, segs=X3L, xf="gn0", bias="shared", scales="value", stats=True, sums=True),
    "halo128_raw": dict(HALO128, segs=R3, bias="shared", scales="value", stats=True),
    "halo128_raw_sums": dict(HALO128, segs=R3, bias="shared", stats=True, sums=True),
    # ---- <64,1,T> halo: the 16x16 layers of 256 channels
    "halo64_act0_res2": dict(HALO64, segs=X3, xf="act0", bias="shared", res=2, scales="value", stats=True),
    "halo64_act0_res2_sums": dict(HALO64, segs=X3, xf="act0", bias="shared", res=2, stats=True, sums=True),
    "halo64_gn0_res2_sums": dict(HALO64, segs=X3, xf="gn0", bias="shared", res=2, scales="value", stats=True,
                                 sums=True),
    "halo64_raw": dict(HALO64, segs=R3, bias="shared", stats=True),
    "halo64_raw_sums": dict(HALO64, segs=R3, bias="shared", scales="value", stats=True, sums=True),
    # ---- up2 with statistics: one slot per (pixel tile, phase)
    "up2_act0": dict(UP2, segs=X3, xf="act0", bias="shared", stats=True),
    "up2_act0_sums": dict(UP2, segs=X3, xf="act0", bias="shared", scales="value", stats=True, sums=True),
    "up2_gn0_sums": dict(UP2, segs=X3, xf="gn0", bias="shared", stats=True, sums=True),
    "up2_raw": dict(UP2, segs=R3, bias="shared", scales="value", stats=True),
    "up2_raw_sums": dict(UP2, segs=R3, bias="shared", stats=True, sums=True),
    # ---- <128,1,T> / <64,1,T> 16x8 pixel tiles: attention qkv / proj (residual), stride-2 downsampling
    "px128_act0": dict(PX128, segs=X1, xf="act0", bias="shared", scales="value"),
    "px128_gn0": dict(PX128, segs=X1, xf="gn0", bias="shared"),
    "px128_res0": dict(PX128, segs=R1, bias="shared", res=0, scales="value", stats=True),
    "px128_res0_sums": dict(PX128, segs=R1, bias="shared", res=0, stats=True, sums=True),
    "s2_128": dict(PX128, segs=RS2, bias="shared", stats=True),
    "s2_128_sums": dict(PX128, segs=RS2, bias="shared", scales="value", stats=True, sums=True),
    "s2_64": dict(PX64, segs=RS2, bias="shared", scales="value", stats=True),
    "px64_raw_sums": dict(PX64, segs=R1, bias="shared", stats=True, sums=True),
    # ---- NB = 2 (8x8 layers): statistics per 32-row quarter, per-sample bias rows and scales inside one tile
    "nb2_act0_sample": dict(NB2, segs=X3, xf="act0", bias="sample", stats=True),
    "nb2_act0_res0_table": dict(NB2, segs=X1, xf="act0", bias="shared", res=0, scales="table", stats=True),
    "nb2_act0_res2": dict(NB2, segs=X3, xf="act0", bias="shared", res=2, scales="value", stats=True),
    "nb2_act0_nostats": dict(NB2, segs=X1, xf="act0", bias="shared", scales="value"),
    "nb2_act0": dict(NB2, segs=[("3x3", 128), ("1x1", 64)], xf="act0", bias="shared", stats=True),
    "nb2_raw_sample": dict(NB2, segs=R3, bias="sample", scales="value", stats=True),
    "nb2_raw_res0_table": dict(NB2, segs=R1, bias="shared", res=0, scales="table", stats=True),
    "nb2_raw_res0": dict(NB2, segs=R1, bias="shared", res=0, scales="value", stats=True),
    "nb2_raw_res2": dict(NB2, segs=R3, bias="shared", res=2, stats=True),
    "nb2_raw_nostats": dict(NB2, segs=R1, bias="shared"),
    "nb2_raw": dict(NB2, segs=R3, bias="shared", scales="value", stats=True),
    "nb2_128_act0": dict(NB2_128, segs=X1, xf="act0", bias="shared", scales="value"),
    "nb2_128_raw": dict(NB2_128, segs=R1, bias="shared"),
    # ---- rows of 128 pixels: the attention GEMMs' fp16, fp32 and per-head outputs
    "row128_f16": dict(ROW128, segs=R1),
    "row128_f32": dict(ROW128, segs=R1, scales="value", out="f32"),
    "row64_f32": dict(ROW64, segs=R1, out="f32"),
    "heads8": dict(HEADS, segs=R1, out="f16x8heads"),
    "heads16": dict(HEADS, segs=R1, scales="value", out="f16x16heads"),
    # ---- <16,2,F>: conv_out, fp32 planar store of 3 / 6 channels
    "out16x2_act0_planar3": dict(OUT16, segs=X3, xf="act0", bias="shared", out="planar3"),
    "out16x2_act0_planar6": dict(OUT16, segs=X3, xf="act0", bias="shared", scales="value", out="planar6"),
    "out16x2_gn0_planar3": dict(OUT16, segs=X3, xf="gn0", bias="shared", scales="value", out="planar3"),
    "out16x2_gn0_planar6": dict(OUT16, segs=X3, xf="gn0", bias="shared", out="planar6"),
    # ---- edge cases outside the plans: the other instantiations and paths of the epilogue
    # <64,2,T>: two stacked sub-tiles summed into one statistics slot; 320 tiles
    "edge_halo64x2": dict(inst=(64, 2), N=20, H=64, W=64, Cout=64, segs=X3, xf="act0", bias="sample", res=2,
                          scales="table", stats=True, sums=True, edge=True),
    # <64,2,F>: the generic planar store (5 of 64 channels), with a residual and statistics of all 64; 320 tiles
    "edge_halo64x2_planar": dict(inst=(64, 2), N=20, H=64, W=64, Cout=64, segs=R3, bias="sample", res=0,
                                 scales="pair", out="planar5", stats=True, sums=True, edge=True),
    # <64,2,F>: fp32 output of a fused operand with one device scale pair; 320 tiles
    "edge_halo64x2_f32": dict(inst=(64, 2), N=20, H=64, W=64, Cout=64, segs=X3, xf="gn0", bias="sample",
                              scales="pair", out="f32", edge=True),
    # <128,1,T>: one device scale pair with a residual and per-sample bias rows
    "edge_halo128_pair": dict(HALO128, segs=X3, xf="act0", bias="sample", res=0, scales="pair", stats=True, sums=True,
                              edge=True),
    # <16,1,F>: dx copies on a ragged 24x24 layer, per-sample bias rows and scales; 288 tiles
    "edge_out16x1": dict(inst=(16, 1), N=48, H=24, W=24, Cout=16, segs=[("3x3", 128)], xf="act0", bias="sample",
                         scales="table", out="planar3", edge=True),
    # dx copies, partial x and y tiles (W 24, H 20 in 16 x 8 tiles); 288 tiles
    "edge_copies64_ragged_xy": dict(inst=(64, 1), N=24, H=20, W=24, Cout=128, segs=[("3x3", 128)], xf="act0",
                                    bias="sample", res=0, scales="table", stats=True, sums=True, edge=True),
    # ... partial x tiles (W 40 in 16-wide tiles) with the nearest-x2 residual; 270 tiles
    "edge_copies128_ragged_x": dict(inst=(128, 1), N=30, H=24, W=40, Cout=128, segs=[("3x3", 128)], xf="gn0",
                                    bias="shared", res=1, scales="table", stats=True, sums=True, edge=True),
    # NB = 8 (4x4 samples), N = 8*33 + 1: per-sample affine rows, bias rows and scales, 2x2-averaged residual; 272 tiles
    "edge_nb8": dict(inst=(64, 1), NB=8, N=265, H=4, W=4, Cout=512, segs=[("3x3", 128)], xf="act0", bias="sample",
                     res=2, scales="table", stats=True, edge=True),
}


class _Geom:
    """Tile geometry of a case"""

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
        self.phases = 4 if self.up2 else 1
        if self.up2:
            self.slots = ops.conv_stats_tiles_up2(self.H, self.W, self.Cout)
            assert self.slots == self.tiles_x * self.tiles_y * 4, self.slots
        else:
            assert ops.conv_tile_config(self.H, self.W, self.Cout, has3) == spec["inst"], \
                ops.conv_tile_config(self.H, self.W, self.Cout, has3)
            self.slots = ops.conv_stats_tiles(self.H, self.W, self.Cout, has3)
            assert self.slots == self.tiles_x * self.tiles_y * (1 if self.NB == 1 else 4), self.slots
        self.tiles = self.tiles_x * self.tiles_y * -(-self.N // self.NB) * (self.Cout // self.BN) * self.phases
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        assert self.tiles >= 2 * sms, f"{self.tiles} tiles on {sms} SMs: fewer than two waves"
        self.Ho, self.Wo = (2 * self.H, 2 * self.W) if self.up2 else (self.H, self.W)

    def locate(self, n, y, x, o):
        """the tile that writes output element (batch entry, y, x, channel)"""
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

    def slot_map(self):
        """[N][Ho][Wo] statistics slot of every output pixel: NB = 1, the pixel tile (times 4 plus the phase for up2);
        NB > 1, the pixel tile times 4 plus the 32-row quarter of the tile row y*TW*NB + (n % NB)*TW + x"""
        y = torch.arange(self.Ho)[:, None]
        x = torch.arange(self.Wo)[None, :]
        if self.NB == 1:
            ys, xs = (y // 2, x // 2) if self.up2 else (y, x)
            ph = (y % 2) * 2 + x % 2 if self.up2 else 0
            slot = ((ys // self.THT) * self.tiles_x + xs // self.TW) * self.phases + ph
            return slot.expand(self.N, self.Ho, self.Wo)
        n = torch.arange(self.N)[:, None, None]
        row = (y % self.TH) * self.TW * self.NB + (n % self.NB) * self.TW + x % self.TW
        return ((y // self.THT) * self.tiles_x + x // self.TW) * 4 + row // 32

    def locate_slot(self, n, slot, pair):
        """the tile (and quarter / phase) that writes statistics slot `slot` of batch entry n"""
        if self.NB == 1:
            t, ph = divmod(slot, self.phases)
            ty, tx = divmod(t, self.tiles_x)
            s = f"tile (tx={tx}, ty={ty}, tn={n}, nt={ph * (self.Cout // self.BN) + 2 * pair // self.BN})"
            if self.MT == 2:
                s += " (sub-tiles 0 and 1)"
            if self.up2:
                s += f" phase (a={ph // 2}, b={ph % 2})"
            return s
        t, q = divmod(slot, 4)
        ty, tx = divmod(t, self.tiles_x)
        return f"tile (tx={tx}, ty={ty}, tn={n // self.NB}, nt={2 * pair // self.BN}) quarter {q}"


def _report(geom, bad, got, want, what):
    """fail with the first mismatching output elements, located"""
    nbad = int(bad.sum())
    if nbad == 0:
        return
    lines = [f"(n={n}, y={y}, x={x}, o={o}) {geom.locate(n, y, x, o)}: got {got[n, y, x, o].item()!r}, "
             f"want {want[n, y, x, o].item()!r}" for n, y, x, o in bad.nonzero()[:8].tolist()]
    pytest.fail(f"{what}: {nbad} of {got.numel()} elements wrong; first:\n  " + "\n  ".join(lines))


def _report_stats(geom, bad, got, want, what):
    """fail with the first mismatching statistics entries [N][slot][pair][sum | sum of squares], located"""
    nbad = int(bad.sum())
    if nbad == 0:
        return
    lines = [f"(n={n}, slot={s}, pair={p}, {'sum of squares' if k else 'sum'}) {geom.locate_slot(n, s, p)}: got "
             f"{got[n, s, p, k].item()!r}, want {want[n, s, p, k].item()!r}"
             for n, s, p, k in bad.nonzero()[:8].tolist()]
    pytest.fail(f"{what}: {nbad} of {got.numel()} statistics wrong; first:\n  " + "\n  ".join(lines))


def _ints(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _sparse_weight(g, Cout, C, k, nnz):
    """[Cout][C][k][k] with nnz entries +-1 per row at random positions, the rest 0"""
    K = C * k * k
    w = torch.zeros(Cout, K, dtype=torch.float64)
    cols = torch.rand(Cout, K, generator=g).topk(nnz, dim=1).indices
    w.scatter_(1, cols, (torch.randint(0, 2, (Cout, nnz), generator=g) * 2 - 1).double())
    return w.view(Cout, C, k, k)


def _conv_sparse(y, w, mode, up2):
    """fp64 conv of y [N][Hs][Ws][C] with the sparse weight w [O][C][k][k] as a sum over its nonzeros, [N][Ho][Wo][O]:
    mode 3x3 pad 1, 1x1, or s2 (stride 2, pad (0, 1, 0, 1)); up2: of the nearest-x2 upsampled y"""
    if up2:
        y = y.repeat_interleave(2, 1).repeat_interleave(2, 2)
    N, Hs, Ws, _ = y.shape
    s, Ho, Wo = (2, Hs // 2, Ws // 2) if mode == "s2" else (1, Hs, Ws)
    if mode == "3x3":
        y = F.pad(y, (0, 0, 1, 1, 1, 1))
    elif mode == "s2":
        y = F.pad(y, (0, 0, 0, 1, 0, 1))
    out = torch.zeros(N, Ho, Wo, w.shape[0], dtype=torch.float64)
    for o, c, ky, kx in w.nonzero().tolist():
        out[..., o] += w[o, c, ky, kx].item() * y[:, ky:ky + s * Ho:s, kx:kx + s * Wo:s, c]
    return out


_MODE = {"3x3": 1, "1x1": 0, "s2": 2}  # ops.MODE_*


def _bits(t):
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[t.dtype])


def _run_case(spec, dev, seed):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    geom = _Geom(spec, dev)
    N, H, W, Cout, Ho, Wo = geom.N, geom.H, geom.W, geom.Cout, geom.Ho, geom.Wo
    xf = spec.get("xf", "raw")

    # ---- operands and the accumulators in fp64: acc[n][y][x][o]
    conv_segs, wparts, acc, l1 = [], [], 0.0, 0.0
    for i, (mode, C) in enumerate(spec["segs"]):
        k = 1 if mode == "1x1" else 3
        Hs, Ws = (2 * H, 2 * W) if mode == "s2" else (H, W)
        x = _ints(g, (N, Hs, Ws, C), -3, 3)
        src = x.half().to(dev)
        y = x
        if i == 0 and xf == "act0":  # y = a x + b, a in {+-1/2, +-1, +-2}, b in Z/2: multiples of 1/2, exact in fp16
            a = torch.tensor([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0])[torch.randint(0, 6, (N, C), generator=g)].double()
            b = _ints(g, (N, C), -4, 4) * 0.5
            y = x * a[:, None, None, :] + b[:, None, None, :]
            conv_segs.append((src, _MODE[mode], torch.stack([a, b], -1).float().contiguous().to(dev), 0, 0))
        elif i == 0 and xf == "gn0":  # gamma = 0: a = 0 and b = beta, whatever the statistics
            beta = _ints(g, (C,), -4, 4) * 0.5
            y = beta.expand(N, Hs, Ws, C)
            sums = torch.stack([torch.randint(-2 ** 34, 2 ** 34, (N, C // 2), generator=g),
                                torch.randint(0, 2 ** 40, (N, C // 2), generator=g)], -1).to(dev)
            gn = ops.GNSpec([sums], [C], torch.zeros(C, device=dev), beta.float().to(dev), 1e-5, H * W)
            conv_segs.append((src, _MODE[mode], gn, 0, 0))
        else:
            conv_segs.append((src, _MODE[mode]))
        w = _sparse_weight(g, Cout, C, k, spec.get("nnz", 6))
        wparts.append(ops.pack_upconv_weight(w) if geom.up2 else ops.pack_conv_weight(w))
        acc = acc + _conv_sparse(y, w, mode, geom.up2)
        # every partial sum of the MMAs is a multiple of 1/2 of magnitude <= l1: exact in fp32 below 2^23
        l1 = l1 + w.abs().sum(dim=(1, 2, 3)).max().item() * y.abs().max().item()
    weight = torch.cat(wparts, -1)
    assert torch.equal(weight.double(), weight.double().round()), "packed weights not integer"
    assert l1 * 2 < 2 ** 24, l1
    v = acc
    kw = {}

    # ---- epilogue: v = (acc + bias) * acc_scale + res_scale * residual
    bias = spec.get("bias")
    if bias:
        rows = N if bias == "sample" else 1
        wide = _ints(g, (rows, Cout + 96), -3, 3)  # a slice of a wider table, like the plans' timestep projections
        v = v + wide[:, None, None, 32:32 + Cout]
        wd = wide.float().to(dev)
        kw.update(ebias=wd[:, 32:32 + Cout], ebias_stride=Cout + 96 if rows > 1 else 0)
    sc = spec.get("scales", "one")
    acc_s, res_s = torch.ones(N, dtype=torch.float64), torch.ones(N, dtype=torch.float64)
    if sc == "value":
        acc_s.fill_(0.25)
        res_s.fill_(0.5)
        kw.update(acc_scale=0.25, res_scale=0.5)
    elif sc == "pair":
        acc_s.fill_(0.5)
        kw.update(scales=torch.tensor([0.5, 1.0], device=dev))
    elif sc == "table":  # rows of 3 floats: the pair, then one unused float
        acc_s = torch.tensor([0.25, 0.5, 1.0], dtype=torch.float64)[torch.arange(N) % 3]
        res_s = torch.tensor([1.0, 0.5], dtype=torch.float64)[torch.arange(N) % 2]
        tab = torch.stack([acc_s, res_s, torch.full((N,), 7.0, dtype=torch.float64)], 1).float()
        kw.update(scales=tab.reshape(-1).to(dev), scales_stride=3)
    v = v * acc_s[:, None, None, None]
    rm = spec.get("res")
    if rm is not None:
        if rm == 0:
            res = _ints(g, (N, Ho, Wo, Cout), -2, 2)
            up = res
        elif rm == 1:
            res = _ints(g, (N, H // 2, W // 2, Cout), -2, 2)
            up = res.repeat_interleave(2, 1).repeat_interleave(2, 2)
        else:
            res = _ints(g, (N, 2 * H, 2 * W, Cout), -2, 2)
            up = res.reshape(N, H, 2, W, 2, Cout).sum(dim=(2, 4)) * 0.25
        v = v + res_s[:, None, None, None] * up
        kw.update(residual=res.half().to(dev), res_mode=rm)
    assert torch.equal(v * 8, (v * 8).round()), "outputs not multiples of 1/8"
    assert v.abs().max().item() <= VMAX, v.abs().max().item()

    # ---- outputs, NaN-filled with one guard sample behind each
    out = spec.get("out", "f16")
    if out.startswith("planar"):
        pc = int(out[6:])
        out_full = torch.full((N + 1, pc, Ho, Wo), NAN, dtype=torch.float32, device=dev)
        kw.update(out_planar=out_full[:-1], out_shape=(N, Ho, Wo, Cout))
        want = v[..., :pc]
    else:
        heads = int(out[4:-5]) if out.endswith("heads") else 1
        out_full = torch.full((N // heads + 1, Ho, Wo, heads * Cout), NAN,
                              dtype=torch.float32 if out == "f32" else torch.float16, device=dev)
        kw.update(out=out_full[:-1], out_heads=heads)
        want = v
    stats_full = sums_full = None
    if spec.get("stats"):
        stats_full = torch.full((N + 1, geom.slots, Cout // 2, 2), NAN, dtype=torch.float32, device=dev)
        kw.update(stats=stats_full[:-1])
        if spec.get("sums"):
            sums_full = torch.zeros(N + 1, Cout // 2, 2, dtype=torch.int64, device=dev)
            kw.update(sums_out=sums_full[:-1])
    op = ops.ConvOp(conv_segs, weight.to(dev), up2=geom.up2, **kw)
    bound = inspect.signature(ops.ConvOp.__init__).bind(None, conv_segs, weight, up2=geom.up2, **kw)
    bound.apply_defaults()
    assert _signature_of_conv(bound.arguments) == _signature_of_case(spec)
    if xf != "raw":  # the epilogue of tile i runs between tile i+1's K stages
        n_sched = sum(C // 64 for _, C in spec["segs"])
        assert 1 <= op.drain_at < n_sched, (op.drain_at, n_sched)

    def launch():
        out_full.fill_(NAN)
        if stats_full is not None:
            stats_full.fill_(NAN)
        if sums_full is not None:
            sums_full.zero_()
        op.launch()
        torch.cuda.synchronize()
        return [t.clone() for t in (out_full, stats_full, sums_full) if t is not None]

    first = launch()
    assert torch.isnan(out_full[-1]).all(), "out: the guard sample behind the output was written"
    got = out_full[:-1].double().cpu()
    if out.startswith("planar"):
        got = got.permute(0, 2, 3, 1)
    elif out.endswith("heads"):
        got = got.reshape(N // heads, Ho, Wo, heads, Cout).permute(0, 3, 1, 2, 4).reshape(N, Ho, Wo, Cout)
    _report(geom, got != want, got, want, "out")

    if stats_full is not None:
        C2 = Cout // 2
        pv = v.reshape(N, Ho, Wo, C2, 2)
        per_px = torch.stack([pv.sum(-1), (pv * pv).sum(-1), pv.abs().sum(-1)], -1)  # [N][Ho][Wo][C/2][3]
        idx = (torch.arange(N)[:, None, None] * geom.slots + geom.slot_map()).reshape(-1)
        tot = torch.zeros(N * geom.slots, C2, 3, dtype=torch.float64)
        tot.index_add_(0, idx, per_px.reshape(-1, C2, 3))
        tot = tot.reshape(N, geom.slots, C2, 3)
        st_want = tot[..., :2]
        # every partial sum the kernel forms: multiples of 1/8 (sums) and 1/64 (squares) below 2^24 units
        assert tot[..., 2].max().item() * 8 < 2 ** 24 and tot[..., 1].max().item() * 64 < 2 ** 24
        assert torch.isnan(stats_full[-1]).all(), "stats: the guard sample was written"
        _report_stats(geom, stats_full[:-1].double().cpu() != st_want, stats_full[:-1].double().cpu(), st_want,
                      "stats")
        if sums_full is not None:
            assert not sums_full[-1].any(), "sums_out: the guard sample was written"
            sums_want = (st_want * ops.STAT_SCALE).sum(1).to(torch.int64)
            gs = sums_full[:-1].cpu()
            bad = gs != sums_want
            assert not bad.any(), f"sums_out: {int(bad.sum())} of {gs.numel()} wrong; first (n, pair, k) " \
                f"{bad.nonzero()[:4].tolist()}"

    second = launch()
    for a, b in zip(first, second):
        assert torch.equal(_bits(a), _bits(b)), "a second launch gives different bits"
    del op
    return geom


@pytest.mark.parametrize("case", list(CASES))
def test_epilogue_exact(cuda_device, case):
    t0 = time.perf_counter()
    geom = _run_case(CASES[case], cuda_device, seed=700 + list(CASES).index(case))
    print(f"{case}: {geom.tiles} tiles, {time.perf_counter() - t0:.2f} s")


# ------------------------------------------------------------------------------------------------------------------
# the plans reach only tabled signatures
# ------------------------------------------------------------------------------------------------------------------
# the option plans of test_engine_options_gpu.py (engine switches -> workloads built with them)
OPTIONS = {
    "default": ({}, None),
    "gn_fold": (dict(GN_FOLD=True), None),
    "gn_fold_producers_only": (dict(GN_FOLD=True, GN_FOLD_PRODUCERS_ONLY=True), ["ddpm_celeba_b16", "iddpm_afhq_b8"]),
    "fuse_min_h_8": (dict(FUSE_MIN_H=8), ["ddpm_celeba_b16", "adm_imagenet_b4"]),
    "skip_in_epilogue": (dict(SKIP_AS_K=False), ["ddpm_celeba_b16", "iddpm_afhq_b8"]),
}


def _record_plan(m, B, dev, monkeypatch):
    """epilogue signatures of every conv launched by one edit evaluation of the plan the current engine switches build
    at batch B (the DeltaBlock's first conv with and without its timestep projection), and by the explicit-delta_h
    path"""
    from asyrp_official_b200 import engine, ops
    seen = set()
    init, launch = ops.ConvOp.__init__, ops.ConvOp.launch
    params = inspect.signature(init)

    def rec_init(self, *a, **k):
        b = params.bind(self, *a, **k)
        b.apply_defaults()
        self._epi_sig = _signature_of_conv(b.arguments)
        init(self, *a, **k)

    def rec_launch(self):
        seen.add(self._epi_sig)
        launch(self)

    with monkeypatch.context() as mp:
        mp.setattr(ops.ConvOp, "__init__", rec_init)
        mp.setattr(ops.ConvOp, "launch", rec_launch)
        eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
        P = eng.plan(B)
        P.t.fill_(700.0)
        eng.state.update(ignore_timestep=False, slerp_t=0.3, use_mask=False)
        for L in P.launches(edit=True):
            L()
        eng.state["ignore_timestep"] = True
        for L in P.delta_ops:
            L()
        for L in P.slerp_ops:
            L()
        torch.cuda.synchronize()
    del P, eng
    return seen


def test_plans_reach_only_tabled_signatures(cuda_device, monkeypatch):
    """every epilogue signature the four benchmark plans launch, under the default engine and the option plans, has an
    exact case in CASES, and every CASES row not marked edge is launched by a plan"""
    import bench
    from asyrp_official_b200 import engine
    seen = {}
    for w, (family, key, B, _, ckpt, _) in bench.WORKLOADS.items():
        m, _ = bench.build_model(family, key, cuda_device, ckpt)
        for opt, (switches, workloads) in OPTIONS.items():
            if workloads is not None and w not in workloads:
                continue
            with monkeypatch.context() as mp:
                for k_, v_ in switches.items():
                    mp.setattr(engine, k_, v_)
                for s in _record_plan(m, B, cuda_device, monkeypatch):
                    seen.setdefault(s, []).append(f"{w}/{opt}")
        del m
        torch.cuda.empty_cache()
    covered = {}
    for name, spec in CASES.items():
        covered.setdefault(_signature_of_case(spec), []).append(name)
    missing = sorted((s for s in seen if s not in covered), key=repr)
    print(f"{len(seen)} signatures launched by the plans, {len(covered)} covered by CASES")
    for s in sorted(seen, key=repr):
        print(f"  {s!r}: {covered.get(s)} <- {seen[s][:3]}")
    assert not missing, f"{len(missing)} epilogue signatures the plans launch have no exact case:\n" + \
        "\n".join(f"    {s!r},  # {', '.join(seen[s][:3])}" for s in missing)
    stale = [n for n, spec in CASES.items() if not spec.get("edge") and _signature_of_case(spec) not in seen]
    assert not stale, f"cases not marked edge whose signature no plan launches: {stale}"
