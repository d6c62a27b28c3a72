"""Placement of the conv epilogue in the transform warps' schedule (ConvParams::drain_at): the transform warps ready the
first drain_at K-schedule entries of tile i+1, then run the epilogue of tile i, then ready the rest of tile i+1.

One case per value the host rule produces and per ring layout: one entry (1x1 chunks, and 3x3 chunks taken as three
dx-shifted copies), both entries of a 128-channel halo conv, 2 of the 4 entries of a halo concat, 3 of the 4 entries of
a halo conv with a 1x1 shortcut in the light ring; across them the epilogue's residual modes 0 / 1 / 2, shared and
per-sample bias, scales, statistics with and without sums_out, and tiles of two samples.  Each case launches at least
3 * SMs + 1 tiles, a count that no CTA count divides, so some CTAs own an odd number of tiles, and runs through the
harness of test_conv_coverage_gpu.py: NaN-filled outputs and statistics with a guard sample behind them, a CPU fp64
reference of the whole descriptor, and a second launch that must give the same bits.
"""
import pytest
import torch

from test_conv_coverage_gpu import _ops, _run_case

pytestmark = pytest.mark.gpu

CASES = {
    # raw 1x1 chunk: no transform, the epilogue runs first; nearest-x2 residual, per-sample bias, stats + sums_out;
    # 416 tiles
    "one_entry_raw_1x1": dict(drain_at=1, inst=(128, 1), N=13, H=64, W=64, Cout=128, segs=[("1x1", 64, None)],
                              ebias="sample", residual=1, res_scale=0.5, acc_scale=1.25, stats=True, sums=True),
    # fused 1x1 chunk, 2x2-average residual; 400 tiles
    "one_entry_fused_1x1": dict(drain_at=1, inst=(128, 1), N=50, H=32, W=32, Cout=128, segs=[("1x1", 64, "affine")],
                                ebias="shared", residual=2, res_scale=0.75, stats=True),
    # two fused 3x3 chunks as three dx-shifted copies each (4 slots hold one entry), ragged x and y tiles; 405 tiles
    "one_entry_copies": dict(drain_at=1, inst=(128, 1), N=45, H=24, W=40, Cout=128, segs=[("3x3", 128, "affine")],
                             ebias="sample", residual=0, res_scale=0.5, stats=True, sums=True),
    # tiles of two samples (8x8, three copies): one entry, per-sample statistics of a mixed tile; 408 tiles
    "one_entry_nb2": dict(drain_at=1, inst=(64, 1), NB=2, N=101, H=8, W=8, Cout=512, segs=[("3x3", 64, "affine")],
                          ebias="sample", stats=True),
    # the 256^2 ResBlock conv: fused 128 -> 128 halo, both entries before the epilogue; 400 tiles
    "two_entries_fused_halo": dict(drain_at=2, inst=(128, 1), N=50, H=32, W=32, Cout=128, segs=[("3x3", 128, "affine")],
                                   ebias="sample", residual=0, res_scale=0.5, acc_scale=0.75, stats=True, sums=True),
    # decoder concat with the GroupNorm finalised in the kernel: 4 halo entries, 2 before the epilogue; 400 tiles
    "two_of_four_gn_concat": dict(drain_at=2, inst=(128, 1), N=50, H=32, W=32, Cout=128,
                                  segs=[("3x3", 128, "gn"), ("3x3", 128, "gn")], gn_ss=True, stats=True, sums=True),
    # <64,2>: two stacked sub-tiles, fused concat of two 64-channel halo chunks; 400 tiles
    "two_entries_64x2_concat": dict(drain_at=2, inst=(64, 2), N=25, H=64, W=64, Cout=64,
                                    segs=[("3x3", 64, "affine"), ("3x3", 64, "affine")], ebias="sample", stats=True),
    # halo conv + 1x1 shortcut in the light ring (H0 L0 H1 L1): 3 entries before the epilogue; 400 tiles
    "three_of_four_halo_shortcut": dict(drain_at=3, inst=(128, 1), N=50, H=32, W=32, Cout=128,
                                        segs=[("3x3", 128, "affine"), ("1x1", 128, None)], ebias="shared",
                                        stats=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_epilogue_placement_across_tiles(cuda_device, case, monkeypatch):
    ops = _ops()
    spec = CASES[case]
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    has3 = any(m == "3x3" for m, _, _ in spec["segs"])
    H, W, Cout, BN = spec["H"], spec["W"], spec["Cout"], spec["inst"][0]
    NB = spec.get("NB", 1)
    if NB == 1:
        tiles = spec["N"] * ops.conv_stats_tiles(H, W, Cout, has3) * (Cout // BN)
    else:
        tiles = -(-spec["N"] // NB) * (Cout // BN)
    assert tiles >= 3 * sms + 1, f"{tiles} tiles on {sms} SMs"
    assert tiles % sms != 0, "every CTA would own the same number of tiles"

    made = []

    class Recorder(ops.ConvOp):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(ops, "ConvOp", Recorder)
    _run_case(spec, cuda_device, seed=500 + list(CASES).index(case))
    assert made[-1].drain_at == spec["drain_at"], (made[-1].drain_at, spec["drain_at"])
