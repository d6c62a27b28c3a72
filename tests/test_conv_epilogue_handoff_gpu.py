"""The conv kernel's staging-tile handoff: the consumer warps write a tile's accumulators into the staging tile and start
the next tile's MMAs while the transform warps run the epilogue from it (two mbarriers, phases counted per CTA tile).

Each case launches at least 3 * SMs + 1 tiles, so that every CTA wraps both staging barriers more than once and some
CTAs own an odd number of tiles, and runs through the harness of test_conv_coverage_gpu.py: NaN-filled outputs and
statistics with a guard sample behind them, a CPU fp64 reference of the whole descriptor, and a second launch that
must give the same bits.
"""
import pytest
import torch

from test_conv_coverage_gpu import _ops, _run_case

pytestmark = pytest.mark.gpu

CASES = {
    # epilogue-bound: one 64-channel 1x1 chunk (4 MMAs per tile) with a residual, per-sample bias, statistics and
    # sums_out, so the epilogue is longer than the K loop; 416 tiles
    "epilogue_bound_1x1": dict(inst=(128, 1), N=13, H=64, W=64, Cout=128, segs=[("1x1", 64, None)], ebias="sample",
                               residual=0, res_scale=0.5, acc_scale=1.25, stats=True, sums=True),
    # mainloop-bound: fused GroupNorm-apply + SiLU halo conv, 128 -> 128 (two 3x3 chunks, as the 256^2 ResBlocks);
    # 400 tiles
    "mainloop_bound_fused_halo": dict(inst=(128, 1), N=50, H=32, W=32, Cout=128, segs=[("3x3", 128, "affine")],
                                      ebias="sample", stats=True, sums=True),
    # raw operands (no transform: the transform warps only run the epilogue), 3x3 halo chunk + 1x1 shortcut chunk
    # through the separate light ring, residual; 400 tiles
    "raw_halo_with_1x1": dict(inst=(128, 1), N=50, H=32, W=32, Cout=128, segs=[("3x3", 64, None), ("1x1", 64, None)],
                              ebias="shared", residual=0, res_scale=0.75, stats=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_staging_handoff_across_tiles(cuda_device, case):
    ops = _ops()
    spec = CASES[case]
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    has3 = any(m == "3x3" for m, _, _ in spec["segs"])
    H, W, Cout = spec["H"], spec["W"], spec["Cout"]
    tiles = spec["N"] * ops.conv_stats_tiles(H, W, Cout, has3) * (Cout // spec["inst"][0])
    assert tiles >= 3 * sms + 1, f"{tiles} tiles on {sms} SMs"
    assert tiles % sms != 0, "every CTA would own the same number of tiles"
    _run_case(spec, cuda_device, seed=300 + list(CASES).index(case))
