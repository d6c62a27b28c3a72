"""conv_gemm_kernel keeps its bits when its warps' register budgets or its epilogue's instruction order change.

One conv per tile instantiation, `PLAIN` and generic, with and without a residual, with a fused GroupNorm-apply + SiLU
operand transform and (where the mode has them) GroupNorm statistics and int64 sums.  Operands are realistic non-integer
values, so the results depend on the summation order of the accumulators and of the statistics.  They are compared, as
SHA-256 of their bytes, with `tests/golden/conv_regsplit.json`, which `tests/golden/make_conv_regsplit.py` wrote from
the build before the transform / epilogue warps got a register budget of their own (`setmaxnreg`) and a second output
row in flight.  Every case has more tiles than an H100 has SMs, so CTAs hand the staging tile over between tiles.
"""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_regsplit.json")

# inst: (BN, MT) the library must choose; plain: which of its two instantiations serves the conv
SHAPES = {
    "plain128": dict(inst=(128, 1), plain=True, N=20, H=32, W=32, Cin=128, Cout=128, k3=True, stats=True, sums=True),
    "plain64x2": dict(inst=(64, 2), plain=True, N=10, H=64, W=64, Cin=64, Cout=64, k3=True, stats=True, sums=True),
    "plain64": dict(inst=(64, 1), plain=True, N=30, H=20, W=24, Cin=64, Cout=64, k3=False, stats=True, sums=True),
    # tiles of two samples (8x8): the generic epilogue's per-sample statistics pass
    "generic64_nb2": dict(inst=(64, 1), plain=False, N=265, H=8, W=8, Cin=64, Cout=128, k3=False, stats=True),
    # fp32 outputs take neither a residual nor statistics
    "generic128_f32": dict(inst=(128, 1), plain=False, N=20, H=32, W=32, Cin=64, Cout=128, k3=False, f32=True),
    "generic64x2_f32": dict(inst=(64, 2), plain=False, N=10, H=64, W=64, Cin=64, Cout=64, k3=False, f32=True),
}
CASES = [(s, r) for s, v in SHAPES.items() for r in ((False,) if v.get("f32") else (False, True))]


def case_id(shape, res):
    return f"{shape}-{'res' if res else 'nores'}"


def _q(rng, shape, lo, hi, scale):
    """multiples of 1/scale: the same values whatever library version draws them"""
    return torch.from_numpy(rng.integers(lo, hi + 1, size=shape).astype(np.float32) / np.float32(scale))


def _sha(t):
    return hashlib.sha256(t.cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def run_case(shape, res, dev):
    """{tensor name: sha256 of its bytes} of one launch"""
    from asyrp_official_b200 import ops
    s = SHAPES[shape]
    N, H, W, Cin, Cout = s["N"], s["H"], s["W"], s["Cin"], s["Cout"]
    assert ops.conv_tile_config(H, W, Cout, s["k3"]) == s["inst"]
    rng = np.random.default_rng([2718, sorted(SHAPES).index(shape), int(res)])
    K = (9 if s["k3"] else 1) * Cin
    x = _q(rng, (N, H, W, Cin), -2048, 2048, 512).half().to(dev)
    w = (_q(rng, (Cout, K), -64, 64, 64) / K ** 0.5).half().to(dev)
    aff = torch.stack([1 + _q(rng, (N, Cin), -2048, 2048, 4096), _q(rng, (N, Cin), -2048, 2048, 4096)], -1)
    aff = aff.contiguous().to(dev)
    bias = _q(rng, (N, Cout), -2048, 2048, 2048).to(dev)
    kw = {}
    if res:
        kw.update(residual=_q(rng, (N, H, W, Cout), -2048, 2048, 512).half().to(dev), res_scale=0.75, acc_scale=0.5)
    if s.get("stats"):
        kw["stats"] = ops.new_stats(N, H, W, Cout, dev, s["k3"])
    if s.get("sums"):
        kw["sums_out"] = ops.new_sums(N, Cout, dev)
    out = torch.full((N, H, W, Cout), float("nan"), device=dev, dtype=torch.float32 if s.get("f32") else torch.float16)
    op = ops.ConvOp([(x, ops.MODE_3x3 if s["k3"] else ops.MODE_1x1, aff, 0, 1)], w, out=out, ebias=bias,
                    ebias_stride=Cout, **kw)
    op.launch()
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    got = {"out": _sha(out)}
    if "stats" in kw:
        got["stats"] = _sha(kw["stats"])
    if "sums_out" in kw:
        got["sums_out"] = _sha(kw["sums_out"])
    return got


def test_cases_cover_every_instantiation():
    assert {(v["inst"], v["plain"]) for v in SHAPES.values()} == {(i, p) for i in ((128, 1), (64, 2), (64, 1))
                                                                 for p in (True, False)}


@pytest.mark.parametrize("shape,res", CASES, ids=[case_id(*c) for c in CASES])
def test_bits_of_parent_build(shape, res, cuda_device):
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert run_case(shape, res, cuda_device) == golden[case_id(shape, res)]
