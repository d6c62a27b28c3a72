"""Time the FID scorer on the GPU, and print the card and its power limit.

FIDInception.features of B images (256 x 256 in, resized to 299 x 299) at B = 1, 16 and 64, and the set statistics of
n = 1 000 and 10 000 feature rows (asyrp_fid_moments: mean and covariance; asyrp_fid_kernel_sum: one n x n sum), with
CUDA events, median of --reps calls after 3 warm-up calls; synthetic weights (the weights do not change the work).
The FLOPs are counted from the layer shapes (2 per multiply-add of every conv; the pools, the pack and the mean are not
counted), so the TF32 TFLOP/s printed are conv FLOPs / time.

    python scripts/fid_timing.py [--reps 10]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import fid, ops, synthetic  # noqa: E402


def conv_flops(m):
    """FLOPs of one image's 94 convs, 2 * Ho * Wo * cout * cin * kh * kw each (cout the layer's width, not the GEMM's
    padded one), from the shapes of the launches of one features() call"""
    total, launch = [0], ops.fid_conv

    def counting(inp, weight, bias, out, kh, kw, stride=1, pad=(0, 0), cstore=None):
        total[0] += 2 * out.shape[1] * out.shape[2] * out.shape[3] * inp.shape[3] * kh * kw
        return launch(inp, weight, bias, out, kh, kw, stride, pad, cstore)
    ops.fid_conv = counting
    try:
        m.features(torch.zeros(1, 3, 256, 256, device=m.device))
    finally:
        ops.fid_conv = launch
    return total[0]


def timed(fn, reps):
    for _ in range(3):
        fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return times[len(times) // 2], times[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
    card = torch.cuda.get_device_name()
    m = fid.FIDInception(synthetic.inception_state_dict(seed=1))
    flops = conv_flops(m)
    print(f"{card} ({limit}): chunk {m.max_rows} images ({fid.ROW_BYTES * m.max_rows / 2 ** 30:.2f} GiB of "
          f"activations); {flops / 1e9:.2f} GFLOP of convs per image")
    for B in (1, 16, 64):
        g = torch.Generator(device=m.device).manual_seed(B)
        x = torch.rand(B, 3, 256, 256, device=m.device, generator=g) * 2 - 1
        med, lo = timed(lambda: m.features(x), a.reps)
        print(f"{card} ({limit}): features, B={B}: median {med:.3f} ms, min {lo:.3f} ms over {a.reps} calls, "
              f"{B / med * 1e3:.1f} images/s, {B * flops / med / 1e9:.1f} TFLOP/s (TF32 convs) at the median")
    for n in (1000, 10000):
        g = torch.Generator(device=m.device).manual_seed(n)
        f = torch.rand(n, fid.DIMS, device=m.device, generator=g)
        med, lo = timed(lambda: ops.fid_moments(f), a.reps)
        print(f"{card} ({limit}): moments, n={n}: median {med:.3f} ms, min {lo:.3f} ms, "
              f"{n * fid.DIMS ** 2 * 2 / med / 1e9:.2f} TFLOP/s (fp64) at the median")
        med, lo = timed(lambda: ops.fid_kernel_sum(f, f, exclude_diag=True), a.reps)
        print(f"{card} ({limit}): kernel sum, n={n} x {n}: median {med:.3f} ms, min {lo:.3f} ms, "
              f"{n * n * fid.DIMS * 2 / med / 1e9:.2f} TFLOP/s (fp64) at the median")


if __name__ == "__main__":
    main()
