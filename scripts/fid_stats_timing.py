"""Time the real-image side of --fid_ref on the GPU, and print the card and its power limit.

Writes --n seeded PNGs at 256 x 256 and at 1024 x 1024 into a temporary directory and runs
`python -m asyrp_official_b200.fid --save-stats` on each folder in this process (images/s, the seconds waiting on the
decoding workers against the seconds of GPU work), times kid_kxx (the n x n kernel sum without the diagonal), and times
kid_subsets at 100 subsets of 1000 rows against a 30 000-row reference (3 x 100 x 1000^2 x 2048 x 2 = 1.23 TFLOP of
fp64 dot products) with CUDA events, median of --reps calls after 2 warm-up calls.  Synthetic weights: the weights
do not change the work.

    python scripts/fid_stats_timing.py [--n 500] [--num_workers 8] [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import fid, ops, synthetic  # noqa: E402


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
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


def write_pngs(folder, n, size, seed):
    from PIL import Image
    os.makedirs(folder)
    g = np.random.default_rng(seed)
    base = g.integers(0, 256, (size // 8, size // 8, 3), dtype=np.uint8)
    for i in range(n):  # smooth-ish content (an upsampled noise field), so PNG decoding is not trivially short
        a = np.repeat(np.repeat(np.roll(base, i, axis=0), 8, 0), 8, 1)
        a = (a.astype(np.int16) + g.integers(-8, 9, a.shape)).clip(0, 255).astype(np.uint8)
        Image.fromarray(a).save(os.path.join(folder, f"{i:05d}.png"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=500)
    ap.add_argument("--num_workers", type=int, default=8)
    ap.add_argument("--batch_size", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
    card = torch.cuda.get_device_name()
    tag = f"{card} ({limit})"
    print(f"{tag}: {os.cpu_count()} host CPUs, --num_workers {a.num_workers}, --batch_size {a.batch_size}")
    sd = synthetic.inception_state_dict(seed=1)
    net = fid.FIDInception(sd)
    with tempfile.TemporaryDirectory() as tmp:
        weights = os.path.join(tmp, "w.pth")
        torch.save(sd, weights)
        for size in (256, 1024):
            folder = os.path.join(tmp, f"real{size}")
            write_pngs(folder, a.n, size, size)
            files = fid.image_files(folder)
            fid.folder_features(net, files[:a.batch_size], a.batch_size, 0)  # warm-up of the shapes
            t0 = time.perf_counter()
            feats, wait, gpu = fid.folder_features(net, files, a.batch_size, a.num_workers)
            t1 = time.perf_counter()
            fid.save_stats(os.path.join(tmp, f"s{size}.npz"), feats)
            t2 = time.perf_counter()
            print(f"{tag}: --save-stats, {a.n} PNGs at {size}^2: {a.n / (t1 - t0):.1f} images/s over the features "
                  f"({t1 - t0:.2f} s: waiting on decoding {wait:.2f} s, GPU {gpu:.2f} s), statistics and file "
                  f"{t2 - t1:.2f} s")
            med, lo = timed(lambda: ops.fid_kernel_sum(feats, feats, exclude_diag=True), a.reps)
            print(f"{tag}: kid_kxx, n={a.n}: median {med:.3f} ms, min {lo:.3f} ms")
        g = torch.Generator(device=net.device).manual_seed(3)
        ref = torch.rand(30000, fid.DIMS, device=net.device, generator=g)
        f = torch.rand(1000, fid.DIMS, device=net.device, generator=g)
        med, lo = timed(lambda: ops.fid_kernel_sum(ref, ref, exclude_diag=True), a.reps)
        print(f"{tag}: kid_kxx, n=30000: median {med:.1f} ms, min {lo:.1f} ms, "
              f"{30000 ** 2 * fid.DIMS * 2 / med / 1e9:.2f} TFLOP/s (fp64) at the median")
        med, lo = timed(lambda: fid.kid_subsets(f, ref, 100, 1000), a.reps)
        flop = 3 * 100 * 1000 ** 2 * fid.DIMS * 2
        print(f"{tag}: kid_subsets 100 x 1000 (set 1000 rows, reference 30000 rows): median {med:.1f} ms, min "
              f"{lo:.1f} ms (index draws and copies included), {flop / med / 1e9:.2f} TFLOP/s (fp64) at the median")
        i1, i2 = fid.kid_subset_indices(1000, 30000, 100, 1000)
        t1, t2 = torch.from_numpy(i1).to(net.device), torch.from_numpy(i2).to(net.device)
        med, lo = timed(lambda: ops.fid_kernel_sum_subsets(ref, ref, t2, t2, exclude_diag=True), a.reps)
        print(f"{tag}: one subset launch (100 x 1000^2 x 2048): median {med:.1f} ms, min {lo:.1f} ms, "
              f"{flop / 3 / med / 1e9:.2f} TFLOP/s (fp64) at the median")


if __name__ == "__main__":
    main()
