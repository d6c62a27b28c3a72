"""Time the k-nearest-neighbour kernels of --prdc on the GPU, against torch.cdist in fp64 on the same card, and print
the card and its power limit.

knn_radii of 30 000 x 2048 (the CelebA-HQ reference set) and knn_counts of 1 000 x 30 000 (a set of edits against it),
seeded uniform features, CUDA events, median of --reps calls after one warm-up call (the torch comparison: one call
after a one-chunk warm-up, on fp64 copies of the features made before the timing).  The work is counted as 3 FLOP per
pair and feature (a subtraction and a fused multiply-add); the data sheet's 34 TFLOP/s FP64 (non-tensor) of the H100
SXM gives the bound printed beside each time.  The torch comparison (cdist in fp64 with compute_mode
'donot_use_mm_for_euclid_dist', squared, then topk or the comparisons, in row chunks of --chunk) is information: it
computes the same quantities but is not the definition (cdist takes a square root).

    python scripts/prdc_timing.py [--reps 3] [--chunk 1000] [--k 5]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import fid, ops  # noqa: E402

FP64_PEAK = 34e12  # FLOP/s, H100 SXM data sheet, FP64 without tensor cores


def timed(fn, reps, warmup=1):
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
        times.append(e0.elapsed_time(e1) / 1e3)
    times.sort()
    return times[len(times) // 2], times[0]


def cdist_sq(a, b):
    return torch.cdist(a, b, compute_mode="donot_use_mm_for_euclid_dist") ** 2


def torch_radii(x, k, chunk):
    return torch.cat([torch.topk(cdist_sq(x[i:i + chunk], x), k + 1, dim=1, largest=False).values[:, k]
                      for i in range(0, x.shape[0], chunk)])


def torch_counts(a, ra, b, rb, chunk):
    b_in_a = torch.zeros(b.shape[0], dtype=torch.int64, device=a.device)
    a_in_b, a_cov = [], []
    for i in range(0, a.shape[0], chunk):
        D = cdist_sq(a[i:i + chunk], b)
        inside = D < ra[i:i + chunk, None]
        b_in_a += inside.sum(0)
        a_cov.append(inside.sum(1))
        a_in_b.append((D < rb[None]).sum(1))
    return b_in_a, torch.cat(a_in_b), torch.cat(a_cov)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=1000)
    ap.add_argument("--k", type=int, default=5)
    a = ap.parse_args()
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
    tag = f"{torch.cuda.get_device_name()} ({limit})"
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3)
    ref = torch.rand(30000, fid.DIMS, device=dev, generator=g)
    f = torch.rand(1000, fid.DIMS, device=dev, generator=g) * 1.02
    n, m, k = ref.shape[0], f.shape[0], a.k
    rr, rf = ops.fid_knn_radii(ref, k), ops.fid_knn_radii(f, k)
    ref64, f64 = ref.double(), f.double()  # the torch comparison runs on fp64 copies, made once outside the timing
    cdist_sq(ref64[:a.chunk], ref64)  # its warm-up: one chunk (a full call is seconds)
    out = {}

    flop = n * n * fid.DIMS * 3
    med, lo = timed(lambda: ops.fid_knn_radii(ref, k), a.reps)
    print(f"{tag}: knn_radii {n} x {fid.DIMS}, k={k}: median {med:.3f} s, min {lo:.3f} s; {flop / med / 1e12:.1f} "
          f"TFLOP/s at the median, the 34 TFLOP/s FP64 bound {flop / FP64_PEAK:.3f} s")
    tmed, _ = timed(lambda: out.update(radii=torch_radii(ref64, k, a.chunk)), 1, warmup=0)
    got = out["radii"]
    print(f"{tag}: torch cdist (fp64) + topk, chunks of {a.chunk} rows: {tmed:.3f} s, one call ({tmed / med:.1f} x); "
          f"max relative difference {((got - rr).abs() / rr).max().item():.2e}, equal: {torch.equal(got, rr)}")

    flop = n * m * fid.DIMS * 3
    med, lo = timed(lambda: ops.fid_knn_counts(ref, rr, f, rf), a.reps)
    print(f"{tag}: knn_counts {n} x {m} x {fid.DIMS}: median {med * 1e3:.2f} ms, min {lo * 1e3:.2f} ms; "
          f"{flop / med / 1e12:.1f} TFLOP/s at the median, the 34 TFLOP/s FP64 bound {flop / FP64_PEAK * 1e3:.2f} ms")
    tmed, _ = timed(lambda: out.update(counts=torch_counts(ref64, rr, f64, rf, a.chunk)), 1, warmup=0)
    mine = ops.fid_knn_counts(ref, rr, f, rf)
    same = all(torch.equal(x.long(), y) for x, y in zip(mine, out["counts"]))
    print(f"{tag}: torch cdist (fp64) + comparisons, chunks of {a.chunk} rows: {tmed * 1e3:.2f} ms, one call "
          f"({tmed / med:.1f} x); counts equal: {same}")
    med, lo = timed(lambda: fid.prdc(ref, f, k, rr), a.reps)
    print(f"{tag}: fid.prdc with the real radii given (fake radii, counts, four values): median {med * 1e3:.2f} ms")


if __name__ == "__main__":
    main()
