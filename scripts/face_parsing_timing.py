"""Time the face-parsing scorer on the GPU, and print the card and its power limit.

FaceParser.seg_consistency of B source images against B edited images (256 x 256 in, resized to 512 x 512, so 2B
images are parsed) at B = 1, 16 and 64, with CUDA events, median of --reps calls after 3 warm-up calls; synthetic
weights (the weights do not change the work).  Reports images parsed per second.

    python scripts/face_parsing_timing.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import face_parsing, synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
    card = torch.cuda.get_device_name()
    m = face_parsing.FaceParser(synthetic.face_parsing_state_dict(seed=1))
    print(f"chunk: {m.max_rows} images ({face_parsing.ROW_BYTES * m.max_rows / 2 ** 30:.2f} GiB of activations)")
    for B in (1, 16, 64):
        g = torch.Generator(device=m.device).manual_seed(B)
        src = torch.rand(B, 3, 256, 256, device=m.device, generator=g) * 2 - 1
        edited = (src + 0.3 * (torch.rand(B, 3, 256, 256, device=m.device, generator=g) * 2 - 1)).clamp(-1, 1)
        for _ in range(3):
            m.seg_consistency(src, edited)
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            m.seg_consistency(src, edited)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        times.sort()
        med, lo = times[len(times) // 2], times[0]
        print(f"{card} ({limit}): FaceParser.seg_consistency, B={B} pairs ({2 * B} images parsed): median {med:.3f} ms, "
              f"min {lo:.3f} ms over {a.reps} calls, {2 * B / med * 1e3:.1f} images/s at the median")


if __name__ == "__main__":
    main()
