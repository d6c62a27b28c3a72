"""Time ArcFace IR-SE50 and the cost of --id_similarity on the GPU, and print the card and its power limit.

  * ArcFace.extract_feats of B = 16, 32 and 96 images (256 x 256 in) with CUDA events, after warm-up calls; synthetic
    weights (the weights do not change the work).
  * `main --run_test` on the CelebA-HQ DDPM (256 x 256, synthetic UNet weights, the smiling DeltaBlock of
    tests/golden/checkpoint) with 16 images in one batch, 40 steps, with and without the flag (and without
    --save_x_origin, so the flag adds the origin trajectory); wall time of run_test after a warm-up run of each.

    python scripts/arcface_timing.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from asyrp_official_b200 import arcface, main as cli, synthetic  # noqa: E402
from asyrp_official_b200.diffusion_latent import Asyrp  # noqa: E402

GFLOP_PER_IMAGE = 12.6  # torch.utils.flop_counter on the reference's Backbone(112, 50, 'ir_se'), multiply-add = 2


def feature_times(reps):
    m = arcface.ArcFace(synthetic.arcface_state_dict(seed=1))
    out = {}
    for B in (16, 32, 96):
        x = torch.rand(B, 3, 256, 256, device=m.device) * 2 - 1
        for _ in range(3):
            m.extract_feats(x)
        times = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            m.extract_feats(x)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        times.sort()
        out[B] = (times[len(times) // 2], times[0])
    return out


def run_test_time(argv):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r.run_test()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()[0]
    card = torch.cuda.get_device_name()
    for B, (med, lo) in feature_times(a.reps).items():
        print(f"{card} ({limit}): ArcFace extract_feats IR-SE50, B={B}: median {med:.3f} ms, min {lo:.3f} ms over "
              f"{a.reps} calls ({GFLOP_PER_IMAGE * B / med:.1f} TFLOP/s at the median)")
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        torch.save(synthetic.arcface_state_dict(seed=1), "ir_se50.pth")
        argv = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/t", "--do_train", "0", "--do_test", "1",
                "--n_test_img", "16", "--bs_train", "16", "--n_inv_step", "40", "--n_train_step", "40",
                "--n_test_step", "40", "--load_random_noise", "--user_defined_t_edit", "500",
                "--user_defined_t_addnoise", "200", "--synthetic_weights", "--train_delta_block", "--get_h_num", "1",
                "--edit_attr", "smiling", "--checkpoint_dir", os.path.join(ROOT, "tests", "golden", "checkpoint"),
                "--manual_checkpoint_name", "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth"]
        flag = argv + ["--id_similarity", "--id_weights", "ir_se50.pth"]
        run_test_time(argv), run_test_time(flag)  # warm-up
        plain, scored = [], []
        for _ in range(2):
            plain.append(run_test_time(argv))
            scored.append(run_test_time(flag))
        print(f"{card} ({limit}): run_test DDPM 256x256, 16 images, 40 steps: {min(plain):.3f} s without the flag, "
              f"{min(scored):.3f} s with --id_similarity (+{min(scored) - min(plain):.3f} s; best of 2)")


if __name__ == "__main__":
    main()
