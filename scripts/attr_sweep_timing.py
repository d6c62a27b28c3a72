"""Time an attribute sweep on one GPU: K attributes x 1 image as one `--run_test --attr_sweep` against K sequential
`--run_test --edit_attr <attribute>` calls, all in one process.

DDPM CelebA-HQ 256x256 with seeded (--synthetic_weights) UNet weights and K seeded DeltaBlocks, 40 steps, t_edit 500,
t_addnoise 0 for every attribute (--user_defined_t_edit / --user_defined_t_addnoise: no CLIP weights needed; no noise
is drawn, so the sweep's rows can be checked against the sequential runs' edits bit for bit).  Each
arm is one whole run_test per call, as a user runs it: model build, weight packing, graph capture, the trajectories
and the PNG.  The arms alternate inside the call after one warm-up of each; each timing is a host clock around work
that ends in a device synchronise, bracketed by CUDA events.  Prints both times, the sweep's speedup and the card's
name, power limit and maximum SM clock read in the same call, as one JSON line.

    python scripts/attr_sweep_timing.py [--k 8] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import main as cli, synthetic  # noqa: E402
from asyrp_official_b200.configs import load_config  # noqa: E402
from asyrp_official_b200.diffusion_latent import Asyrp  # noqa: E402
from asyrp_official_b200.modules import DDPM  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, e0.elapsed_time(e1) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attr_sweep_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    attrs = [f"attr{i}" for i in range(args.k)]
    work = tempfile.mkdtemp(prefix="attr_sweep_timing_")
    os.chdir(work)
    os.makedirs("checkpoint")
    m = DDPM(load_config("celeba.yml"))
    m.setattr_layers(args.k)
    synthetic.randomize_(m, seed=77, style="jittered")
    for i, a in enumerate(attrs):
        torch.save({"0": {n: v.clone() for n, v in getattr(m, f"layer_{i}").state_dict().items()}},
                   f"checkpoint/{a}_0.pth")
    del m
    base = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/timing", "--do_train", "0", "--do_test", "1",
            "--n_test_img", "1", "--n_train_img", "0", "--bs_train", "1", "--t_0", "999",
            "--n_inv_step", str(args.steps), "--n_train_step", str(args.steps), "--n_test_step", str(args.steps),
            "--load_random_noise", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0",
            "--synthetic_weights", "--seed", "1234", "--train_delta_block", "--get_h_num", "1"]

    def run(extra):
        a, config = cli.parse_args_and_config(base + extra)
        return Asyrp(a, config, device=dev).run_test()

    def sweep():
        return run(["--attr_sweep", " ".join(attrs), "--manual_checkpoint_name", "attribute_0.pth"])

    def sequential():
        return [run(["--edit_attr", a, "--manual_checkpoint_name", f"{a}_0.pth"]) for a in attrs]

    timed(sweep)
    timed(lambda: run(["--edit_attr", attrs[0], "--manual_checkpoint_name", f"{attrs[0]}_0.pth"]))
    t_sweep, t_seq, ev_sweep, ev_seq = [], [], [], []
    same = None
    for _ in range(args.reps):
        res_s, w, e = timed(sweep)
        t_sweep.append(w)
        ev_sweep.append(e)
        res_q, w, e = timed(sequential)
        t_seq.append(w)
        ev_seq.append(e)
        rows = next(iter(res_s.values()))
        same = all(torch.equal(rows[k], next(iter(r.values()))[0]) for k, r in enumerate(res_q))
    print(json.dumps({
        "workload": f"DDPM CelebA-HQ 256x256, {args.steps} steps, t_edit 500, t_addnoise 0, {args.k} attributes x 1 "
                    "image, synthetic weights, seeded DeltaBlocks",
        "sweep_s": [round(v, 3) for v in t_sweep], "sequential_s": [round(v, 3) for v in t_seq],
        "sweep_event_s": [round(v, 3) for v in ev_sweep], "sequential_event_s": [round(v, 3) for v in ev_seq],
        "speedup_best": round(min(t_seq) / min(t_sweep), 2), "rows_equal_sequential": same,
        "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
