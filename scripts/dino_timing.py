"""Time `--dino_structure` on the GPU and print the card and its power limit.

  - features: DINO.features per image for ViT-S/8 and ViT-B/8 (seeded weights, 12 blocks, 224^2 from 256^2 input),
    batches of 16, median of --reps (host clock around work that ends in a device synchronise, after a warm-up);
  - attention: asyrp_dino_attention at T = 785 (ViT-*/8 at 224^2), 16 images, 6 and 12 heads, CUDA events over 20
    launches, against the 4 B heads T^2 64 FLOPs of QK^T and PV (TF32 peak 495 TFLOP/s, dense, data sheet);
  - distance: asyrp_dino_selfsim_distance of 16 pairs at T = 785 for D = 384 and 768, CUDA events over 20 launches;
  - overhead: DINO.scores of 16 edited rows against 4 origin images (ViT-B/8) next to one 16-row, 40-step DDPM
    CelebA-HQ 256^2 edit replay (seeded weights, t_edit 500), the two alternated, medians of --reps.

    python scripts/dino_timing.py [--reps 5] [--out results/dino_timing.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace as NS

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import dino, modules, ops, synthetic  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

S, ROWS, IMAGES, STEPS, T = 256, 16, 4, 40, 785
TF32_PEAK = 495e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def events(fn, n=20):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dino_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(ROWS, 3, S, S, generator=g) * 2 - 1).to(dev)
    res = {"gpu": gpu_info(), "torch": torch.__version__, "input": S, "batch": ROWS}
    nets = {}
    for name, dim in (("vits8", 384), ("vitb8", 768)):
        net = nets[name] = dino.DINO(synthetic.dino_state_dict(seed=1, dim=dim, depth=12, patch=8, grid=28),
                                     device=dev)
        net.features(x)
        res[f"{name}_features_ms_per_image"] = 1e3 * median([clock(lambda: net.features(x)) for _ in range(a.reps)]) \
            / ROWS
    for heads in (6, 12):
        D = 64 * heads
        qkv = torch.randn(ROWS, T, 3 * D, device=dev)
        out = torch.empty(ROWS, T, D, device=dev)
        ms = events(lambda: ops.dino_attention(qkv, out, heads))
        flops = 4.0 * ROWS * heads * T * T * 64
        res[f"attention_h{heads}_ms"] = ms
        res[f"attention_h{heads}_tflops"] = flops / (ms * 1e-3) / 1e12
        res[f"attention_h{heads}_share_of_tf32_peak"] = flops / (ms * 1e-3) / TF32_PEAK
        keys = torch.randn(2 * ROWS * T, D, device=dev)
        ia = torch.arange(ROWS, device=dev) * T
        ib = ia + ROWS * T
        dist = torch.empty(ROWS, dtype=torch.float64, device=dev)
        res[f"distance_d{D}_ms"] = events(lambda: ops.dino_selfsim_distance(keys, ia, ib, T, dist))
        del qkv, out, keys
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    eng = m.engine
    seq, seq_next = make_sequences(999, STEPS)
    sch = Schedule(osmp.make_betas(), seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0))
    replay = lambda: eng.sample(x, sch)  # noqa: E731
    net = nets["vitb8"]
    score = lambda: net.scores(x[:IMAGES], x)  # noqa: E731
    replay()
    score()
    t_replay, t_score = [], []
    for _ in range(a.reps):
        t_replay.append(clock(replay))
        t_score.append(clock(score))
    res["replay_ms"] = 1e3 * median(t_replay)
    res["vitb8_scores_ms"] = 1e3 * median(t_score)
    res["scores_share_of_replay"] = median(t_score) / median(t_replay)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
