"""Time a run_test-style hs_coeff sweep on one GPU: one replay per tuple (the reference's save_image loop) against the
tuples run as rows of one batch (Asyrp.save_image's chunked sweep).

DDPM CelebA-HQ 256x256, 40 steps, t_edit 500, t_addnoise 200, the shipped `smiling` DeltaBlock on seeded UNet weights;
--delta_interpolation --num_delta 5 (tuples (1, v) for v in linspace(0, 1, 5)) at bs_train 1 and 4.  Both arms use
the same x_T and the same per-tuple noise; the arms alternate inside one call, device-timed with CUDA events after a
warm-up sweep of each.  Prints edited images/s of both arms, max|Δ| between their images (0: bit-identical), and the
card's name, power limit and maximum SM clock read in the same call.

    python scripts/hs_sweep_timing.py [--bs 1 4] [--reps 3] [--max_rows 16]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import modules, synthetic  # noqa: E402
from asyrp_official_b200.diffusion_latent import chunk_noise, pad_rows, plan_sweep  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

CKPT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "checkpoint",
                    "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--num_delta", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max_rows", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hs_sweep_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    m.layer_0.load_state_dict(torch.load(CKPT, map_location="cpu", weights_only=True)["0"])
    m.refresh_weights()
    eng = m.engine
    seq, seq_next = make_sequences(999, 40)
    betas = osmp.make_betas()
    tuples = [(1.0, float(v)) for v in np.linspace(0.0, 1.0, a.num_delta)]
    scheds = [Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=200, hs_coeff=t) for t in tuples]
    n_sto = scheds[0].n_stochastic
    K = len(tuples)
    info = gpu_info()
    results = []
    for B in a.bs:
        g = torch.Generator(device=dev).manual_seed(1000 + B)
        x = torch.randn(B, 3, 256, 256, device=dev, generator=g)
        noise = [torch.randn(n_sto, B, 3, 256, 256, device=dev, generator=g) for _ in range(K)]
        tpc, chunks = plan_sweep(K, B, a.max_rows)

        def sequential():
            return [eng.sample(x, scheds[k], noise=noise[k]) for k in range(K)]

        def batched():
            out = []
            for ch in chunks:
                rows_x = pad_rows(x.repeat(len(ch), 1, 1, 1), tpc * B)
                it = iter([noise[k] for k in ch])
                z = chunk_noise(len(ch), tpc, B, lambda: next(it))
                tab = pad_rows(torch.tensor([tuples[k] for k in ch for _ in range(B)], dtype=torch.float32), tpc * B)
                x0 = eng.sample(rows_x, scheds[ch[0]], noise=z, hs_coeffs=tab)
                out += [x0[j * B:(j + 1) * B] for j in range(len(ch))]
            return out

        arms = {"sequential": sequential, "batched": batched}
        outs = {name: f() for name, f in arms.items()}  # warm-up: plans, graphs
        torch.cuda.synchronize()
        diff = max((p - q).abs().max().item() for p, q in zip(outs["sequential"], outs["batched"]))
        times = {name: [] for name in arms}
        for _ in range(a.reps):
            for name, f in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / 1e3)
        r = {"bs": B, "tuples": K, "rows_per_replay": tpc * B, "chunks": len(chunks), "max_abs_diff": diff}
        for name in arms:
            t = float(np.median(times[name]))
            r[f"{name}_s"] = round(t, 4)
            r[f"{name}_img_per_s"] = round(K * B / t, 3)
        r["speedup"] = round(r["sequential_s"] / r["batched_s"], 3)
        results.append(r)
        print(f"bs {B}: {K} tuples, sequential {r['sequential_img_per_s']} img/s, batched ({len(chunks)} replay(s) of "
              f"{tpc * B} rows) {r['batched_img_per_s']} img/s, x{r['speedup']}, max|diff| {diff}", flush=True)
    print(json.dumps({"gpu": info, "workload": "DDPM CelebA-HQ 256, 40 steps, t_edit 500, t_addnoise 200, smiling",
                      "results": results}))


if __name__ == "__main__":
    main()
