"""Time h-space direction discovery and editing with a found direction on the GPU, and print the card and its power
limit.

Model: DDPM CelebA-HQ 256² on seeded weights, the 40-step generative grid (t_0 = 999).  Discovery of the top K = 8
principal components at n = 256 and 1024 samples, each part timed on its own (host clock around work that ends in a
device synchronise, after one warm-up of each shape):
  - generation: the plain pass from x_T with h recorded at every step, 16 rows per replay, copied into one
    [steps][n][d] buffer, as Asyrp.run_h_directions runs it;
  - Gram: the mean (h_combine) and the centred Gram (h_gram) of every step;
  - eigh: numpy.linalg.eigh of every step's Gram on the host, fp64;
  - projection: the K principal directions (h_combine) of every step.
Editing: one 40-step edit trajectory of 16 rows (t_edit 500, t_addnoise 200), median of --reps replays, with an
additive direction (h2 = c0 h + α d) against the shipped `smiling` DeltaBlock on the same weights.

    python scripts/h_directions_timing.py [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time
from types import SimpleNamespace as NS

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import modules, ops, synthetic  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

CKPT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "checkpoint",
                    "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth")
K = 8
BS = 16


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def model(dev, n_delta):
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    if n_delta:
        m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    if n_delta:
        m.layer_0.load_state_dict(torch.load(CKPT, map_location="cpu", weights_only=True)["0"])
        m.refresh_weights()
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("h_directions_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    print(f"card: {gpu_info()} (name, power limit, max SM clock)")
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 40)
    plain = Schedule(betas, seq, seq_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False)
    m = model(dev, 0)
    eng = m.engine
    g = torch.Generator(device=dev).manual_seed(7)
    steps = len(plain.steps)
    eng.sample(torch.randn(BS, 3, 256, 256, device=dev, generator=g), plain, record_h=True)  # warm-up / capture
    d = int(np.prod(eng.last_records["h"].shape[2:]))
    for n in (256, 1024):
        x_T = torch.randn(n, 3, 256, 256, device=dev, generator=g)
        X = torch.empty(steps, n, d, dtype=torch.float32, device=dev)

        def generate():
            for k in range(0, n, BS):
                eng.sample(x_T[k:k + BS], plain, record_h=True)
                X[:, k:k + BS].copy_(eng.last_records["h"].reshape(steps, BS, d))
        _, t_gen = clock(generate)
        w_mean = torch.full((1, n), 1.0 / n, dtype=torch.float64, device=dev)
        ops.h_gram(X[0], ops.h_combine(X[0], w_mean)[0])  # warm-up
        mus = []

        def grams():
            out = []
            for k in range(steps):
                mu = ops.h_combine(X[k], w_mean)[0]
                mus.append(mu)
                out.append(ops.h_gram(X[k], mu))
            return out
        Gs, t_gram = clock(grams)
        Gh = [G.cpu().numpy() for G in Gs]
        t0 = time.perf_counter()
        eig = [np.linalg.eigh(G) for G in Gh]
        t_eigh = time.perf_counter() - t0
        W = [torch.from_numpy(np.ascontiguousarray((U[:, ::-1][:, :K] / np.sqrt(lam[::-1][:K])).T)).to(dev)
             for lam, U in eig]

        def project():
            return [ops.h_combine(X[k], W[k], mus[k]) for k in range(steps)]
        V, t_proj = clock(project)
        unit = max(abs(float(v.norm(dim=1).max()) - 1.0) for v in V)
        print(f"discovery n={n} d={d} steps={steps} K={K}: generation with record_h {t_gen:.2f} s "
              f"({-(-n // BS)} replays of {BS} rows), Gram {t_gram * 1e3:.1f} ms, eigh (host) {t_eigh * 1e3:.1f} ms, "
              f"projection {t_proj * 1e3:.1f} ms; max | |v_k| - 1 | = {unit:.2e}")
        del X, Gs, V
        torch.cuda.empty_cache()
    # editing throughput, batch 16
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=200, hs_coeff=(1.0, 1.0))
    x_T = torch.randn(BS, 3, 256, 256, device=dev, generator=g)
    noise = torch.randn(sch.n_stochastic, BS, 3, 256, 256, device=dev, generator=g)
    D = torch.randn(sch.n_edit, 512, 8, 8, device=dev, generator=g)
    table = torch.tensor([[1.0, 0.5 * (i % 4)] for i in range(BS)])

    def median(fn):
        fn()
        ts = sorted(clock(fn)[1] for _ in range(a.reps))
        return ts[len(ts) // 2]
    t_add = median(lambda: eng.sample(x_T, sch, noise=noise, h_direction=D, hs_coeffs=table))
    del m, eng
    torch.cuda.empty_cache()
    m = model(dev, 1)
    eng = m.engine
    t_db = median(lambda: eng.sample(x_T, sch, noise=noise))
    print(f"editing, {BS} rows, 40 steps ({sch.n_edit} edit steps): additive direction {t_add * 1e3:.1f} ms, "
          f"DeltaBlock {t_db * 1e3:.1f} ms ({t_add / t_db:.3f}x)")


if __name__ == "__main__":
    main()
