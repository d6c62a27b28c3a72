"""Time DiffStyle's generation on one GPU: P content / style pairs as rows of batched replays against one replay per
pair, in one process.

DDPM CelebA-HQ 256x256 with seeded synthetic UNet weights, 40 steps (--n_inv_step 40 from t_0 999), t_edit 400,
t_noise 200, dt_lambda 0.9985 from dt_end 950, one hs_coeff per pair (0.9).  The style latents and content h are seeded
random tensors: the timing does not depend on their values, and no inversion is timed.  The batched arm runs the P rows
in replays of --rows rows; the other arm runs P replays of one row.  Each arm is warmed up once (graph capture), then
the arms alternate --reps times; each timing is a host clock around the replays ending in a device synchronise.
Prints pairs/s of both arms, the speedup and the card's name, power limit and maximum SM clock, as one JSON line.

    python scripts/diff_style_timing.py [--pairs 16] [--rows 16] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import synthetic  # noqa: E402
from asyrp_official_b200.modules import DDPM  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from asyrp_official_b200.configs import load_config  # noqa: E402
from asyrp_official_b200.utils.diffusion_utils import get_beta_schedule  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--rows", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diff_style_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    config = load_config("celeba.yml")
    model = DDPM(config)
    synthetic.randomize_(model, seed=1234)
    eng = model.to(dev).engine
    betas = torch.from_numpy(get_beta_schedule(beta_start=config.diffusion.beta_start,
                                               beta_end=config.diffusion.beta_end,
                                               num_diffusion_timesteps=config.diffusion.num_diffusion_timesteps)).float()
    seq, seq_next = make_sequences(999, 40)
    sch = Schedule(betas, seq, seq_next, t_edit=400, t_addnoise=200, hs_coeff=(0.9,), dt_lambda=0.9985, dt_end=950)
    g = torch.Generator().manual_seed(0)
    S, C, hh = config.data.image_size, 512, 8
    x_T = torch.randn(a.pairs, 3, S, S, generator=g).to(dev)
    dh = torch.randn(sch.n_edit, a.pairs, C, hh, hh, generator=g).to(dev)
    nz = torch.randn(sch.n_stochastic, a.pairs, 3, S, S, generator=g).to(dev)

    def run(rows):
        out = []
        for k in range(0, a.pairs, rows):
            sl = slice(k, min(k + rows, a.pairs))
            n = sl.stop - sl.start
            if n < rows:  # the last replay padded to the captured row count
                pad = lambda t, d: torch.cat([t, t.narrow(d, t.shape[d] - 1, 1).expand(  # noqa: E731
                    *[rows - n if i == d else -1 for i in range(t.dim())])], dim=d)
                out.append(eng.sample(pad(x_T[sl], 0), sch, noise=pad(nz[:, sl], 1).contiguous(),
                                      delta_hs=pad(dh[:, sl], 1).contiguous())[:n])
            else:
                out.append(eng.sample(x_T[sl], sch, noise=nz[:, sl].contiguous(), delta_hs=dh[:, sl].contiguous()))
        return torch.cat(out)

    def timed(rows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = run(rows)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    batched_out = run(a.rows)  # warm-up: plans and graph captures
    single_out = run(1)
    same = bool(torch.equal(batched_out, single_out))
    tb, ts = [], []
    for _ in range(a.reps):
        tb.append(timed(a.rows)[0])
        ts.append(timed(1)[0])
    res = {"workload": "diff_style DDPM CelebA-HQ 256x256, 40 steps, t_edit 400, t_noise 200", "pairs": a.pairs,
           "rows_per_replay": a.rows, "batched_pairs_per_s": a.pairs / min(tb), "single_pairs_per_s": a.pairs / min(ts),
           "speedup": min(ts) / min(tb), "batched_s": tb, "single_s": ts, "rows_equal_single_replays": same,
           "gpu": gpu_info()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
