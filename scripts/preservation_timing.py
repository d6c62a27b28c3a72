"""Time --content_preservation on the GPU beside the edit trajectory it scores, and print the card and its power limit.

One batch at the default workload's shape: B = 16 origin rows of 256 x 256 and 16 or 80 edited rows (--delta_interpolation
with five strengths gives 80).  Three times, CUDA events, median of --reps calls after a warm-up call of each:
  - ContentPreservation.scores(origin, edited): the copies, quantiser, pyramids, SSE, five SSIM levels, LPIPS-Alex on
    both and the host combination;
  - the SSIM kernels alone: asyrp_ssim_level at the five levels of the prepared pyramids;
  - the 40-step edit trajectory (DDPM CelebA-HQ, t_edit 500, t_addnoise 200, the shipped `smiling` DeltaBlock on
    seeded UNet weights) of the same rows, as Asyrp.save_image runs it: replays of --max_rows rows.

    python scripts/preservation_timing.py [--reps 5] [--max_rows 16]
"""
import argparse
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import modules, ops, preservation as pv, synthetic  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

CKPT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "checkpoint",
                    "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
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
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max_rows", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("preservation_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    print(f"card: {gpu_info()} (name, power limit, max SM clock)")
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    m.layer_0.load_state_dict(torch.load(CKPT, map_location="cpu", weights_only=True)["0"])
    m.refresh_weights()
    eng = m.engine
    seq, seq_next = make_sequences(999, 40)
    sch = Schedule(osmp.make_betas(), seq, seq_next, t_edit=500, t_addnoise=200, hs_coeff=(1.0, 1.0))
    B, S = 16, 256
    g = torch.Generator(device=dev).manual_seed(7)
    x_T = torch.randn(a.max_rows, 3, S, S, device=dev, generator=g)
    noise = torch.randn(sch.n_stochastic, a.max_rows, 3, S, S, device=dev, generator=g) if sch.n_stochastic else None
    origin = eng.sample(x_T[:B], Schedule(osmp.make_betas(), seq, seq_next, t_edit=10 ** 9, t_addnoise=0,
                                          hs_coeff=(1.0,), edit=False)).cpu()
    edited = eng.sample(x_T, sch, noise=noise).cpu()[:B]
    scorer = pv.ContentPreservation(synthetic.lpips_state_dict(seed=1234), device=dev)
    for n in (16, 80):
        ed = torch.cat([(edited + 0.02 * k * torch.randn(edited.shape)).clamp(-1, 1) for k in range(n // B)])
        t_score = timed(lambda: scorer.scores(origin, ed), a.reps)
        s, _ = scorer._prepare(origin, "ref")
        e, _ = scorer._prepare(ed, "timing")
        stats = torch.empty(pv.LEVELS, n, 3, 2, dtype=torch.float64, device=dev)

        def ssim():
            for lvl in range(pv.LEVELS):
                ops.ssim_level(s.levels[lvl], e.levels[lvl], stats[lvl])
        t_ssim = timed(ssim, a.reps)
        replays = -(-n // a.max_rows)

        def trajectory():
            for _ in range(replays):
                eng.sample(x_T, sch, noise=noise)
        t_traj = timed(trajectory, a.reps)
        print(f"B={B} origin rows, {n} edited rows, {S}x{S}: scorer {t_score:.2f} ms, SSIM kernels (5 levels) "
              f"{t_ssim:.3f} ms, 40-step trajectory ({replays} replay(s) of {a.max_rows} rows) {t_traj:.1f} ms; "
              f"scorer / trajectory {t_score / t_traj:.3%}")


if __name__ == "__main__":
    main()
