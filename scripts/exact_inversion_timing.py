"""Time `--exact_inversion` on the GPU and print the card and its power limit.

Model: DDPM CelebA-HQ 256² on seeded weights with one seeded DeltaBlock, the 40-step grid (t_0 = 999).
  - update kernel: ops.ddim_update_anchored against ops.ddim_update on the 16 x 3 x 256² state with B = 16 anchored
    images, CUDA events around one replay of a graph of 200 launches each, against the bytes each moves over 3.35 TB/s;
  - anchors: the recording inversion (UNetEngine.anchors, 40 evaluations) against the plain inversion replay (39), B
    images, median of --reps (host clock around work that ends in a device synchronise, after one warm-up);
  - one --run_test batch (save_image, B images x 4 hs_coeff tuples, t_edit 500, t_addnoise 0, --save_x_origin):
    today's path (an origin pass from the cached x_T, then the edits) against the anchored one (anchor_batch, then the
    anchored edits), the two alternated, median of --reps.

    python scripts/exact_inversion_timing.py [--reps 3] [--images 4] [--out results/exact_inversion_timing.json]
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
from asyrp_official_b200 import main as cli, ops  # noqa: E402
from asyrp_official_b200.diffusion_latent import Asyrp  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402

S, STEPS, N_KERNEL, TUPLES = 256, 40, 16, 4
HBM = 3.35e12


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


def graph_ms(fn, dev, n=200):
    """device time of one of n back-to-back launches captured in one graph"""
    st = torch.cuda.Stream(device=dev)
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(10):
            fn()
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(n):
            fn()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("exact_inversion_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "torch": torch.__version__}
    # ---- the update kernel at the benchmark's shape
    g = torch.Generator().manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev)  # noqa: E731
    x, et, em = rnd(N_KERNEL, 3, S, S), rnd(N_KERNEL, 3, S, S), rnd(N_KERNEL, 3, S, S)
    A0, A1, E0 = rnd(N_KERNEL, 3, S, S), rnd(N_KERNEL, 3, S, S), rnd(N_KERNEL, 3, S, S)
    at, an, c2 = 0.35, 0.52, 0.61
    t_anch = graph_ms(lambda: ops.ddim_update_anchored(x, et, em, x, None, A0, A1, E0, at, an, c2), dev)
    t_ddim = graph_ms(lambda: ops.ddim_update(x, et, em, None, x, None, at, an, 0.0, c2), dev)
    b_anch, b_ddim = 4.0 * 7 * x.numel(), 4.0 * 4 * x.numel()
    res.update({"kernel_rows": N_KERNEL, "anchored_us": 1e3 * t_anch, "ddim_update_us": 1e3 * t_ddim,
                "anchored_bytes": b_anch, "ddim_update_bytes": b_ddim,
                "anchored_TBps": b_anch / (t_anch * 1e-3) / 1e12, "ddim_update_TBps": b_ddim / (t_ddim * 1e-3) / 1e12,
                "anchored_share_of_hbm": b_anch / (t_anch * 1e-3) / HBM,
                "ddim_update_share_of_hbm": b_ddim / (t_ddim * 1e-3) / HBM})
    del x, et, em, A0, A1, E0
    # ---- a runner on DDPM CelebA-HQ 256² with seeded weights
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            args, cfg = cli.parse_args_and_config(
                ["--run_test", "--config", "celeba.yml", "--exp", "./runs/t", "--bs_train", str(a.images),
                 "--n_inv_step", str(STEPS), "--n_test_step", str(STEPS), "--n_train_step", str(STEPS),
                 "--synthetic_weights", "--seed", "1234", "--train_delta_block", "--get_h_num", "1",
                 "--max_rows_per_replay", "16", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0"])
            r = Asyrp(args, cfg, device=dev)
            r.t_edit, r.t_addnoise = 500, 0
            model = r.load_pretrained_model()
            model.setattr_layers(1)
            model = model.to(dev)
            eng = model.engine
            seq, seq_next = make_sequences(999, STEPS)
            inv = Schedule.inversion(r.betas, seq, seq_next)
            x0 = (torch.rand(a.images, 3, S, S, generator=g) * 2 - 1).to(dev)
            plain_inv = lambda: eng.sample(x0, inv)  # noqa: E731
            rec_inv = lambda: eng.anchors(x0, inv)  # noqa: E731
            plain_inv()
            rec_inv()
            t_pi, t_ri = [], []
            for _ in range(a.reps):
                t_pi.append(clock(plain_inv))
                t_ri.append(clock(rec_inv))
            x_lat = plain_inv()
            coeffs = [(1.0, 0.25 * (k + 1)) for k in range(TUPLES)]
            kw = dict(save_x_origin=True, hs_coeff=coeffs, folder_dir="out", file_name="b")
            today = lambda: r.save_image(model, x_lat, seq, seq_next, **kw)  # noqa: E731
            anchored = lambda: _anchored(r, model, x0, seq, seq_next, kw)  # noqa: E731
            today()
            anchored()
            t_today, t_exact = [], []
            for _ in range(a.reps):
                t_today.append(clock(today))
                t_exact.append(clock(anchored))
        finally:
            os.chdir(cwd)
    res.update({"images": a.images, "steps": STEPS, "tuples": TUPLES,
                "plain_inversion_ms": 1e3 * median(t_pi), "recording_inversion_ms": 1e3 * median(t_ri),
                "batch_today_ms": 1e3 * median(t_today), "batch_exact_ms": 1e3 * median(t_exact),
                "plain_inversion_ms_all": [1e3 * t for t in t_pi], "recording_inversion_ms_all": [1e3 * t for t in t_ri],
                "batch_today_ms_all": [1e3 * t for t in t_today], "batch_exact_ms_all": [1e3 * t for t in t_exact]})
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


def _anchored(r, model, x0, seq, seq_next, kw):
    """one --exact_inversion batch: the anchors of the input images, then save_image from their x_T"""
    anc = r.anchor_batch(model, x0)
    return r.save_image(model, anc.x_T, seq, seq_next, anchors=anc, **kw)


if __name__ == "__main__":
    main()
