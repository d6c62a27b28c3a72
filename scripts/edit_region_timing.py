"""Time `--edit_region` on the GPU and print the card and its power limit.

Model: DDPM CelebA-HQ 256² on seeded weights with one seeded DeltaBlock, the 40-step generative grid (t_0 = 999,
t_edit 500, t_addnoise 0), 16 rows per replay: 4 images x 4 hs_coeff tuples, as save_image runs them.
  - replay: one edit trajectory with and without the region blend, the two alternated, median of --reps replays (host
    clock around work that ends in a device synchronise, after one warm-up of each);
  - blend kernel: ops.blend_rows on the 16 x 3 x 256² state with 4 masks and reference images, CUDA events around
    one replay of a graph of 200 launches, against the bytes it moves (read x, ref, mask; write x) over 3.35 TB/s;
  - mask build: the mask of one batch of 4 images (the face parser's labels of the origin x0, select, dilate r = 4,
    feather sigma = 2), median of --reps, and the mask kernels alone.

    python scripts/edit_region_timing.py [--reps 5] [--out results/edit_region_timing.json]
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
from asyrp_official_b200 import face_parsing, modules, ops, region, synthetic  # noqa: E402
from asyrp_official_b200.schedule import Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

B, TUPLES, S, STEPS = 4, 4, 256, 40
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("edit_region_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    eng = m.engine
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, STEPS)
    edit = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0))
    origin = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0,), edit=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, S, S, generator=g).to(dev)
    x0 = eng.sample(x, origin, record_process=True)
    ref = eng.last_records["x"].clone()
    parser = face_parsing.FaceParser(synthetic.face_parsing_state_dict(seed=5), device=dev)
    classes = region.parse_classes("hair hat")
    mask = region.region_masks(parser, x0, classes, 4, 2.0)
    rows = x.repeat(TUPLES, 1, 1, 1)
    table = torch.tensor([[1.0, 0.25 * (k + 1)] for k in range(TUPLES) for _ in range(B)])
    plain = lambda: eng.sample(rows, edit, hs_coeffs=table)  # noqa: E731
    blended = lambda: eng.sample(rows, edit, hs_coeffs=table, blend=(mask, ref))  # noqa: E731
    plain()
    blended()
    t_plain, t_blend = [], []
    for _ in range(a.reps):
        t_plain.append(clock(plain))
        t_blend.append(clock(blended))
    # the blend kernel alone at the replay's shape
    xs = torch.randn(B * TUPLES, 3, S, S, device=dev)
    r0 = ref[0].contiguous()
    n = 200
    st = torch.cuda.Stream(device=dev)
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(10):
            ops.blend_rows(xs, r0, mask)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()  # n launches back to back, as the trajectory graph issues them: no host overhead
    with torch.cuda.graph(graph):
        for _ in range(n):
            ops.blend_rows(xs, r0, mask)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    k_ms = e0.elapsed_time(e1) / n
    nbytes = 4 * (2 * xs.numel() + r0.numel() + mask.numel())
    # mask build per batch
    t_mask, t_kernels = [], []
    lab = parser.labels(x0)
    for _ in range(a.reps):
        t_mask.append(clock(lambda: region.region_masks(parser, x0, classes, 4, 2.0)))
        t_kernels.append(clock(lambda: region.masks_from_labels(lab, classes, S, 4, 2.0)))
    res = {
        "gpu": gpu_info(), "torch": torch.__version__, "rows": B * TUPLES, "images": B, "steps": STEPS,
        "replay_ms": 1e3 * median(t_plain), "replay_blend_ms": 1e3 * median(t_blend),
        "replay_launches": None, "blend_kernel_ms": k_ms, "blend_bytes": nbytes,
        "blend_bytes_over_hbm_ms": 1e3 * nbytes / HBM, "blend_share_of_hbm": (nbytes / HBM) / (k_ms * 1e-3),
        "blend_steps_share_of_replay": STEPS * k_ms / (1e3 * median(t_plain)),
        "mask_build_ms": 1e3 * median(t_mask), "mask_kernels_ms": 1e3 * median(t_kernels),
        "replay_ms_all": [1e3 * t for t in t_plain], "replay_blend_ms_all": [1e3 * t for t in t_blend],
        "mask_fraction": float(mask.mean()),
    }
    eng.sample(rows, edit, hs_coeffs=table, blend=(mask, ref))
    res["replay_launches"] = eng.last_launches
    eng.sample(rows, edit, hs_coeffs=table)
    res["replay_launches_plain"] = eng.last_launches
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
