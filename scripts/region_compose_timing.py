"""Time `--region_compose` on the GPU and print the card and its power limit.

  - compose kernel: ops.compose_rows at 256², b = 16 images, C = 3, K in {1, 2, 3, 4} attributes, CUDA events around
    one replay of a graph of 200 launches, against the bytes it moves, (2K + 1) C 4 + 4K per pixel (read the K rows,
    the origin and the K masks; write the K rows), over the 3.35 TB/s data-sheet bound; ops.blend_rows on the same 16
    images as the K = 1 yardstick;
  - replay: DDPM CelebA-HQ 256² on seeded weights with K = 3 seeded DeltaBlocks, the 40-step generative grid, the rows
    --max_rows_per_replay 16 gives (K b = 15: b = 5 images), each attribute its own t_edit / t_addnoise; the same
    RowSchedule with and without compose=, the two alternated, median of --reps replays (host clock around work that
    ends in a device synchronise, after one warm-up of each).

    python scripts/region_compose_timing.py [--reps 5] [--out results/region_compose_timing.json]
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
from asyrp_official_b200 import modules, ops, synthetic  # noqa: E402
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences  # noqa: E402
from oracle import ddpm as od, sampler as osmp  # noqa: E402

S, C, STEPS = 256, 3, 40
B_KERNEL = 16
K_REPLAY, B_REPLAY = 3, 5
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
    """the time of one fn() launch: n launches captured back to back in one graph (no host overhead), CUDA events"""
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("region_compose_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "torch": torch.__version__, "kernel": {}}
    # the kernels alone
    ref = torch.randn(B_KERNEL, C, S, S, device=dev)
    for K in (1, 2, 3, 4):
        x = torch.randn(K * B_KERNEL, C, S, S, device=dev)
        masks = torch.rand(K, B_KERNEL, S, S, device=dev) / K
        ms = graph_ms(lambda: ops.compose_rows(x, ref, masks), dev)
        nbytes = B_KERNEL * S * S * ((2 * K + 1) * C * 4 + 4 * K)
        res["kernel"][f"compose_K{K}"] = {"ms": ms, "bytes": nbytes, "TB_per_s": nbytes / (ms * 1e-3) / 1e12,
                                          "share_of_3.35TB_per_s": nbytes / HBM / (ms * 1e-3)}
    x = torch.randn(B_KERNEL, C, S, S, device=dev)
    mask = torch.rand(B_KERNEL, S, S, device=dev)
    ms = graph_ms(lambda: ops.blend_rows(x, ref, mask), dev)
    nbytes = B_KERNEL * S * S * (3 * C * 4 + 4)
    res["kernel"]["blend_K1"] = {"ms": ms, "bytes": nbytes, "TB_per_s": nbytes / (ms * 1e-3) / 1e12,
                                 "share_of_3.35TB_per_s": nbytes / HBM / (ms * 1e-3)}
    del x, ref, mask
    # the whole trajectory
    cfg = od.CELEBA_CFG
    m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                        data=NS(image_size=cfg["image_size"])))
    m.setattr_layers(K_REPLAY)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    eng = m.engine
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, STEPS)
    times = [(500, 0), (600, 300), (400, 0)][:K_REPLAY]
    coeffs = [tuple([1.0] + [1.0 if j == k else 0.0 for j in range(K_REPLAY)]) for k in range(K_REPLAY)]
    rs = RowSchedule(betas, seq, seq_next, [times[k][0] for k in range(K_REPLAY) for _ in range(B_REPLAY)],
                     [times[k][1] for k in range(K_REPLAY) for _ in range(B_REPLAY)],
                     [coeffs[k] for k in range(K_REPLAY) for _ in range(B_REPLAY)])
    origin = Schedule(betas, seq, seq_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False)
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(B_REPLAY, 3, S, S, generator=g).to(dev)
    eng.sample(x_T, origin, record_process=True)
    ref = eng.last_records["x"].clone()
    masks = torch.rand(K_REPLAY, B_REPLAY, S, S, generator=g).to(dev) / K_REPLAY
    rows = x_T.repeat(K_REPLAY, 1, 1, 1)
    z = torch.randn(rs.n_stochastic, B_REPLAY, 3, S, S, generator=g).to(dev).repeat(1, K_REPLAY, 1, 1, 1)
    plain = lambda: eng.sample(rows, rs, noise=z)  # noqa: E731
    composed = lambda: eng.sample(rows, rs, noise=z, compose=(masks, ref))  # noqa: E731
    plain()
    launches_plain = eng.last_launches
    composed()
    launches_compose = eng.last_launches
    t_plain, t_comp = [], []
    for _ in range(a.reps):
        t_plain.append(clock(plain))
        t_comp.append(clock(composed))
    res.update({"replay_rows": K_REPLAY * B_REPLAY, "replay_K": K_REPLAY, "replay_images": B_REPLAY, "steps": STEPS,
                "replay_ms": 1e3 * median(t_plain), "replay_compose_ms": 1e3 * median(t_comp),
                "replay_ms_all": [1e3 * t for t in t_plain], "replay_compose_ms_all": [1e3 * t for t in t_comp],
                "replay_launches": launches_plain, "replay_launches_compose": launches_compose})
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
