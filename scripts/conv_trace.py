"""Pipeline timeline of one conv launch (diagnostic build of the library with -DASYRP_TRACE).

    ASYRP_LIB_SUFFIX=_trace ASYRP_EXTRA_NVCC_FLAGS=-DASYRP_TRACE python -m asyrp_official_b200.build   # build container
    ASYRP_LIB_SUFFIX=_trace python scripts/conv_trace.py SPEC [--out gpurun_out/trace.npz]              # GPU box
    SPEC = H,Cin,Cout[,nseg[,fused[,n1x1]]]  (batch 16; n1x1: number of extra 1x1 segments of Cin channels)

Every role of conv_gemm_kernel stamps clock64() at its hand-off points (csrc/conv_gemm.cu ASYRP_TRACE_STAMP):
  0 A-producer: slot free, TMA issued      1 transform: stage landed      2 transform: stage done
  3 MMA: waits for the stage               4 MMA: stage ready             9 MMA: all MMAs of the stage issued
  5 MMA: tile start                        6 MMA: accumulator free        7 epilogue: accumulator full   8 epilogue: drained
The script saves the raw stamps and prints, per CTA, where the tensor pipe's idle time between stages comes from."""
import argparse, ctypes as C, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import ops, _lib
ap = argparse.ArgumentParser()
ap.add_argument("spec")
ap.add_argument("--out", default="gpurun_out/trace.npz")
a = ap.parse_args()
dev = torch.device("cuda:0")
N = 16
f = [int(v) for v in a.spec.split(",")]
H, Cin, Cout = f[:3]
nseg = f[3] if len(f) > 3 else 1
fused = f[4] if len(f) > 4 else 0
n1 = f[5] if len(f) > 5 else 0
segs = []
for _ in range(nseg):
    x = torch.randn(N, H, H, Cin, device=dev).half()
    aff = torch.stack([torch.ones(N, Cin, device=dev), torch.zeros(N, Cin, device=dev)], -1).contiguous()
    segs.append((x, ops.MODE_3x3, aff, 0, 1) if fused else (x, ops.MODE_3x3))
for _ in range(n1):
    segs.append((torch.randn(N, H, H, Cin, device=dev).half(), ops.MODE_1x1))
K = 9 * Cin * nseg + Cin * n1
w = (torch.randn(Cout, K, device=dev) / K ** 0.5).half()
out = torch.empty(N, H, H, Cout, device=dev, dtype=torch.float16)
op = ops.ConvOp(segs, w, out=out, stats=ops.new_stats(N, H, H, Cout, dev, True))
lib = _lib.load()
ROLES, LEN = 10, 128
buf = torch.zeros(132 * ROLES * LEN, dtype=torch.int64, device=dev)
lib.asyrp_conv_set_trace.restype = C.c_int
lib.asyrp_conv_set_trace.argtypes = [C.c_void_p, C.c_void_p]
for _ in range(3):
    op.launch()
torch.cuda.synchronize()
grid = lib.asyrp_conv_set_trace(op._h, buf.data_ptr())
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); op.launch(); e1.record(); torch.cuda.synchronize()
us = e0.elapsed_time(e1) * 1e3
t = buf.cpu().numpy().reshape(132, ROLES, LEN)[:grid]
os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
np.savez_compressed(a.out, t=t, spec=a.spec, us=us, grid=grid)
print(f"{a.spec}: {us:.1f} us, grid {grid}, {2.0 * N * H * H * Cout * K / us / 1e6:.0f} TF/s")
for cta in (0, 1, grid // 2, grid - 1):
    r = t[cta]
    ns = int((r[4] > 0).sum()); nt = int((r[5] > 0).sum())
    t0 = r[5][0]
    span = r[8][nt - 1] - t0
    wait = (r[4][:ns] - r[3][:ns])
    acc_wait = (r[6][:nt] - r[5][:nt])
    issue = (r[9][:ns] - r[4][:ns])
    xf = (r[2][:ns] - r[1][:ns])
    land = (r[1][:ns] - r[0][:ns])
    print(f"CTA {cta}: {nt} tiles, {ns} stages, span {span} clk = {span / max(nt, 1):.0f} per tile; MMA warp waits: stage-ready "
          f"{wait.sum()} ({wait.sum() / span * 100:.1f}%), accumulator {acc_wait.sum()} ({acc_wait.sum() / span * 100:.1f}%); "
          f"issue per stage {issue.mean():.0f}; transform per stage {xf.mean():.0f} (max {xf.max()}); TMA issue->landed "
          f"{land.mean():.0f} (max {land.max()})")
