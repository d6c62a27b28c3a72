"""Pipeline timeline of one conv launch (diagnostic build of the library with -DASYRP_TRACE).

    ASYRP_LIB_SUFFIX=_trace ASYRP_EXTRA_NVCC_FLAGS=-DASYRP_TRACE python -m asyrp_official_b200.build   # build container
    ASYRP_LIB_SUFFIX=_trace python scripts/conv_trace.py SPEC [--out gpurun_out/trace.npz]              # GPU box
    SPEC = H,Cin,Cout[,nseg[,fused[,n1x1]]]  (batch 16; n1x1: number of extra 1x1 segments of Cin channels)

Every role of conv_gemm_kernel stamps clock64() at its hand-off points (csrc/conv_gemm.cu ASYRP_TRACE_STAMP):
  0 A-producer: slot free, TMA issued      1 transform: stage landed      2 transform: stage done
  3 MMA: waits for the stage               4 MMA: stage ready             9 MMA: all MMAs of the stage issued
  5 MMA: tile start                        6 MMA: staging tile free (the previous tile's epilogue has read it)
  7 epilogue: staging tile full            8 epilogue: staging tile drained
  10 MMA: clocks the stage spent waiting for weight stages (a duration, not a time stamp)
  11 transform: stage transformed, before the proxy fence (stages without a transform have no stamp)
A library built before the staging handoff has 10 roles (--roles 10) and no stamp 6 or 10; one built before the fence
stamp has 11 (--roles 11).

Per CTA the script prints, as shares of the CTA's span (first tile start to last drain):
  * tile boundaries: from the last MMA issue of tile i to the first stage of tile i+1 being ready (includes the last
    wgmma group's execution), split into the wait for the staging tile and the rest (staging write, A-stage wait);
  * A waits: the MMA warps waiting for a ready activation stage inside a tile;
  * B waits: the MMA warps waiting for a weight stage;
  * the epilogue's length per tile, the transform warps' clocks per stage, and how many of them the proxy fence after
    the transform takes."""
import argparse, ctypes as C, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import ops, _lib
ap = argparse.ArgumentParser()
ap.add_argument("spec")
ap.add_argument("--out", default="gpurun_out/trace.npz")
ap.add_argument("--roles", type=int, default=12,
                help="trace roles of the library (10 before the staging handoff, 11 before the fence stamp)")
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
ROLES, LEN = a.roles, 128
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
np.savez_compressed(a.out, t=t, spec=a.spec, us=us, grid=grid, roles=ROLES)
print(f"{a.spec}: {us:.1f} us, grid {grid}, {2.0 * N * H * H * Cout * K / us / 1e6:.0f} TF/s")
# K stages per tile: one per 64-channel chunk (halo tiles, 1x1 chunks), three dx-shifted copies per 3x3 chunk otherwise
halo = H % 16 == 0
spt = (Cin // 64) * (nseg * (1 if halo else 3) + n1)
rows = []
for cta in range(grid):
    r = t[cta]
    nt = int((r[5] > 0).sum())
    nts = min(nt, LEN // spt)  # tiles whose stages are all stamped
    ns = nts * spt
    span = r[8][nt - 1] - r[5][0]
    first = np.arange(1, nts) * spt          # first stage of tiles 1..nts-1
    gap = r[4][first] - r[9][first - 1]      # last MMA issue of tile i -> first stage of tile i+1 ready
    st_wait = (r[6][:nts - 1] - r[9][first - 1]) if ROLES > 10 else np.zeros(0)
    inner = np.setdiff1d(np.arange(ns), np.arange(0, ns, spt))
    a_wait = r[4][inner] - r[3][inner]
    b_wait = r[10][:ns] if ROLES > 10 else np.zeros(0)
    epi = r[8][:nt] - r[7][:nt]
    # shares of the stamped part of the span (stage stamps stop at LEN)
    cov = (r[9][ns - 1] - r[5][0]) if nts < nt else span
    fenced = (r[11][:ns] > 0) if ROLES > 11 else np.zeros(ns, bool)
    fence = (r[2][:ns] - r[11][:ns])[fenced].mean() if fenced.any() else 0.0
    rows.append((nt, span / nt, gap.sum() / cov, st_wait.sum() / cov, a_wait.sum() / cov, b_wait.sum() / cov,
                 epi.mean(), (r[2][:ns] - r[1][:ns]).mean(), fence))
R = np.array(rows)
print("CTA  tiles  clk/tile  boundary%  (staging wait%)  A-wait%  B-wait%  epilogue clk  transform clk/stage  fence clk")
for cta in sorted({0, 1, grid // 2, grid - 1}):
    nt, pt, g, s, aw, bw, ep, xf, fc = R[cta]
    print(f"{cta:3d} {nt:6.0f} {pt:9.0f} {100 * g:9.1f}  ({100 * s:5.1f})       {100 * aw:6.1f}  {100 * bw:6.1f}  {ep:12.0f}  "
          f"{xf:8.0f}  {fc:8.0f}")
nt, pt, g, s, aw, bw, ep, xf, fc = R.mean(0)
print(f"all {nt:6.1f} {pt:9.0f} {100 * g:9.1f}  ({100 * s:5.1f})       {100 * aw:6.1f}  {100 * bw:6.1f}  {ep:12.0f}  {xf:8.0f}  "
      f"{fc:8.0f}")
