"""Micro-benchmark: 3x3 conv -> 128 channels @256x256, batch 16, K swept via Cin; fused (GN+SiLU operand) vs unfused."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import ops
dev = torch.device("cuda:0")
N, H, W, Cout = 16, 256, 256, 128
for fused in (0, 1):
    for Cin in (64, 128, 256, 512):
        x = torch.randn(N, H, W, Cin, device=dev).half()
        w = (torch.randn(Cout, 9 * Cin, device=dev) / (3 * Cin ** 0.5)).half()
        out = torch.empty(N, H, W, Cout, device=dev, dtype=torch.float16)
        aff = torch.stack([torch.ones(N, Cin, device=dev), torch.zeros(N, Cin, device=dev)], -1).contiguous()
        seg = (x, ops.MODE_3x3, aff, 0, 1) if fused else (x, ops.MODE_3x3)
        st = ops.new_stats(N, H, W, Cout, dev, True)
        op = ops.ConvOp([seg], w, out=out, stats=st)
        for _ in range(3): op.launch()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): op.launch()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        fl = 2.0 * N * H * W * Cout * 9 * Cin
        tiles = N * H * W / 256
        print(f"fused={fused} Cin={Cin:4d} stages/tile={Cin//64:2d}  {ms*1e3:8.1f} us  {fl/ms/1e9:7.1f} TF/s   per-tile {ms*1e3*132/tiles:6.2f} us")
