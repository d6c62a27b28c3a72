"""One eager UNet evaluation (edit step: encoder + DeltaBlock + two decoders) at the bench workload — a short
command to wrap in a profiler."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import WORKLOADS, build_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="ddpm_celeba_b16")
ap.add_argument("--batch", type=int, default=None)
ap.add_argument("--reps", type=int, default=1)
a = ap.parse_args()
family, key, batch, _, ckpt, _ = WORKLOADS[a.workload]
batch = a.batch or batch
dev = torch.device("cuda:0")
m, _ = build_model(family, key, dev, ckpt)
P = m.engine.plan(batch)
P.x.normal_()
P.t.fill_(999.0)
P.set_coeffs((1.0, 1.0))
P.run_temb()
for _ in range(a.reps):
    P.run_encoder()
    P.run_edit()
    P.run_decoder()
torch.cuda.synchronize()
print("done", len(P.launches(True)), "launches; pool MiB", P.pool.total / 2**20)
