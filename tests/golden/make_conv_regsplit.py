"""Writes conv_regsplit.json: SHA-256 of the outputs and statistics of tests/test_conv_regsplit_gpu.py's cases.

    python tests/golden/make_conv_regsplit.py [--out tests/golden/conv_regsplit.json]      # on an H100

Run it with the library build whose bits are to be kept (ASYRP_LIB_SUFFIX selects a build beside the product one).  The
committed file comes from the last build whose conv_gemm_kernel ran 576 threads at one register limit.
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]
import test_conv_regsplit_gpu as t  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=os.path.join(HERE, "conv_regsplit.json"))
a = ap.parse_args()
dev = torch.device("cuda:0")
golden = {t.case_id(s, r): t.run_case(s, r, dev) for s, r in t.CASES}
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(golden, f, indent=1, sort_keys=True)
    f.write("\n")
print(f"{a.out}: {len(golden)} cases")
