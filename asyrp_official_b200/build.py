"""Build libasyrp_b200.so in-tree with nvcc for sm_90a (H100).

The shared library is the C-ABI boundary (include/asyrp_b200.h).  It is built into the package directory
so that it travels with the repository snapshot to the GPU box; nothing is JIT-compiled at import time.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# ASYRP_LIB_SUFFIX / ASYRP_EXTRA_NVCC_FLAGS: diagnostic builds next to the product library (scripts/conv_trace.py)
SUFFIX = os.environ.get("ASYRP_LIB_SUFFIX", "")
LIB = os.path.join(HERE, f"libasyrp_b200{SUFFIX}.so")
SOURCES = ["common.cu", "conv_gemm.cu", "pointwise.cu", "attention.cu", "lpips.cu", "clip_text.cu", "clip_image.cu",
           "arcface.cu", "face_parsing.cu", "fid.cu", "prdc.cu", "preservation.cu",
           "hspace.cu", "region.cu", "inversion.cu", "dino.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-cudart", "static",
]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if not f.endswith(".o")] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile every CUDA source into libasyrp_b200.so (no-op when up to date)."""
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(CSRC, src.replace(".cu", f"{SUFFIX}.o"))
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("ASYRP_EXTRA_NVCC_FLAGS", "").split(), "-c", path, "-o", obj] + \
            (["-Xptxas", "-v"] if verbose else [])
        subprocess.run(cmd, check=True)
        objs.append(obj)
    subprocess.run([nvcc, "-shared", *NVCC_FLAGS[:2], "-cudart", "static", "-o", LIB, *objs], check=True)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
