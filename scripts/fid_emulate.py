"""CPU emulation of the FID Inception-v3 kernels' roundings, to bound their error against fp64 (DESIGN.md §2).

Same method as arcface_emulate.py: activations in fp32, both operands of every conv rounded to TF32 with fp32
accumulation (the TF32 implicit GEMM on the GPU); the input pack, the pools and the global mean plain fp32.  The BN is
applied after the conv here, where the GPU folds it into the weights before rounding them: the same number of TF32
roundings per product.  The full synthetic network (synthetic.inception_state_dict, seeds 7 and 8, oracle.fid's
formulas) on sets of 8 smooth images in [-1, 1] (64 x 64, resized to 299 x 299).  Prints

  * the max-abs error of the pool features, absolute and relative to max |feature|,
  * FID and KID of a set against a small edit of it (+ 0.1 of other smooth images), against unrelated images, and
    against itself, in fp64 (moments and statistics from fp64 features) with the absolute error of the emulated ones.

    python scripts/fid_emulate.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from arcface_emulate import emulated  # noqa: E402
from asyrp_official_b200 import synthetic  # noqa: E402
from asyrp_official_b200.fid import frechet_distance, kid_from_sums  # noqa: E402
from clip_image_emulate import smooth_images  # noqa: E402
from oracle import fid as ofid  # noqa: E402

N, S = 8, 64


def kid(f1, f2):
    f1, f2 = np.asarray(f1, dtype=np.float64), np.asarray(f2, dtype=np.float64)
    d = f1.shape[1]
    kxx, kyy, kxy = ((a @ b.T / d + 1) ** 3 for a, b in ((f1, f1), (f2, f2), (f1, f2)))
    return kid_from_sums(kxx.sum() - np.trace(kxx), kyy.sum() - np.trace(kyy), kxy.sum(), len(f1), len(f2))


def scores(f1, f2):
    return frechet_distance(*ofid.moments(f1), *ofid.moments(f2)), kid(f1, f2)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    worst = [0.0, 0.0, 0.0]
    for seed in (7, 8):
        sd = synthetic.inception_state_dict(seed=seed)
        m64, m32 = ofid.fid_inception(sd), ofid.fid_inception(sd, dtype=torch.float32)
        src = smooth_images(N, S, seed)
        sets = {"edit 0.1": (src + 0.1 * smooth_images(N, S, seed + 100)).clamp(-1, 1),
                "unrelated": smooth_images(N, S, seed + 200), "itself": src}
        f64 = {k: ofid.features(m64, ofid.preprocess(v)) for k, v in {"src": src, **sets}.items()}
        with emulated():
            f32 = {k: ofid.features(m32, ofid.preprocess(v, dtype=torch.float32)).double()
                   for k, v in {"src": src, **sets}.items()}
        err = max((f32[k] - f64[k]).abs().max().item() for k in f64)
        mx = max(f64[k].abs().max().item() for k in f64)
        print(f"seed {seed}: features max-abs {err:.3e} (rel {err / mx:.3e}, max|f| {mx:.2f})")
        worst[0] = max(worst[0], err)
        for name in sets:
            (fd, kd), (fe, ke) = scores(f64["src"], f64[name]), scores(f32["src"], f32[name])
            print(f"    {name:10s}: FID {fd:.6g} (abs err {abs(fe - fd):.3e}), KID {kd:.6g} (abs err {abs(ke - kd):.3e})")
            worst[1], worst[2] = max(worst[1], abs(fe - fd)), max(worst[2], abs(ke - kd))
    print(f"worst: features max-abs {worst[0]:.3e}, FID abs err {worst[1]:.3e}, KID abs err {worst[2]:.3e}")


if __name__ == "__main__":
    main()
