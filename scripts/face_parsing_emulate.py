"""CPU emulation of the face-parsing kernels' roundings, to bound their error against fp64 (DESIGN.md §2).

Same method as arcface_emulate.py: activations in fp32, both operands of every conv over a map larger than 1x1 (the
stem, the ResNet, the ARM / head / FFM convs and the class layer: the TF32 implicit GEMM on the GPU) rounded to TF32
with fp32 accumulation; the input pack, max-pool, the gates' 1x1 layers on the pooled vectors, the upsampling and the
argmax plain fp32.  The full synthetic BiSeNet (synthetic.face_parsing_state_dict, seeds 7 and 8, oracle.face_parsing's
formulas), smooth images in [-1, 1] and the same images scaled by 1e3 (clamped by the input stage).  Prints

  * the max-abs error of the 64 x 64 logits, absolute and relative to max |logit|,
  * the fraction of the 512^2 labels that differ from fp64's, and the fraction of pixels whose fp64 top-2 margin is
    at most twice the upsampled logits' max-abs error (the only pixels whose label may flip),
  * the absolute error of SC for an edit and for an image against itself.

    python scripts/face_parsing_emulate.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from arcface_emulate import emulated  # noqa: E402
from asyrp_official_b200 import synthetic  # noqa: E402
from clip_image_emulate import smooth_images  # noqa: E402
from oracle import face_parsing as of  # noqa: E402


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    worst = {}
    for seed in (7, 8):
        sd = synthetic.face_parsing_state_dict(seed=seed)
        src = smooth_images(2, 256, seed)
        for scale in (1.0, 1e3):
            x = src * scale
            y = (src + 0.3 * smooth_images(2, 256, seed + 100)) * scale
            l64, u64 = of.logits(sd, x), of.logits(sd, y)
            with emulated():
                l32, u32 = of.logits(sd, x, dtype=torch.float32).double(), of.logits(sd, y, dtype=torch.float32).double()
            err = max((l32 - l64).abs().max().item(), (u32 - u64).abs().max().item())
            up_err = max((of.upsample(l32) - of.upsample(l64)).abs().max().item(),
                         (of.upsample(u32) - of.upsample(u64)).abs().max().item())
            lab64, lab32 = of.upsample(l64).argmax(1), of.upsample(l32).argmax(1)
            flips = (lab64 != lab32).double().mean().item()
            low = (of.top2_margin(l64) <= 2 * up_err).double().mean().item()
            sc64 = (of.upsample(u64).argmax(1) == lab64).double().mean((1, 2))
            sc32 = (of.upsample(u32).argmax(1) == lab32).double().mean((1, 2))
            print(f"seed {seed} |x| ~ {scale:g}: logits max-abs {err:.3e} (rel {err / l64.abs().max().item():.3e}, "
                  f"max|logit| {l64.abs().max().item():.2f}), upsampled {up_err:.3e}; label flips {flips:.3e}, "
                  f"margin <= 2 err {low:.3e}; SC {[round(v, 4) for v in sc64.tolist()]} abs err "
                  f"{(sc32 - sc64).abs().max().item():.3e}")
            w = worst.setdefault(scale, [0.0, 0.0, 0.0])
            w[0], w[1], w[2] = max(w[0], err), max(w[1], low), max(w[2], (sc32 - sc64).abs().max().item())
    for scale, (err, low, dsc) in worst.items():
        print(f"worst |x| ~ {scale:g}: logits max-abs {err:.3e}, low-margin fraction {low:.3e}, SC abs err {dsc:.3e}")


if __name__ == "__main__":
    main()
