"""CPU emulation of the ArcFace kernels' roundings, to bound their error against fp64 (DESIGN.md §2).

Same method as clip_image_emulate.py: activations in fp32, both operands of every 3x3 / shortcut conv and of the
25088 -> 512 linear layer rounded to TF32 with fp32 accumulation; the crop and pool, BatchNorm, PReLU, the
squeeze-excitation gate (its 1x1 convs act on a 1x1 map: plain fp32 on the GPU), l2_norm and the dot product plain
fp32.  The full synthetic IR-SE50 (synthetic.arcface_state_dict, seeds 7 and 8, oracle.arcface's formulas), smooth
images in [-1, 1] and the same images scaled by 1e3 (synthetic UNet weights give |x_0| ~ 1e3).  Prints

  * the max-abs error of the unit features (relative to max |f|, which is the same as absolute up to ~1/sqrt(512)),
  * the absolute error of ID = 1 - IDLoss for edits of decreasing size, and for an image against itself.

    python scripts/arcface_emulate.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import synthetic  # noqa: E402
from clip_image_emulate import smooth_images  # noqa: E402
from clip_text_emulate import tf32  # noqa: E402
from oracle import arcface as oa  # noqa: E402


class emulated:
    """within the block: convs over maps larger than 1x1 and every product with a 2-D weight on TF32 operands"""

    def __enter__(self):
        self.mm, self.conv = torch.Tensor.__matmul__, torch.nn.functional.conv2d
        mm, conv = self.mm, self.conv
        torch.Tensor.__matmul__ = lambda a, b: mm(tf32(a), tf32(b)) if b.dim() == 2 else mm(a, b)
        torch.nn.functional.conv2d = lambda x, w, *a, **k: (conv(tf32(x), tf32(w), *a, **k) if x.shape[-1] > 1
                                                           else conv(x, w, *a, **k))

    def __exit__(self, *exc):
        torch.Tensor.__matmul__, torch.nn.functional.conv2d = self.mm, self.conv


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for seed in (7, 8):
        sd = synthetic.arcface_state_dict(seed=seed)
        src = smooth_images(2, 256, seed)
        for scale in (1.0, 1e3):
            x = src * scale
            f64 = oa.extract_feats(sd, x)
            with emulated():
                f32 = oa.extract_feats(sd, x, dtype=torch.float32).double()
            e = ((f32 - f64).abs().max() / f64.abs().max()).item()
            self_id = (f32 * f32).sum(-1)
            print(f"seed {seed} |x| ~ {scale:g}: features rel max-abs {e:.3e}, |1 - ID(x, x)| "
                  f"{(1 - self_id).abs().max().item():.3e}")
            for delta in (1.0, 3e-1, 1e-1, 1e-2):
                y = (src + delta * smooth_images(2, 256, seed + 100)) * scale
                g64 = oa.extract_feats(sd, y)
                with emulated():
                    g32 = oa.extract_feats(sd, y, dtype=torch.float32).double()
                id64, id32 = (g64 * f64).sum(-1), (g32 * f32).sum(-1)
                print(f"    edit {delta:g}: ID {[round(v, 4) for v in id64.tolist()]}  abs err "
                      f"{(id32 - id64).abs().max().item():.3e}")


if __name__ == "__main__":
    main()
