"""CPU emulation of the CLIP image kernels' roundings, to bound their error against fp64 (DESIGN.md §2).

Same method as clip_text_emulate.py: activations in fp32, both operands of every linear layer (the patch embedding
included) rounded to TF32 with fp32 accumulation; preprocessing, LayerNorm, attention, pooling and the directions
plain fp32.  Seeded synthetic ViT-B/16 and ViT-B/32 towers (oracle.clip_image's formulas), smooth images in [-1, 1]
and the same images scaled to |x| ~ 1e3 (synthetic UNet weights produce such images).  Prints

  * the relative max-abs error of encode_image's features, and
  * the absolute error of S_dir (the directional similarity, text direction from the emulated text tower) for edits
    of decreasing size, against |df|/|f| (the relative size of the feature change the edit causes).

    python scripts/clip_image_emulate.py
"""
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import synthetic  # noqa: E402
from clip_text_emulate import tf32  # noqa: E402
from oracle import clip_image as oci  # noqa: E402
from oracle import clip_text as oct  # noqa: E402

TEMPLATES = ["a bad photo of a {}.", "a photo of the hard to see {}.", "a rendering of a {}.", "the {}."]
SRC, TRG = "face", "smiling face"


class emulated:
    """within the block: every linear layer (2-D weight operand) and conv2d on TF32-rounded operands"""

    def __enter__(self):
        self.mm, self.conv = torch.Tensor.__matmul__, torch.nn.functional.conv2d
        mm, conv = self.mm, self.conv
        torch.Tensor.__matmul__ = lambda a, b: mm(tf32(a), tf32(b)) if b.dim() == 2 else mm(a, b)
        torch.nn.functional.conv2d = lambda x, w, *a, **k: conv(tf32(x), tf32(w), *a, **k)

    def __exit__(self, *exc):
        torch.Tensor.__matmul__, torch.nn.functional.conv2d = self.mm, self.conv


def smooth_images(B, S, seed):
    """sums of a few low-frequency sinusoids per channel, in [-1, 1]"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, S), torch.linspace(0, 1, S), indexing="ij")
    out = torch.zeros(B, 3, S, S)
    for _ in range(4):
        fy, fx, ph = (torch.rand(B, 3, 1, 1, generator=g) * 6 for _ in range(3))
        out += torch.sin(fy * yy * 3.14 + fx * xx * 3.14 + ph)
    return (out / 4).clamp(-1, 1)


def main():
    with tempfile.TemporaryDirectory() as d:
        gz = os.path.join(d, "bpe.txt.gz")
        n = synthetic.write_clip_vocab(gz, synthetic.clip_bpe_merges([t.format(SRC + " " + TRG) for t in TEMPLATES]))
        tok = oct.SimpleTokenizer(gz)
    for name, patch, grid in (("ViT-B/16", 16, 14), ("ViT-B/32", 32, 7)):
        for seed in (1, 2):
            sd = synthetic.clip_image_state_dict(seed=seed, width=768, layers=12, patch=patch, grid=grid,
                                                 embed_dim=512)
            sd.update(synthetic.clip_text_state_dict(seed=seed, width=512, layers=12, vocab=n, embed_dim=512))
            text64 = oci.compute_text_direction(sd, tok, TEMPLATES, SRC, TRG)
            with emulated():
                text32 = oci.compute_text_direction(sd, tok, TEMPLATES, SRC, TRG, dtype=torch.float32)
            src = smooth_images(2, 256, seed)
            for scale in (1.0, 1e3):
                x = src * scale
                f64 = oci.encode_image(sd, x)
                with emulated():
                    f32 = oci.encode_image(sd, x, dtype=torch.float32).double()
                e = ((f32 - f64).abs().max() / f64.abs().max()).item()
                print(f"{name} seed {seed} |x| ~ {scale:g}: features rel max-abs {e:.3e}")
                for delta in (3e-1, 1e-1, 3e-2, 1e-2):
                    y = (src + delta * smooth_images(2, 256, seed + 100)) * scale
                    g64 = oci.encode_image(sd, y)
                    with emulated():
                        g32 = oci.encode_image(sd, y, dtype=torch.float32).double()
                    ratio = ((g64 - f64).norm(dim=-1) / f64.norm(dim=-1)).min().item()
                    unit = lambda f: f / f.norm(dim=-1, keepdim=True)  # noqa: E731
                    s64 = torch.nn.CosineSimilarity()(oci.edit_direction(unit(f64), unit(g64)), text64)
                    s32 = torch.nn.CosineSimilarity()(oci.edit_direction(unit(f32), unit(g32)), text32.double())
                    print(f"    edit {delta:g}: |df|/|f| >= {ratio:.3e}  S_dir abs err {(s32 - s64).abs().max().item():.3e}"
                          f"  (err * |df|/|f| = {(s32 - s64).abs().max().item() * ratio:.3e})")


if __name__ == "__main__":
    main()
