"""CPU emulation of the CLIP text kernels' roundings, to bound their error against fp64 (DESIGN.md §2).

The kernels keep activations in fp32 and round both operands of every linear layer to TF32 (10-bit mantissa, round
to nearest, ties away: cvt.rna.tf32.f32), accumulating in fp32; LayerNorm, attention, pooling and the cosine are
plain fp32.  This script evaluates encode_text that way (oracle.clip_text's formulas, fp32, with the GEMM operands
rounded) and in fp64, on the seeded synthetic towers the GPU tests use, and prints the relative max-abs error of the
features and the absolute error of the source/target cosine.

    python scripts/clip_text_emulate.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import synthetic  # noqa: E402
from oracle import clip_text as oct  # noqa: E402

PROMPTS = ["face", "smiling face", "person", "person with blond hair", "photo", "painting by gogh", "a photo of a "
           "red sports car on the street", "Person with curly hair and a very long beard, in a garden"]


def tf32(x):
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)  # |x| rounded to 10 mantissa bits, ties away from zero


def emulated_encode(sd, ids):
    orig = torch.Tensor.__matmul__

    def mm(a, b):  # every linear layer (weight operand 2-D); the attention's batched products stay fp32
        if b.dim() == 2:
            return orig(tf32(a), tf32(b))
        return orig(a, b)

    torch.Tensor.__matmul__ = mm
    try:
        return oct.encode_text(sd, ids, dtype=torch.float32)
    finally:
        torch.Tensor.__matmul__ = orig


def main():
    merges = synthetic.clip_bpe_merges(PROMPTS)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        gz = os.path.join(d, "bpe.txt.gz")
        n = synthetic.write_clip_vocab(gz, merges)
        ids = oct.SimpleTokenizer(gz).tokenize(PROMPTS)
    half = len(PROMPTS) // 2
    for width, layers in ((512, 12), (768, 12), (128, 2)):
        for seed in (1, 2, 3):
            sd = synthetic.clip_text_state_dict(seed=seed, width=width, layers=layers, vocab=n, embed_dim=512)
            ref = oct.encode_text(sd, ids, dtype=torch.float64)
            out = emulated_encode(sd, ids).double()
            e = ((out - ref).abs().max() / ref.abs().max()).item()
            ce = (oct.cosine(out[:half], out[half:]) - oct.cosine(ref[:half], ref[half:])).abs().max().item()
            print(f"width {width} layers {layers} seed {seed}: features rel max-abs {e:.3e}  cosine abs {ce:.3e}")


if __name__ == "__main__":
    main()
