"""Time one CLIPText.text_cosine call of two prompts (one source, one target) at the ViT-B/16 text size (512 wide,
12 layers, 77 tokens) with CUDA events, after warm-up calls: tokenizing, the encoder, the cosine and the copy of the
result to the host.  Synthetic weights and vocabulary; the vocabulary size does not change the work.

    python scripts/clip_text_timing.py [--reps 20]
"""
import argparse
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asyrp_official_b200 import clip_text, synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    src, trg = "face", "smiling face"
    with tempfile.TemporaryDirectory() as d:
        gz = os.path.join(d, "bpe.txt.gz")
        n = synthetic.write_clip_vocab(gz, synthetic.clip_bpe_merges([src, trg]))
        m = clip_text.CLIPText(synthetic.clip_text_state_dict(seed=1, vocab=n), gz)
    for _ in range(3):
        m.text_cosine(src, trg)
    times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        m.text_cosine(src, trg)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    print(f"{torch.cuda.get_device_name()}: text_cosine of 2 prompts, median {times[len(times) // 2]:.3f} ms, "
          f"min {times[0]:.3f} ms over {a.reps} calls")


if __name__ == "__main__":
    main()
