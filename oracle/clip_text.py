"""CPU oracle of CLIP's text tower: a plain restatement of OpenAI CLIP's encode_text (model.py: the residual
attention blocks, the causal mask, ln_final at the end-of-text token, text_projection), of its SimpleTokenizer +
tokenize, and of the CosineSimilarity(dim=1, eps=1e-6) Asyrp.set_t_edit_t_addnoise takes (diffusion_latent.py:1327).
Test infrastructure only; evaluated in fp32 or fp64 (the `dtype` argument)."""
import gzip
import html
import math
import re

import torch

PAT = r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+"""


def layer_norm(x, w, b):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, 1e-5)


def quick_gelu(z):
    return z * torch.sigmoid(1.702 * z)


def causal_attention(x, in_w, in_b, out_w, out_b, heads):
    """nn.MultiheadAttention(width, heads)(x, x, x, attn_mask=triu(-inf, 1)) on x [P][T][w]"""
    P, T, w = x.shape
    dh = w // heads
    q, k, v = (x @ in_w.t() + in_b).split(w, dim=-1)
    q, k, v = (t.reshape(P, T, heads, dh).transpose(1, 2) for t in (q, k, v))
    s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
    mask = torch.full((T, T), float("-inf"), dtype=x.dtype).triu(1)
    a = torch.softmax(s + mask, dim=-1) @ v
    return a.transpose(1, 2).reshape(P, T, w) @ out_w.t() + out_b


def encode_text(sd, ids, dtype=torch.float64):
    """CLIP's encode_text on token ids [P][T] with a CLIP state dict (text-tower keys): [P][embed_dim]"""
    g = {k: v.to(dtype) for k, v in sd.items() if not k.startswith("visual.")}
    width = g["ln_final.weight"].shape[0]
    heads = width // 64
    layers = len({k.split(".")[2] for k in g if k.startswith("transformer.resblocks.")})
    ids = torch.as_tensor(ids).long()
    x = g["token_embedding.weight"][ids] + g["positional_embedding"]
    for i in range(layers):
        p = f"transformer.resblocks.{i}."
        x = x + causal_attention(layer_norm(x, g[p + "ln_1.weight"], g[p + "ln_1.bias"]), g[p + "attn.in_proj_weight"],
                                 g[p + "attn.in_proj_bias"], g[p + "attn.out_proj.weight"], g[p + "attn.out_proj.bias"],
                                 heads)
        h = layer_norm(x, g[p + "ln_2.weight"], g[p + "ln_2.bias"])
        h = quick_gelu(h @ g[p + "mlp.c_fc.weight"].t() + g[p + "mlp.c_fc.bias"])
        x = x + h @ g[p + "mlp.c_proj.weight"].t() + g[p + "mlp.c_proj.bias"]
    x = layer_norm(x, g["ln_final.weight"], g["ln_final.bias"])
    return x[torch.arange(x.shape[0]), ids.argmax(dim=-1)] @ g["text_projection"]


def cosine(a, b):
    return torch.nn.CosineSimilarity(dim=1, eps=1e-6)(a, b)


# ---------------------------------------------------------------------------------------------------------------------
def bytes_to_unicode():
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


class SimpleTokenizer:
    """SimpleTokenizer without ftfy"""

    def __init__(self, bpe_path):
        import regex
        self.byte_encoder = bytes_to_unicode()
        merges = gzip.open(bpe_path).read().decode("utf-8").split("\n")
        merges = [tuple(m.split()) for m in merges[1:49152 - 256 - 2 + 1]]
        vocab = list(bytes_to_unicode().values())
        vocab = vocab + [v + "</w>" for v in vocab] + ["".join(m) for m in merges] + ["<|startoftext|>",
                                                                                      "<|endoftext|>"]
        self.encoder = dict(zip(vocab, range(len(vocab))))
        self.bpe_ranks = dict(zip(merges, range(len(merges))))
        self.pat = regex.compile(PAT, regex.IGNORECASE)

    def bpe(self, token):
        word = tuple(token[:-1]) + (token[-1] + "</w>",)
        while len(word) > 1:
            pairs = set(zip(word, word[1:]))
            bigram = min(pairs, key=lambda p: self.bpe_ranks.get(p, float("inf")))
            if bigram not in self.bpe_ranks:
                break
            first, second = bigram
            new, i = [], 0
            while i < len(word):
                try:
                    j = word.index(first, i)
                except ValueError:
                    new.extend(word[i:])
                    break
                new.extend(word[i:j])
                i = j
                if i < len(word) - 1 and word[i + 1] == second:
                    new.append(first + second)
                    i += 2
                else:
                    new.append(word[i])
                    i += 1
            word = tuple(new)
        return word

    def encode(self, text):
        text = re.sub(r"\s+", " ", html.unescape(html.unescape(text)).strip()).strip().lower()
        out = []
        for token in self.pat.findall(text):
            token = "".join(self.byte_encoder[b] for b in token.encode("utf-8"))
            out.extend(self.encoder[t] for t in self.bpe(token))
        return out

    def tokenize(self, texts, context_length=77):
        sot, eot = self.encoder["<|startoftext|>"], self.encoder["<|endoftext|>"]
        result = torch.zeros(len(texts), context_length, dtype=torch.long)
        for i, t in enumerate(texts):
            tokens = [sot] + self.encode(t) + [eot]
            if len(tokens) > context_length:
                raise RuntimeError(f"Input {t} is too long for context length {context_length}")
            result[i, :len(tokens)] = torch.tensor(tokens)
        return result
