"""CLIP's text tower on the engine's kernels: the tokenizer, the weight loader and `CLIPText`, which gives the
text-direction cosine Asyrp.set_t_edit_t_addnoise chooses t_edit from (diffusion_latent.py:1319-1329).

    tokenize       OpenAI CLIP's SimpleTokenizer + clip.tokenize(truncate=False): html.unescape twice, whitespace
                   collapsed, lower-cased, CLIP's pre-tokenisation regex, byte-level BPE over the merges of
                   bpe_simple_vocab_16e6.txt.gz; [SOT] + tokens + [EOT], zero-padded to the context length.  ftfy's
                   mojibake repair (the first step of CLIP's basic_clean) is skipped: ftfy is not a dependency, and it
                   changes nothing on ASCII prompts.
    encode_text    x = token_embedding[ids] + positional_embedding; per residual block
                   x += out_proj(causal_mha(ln_1(x))), x += c_proj(quick_gelu(c_fc(ln_2(x)))); the feature is
                   ln_final(x[eot]) @ text_projection, eot = the first argmax of the ids (the end-of-text token).
    text_cosine    torch.nn.CosineSimilarity(dim=1, eps=1e-6) of the source and target features.

Weights: CLIP's downloaded TorchScript archive (e.g. ~/.cache/clip/ViT-B-16.pt) or a torch.save of its state dict;
only the text-tower keys are used (INTEGRATION.md lists them).  Every arithmetic operation is a kernel of
libasyrp_b200.so (csrc/clip_text.cu): fp32 activations, the linear layers on the TF32 tensor cores.
"""
import functools
import gzip
import html
import re

import torch

from . import _lib, ops

CONTEXT_LENGTH = 77
HEAD_DIM = 64
SOT, EOT = "<|startoftext|>", "<|endoftext|>"
# not part of the text tower: skipped by the loader
IGNORED_KEYS = ("logit_scale", "input_resolution", "context_length", "vocab_size")
IGNORED_PREFIXES = ("visual.",)
BLOCK_KEYS = ("ln_1.weight", "ln_1.bias", "attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight",
              "attn.out_proj.bias", "ln_2.weight", "ln_2.bias", "mlp.c_fc.weight", "mlp.c_fc.bias",
              "mlp.c_proj.weight", "mlp.c_proj.bias")
_PAT = r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+"""


# ---------------------------------------------------------------------------------------------------------------------
# tokenizer
def byte_symbols():
    """byte -> printable unicode symbol of byte-level BPE: the 188 printable Latin-1 bytes map to themselves, the
    other 68 to chr(256), chr(257), ... in byte order.  The dict's order (printable bytes first, then the others) is
    the order of the first 256 vocabulary entries."""
    keep = [*range(ord("!"), ord("~") + 1), *range(ord("¡"), ord("¬") + 1), *range(ord("®"), ord("ÿ") + 1)]
    rest = [b for b in range(256) if b not in keep]
    return {**{b: chr(b) for b in keep}, **{b: chr(256 + i) for i, b in enumerate(rest)}}


def read_merges(path):
    """the BPE merges of a bpe_simple_vocab_16e6.txt.gz-style file: lines 1 .. 49152-256-2 (line 0 is a header)"""
    with gzip.open(path, "rt", encoding="utf-8") as f:
        lines = f.read().split("\n")
    return [tuple(line.split()) for line in lines[1:49152 - 256 - 2 + 1]]


def clean_text(text):
    """CLIP's basic_clean without ftfy, whitespace_clean, lower-casing"""
    text = html.unescape(html.unescape(text)).strip()
    return re.sub(r"\s+", " ", text).strip().lower()


class Tokenizer:
    """CLIP's SimpleTokenizer over a merges file"""

    def __init__(self, vocab_path):
        import regex
        self.byte_encoder = byte_symbols()
        merges = read_merges(vocab_path)
        symbols = list(self.byte_encoder.values())
        vocab = symbols + [s + "</w>" for s in symbols] + ["".join(m) for m in merges] + [SOT, EOT]
        self.encoder = {tok: i for i, tok in enumerate(vocab)}
        self.ranks = {m: i for i, m in enumerate(merges)}
        self.sot, self.eot = self.encoder[SOT], self.encoder[EOT]
        self.pattern = regex.compile(_PAT, regex.IGNORECASE)
        self._bpe = functools.lru_cache(maxsize=None)(self._bpe_uncached)

    def __len__(self):
        return len(self.encoder)

    def _bpe_uncached(self, token):
        if token in (SOT, EOT):
            return (token,)
        word = list(token[:-1]) + [token[-1] + "</w>"]
        while len(word) > 1:
            pairs = {(a, b) for a, b in zip(word, word[1:])}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            merged, i = [], 0
            while i < len(word):  # merge every non-overlapping occurrence, left to right
                if i + 1 < len(word) and (word[i], word[i + 1]) == best:
                    merged.append(word[i] + word[i + 1])
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        return tuple(word)

    def encode(self, text):
        ids = []
        for token in self.pattern.findall(clean_text(text)):
            sym = "".join(self.byte_encoder[b] for b in token.encode("utf-8"))
            ids.extend(self.encoder[piece] for piece in self._bpe(sym))
        return ids

    def tokenize(self, texts, context_length=CONTEXT_LENGTH):
        """clip.tokenize(texts, context_length, truncate=False): int64 [len(texts)][context_length]"""
        if isinstance(texts, str):
            texts = [texts]
        out = torch.zeros(len(texts), context_length, dtype=torch.long)
        for i, text in enumerate(texts):
            ids = [self.sot] + self.encode(text) + [self.eot]
            if len(ids) > context_length:
                raise RuntimeError(f"Input {text} is too long for context length {context_length}")
            out[i, :len(ids)] = torch.tensor(ids)
        return out


# ---------------------------------------------------------------------------------------------------------------------
# weights
def block_key_shapes(width, layers):
    """name -> shape of every tensor of CLIP's Transformer (transformer.resblocks.*), the same in both towers"""
    per = {"ln_1.weight": (width,), "ln_1.bias": (width,), "attn.in_proj_weight": (3 * width, width),
           "attn.in_proj_bias": (3 * width,), "attn.out_proj.weight": (width, width), "attn.out_proj.bias": (width,),
           "ln_2.weight": (width,), "ln_2.bias": (width,), "mlp.c_fc.weight": (4 * width, width),
           "mlp.c_fc.bias": (4 * width,), "mlp.c_proj.weight": (width, 4 * width), "mlp.c_proj.bias": (width,)}
    return {f"transformer.resblocks.{i}.{k}": s for i in range(layers) for k, s in per.items()}


def text_key_shapes(width, layers, context, vocab, embed_dim):
    """name -> shape of every text-tower tensor of a CLIP state dict"""
    shapes = {"token_embedding.weight": (vocab, width), "positional_embedding": (context, width),
              "ln_final.weight": (width,), "ln_final.bias": (width,), "text_projection": (width, embed_dim)}
    shapes.update(block_key_shapes(width, layers))
    return shapes


def _read(path):
    """CLIP's TorchScript archive (torch.jit.load) or a plain torch.save state dict, as clip.load tries them"""
    try:
        return torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return torch.load(path, map_location="cpu", weights_only=True)


def load_state_dict(sd_or_path, vocab_size=None):
    """Validate the text tower of a CLIP state dict (or of the archive / torch.save at a path) and return
    (dims, tensors): dims = {width, heads, layers, context, vocab, embed_dim} derived as CLIP's build_model does,
    tensors = the text-tower keys cast to fp32 on the host.

    visual.*, logit_scale, input_resolution, context_length and vocab_size are ignored.  Raises ValueError on a
    missing, mis-shaped or unknown text key, on a width that is not a multiple of 64 (the heads are width/64), and
    when vocab_size (the tokenizer's) differs from the token_embedding rows."""
    sd = sd_or_path if isinstance(sd_or_path, dict) else _read(sd_or_path)
    sd = {k: torch.as_tensor(v) for k, v in sd.items()
          if k not in IGNORED_KEYS and not k.startswith(IGNORED_PREFIXES)}
    for k in ("token_embedding.weight", "positional_embedding", "ln_final.weight", "text_projection"):
        if k not in sd:
            raise ValueError(f"CLIP state dict: missing key {k!r}")
    width = sd["ln_final.weight"].shape[0]
    blocks = {k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")}
    if not all(b.isdigit() for b in blocks):
        raise ValueError(f"CLIP state dict: unexpected residual-block names {sorted(blocks)}")
    dims = dict(width=width, heads=width // HEAD_DIM, layers=len(blocks), context=sd["positional_embedding"].shape[0],
                vocab=sd["token_embedding.weight"].shape[0], embed_dim=sd["text_projection"].shape[-1])
    if width % HEAD_DIM or dims["embed_dim"] % 64 or dims["layers"] == 0:
        raise ValueError(f"CLIP state dict: width {width} and embed_dim {dims['embed_dim']} must be multiples of 64, "
                         f"with at least one residual block")
    if dims["context"] > 128:
        raise ValueError(f"CLIP state dict: context length {dims['context']} > 128 is not supported")
    if vocab_size is not None and vocab_size != dims["vocab"]:
        raise ValueError(f"CLIP vocabulary has {vocab_size} tokens but token_embedding has {dims['vocab']} rows")
    expected = text_key_shapes(width, dims["layers"], dims["context"], dims["vocab"], dims["embed_dim"])
    out = {}
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f"CLIP state dict: missing key {k!r}")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"CLIP state dict: {k!r} has shape {tuple(sd[k].shape)}, expected {shape}")
        out[k] = sd[k].detach().float().cpu().contiguous()
    unknown = sorted(set(sd) - set(expected))
    if unknown:
        raise ValueError(f"CLIP state dict: unexpected keys {unknown} (expected CLIP's text-tower layout)")
    return dims, out


# ---------------------------------------------------------------------------------------------------------------------
def residual_blocks(sd, layers, heads, x, causal):
    """CLIP's Transformer on x [P][T][w] (device, fp32), in place: per block x += out_proj(mha(ln_1(x))),
    x += c_proj(quick_gelu(c_fc(ln_2(x)))), with the weights sd[f"transformer.resblocks.{i}.{key}"].  The attention is
    causal in the text tower and full in the image tower."""
    P, T, w = x.shape
    h = torch.empty_like(x)
    qkv = x.new_empty(P, T, 3 * w)
    mlp = x.new_empty(P, T, 4 * w)
    for i in range(layers):
        b = {k: sd[f"transformer.resblocks.{i}.{k}"] for k in BLOCK_KEYS}
        ops.clip_layernorm(x, b["ln_1.weight"], b["ln_1.bias"], h)
        ops.clip_linear(h, b["attn.in_proj_weight"], b["attn.in_proj_bias"], qkv)
        ops.clip_attention(qkv, h, heads, causal=causal)
        ops.clip_linear(h, b["attn.out_proj.weight"], b["attn.out_proj.bias"], x, ops.CLIP_EPI_RESIDUAL, residual=x)
        ops.clip_layernorm(x, b["ln_2.weight"], b["ln_2.bias"], h)
        ops.clip_linear(h, b["mlp.c_fc.weight"], b["mlp.c_fc.bias"], mlp, ops.CLIP_EPI_QUICK_GELU)
        ops.clip_linear(mlp, b["mlp.c_proj.weight"], b["mlp.c_proj.bias"], x, ops.CLIP_EPI_RESIDUAL, residual=x)


class CLIPText:
    """CLIPText(weights, vocab_path).text_cosine(src_txts, trg_txts) -> fp32 [n] on the host, the cosine of each
    source / target pair's encode_text features.  Every operation is a kernel of libasyrp_b200.so; a prompt's
    features are bit-identical whatever batch it is encoded in."""

    def __init__(self, state_dict_or_path, vocab_path, device=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("CLIPText needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        self.tokenizer = Tokenizer(vocab_path)
        self.dims, sd = load_state_dict(state_dict_or_path, vocab_size=len(self.tokenizer))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.sd = {k: v.to(self.device) for k, v in sd.items()}
        # x @ text_projection is a linear layer with weight text_projection^T
        self.proj = sd["text_projection"].t().contiguous().to(self.device)

    def tokenize(self, texts):
        return self.tokenizer.tokenize(texts, self.dims["context"])

    @torch.no_grad()
    def encode_text(self, token_ids):
        """token_ids [P][context] (clip.tokenize's layout) -> fp32 [P][embed_dim] on the device"""
        d, sd = self.dims, self.sd
        ids = torch.as_tensor(token_ids)
        if ids.dim() != 2 or ids.shape[1] != d["context"]:
            raise ValueError(f"token ids must be [P][{d['context']}], got {tuple(ids.shape)}")
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= d["vocab"]):
            raise ValueError(f"token ids must lie in [0, {d['vocab']})")
        P, T, w = ids.shape[0], d["context"], d["width"]
        f32 = dict(dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ids = ids.to(torch.int32).contiguous().to(self.device)
            x = torch.empty(P, T, w, **f32)
            ops.clip_embed(ids, sd["token_embedding.weight"], sd["positional_embedding"], x)
            residual_blocks(sd, d["layers"], d["heads"], x, causal=True)
            pooled = torch.empty(P, w, **f32)
            ops.clip_pool(x, ids, sd["ln_final.weight"], sd["ln_final.bias"], pooled)
            feats = torch.empty(P, d["embed_dim"], **f32)
            ops.clip_linear(pooled, self.proj, None, feats)
        return feats

    @torch.no_grad()
    def text_cosine(self, src_txts, trg_txts):
        """CosineSimilarity(dim=1, eps=1e-6)(encode_text(tokenize(src)), encode_text(tokenize(trg))): fp32 [n] on the
        host, one entry per pair; both sides run as one batch"""
        src = [src_txts] if isinstance(src_txts, str) else list(src_txts)
        trg = [trg_txts] if isinstance(trg_txts, str) else list(trg_txts)
        if len(src) != len(trg) or not src:
            raise ValueError(f"need as many source as target texts, got {len(src)} and {len(trg)}")
        n = len(src)
        feats = self.encode_text(self.tokenize(src + trg))
        cos = torch.empty(n, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ops.clip_cosine(feats[:n], feats[n:], cos)
        return cos.cpu()
