"""Seeded synthetic weights for benchmarks and smoke tests (no network => no pretrained checkpoints).

Every parameter is drawn from its own generator seeded by crc32(name) ^ seed, with the distributions torch's
Conv2d / Linear / GroupNorm constructors use — but never zeroed (the ADM family's zero_module() layers would make
a random-init network output exactly 0, SURVEY.md §0)."""
import math
import zlib

import torch


def randomize_(model, seed=1234, style="torch_default"):
    """in-place, deterministic, construction-order independent re-initialisation of all parameters"""
    sd = model.state_dict()
    model.load_state_dict(_draw({k: tuple(v.shape) for k, v in sd.items()}, seed, style))
    return model


def lpips_state_dict(seed=1234):
    """seeded LPIPS-Alex weights in the lpips package's state-dict layout (asyrp_official_b200.lpips): the backbone
    drawn as above, the lin weights |U(-1/sqrt(C), 1/sqrt(C))| (the trained ones are non-negative)"""
    from .lpips import state_dict_shapes
    sd = _draw(state_dict_shapes(), seed, "torch_default")
    return {k: (v.abs() if k.startswith("lin") else v) for k, v in sd.items()}


def clip_text_state_dict(seed=1234, width=512, layers=12, context=77, vocab=49408, embed_dim=512):
    """seeded CLIP text-tower weights in CLIP's state-dict layout (asyrp_official_b200.clip_text), at the scales of
    CLIP's initialize_parameters: token embedding N(0, .02^2), positional N(0, .01^2), in_proj / text_projection
    std width^-1/2, out_proj / c_proj std width^-1/2 (2 layers)^-1/2, c_fc std (2 width)^-1/2.  No term is zero:
    the biases are N(0, .02^2) and the LayerNorm affines 1 + N(0, .1^2) / N(0, .02^2), so a dropped term shows."""
    from .clip_text import text_key_shapes
    std = {"token_embedding.weight": 0.02, "positional_embedding": 0.01, "text_projection": width ** -0.5}
    return _draw_clip(text_key_shapes(width, layers, context, vocab, embed_dim), "", std, width, layers, seed)


def clip_image_state_dict(seed=1234, width=768, layers=12, patch=16, grid=14, embed_dim=512):
    """seeded CLIP image-tower (VisionTransformer) weights under visual.* in CLIP's state-dict layout
    (asyrp_official_b200.clip_image), at CLIP's init scales: class_embedding, positional_embedding and proj std
    width^-1/2, conv1 torch's Conv2d default U(-b, b), b = (3 patch^2)^-1/2, the blocks as in clip_text_state_dict.
    No term is zero: biases N(0, .02^2), LayerNorm affines 1 + N(0, .1^2) / N(0, .02^2).  Defaults: ViT-B/16."""
    from .clip_image import image_key_shapes
    std = {"class_embedding": width ** -0.5, "positional_embedding": width ** -0.5, "proj": width ** -0.5}
    sd = _draw_clip(image_key_shapes(width, layers, patch, grid, embed_dim), "visual.", std, width, layers, seed)
    sd["visual.conv1.weight"] = (2 * sd["visual.conv1.weight"] - 1) * (3 * patch * patch) ** -0.5
    return sd


def arcface_state_dict(seed=1234):
    """seeded ArcFace Backbone(112, 50, 'ir_se') weights in its state-dict layout (asyrp_official_b200.arcface), every
    term non-degenerate: convs U(-b, b) with b = 1.5 fan_in^-1/2 (at torch's default b = fan_in^-1/2 the BatchNorm
    shifts drown an image in [-1, 1] and unrelated images score ID ~.997; at Kaiming's (6 / fan_in)^1/2 the 24 blocks
    amplify TF32 rounding into a different feature), the linear layer and its bias U(-b, b), b = fan_in^-1/2; BatchNorms
    weight 1 + N(0, .1^2), bias, running_mean N(0, .1^2), running_var exp(N(0, .2^2)) > 0; PReLU slopes
    .25 + N(0, .05^2); num_batches_tracked 0 (ignored by eval-mode BatchNorm)"""
    from .arcface import _bn_prefixes, state_dict_shapes
    sd = {}
    for name, shp in state_dict_shapes().items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        if name == "output_layer.3.bias":
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * (512 * 49) ** -0.5
        elif name == "output_layer.3.weight":
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * shp[1] ** -0.5
        elif len(shp) >= 2:
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * 1.5 * math.prod(shp[1:]) ** -0.5
        elif name.endswith("running_var"):
            sd[name] = torch.exp(0.2 * torch.randn(shp, generator=g))
        elif name.endswith(".weight") and ".res_layer.2." in name or name == "input_layer.2.weight":
            sd[name] = 0.25 + 0.05 * torch.randn(shp, generator=g)
        elif name.endswith(".weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[name] = 0.1 * torch.randn(shp, generator=g)
    for prefix in _bn_prefixes():
        sd[prefix + ".num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return sd


def face_parsing_state_dict(seed=1234, n_classes=19, aux=True):
    """seeded face-parsing BiSeNet(n_classes) weights in its state-dict layout (asyrp_official_b200.face_parsing),
    scaled so that activations stay O(1) through the 18 layers: convs U(-b, b) with b = gain * (3 / fan_in)^1/2, gain
    2^1/2 (He's, for the ReLU) except the blocks' conv2 and the downsample convs (gain 1 / 2^1/2, so that a residual
    sum of two O(1) terms stays O(1)) and the class layer (gain 4, so that class margins are a few units and the labels
    follow the image rather than noise); BatchNorms weight 1 + N(0, .1^2), bias and running_mean N(0, .1^2),
    running_var exp(N(0, .2^2)); num_batches_tracked 0.  aux: include the two auxiliary heads."""
    from .face_parsing import aux_head_shapes, state_dict_shapes
    shapes = {**state_dict_shapes(n_classes), **(aux_head_shapes(n_classes) if aux else {})}
    sd = {}
    for name, shp in shapes.items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        if len(shp) >= 2:
            gain = 2 ** 0.5
            if name.endswith("conv2.weight") and ".layer" in name or ".downsample." in name:
                gain = 2 ** -0.5
            elif name.endswith("conv_out.weight"):
                gain = 4.0
            b = gain * (3.0 / math.prod(shp[1:])) ** 0.5
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * b
        elif name.endswith("running_var"):
            sd[name] = torch.exp(0.2 * torch.randn(shp, generator=g))
        elif name.endswith(".weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[name] = 0.1 * torch.randn(shp, generator=g)
    for name in list(sd):
        if name.endswith("running_var"):
            sd[name[:-len("running_var")] + "num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return sd


def inception_state_dict(seed=1234, fc=True):
    """seeded FID Inception-v3 weights in its state-dict layout (asyrp_official_b200.fid), scaled so that activations
    stay O(1) through the 94 BasicConv2d layers and the features follow the image: convs U(-b, b) with
    b = 2^1/2 (3 / fan_in)^1/2 (He's, for the ReLU); BatchNorms weight 1 + N(0, .1^2), bias and running_mean
    N(0, .1^2), running_var exp(N(0, .2^2)); num_batches_tracked 0.  fc: include the (ignored) fc layer."""
    from .fid import FC, state_dict_shapes
    shapes = {**state_dict_shapes(), **(FC if fc else {})}
    sd = {}
    for name, shp in shapes.items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        if len(shp) >= 2:
            b = (2 ** 0.5) * (3.0 / math.prod(shp[1:])) ** 0.5
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * b
        elif name.endswith("running_var"):
            sd[name] = torch.exp(0.2 * torch.randn(shp, generator=g))
        elif name.endswith(".weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[name] = 0.1 * torch.randn(shp, generator=g)
    for name in list(sd):
        if name.endswith("running_var"):
            sd[name[:-len("running_var")] + "num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return sd


def dino_state_dict(seed=1234, dim=384, depth=12, patch=8, grid=28):
    """seeded DINO VisionTransformer weights in its state-dict layout (asyrp_official_b200.dino; default ViT-S/8 at
    224^2): linear and conv weights U(-b, b) with b = fan_in^-1/2 (torch's default), biases N(0, .02^2), LayerNorm
    weights 1 + N(0, .1^2) and biases N(0, .1^2), cls_token and pos_embed N(0, .02^2) (DINO's trunc_normal_ std)"""
    from .dino import key_shapes
    sd = {}
    for name, shp in key_shapes(dim, depth, patch, grid).items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        if name in ("cls_token", "pos_embed"):
            sd[name] = 0.02 * torch.randn(shp, generator=g)
        elif len(shp) >= 2:
            sd[name] = (torch.rand(shp, generator=g) * 2 - 1) * math.prod(shp[1:]) ** -0.5
        elif "norm" in name and name.endswith(".weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif "norm" in name:
            sd[name] = 0.1 * torch.randn(shp, generator=g)
        else:
            sd[name] = 0.02 * torch.randn(shp, generator=g)
    return sd


def _draw_clip(shapes, prefix, std, width, layers, seed):
    """CLIP weights of `shapes` (names without `prefix`), each from its own generator seeded by crc32(prefix + name)"""
    std = {**std, "attn.in_proj_weight": width ** -0.5, "attn.out_proj.weight": width ** -0.5 * (2 * layers) ** -0.5,
           "mlp.c_fc.weight": (2 * width) ** -0.5, "mlp.c_proj.weight": width ** -0.5 * (2 * layers) ** -0.5}
    sd = {}
    for name, shp in shapes.items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32((prefix + name).encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        key = name.split(".", 3)[-1] if name.startswith("transformer.") else name
        if key == "conv1.weight":  # U(0, 1), scaled by the caller
            sd[prefix + name] = torch.rand(shp, generator=g)
            continue
        z = torch.randn(shp, generator=g)
        if key in std:
            sd[prefix + name] = z * std[key]
        elif key.startswith("ln") and key.endswith(".weight"):
            sd[prefix + name] = 1.0 + 0.1 * z
        else:  # biases
            sd[prefix + name] = 0.02 * z
    return sd


def clip_bpe_merges(texts):
    """BPE merges that build every word of texts (after CLIP's cleaning and pre-tokenisation) left to right from its
    byte symbols: a small vocabulary for tests and smoke runs in place of bpe_simple_vocab_16e6.txt.gz"""
    import regex

    from .clip_text import _PAT, byte_symbols, clean_text
    enc, merges, seen = byte_symbols(), [], set()
    for text in texts:
        for token in regex.findall(_PAT, clean_text(text), regex.IGNORECASE):
            sym = [enc[b] for b in token.encode("utf-8")]
            sym[-1] += "</w>"
            cur = sym[0]
            for s in sym[1:]:
                if (cur, s) not in seen:
                    seen.add((cur, s))
                    merges.append((cur, s))
                cur += s
    return merges


def write_clip_vocab(path, merges):
    """write merges as a bpe_simple_vocab_16e6.txt.gz-style file (a header line, then one 'a b' merge per line);
    returns the vocabulary size: 512 byte symbols + the merges + 2"""
    import gzip
    with gzip.open(path, "wt", encoding="utf-8") as f:
        f.write("\n".join(["#version: 0.2"] + [f"{a} {b}" for a, b in merges]))
    return 512 + len(merges) + 2


def _draw(shapes, seed, style):
    fan = {k[:-7]: math.prod(v[1:]) for k, v in shapes.items() if k.endswith(".weight") and len(v) >= 2}
    new = {}
    for name, shp in shapes.items():
        g = torch.Generator()
        g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        base = name.rsplit(".", 1)[0]
        if len(shp) >= 2:
            if style == "torch_default":
                t = (torch.rand(shp, generator=g) * 2 - 1) * (1.0 / math.sqrt(fan[base]))
            else:
                t = torch.randn(shp, generator=g) / math.sqrt(fan[base])
        elif base in fan:
            t = (torch.rand(shp, generator=g) * 2 - 1) * (1.0 / math.sqrt(fan[base]))
        elif name.endswith(".weight"):
            t = torch.ones(shp) if style == "torch_default" else 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            t = torch.zeros(shp) if style == "torch_default" else 0.1 * torch.randn(shp, generator=g)
        new[name] = t.float()
    return new
