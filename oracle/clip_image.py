"""CPU oracle of CLIP's image tower and of the directional similarity of the reference's CLIPLoss: a plain restatement
of CLIPLoss.preprocess (losses/clip_loss.py:39-41, with torchvision 0.10's tensor Resize: bicubic, A = -0.75,
align_corners=False, no antialiasing, taps clamped at the edges), OpenAI CLIP's VisionTransformer.forward,
get_image_features, compute_text_direction and clip_directional_loss (:102-117,170-180).  Test infrastructure only;
evaluated in fp32 or fp64 (the `dtype` argument)."""
import math

import torch

from oracle import clip_text as oct

MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


def _cubic_weights(t):
    """PyTorch's cubic convolution coefficients (A = -0.75) of the four taps floor-1 .. floor+2 at fraction t"""
    A = -0.75

    def c1(x):
        return ((A + 2) * x - (A + 3)) * x * x + 1

    def c2(x):
        return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A
    return torch.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], dim=-1)


def resize_bicubic(x, R):
    """F.interpolate(x, (R, R), mode="bicubic", align_corners=False, antialias=False) of x [B][C][S][S], written out"""
    S = x.shape[-1]
    o = torch.arange(R, dtype=x.dtype)
    real = (o + 0.5) * (S / R) - 0.5
    f = torch.floor(real)
    w = _cubic_weights(real - f)                                     # [R][4]
    idx = (f.long()[:, None] + torch.arange(-1, 3)[None]).clamp(0, S - 1)  # [R][4]
    rows = x[..., idx, :]                                            # [B][C][R][4][S]
    rows = (rows * w[:, :, None]).sum(-2)                            # [B][C][R][S]
    cols = rows[..., idx]                                            # [B][C][R][R][4]
    return (cols * w).sum(-1)


def preprocess(x, R):
    """CLIPLoss.preprocess of images x [B][3][S][S] in [-1, 1]: (x+1)/2, bicubic resize to R, CenterCrop (identity),
    CLIP's Normalize"""
    y = resize_bicubic((x + 1) / 2, R)
    mean = torch.tensor(MEAN, dtype=x.dtype)[:, None, None]
    std = torch.tensor(STD, dtype=x.dtype)[:, None, None]
    return (y - mean) / std


def full_attention(x, in_w, in_b, out_w, out_b, heads):
    """nn.MultiheadAttention(width, heads)(x, x, x) on x [B][T][w]"""
    B, T, w = x.shape
    dh = w // heads
    q, k, v = (x @ in_w.t() + in_b).split(w, dim=-1)
    q, k, v = (t.reshape(B, T, heads, dh).transpose(1, 2) for t in (q, k, v))
    a = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(dh), dim=-1) @ v
    return a.transpose(1, 2).reshape(B, T, w) @ out_w.t() + out_b


def dims_of(sd):
    g = {k[7:]: v for k, v in sd.items() if k.startswith("visual.")}
    width, patch = g["conv1.weight"].shape[0], g["conv1.weight"].shape[-1]
    grid = round((g["positional_embedding"].shape[0] - 1) ** 0.5)
    layers = len({k.split(".")[2] for k in g if k.startswith("transformer.resblocks.")})
    return dict(width=width, patch=patch, grid=grid, layers=layers, heads=width // 64)


def encode_image(sd, images, dtype=torch.float64):
    """CLIPLoss.encode_images: preprocess, then VisionTransformer.forward with the visual.* keys of a CLIP state dict:
    [B][embed_dim]"""
    d = dims_of(sd)
    g = {k[7:]: v.to(dtype) for k, v in sd.items() if k.startswith("visual.")}
    x = preprocess(images.to(dtype), d["grid"] * d["patch"])
    x = torch.nn.functional.conv2d(x, g["conv1.weight"], stride=d["patch"])  # [B][w][G][G]
    x = x.flatten(2).transpose(1, 2)                                        # [B][G*G][w]
    cls = g["class_embedding"].expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], dim=1) + g["positional_embedding"]
    x = oct.layer_norm(x, g["ln_pre.weight"], g["ln_pre.bias"])
    for i in range(d["layers"]):
        p = f"transformer.resblocks.{i}."
        x = x + full_attention(oct.layer_norm(x, g[p + "ln_1.weight"], g[p + "ln_1.bias"]), g[p + "attn.in_proj_weight"],
                               g[p + "attn.in_proj_bias"], g[p + "attn.out_proj.weight"], g[p + "attn.out_proj.bias"],
                               d["heads"])
        h = oct.layer_norm(x, g[p + "ln_2.weight"], g[p + "ln_2.bias"])
        h = oct.quick_gelu(h @ g[p + "mlp.c_fc.weight"].t() + g[p + "mlp.c_fc.bias"])
        x = x + h @ g[p + "mlp.c_proj.weight"].t() + g[p + "mlp.c_proj.bias"]
    return oct.layer_norm(x[:, 0], g["ln_post.weight"], g["ln_post.bias"]) @ g["proj"]


def get_image_features(sd, images, dtype=torch.float64):
    f = encode_image(sd, images, dtype)
    return f / f.norm(dim=-1, keepdim=True)


def compute_text_direction(sd, tokenizer, templates, source_class, target_class, dtype=torch.float64):
    """normalize(mean over templates of trg / |trg| - src / |src|) of the text features: [1][embed_dim]"""
    def feats(cls):
        f = oct.encode_text(sd, tokenizer.tokenize([t.format(cls) for t in templates]), dtype)
        return f / f.norm(dim=-1, keepdim=True)
    d = (feats(target_class) - feats(source_class)).mean(dim=0, keepdim=True)
    return d / d.norm(dim=-1, keepdim=True)


def edit_direction(src_feats, trg_feats):
    """clip_directional_loss's edit direction from normalised image features"""
    e = trg_feats - src_feats
    return e / (e.norm(dim=-1, keepdim=True) + 1e-7)


def directional_similarity(sd, tokenizer, templates, src_img, source_class, target_img, target_class,
                           dtype=torch.float64):
    """1 - DirectionLoss('cosine') per row, i.e. CosineSimilarity()(edit direction, text direction): [B]"""
    text = compute_text_direction(sd, tokenizer, templates, source_class, target_class, dtype)
    e = edit_direction(get_image_features(sd, src_img, dtype), get_image_features(sd, target_img, dtype))
    return torch.nn.CosineSimilarity()(e, text)


def clip_directional_loss(sd, tokenizer, templates, src_img, source_class, target_img, target_class,
                          dtype=torch.float64):
    return (1 - directional_similarity(sd, tokenizer, templates, src_img, source_class, target_img, target_class,
                                       dtype)).mean()
