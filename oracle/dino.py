"""fp64 numpy restatement of asyrp_official_b200.dino: DINO's input transform and patch matrix, the VisionTransformer
backbone, the last block's keys, the self-similarity structure distance and the CLS cosine.  Weights are the DINO
state dict as numpy arrays (any float dtype); every computation is in fp64."""
import math

import numpy as np

MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])


def aa_weights(n_in, n_out):
    """[n_out][n_in] matrix of PyTorch's antialiased bilinear resize along one axis (align_corners=False): output i
    takes the triangle weights around centre scale (i + 0.5), support max(1, scale), normalised by their sum"""
    scale = n_in / n_out
    support = max(scale, 1.0)
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    W = np.zeros((n_out, n_in))
    for i in range(n_out):
        c = scale * (i + 0.5)
        lo = max(int(c - support + 0.5), 0)
        hi = min(int(c + support + 0.5), n_in)
        w = np.array([max(0.0, 1.0 - abs((j - c + 0.5) * inv)) for j in range(lo, hi)])
        if w.sum() != 0:
            W[i, lo:hi] = w / w.sum()
    return W


def preprocess(x, resolution):
    """x [B][3][S][S] in [-1, 1] -> (x + 1) / 2, antialiased bilinear resize to resolution, ImageNet Normalize"""
    x = (np.asarray(x, dtype=np.float64) + 1.0) / 2.0
    W = aa_weights(x.shape[-1], resolution)
    y = np.einsum("ij,bcjk,lk->bcil", W, x, W)
    return (y - MEAN[None, :, None, None]) / STD[None, :, None, None]


def pack(x, grid, patch):
    """the patch matrix [B*grid^2][3*patch^2] (c, ky, kx) columns, without the GEMM's zero padding"""
    y = preprocess(x, grid * patch)
    B = y.shape[0]
    y = y.reshape(B, 3, grid, patch, grid, patch).transpose(0, 2, 4, 1, 3, 5)
    return y.reshape(B * grid * grid, 3 * patch * patch)


def layernorm(x, g, b, eps=1e-6):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * g + b


def gelu(x):
    erf = np.vectorize(math.erf)
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def attention(qkv, heads):
    """non-causal softmax attention, head size 64, scale 1/8: qkv [B][T][3D] -> [B][T][D]"""
    B, T, D3 = qkv.shape
    D = D3 // 3
    q, k, v = (qkv[..., i * D:(i + 1) * D].reshape(B, T, heads, D // heads).transpose(0, 2, 1, 3) for i in range(3))
    s = q @ k.transpose(0, 1, 3, 2) * (D // heads) ** -0.5
    s = np.exp(s - s.max(-1, keepdims=True))
    p = s / s.sum(-1, keepdims=True)
    return (p @ v).transpose(0, 2, 1, 3).reshape(B, T, D)


def forward(sd, x):
    """(keys [B][T][D] of the last block, final-norm tokens [B][T][D]) of images x [B][3][S][S] in [-1, 1]"""
    sd = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    conv = sd["patch_embed.proj.weight"]
    D, P = conv.shape[0], conv.shape[-1]
    T = sd["pos_embed"].shape[1]
    G = round(math.sqrt(T - 1))
    B = x.shape[0]
    emb = pack(x, G, P) @ conv.reshape(D, -1).T + sd["patch_embed.proj.bias"]
    h = np.concatenate([np.broadcast_to(sd["cls_token"].reshape(1, 1, D), (B, 1, D)), emb.reshape(B, G * G, D)], 1)
    h = h + sd["pos_embed"]
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    keys = None
    for i in range(depth):
        p = f"blocks.{i}."
        qkv = layernorm(h, sd[p + "norm1.weight"], sd[p + "norm1.bias"]) @ sd[p + "attn.qkv.weight"].T + \
            sd[p + "attn.qkv.bias"]
        keys = qkv[..., D:2 * D]
        h = h + attention(qkv, D // 64) @ sd[p + "attn.proj.weight"].T + sd[p + "attn.proj.bias"]
        t = layernorm(h, sd[p + "norm2.weight"], sd[p + "norm2.bias"])
        h = h + gelu(t @ sd[p + "mlp.fc1.weight"].T + sd[p + "mlp.fc1.bias"]) @ sd[p + "mlp.fc2.weight"].T + \
            sd[p + "mlp.fc2.bias"]
    return keys, layernorm(h, sd["norm.weight"], sd["norm.bias"])


def selfsim(k, eps=1e-8):
    """S = k^ k^T, k^ = k / max(|k|, eps), for keys [T][D]"""
    k = np.asarray(k, dtype=np.float64)
    kh = k / np.maximum(np.linalg.norm(k, axis=-1, keepdims=True), eps)
    return kh @ kh.T


def structure_distance(ka, kb, eps=1e-8):
    """(1/T^2) sum_ij (S(a)_ij - S(b)_ij)^2"""
    return float(np.mean((selfsim(ka, eps) - selfsim(kb, eps)) ** 2))


def cls_cos(a, b, eps=1e-8):
    """CosineSimilarity(eps) of two CLS embeddings [D]: sum a/max(|a|, eps) * b/max(|b|, eps)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float((a / max(np.linalg.norm(a), eps)) @ (b / max(np.linalg.norm(b), eps)))
