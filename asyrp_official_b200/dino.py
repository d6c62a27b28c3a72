"""A DINO ViT on the engine's kernels and the two scores `--dino_structure` reports for an edit (or a DiffStyle result)
against its source image: the structure distance of Splice (Tumanyan et al. 2022) and Plug-and-Play (Tumanyan et al.
2023), and the cosine of DINO's CLS embeddings for appearance.

    input       x in [-1, 1] -> (x + 1) / 2 -> torchvision Resize(R) on a float tensor, i.e.
                F.interpolate(mode="bilinear", align_corners=False, antialias=True), R = G * P -> ImageNet Normalize
    network     facebookresearch/dino's VisionTransformer, backbone only, eval mode: a P x P stride-P conv with bias as
                one linear layer over the patch matrix; x = [cls_token ; patches] + pos_embed; per block
                x += proj(attn(norm1(x))), x += fc2(GELU(fc1(norm2(x)))) (LayerNorm eps 1e-6, exact erf GELU, qkv with
                bias, scale 64^-0.5); a final norm
    structure   k = the keys of the last block (the key third of its qkv, heads concatenated, CLS included) [T][D];
                k^ = k / max(|k|, 1e-8), S(x) = k^ k^T, D(a, b) = (1/T^2) sum_ij (S(a)_ij - S(b)_ij)^2 (Splice's
                mse_loss of the two self-similarity matrices); D(a, a) = 0 exactly
    appearance  cls_cos(a, b) = CosineSimilarity(eps 1e-8) of the final-norm CLS tokens (DINO's forward output)

Weights: a plain torch.save of the VisionTransformer state dict (--dino_weights, e.g. dino_vitbase8_pretrain.pth);
D, the depth and P are read from the shapes and heads = D / 64.  ViT-S/8, S/16, B/8 and B/16 load; no real checkpoint
has been loaded in this build's tests, which use random weights of the same layout.  Every arithmetic operation is a
kernel of libasyrp_b200.so (csrc/dino.cu, and the CLIP towers' linear layers and token kernels): fp32 activations,
the linear layers and the attention on the TF32 tensor cores.
"""
import torch

from . import _lib, ops

HEAD_DIM = 64
MAX_TOKENS = 1025  # asyrp_dino_attention, asyrp_dino_selfsim_distance
LN_EPS = 1e-6
NORM_EPS = 1e-8  # k / max(|k|, eps), and CosineSimilarity's eps
# device memory of the scored rows: rows are scored in chunks of ACTIVATION_BUDGET // row_bytes(dims) images
ACTIVATION_BUDGET = 1 << 30
BLOCK_KEYS = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
              "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias")


def key_shapes(dim, depth, patch, grid):
    """name -> shape of every tensor of a DINO VisionTransformer state dict (mlp_ratio 4)"""
    shapes = {"cls_token": (1, 1, dim), "pos_embed": (1, grid * grid + 1, dim),
              "patch_embed.proj.weight": (dim, 3, patch, patch), "patch_embed.proj.bias": (dim,),
              "norm.weight": (dim,), "norm.bias": (dim,)}
    per = {"norm1.weight": (dim,), "norm1.bias": (dim,), "attn.qkv.weight": (3 * dim, dim),
           "attn.qkv.bias": (3 * dim,), "attn.proj.weight": (dim, dim), "attn.proj.bias": (dim,),
           "norm2.weight": (dim,), "norm2.bias": (dim,), "mlp.fc1.weight": (4 * dim, dim),
           "mlp.fc1.bias": (4 * dim,), "mlp.fc2.weight": (dim, 4 * dim), "mlp.fc2.bias": (dim,)}
    shapes.update({f"blocks.{i}.{k}": s for i in range(depth) for k, s in per.items()})
    return shapes


def load_state_dict(sd_or_path):
    """Validate a DINO VisionTransformer state dict (or the torch.save at a path) and return (dims, tensors): dims =
    {dim, heads, depth, patch, grid, tokens, resolution}, tensors fp32 on the host.  Raises ValueError naming the key
    on a missing, mis-shaped or unknown key, a `module.` / `backbone.` prefix (a DDP or training-wrapper checkpoint),
    a width that is not a multiple of 64, and more than 1025 tokens."""
    sd = sd_or_path
    if not isinstance(sd, dict):
        try:
            sd = torch.load(sd_or_path, map_location="cpu", weights_only=True)
        except Exception as e:  # a file torch.load cannot read
            raise ValueError(f"DINO state dict: cannot read {sd_or_path!r}: {e}") from None
        if not isinstance(sd, dict):
            raise ValueError(f"DINO state dict: {sd_or_path!r} holds a {type(sd).__name__}, not a state dict")
    for k in sd:
        if not isinstance(k, str):
            raise ValueError(f"DINO state dict: key {k!r} is not a name")
        if k.startswith(("module.", "backbone.")):
            raise ValueError(f"DINO state dict: key {k!r} has a {k.split('.')[0]}. prefix; save the backbone's own "
                             "state dict (strip the prefix)")
    for k in ("patch_embed.proj.weight", "pos_embed"):
        if k not in sd:
            raise ValueError(f"DINO state dict: missing key {k!r}")
    conv, pos = torch.as_tensor(sd["patch_embed.proj.weight"]), torch.as_tensor(sd["pos_embed"])
    if conv.dim() != 4 or conv.shape[1] != 3 or conv.shape[2] != conv.shape[3] or conv.shape[2] == 0:
        raise ValueError(f"DINO state dict: 'patch_embed.proj.weight' has shape {tuple(conv.shape)}, expected "
                         "[D][3][P][P]")
    dim, patch = conv.shape[0], conv.shape[2]
    if dim == 0 or dim % HEAD_DIM:
        raise ValueError(f"DINO state dict: 'patch_embed.proj.weight' gives D = {dim}, which must be a positive "
                         f"multiple of {HEAD_DIM} (heads = D / {HEAD_DIM})")
    if pos.dim() != 3 or pos.shape[0] != 1 or pos.shape[2] != dim:
        raise ValueError(f"DINO state dict: 'pos_embed' has shape {tuple(pos.shape)}, expected [1][T][{dim}]")
    T = pos.shape[1]
    grid = round(max(T - 1, 0) ** 0.5)
    if T < 2 or grid * grid + 1 != T:
        raise ValueError(f"DINO state dict: 'pos_embed' has {T} tokens; expected 1 + G^2")
    if T > MAX_TOKENS:
        raise ValueError(f"DINO state dict: 'pos_embed' has {T} tokens, above {MAX_TOKENS} (1 + 32^2)")
    blocks = set()
    for k in sd:
        if k.startswith("blocks."):
            b = k.split(".")[1]
            if not b.isdigit():
                raise ValueError(f"DINO state dict: unexpected key {k!r}")
            blocks.add(int(b))
    depth = max(blocks) + 1 if blocks else 0
    if depth == 0:
        raise ValueError("DINO state dict: missing key 'blocks.0.attn.qkv.weight' (no transformer block)")
    expected = key_shapes(dim, depth, patch, grid)
    out = {}
    for k, shape in expected.items():
        if k not in sd:
            raise ValueError(f"DINO state dict: missing key {k!r}")
        v = torch.as_tensor(sd[k])
        if tuple(v.shape) != shape:
            raise ValueError(f"DINO state dict: {k!r} has shape {tuple(v.shape)}, expected {shape}")
        out[k] = v.detach().float().cpu().contiguous()
    unknown = sorted(set(sd) - set(expected))
    if unknown:
        raise ValueError(f"DINO state dict: unexpected key {unknown[0]!r} (expected DINO's VisionTransformer layout; "
                         "a head or a projector is not part of the backbone)")
    dims = dict(dim=dim, heads=dim // HEAD_DIM, depth=depth, patch=patch, grid=grid, tokens=T,
                resolution=grid * patch)
    return dims, out


def row_bytes(dims):
    """device bytes of one image's activations in DINO.features: the patch matrix, the patch embeddings, the residual
    stream, the normalised / attention rows, qkv and the MLP hidden rows"""
    g2, T, D = dims["grid"] ** 2, dims["tokens"], dims["dim"]
    return 4 * (g2 * (ops.clip_image_kpad(dims["patch"]) + D) + T * D * (1 + 1 + 3 + 4))


class DINO:
    """DINO(weights).features(x) -> (keys, cls) for images x [B][3][S][S] in [-1, 1]; scores(origin, edited) -> fp64
    [n][B][2] (structure distance, CLS cosine).  Every operation is a kernel of libasyrp_b200.so; an image's features
    are the same bits whatever batch or chunk it is in.  max_rows: images per features call in scores (default
    ACTIVATION_BUDGET // row_bytes)."""

    def __init__(self, state_dict_or_path, device=None, max_rows=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("DINO needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        self.dims, sd = load_state_dict(state_dict_or_path)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        d = self.dims
        # the patch conv over non-overlapping patches is a linear layer over the patch matrix, K zero-padded
        w = torch.zeros(d["dim"], ops.clip_image_kpad(d["patch"]))
        w[:, :3 * d["patch"] ** 2] = sd.pop("patch_embed.proj.weight").reshape(d["dim"], -1)
        self.conv = w.to(self.device)
        self.sd = {k: v.to(self.device) for k, v in sd.items()}
        self.sd["cls_token"] = self.sd["cls_token"].reshape(-1)
        self.sd["pos_embed"] = self.sd["pos_embed"].reshape(d["tokens"], d["dim"])
        self.max_rows = max(1, int(max_rows) if max_rows is not None else ACTIVATION_BUDGET // row_bytes(d))

    @torch.no_grad()
    def features(self, x):
        """x fp32 [B][3][S][S] in [-1, 1] (square) -> (keys, cls) on the device: keys the last block's keys, a strided
        view [B][T][D] into its qkv buffer (row stride 3D), cls fp32 [B][D] the final-norm CLS tokens"""
        d, sd = self.dims, self.sd
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != x.shape[3] or x.shape[0] == 0:
            raise ValueError(f"images must be [B][3][S][S] (square), got {tuple(x.shape)}")
        B, G, D, T = x.shape[0], d["grid"], d["dim"], d["tokens"]
        f32 = dict(dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            x = x.to(**f32).contiguous()
            patches = torch.empty(B * G * G, self.conv.shape[1], **f32)
            ops.dino_pack(x, patches, G, d["patch"])
            emb = torch.empty(B * G * G, D, **f32)
            ops.clip_linear(patches, self.conv, sd["patch_embed.proj.bias"], emb)
            del patches
            h = torch.empty(B, T, D, **f32)
            ops.clip_image_tokens(emb, sd["cls_token"], sd["pos_embed"], h)
            del emb
            t = torch.empty_like(h)
            qkv = torch.empty(B, T, 3 * D, **f32)
            mlp = torch.empty(B, T, 4 * D, **f32)
            for i in range(d["depth"]):
                b = {k: sd[f"blocks.{i}.{k}"] for k in BLOCK_KEYS}
                ops.dino_layernorm(h, b["norm1.weight"], b["norm1.bias"], t, eps=LN_EPS)
                ops.clip_linear(t, b["attn.qkv.weight"], b["attn.qkv.bias"], qkv)
                ops.dino_attention(qkv, t, d["heads"])
                ops.clip_linear(t, b["attn.proj.weight"], b["attn.proj.bias"], h, ops.CLIP_EPI_RESIDUAL, residual=h)
                ops.dino_layernorm(h, b["norm2.weight"], b["norm2.bias"], t, eps=LN_EPS)
                ops.clip_linear(t, b["mlp.fc1.weight"], b["mlp.fc1.bias"], mlp, ops.CLIP_EPI_GELU)
                ops.clip_linear(mlp, b["mlp.fc2.weight"], b["mlp.fc2.bias"], h, ops.CLIP_EPI_RESIDUAL, residual=h)
            cls = torch.empty(B, D, **f32)
            ops.dino_layernorm(h.view(B, T * D)[:, :D], sd["norm.weight"], sd["norm.bias"], cls, eps=LN_EPS)
        return qkv[:, :, D:2 * D], cls

    @torch.no_grad()
    def scores(self, origin, edited):
        """fp64 [n][B][2] on the host: (structure distance, cls_cos) of edited row j against origin row j % B, for
        origin [B][3][S][S] and edited [n B][3][S'][S'] in [-1, 1].  The origin features are computed once; both sides
        run in chunks of max_rows images, and each row's values do not depend on the chunking."""
        B, N = origin.shape[0], edited.shape[0]
        if B == 0 or N == 0 or N % B:
            raise ValueError(f"edited images ({N}) must be a positive whole multiple of the origin images ({B})")
        T, D, m = self.dims["tokens"], self.dims["dim"], self.max_rows
        f32 = dict(dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            # the origin keys and CLS rows stay resident; each chunk's keys follow them in one key buffer
            keys = torch.empty((B + min(m, N)) * T, D, **f32)
            cls_o = torch.empty(B, D, **f32)
            for s in range(0, B, m):
                k, c = self.features(origin[s:s + m])
                keys[s * T:(s + k.shape[0]) * T].view(k.shape[0], T, D).copy_(k)
                cls_o[s:s + k.shape[0]] = c
            dist = torch.empty(N, dtype=torch.float64, device=self.device)
            cos = torch.empty(N, **f32)
            for s in range(0, N, m):
                k, c = self.features(edited[s:s + m])
                n = k.shape[0]
                keys[B * T:(B + n) * T].view(n, T, D).copy_(k)
                j = torch.arange(s, s + n, device=self.device)
                ops.dino_selfsim_distance(keys, (j % B) * T, (B + j - s) * T, T, dist[s:s + n], eps=NORM_EPS)
                ops.clip_cosine(cls_o[j % B].contiguous(), c, cos[s:s + n], eps=NORM_EPS)
        return torch.stack([dist, cos.double()], dim=1).view(N // B, B, 2).cpu()
