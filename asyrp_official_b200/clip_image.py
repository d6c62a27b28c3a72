"""CLIP's image tower on the engine's kernels, and the directional similarity of the reference's CLIPLoss
(losses/clip_loss.py:102-117,170-180), the quantity `--DirectionalClipSmilarity` reports for each edit.

    preprocess     CLIPLoss.preprocess: Normalize(-1, 2), i.e. (x+1)/2; Resize(R, BICUBIC) as torchvision 0.10 resizes
                   a tensor (F.interpolate(mode="bicubic", align_corners=False), no antialiasing); CenterCrop(R), the
                   identity on the square images this takes; Normalize with CLIP's mean and std.
    encode_image   VisionTransformer.forward: conv1 (patch embedding, no bias) as one linear layer over the patch
                   matrix; x = [class_embedding ; patches] + positional_embedding; ln_pre; the residual blocks with full
                   attention; ln_post(x[:, 0]) @ proj.
    directional    get_image_features (each feature over its norm), edit direction (trg - src) / (|.| + 1e-7);
                   compute_text_direction: the templates formatted with each class text, each feature over its norm,
                   mean of trg - src over the templates, over its norm; S_dir = CosineSimilarity(eps=1e-8) of the two,
                   clip_directional_loss = 1 - mean S_dir.

Weights: the same --clip_weights file as clip_text (CLIP's TorchScript archive or a torch.save of its state dict);
only the visual.* keys of a ViT are used (INTEGRATION.md lists them); the ResNet family (RN50, ...) is not supported.
Every arithmetic operation is a kernel of libasyrp_b200.so (csrc/clip_image.cu, csrc/clip_text.cu): fp32 activations,
the linear layers on the TF32 tensor cores.
"""
import ast
import os

import torch

from . import _lib, clip_text, ops

PREFIX = "visual."
MAX_TOKENS = 257  # asyrp_clip_attention_full
IMAGE_EPS = 1e-7  # clip_directional_loss: edit_direction /= (norm + 1e-7)
COSINE_EPS = 1e-8  # DirectionLoss('cosine'): torch.nn.CosineSimilarity()'s default


def image_key_shapes(width, layers, patch, grid, embed_dim):
    """name -> shape of every visual.* tensor of a ViT CLIP state dict (without the prefix)"""
    shapes = {"conv1.weight": (width, 3, patch, patch), "class_embedding": (width,),
              "positional_embedding": (grid * grid + 1, width), "ln_pre.weight": (width,), "ln_pre.bias": (width,),
              "ln_post.weight": (width,), "ln_post.bias": (width,), "proj": (width, embed_dim)}
    shapes.update(clip_text.block_key_shapes(width, layers))
    return shapes


def load_state_dict(sd_or_path):
    """Validate the image tower of a CLIP state dict (or of the archive / torch.save at a path) and return
    (dims, tensors): dims = {width, heads, layers, patch, grid, resolution, embed_dim} derived as CLIP's build_model
    does, tensors = the visual.* tensors without the prefix, fp32 on the host.  Keys outside visual.* are ignored.

    Raises ValueError on a missing, mis-shaped or unknown visual key, on the ModifiedResNet layout (visual.layer1.*),
    on a width or embed_dim that is not a multiple of 64, on more than 257 tokens, and when the text tower's
    text_projection (when the state dict holds one) has another embed_dim."""
    sd = sd_or_path if isinstance(sd_or_path, dict) else clip_text._read(sd_or_path)
    text_proj = sd.get("text_projection")
    vis = {k[len(PREFIX):]: torch.as_tensor(v) for k, v in sd.items() if k.startswith(PREFIX)}
    if any(k.startswith("layer1.") for k in vis):
        raise ValueError("CLIP state dict: the ModifiedResNet image tower (RN50 family) is not supported; use a ViT "
                         "model (ViT-B/32, ViT-B/16, ViT-L/14)")
    for k in ("conv1.weight", "positional_embedding", "proj"):
        if k not in vis:
            raise ValueError(f"CLIP state dict: missing key {PREFIX + k!r}")
    conv, pos, proj = vis["conv1.weight"], vis["positional_embedding"], vis["proj"]
    if conv.dim() != 4 or pos.dim() != 2 or proj.dim() != 2:
        raise ValueError(f"CLIP state dict: visual.conv1.weight {tuple(conv.shape)}, visual.positional_embedding "
                         f"{tuple(pos.shape)} and visual.proj {tuple(proj.shape)} must be 4-, 2- and 2-D")
    blocks = {k.split(".")[2] for k in vis if k.startswith("transformer.resblocks.")}
    if not all(b.isdigit() for b in blocks):
        raise ValueError(f"CLIP state dict: unexpected visual residual-block names {sorted(blocks)}")
    width, patch = conv.shape[0], conv.shape[-1]
    grid = round((pos.shape[0] - 1) ** 0.5)
    dims = dict(width=width, heads=width // clip_text.HEAD_DIM, layers=len(blocks), patch=patch, grid=grid,
                resolution=grid * patch, embed_dim=proj.shape[1])
    if width % clip_text.HEAD_DIM or dims["embed_dim"] % 64 or dims["layers"] == 0:
        raise ValueError(f"CLIP state dict: visual width {width} and embed_dim {dims['embed_dim']} must be multiples "
                         f"of 64, with at least one residual block")
    if grid * grid + 1 != pos.shape[0] or pos.shape[0] > MAX_TOKENS:
        raise ValueError(f"CLIP state dict: visual.positional_embedding has {pos.shape[0]} rows; expected 1 + grid^2 "
                         f"<= {MAX_TOKENS}")
    if text_proj is not None and tuple(text_proj.shape)[-1] != dims["embed_dim"]:
        raise ValueError(f"CLIP state dict: the image tower's embed_dim {dims['embed_dim']} differs from the text "
                         f"tower's {tuple(text_proj.shape)[-1]}")
    expected = image_key_shapes(width, dims["layers"], patch, grid, dims["embed_dim"])
    out = {}
    for k, shape in expected.items():
        if k not in vis:
            raise ValueError(f"CLIP state dict: missing key {PREFIX + k!r}")
        if tuple(vis[k].shape) != shape:
            raise ValueError(f"CLIP state dict: {PREFIX + k!r} has shape {tuple(vis[k].shape)}, expected {shape}")
        out[k] = vis[k].detach().float().cpu().contiguous()
    unknown = sorted(PREFIX + k for k in set(vis) - set(expected))
    if unknown:
        raise ValueError(f"CLIP state dict: unexpected keys {unknown} (expected CLIP's VisionTransformer layout)")
    return dims, out


def read_templates(path):
    """imagenet_templates of the reference's utils/text_templates.py: the list literal assigned to that name, read with
    ast (the file is parsed, never imported or executed)"""
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found: pass --text_templates <file defining imagenet_templates> (the "
                                "reference's utils/text_templates.py)")
    with open(path, encoding="utf-8") as f:
        tree = ast.parse(f.read(), filename=path)
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "imagenet_templates"
                                                for t in node.targets):
            templates = ast.literal_eval(node.value)
            if not templates or not all(isinstance(t, str) for t in templates):
                raise ValueError(f"{path}: imagenet_templates must be a non-empty list of strings")
            return list(templates)
    raise ValueError(f"{path} assigns no imagenet_templates literal")


# ---------------------------------------------------------------------------------------------------------------------
class CLIPImage:
    """CLIPImage(weights).encode_image(x) -> fp32 [B][embed_dim] on the device for images x [B][3][S][S] in [-1, 1].
    Every operation is a kernel of libasyrp_b200.so; an image's features are bit-identical whatever batch it is in."""

    def __init__(self, state_dict_or_path, device=None):
        if not torch.cuda.is_available():
            raise _lib.AsyrpError("CLIPImage needs a CUDA device (sm_90a); there is no CPU path")
        _lib.load()
        self.dims, sd = load_state_dict(state_dict_or_path)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.sd = {k: v.to(self.device) for k, v in sd.items()}
        d = self.dims
        # conv1 over non-overlapping patches is a linear layer over the patch matrix, K zero-padded for the GEMM
        w = torch.zeros(d["width"], ops.clip_image_kpad(d["patch"]))
        w[:, :3 * d["patch"] ** 2] = sd["conv1.weight"].reshape(d["width"], -1)
        self.conv = w.to(self.device)
        self.proj = sd["proj"].t().contiguous().to(self.device)  # x @ proj is a linear layer with weight proj^T

    @torch.no_grad()
    def encode_image(self, x):
        """x fp32 [B][3][S][S] in [-1, 1] (square) -> fp32 [B][embed_dim] on the device"""
        d, sd = self.dims, self.sd
        x = torch.as_tensor(x)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] != x.shape[3] or x.shape[0] == 0:
            raise ValueError(f"images must be [B][3][S][S] (square), got {tuple(x.shape)}")
        B, G, w = x.shape[0], d["grid"], d["width"]
        T = G * G + 1
        f32 = dict(dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            x = x.to(**f32).contiguous()
            patches = torch.empty(B * G * G, self.conv.shape[1], **f32)
            ops.clip_image_patches(x, patches, G, d["patch"])
            emb = torch.empty(B * G * G, w, **f32)
            ops.clip_linear(patches, self.conv, None, emb)
            h = torch.empty(B, T, w, **f32)
            ops.clip_image_tokens(emb, sd["class_embedding"], sd["positional_embedding"], h)
            ops.clip_layernorm(h, sd["ln_pre.weight"], sd["ln_pre.bias"], h)
            clip_text.residual_blocks(sd, d["layers"], d["heads"], h, causal=False)
            pooled = torch.empty(B, w, **f32)
            ops.clip_layernorm_rows(h, sd["ln_post.weight"], sd["ln_post.bias"], pooled)
            feats = torch.empty(B, d["embed_dim"], **f32)
            ops.clip_linear(pooled, self.proj, None, feats)
        return feats


class CLIPLoss:
    """The directional term of the reference's CLIPLoss on both CLIP towers.  CLIPLoss(weights, vocab_path, templates)
    with templates the imagenet_templates list (read_templates)."""

    def __init__(self, state_dict_or_path, vocab_path, templates, device=None):
        sd = state_dict_or_path if isinstance(state_dict_or_path, dict) else clip_text._read(state_dict_or_path)
        self.text = clip_text.CLIPText(sd, vocab_path, device=device)
        self.image = CLIPImage(sd, device=device)
        self.device = self.image.device
        if self.text.dims["embed_dim"] != self.image.dims["embed_dim"]:
            raise ValueError(f"CLIP text embed_dim {self.text.dims['embed_dim']} != image embed_dim "
                             f"{self.image.dims['embed_dim']}")
        self.templates = list(templates)
        if not self.templates:
            raise ValueError("CLIPLoss needs at least one text template")
        self.target_direction = {}  # (source_class, target_class) -> [1][embed_dim] on the device

    def compose_text_with_templates(self, text):
        return [template.format(text) for template in self.templates]

    @torch.no_grad()
    def compute_text_direction(self, source_class, target_class):
        """normalize(mean_t(f(t(trg))/|f(t(trg))| - f(t(src))/|f(t(src))|)) over the templates t: [1][embed_dim]"""
        n = len(self.templates)
        feats = self.text.encode_text(self.text.tokenize(self.compose_text_with_templates(source_class) +
                                                         self.compose_text_with_templates(target_class)))
        out = torch.empty(1, feats.shape[1], dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ops.clip_direction(feats[:n], feats[n:], out, n, 0.0)
        return out

    @torch.no_grad()
    def directional_similarity(self, src_img, source_class, target_img, target_class):
        """S_dir = CosineSimilarity(eps 1e-8)(edit direction, text direction): fp32 [len(target_img)] on the host.
        target_img may hold k * B rows for B source images: row j is paired with source row j % B, so a batch edited
        at several strengths encodes its sources once.  The text direction is cached per (source, target) pair."""
        key = (source_class, target_class)
        if key not in self.target_direction:
            self.target_direction[key] = self.compute_text_direction(source_class, target_class)
        B, N = src_img.shape[0], target_img.shape[0]
        if B == 0 or N % B:
            raise ValueError(f"target images ({N}) must be a whole multiple of the source images ({B})")
        feats = self.image.encode_image(torch.cat([torch.as_tensor(src_img).to(self.device),
                                                   torch.as_tensor(target_img).to(self.device)]))
        src = feats[:B].repeat(N // B, 1)
        edit = torch.empty_like(src)
        cos = torch.empty(N, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ops.clip_direction(src, feats[B:].contiguous(), edit, 1, IMAGE_EPS)
            ops.clip_cosine(edit, self.target_direction[key].expand(N, -1).contiguous(), cos, eps=COSINE_EPS)
        return cos.cpu()

    def clip_directional_loss(self, src_img, source_class, target_img, target_class):
        """the reference's value: 1 - mean of directional_similarity"""
        return 1.0 - self.directional_similarity(src_img, source_class, target_img, target_class).double().mean().item()

