"""CPU oracle of the reference's IDLoss (losses/id_loss.py) and ArcFace Backbone(112, 50, 'ir_se') in eval mode
(models/insight_face/model_irse.py, helpers.py), restated from the architecture on the raw (unfolded) state dict:
crop x[:, :, 35:223, 32:220], AdaptiveAvgPool2d((112, 112)) written out bin by bin, the input layer, 24 bottleneck
IR-SE blocks, the output layer (BN2d, flatten NCHW, linear, BN1d), l2_norm and IDLoss.  Test infrastructure only;
evaluated in fp32 or fp64 (the `dtype` argument)."""
import torch
import torch.nn.functional as F

BLOCKS = tuple([(64, 64, 2)] + [(64, 64, 1)] * 2 + [(64, 128, 2)] + [(128, 128, 1)] * 3 + [(128, 256, 2)] +
               [(256, 256, 1)] * 13 + [(256, 512, 2)] + [(512, 512, 1)] * 2)
EPS = 1e-5


def crop(x):
    return x[:, :, 35:223, 32:220]


def adaptive_avg_pool(x, out=112):
    """AdaptiveAvgPool2d((out, out)): bin i covers [floor(S i / out), ceil(S (i+1) / out))"""
    S_h, S_w = x.shape[-2:]

    def bins(S):
        return [((S * i) // out, -(-(S * (i + 1)) // out)) for i in range(out)]
    rows = torch.stack([x[..., a:b, :].mean(-2) for a, b in bins(S_h)], -2)
    return torch.stack([rows[..., a:b].mean(-1) for a, b in bins(S_w)], -1)


def preprocess(x, dtype=torch.float64):
    """IDLoss.extract_feats before the backbone: [B][3][112][112]"""
    return adaptive_avg_pool(crop(torch.as_tensor(x).to(dtype)))


def _g(sd, dtype):
    return {k: v.to(dtype) for k, v in sd.items() if not k.endswith("num_batches_tracked")}


def batch_norm(x, g, prefix):
    shape = (1, -1) + (1,) * (x.dim() - 2)
    scale = g[prefix + ".weight"] / torch.sqrt(g[prefix + ".running_var"] + EPS)
    return (x - g[prefix + ".running_mean"].view(shape)) * scale.view(shape) + g[prefix + ".bias"].view(shape)


def prelu(x, a):
    return torch.where(x > 0, x, a.view(1, -1, 1, 1) * x)


def se(x, g, prefix):
    m = x.mean((2, 3), keepdim=True)
    h = torch.relu(F.conv2d(m, g[prefix + ".fc1.weight"]))
    return x * torch.sigmoid(F.conv2d(h, g[prefix + ".fc2.weight"]))


def block(x, g, i, cin, depth, stride):
    p = f"body.{i}."
    if cin == depth:
        sc = x[:, :, ::stride, ::stride]  # MaxPool2d(1, stride)
    else:
        sc = batch_norm(F.conv2d(x, g[p + "shortcut_layer.0.weight"], stride=stride), g, p + "shortcut_layer.1")
    r = batch_norm(x, g, p + "res_layer.0")
    r = prelu(F.conv2d(r, g[p + "res_layer.1.weight"], padding=1), g[p + "res_layer.2.weight"])
    r = batch_norm(F.conv2d(r, g[p + "res_layer.3.weight"], stride=stride, padding=1), g, p + "res_layer.4")
    return se(r, g, p + "res_layer.5") + sc


def backbone(sd, x, dtype=torch.float64):
    """Backbone.forward of [B][3][112][112] -> [B][512] unit vectors (l2_norm, no epsilon)"""
    g = _g(sd, dtype)
    x = x.to(dtype)
    h = prelu(batch_norm(F.conv2d(x, g["input_layer.0.weight"], padding=1), g, "input_layer.1"),
              g["input_layer.2.weight"])
    for i, (cin, depth, stride) in enumerate(BLOCKS):
        h = block(h, g, i, cin, depth, stride)
    h = batch_norm(h, g, "output_layer.0").reshape(h.shape[0], -1)  # Dropout: identity in eval; flatten NCHW
    h = h @ g["output_layer.3.weight"].t() + g["output_layer.3.bias"]
    h = batch_norm(h, g, "output_layer.4")
    return h / torch.norm(h, 2, 1, True)


def extract_feats(sd, x, dtype=torch.float64):
    return backbone(sd, preprocess(x, dtype), dtype)


def id_loss(sd, x, x_hat, dtype=torch.float64):
    """IDLoss.forward: 1 - x_hat_feats[i] . x_feats[i] per row"""
    return 1 - (extract_feats(sd, x_hat, dtype) * extract_feats(sd, x, dtype)).sum(-1)


def id_similarity(sd, src, edited, dtype=torch.float64):
    """1 - IDLoss with edited row j paired with source row j % B"""
    B = src.shape[0]
    fs, fe = extract_feats(sd, src, dtype), extract_feats(sd, edited, dtype)
    return (fe * fs.repeat(edited.shape[0] // B, 1)).sum(-1)
