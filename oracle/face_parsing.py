"""CPU oracle of the face-parsing BiSeNet (BiSeNet(n_classes=19), eval mode) and of the segmentation consistency (SC)
of an edit, restated as torch.nn.functional calls on the raw (unfolded) state dict.  Test infrastructure only;
evaluated in fp64 by default (the `dtype` argument).  The network and the metric are this project's definition
(asyrp_official_b200/face_parsing.py): the reference has no segmentation network.

  input     clamp to [-1, 1], map to [0, 1], bilinear resize to 512 x 512 (align_corners=False), ImageNet mean / std
  backbone  cp.resnet: ResNet-18 (conv1 7x7/2 + bn1 + ReLU, max-pool 3x3/2 pad 1, layer1..4) -> feat8, feat16, feat32
  context   avg = ConvBNReLU1x1(mean_hw(feat32)); s32 = arm32(feat32) + avg; up32 = conv_head32(nearest2x(s32));
            s16 = arm16(feat16) + up32; up16 = conv_head16(nearest2x(s16)); ARM(x) = f * sigmoid(bn_atten(conv_atten(
            mean_hw(f)))), f = ConvBNReLU3x3(x)
  ffm       f = convblk(cat[feat8, up16]); out = f * sigmoid(conv2(relu(conv1(mean_hw(f))))) + f
  head      conv_out.conv (ConvBNReLU3x3), conv_out.conv_out (1x1) -> logits at 64 x 64, bilinear align_corners=True to
            512 x 512, argmax over classes
  SC        fraction of the 512^2 pixels whose label equals the label of the source row j % B
"""
import torch
import torch.nn.functional as F

EPS = 1e-5
SIZE = 512
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
LAYERS = ((64, 1), (128, 2), (256, 2), (512, 2))  # (channels, stride of block 0) of layer1..4


def _g(sd, dtype):
    return {k: v.to(dtype) for k, v in sd.items() if not k.endswith("num_batches_tracked")}


def bn(x, g, prefix):
    shape = (1, -1) + (1,) * (x.dim() - 2)
    scale = g[prefix + ".weight"] / torch.sqrt(g[prefix + ".running_var"] + EPS)
    return (x - g[prefix + ".running_mean"].view(shape)) * scale.view(shape) + g[prefix + ".bias"].view(shape)


def conv_bn_relu(x, g, prefix, stride=1):
    w = g[prefix + ".conv.weight"]
    return torch.relu(bn(F.conv2d(x, w, stride=stride, padding=w.shape[-1] // 2), g, prefix + ".bn"))


def preprocess(x, dtype=torch.float64):
    """[B][3][H][W] in [-1, 1] -> the normalised [B][3][512][512] the backbone reads"""
    x = torch.as_tensor(x).to(dtype).clamp(-1, 1) * 0.5 + 0.5
    x = F.interpolate(x, (SIZE, SIZE), mode="bilinear", align_corners=False)
    mean = torch.tensor(MEAN, dtype=dtype).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=dtype).view(1, 3, 1, 1)
    return (x - mean) / std


def basic_block(x, g, prefix, stride):
    r = torch.relu(bn(F.conv2d(x, g[prefix + ".conv1.weight"], stride=stride, padding=1), g, prefix + ".bn1"))
    r = bn(F.conv2d(r, g[prefix + ".conv2.weight"], padding=1), g, prefix + ".bn2")
    sc = x
    if prefix + ".downsample.0.weight" in g:
        sc = bn(F.conv2d(x, g[prefix + ".downsample.0.weight"], stride=stride), g, prefix + ".downsample.1")
    return torch.relu(sc + r)


def resnet(g, x, prefix="cp.resnet"):
    """(feat8, feat16, feat32) of the normalised [B][3][512][512] input; g: the state dict in the oracle's dtype"""
    h = torch.relu(bn(F.conv2d(x, g[prefix + ".conv1.weight"], stride=2, padding=3), g, prefix + ".bn1"))
    h = F.max_pool2d(h, 3, 2, 1)
    feats = []
    for li, (_, stride) in enumerate(LAYERS):
        for b in range(2):
            h = basic_block(h, g, f"{prefix}.layer{li + 1}.{b}", stride if b == 0 else 1)
        feats.append(h)
    return feats[1], feats[2], feats[3]


def arm(x, g, prefix):
    f = conv_bn_relu(x, g, prefix + ".conv")
    a = bn(F.conv2d(f.mean((2, 3), keepdim=True), g[prefix + ".conv_atten.weight"]), g, prefix + ".bn_atten")
    return f * torch.sigmoid(a)


def logits(sd, x, dtype=torch.float64):
    """the main head's logits [B][n_classes][64][64] of images x [B][3][H][W] in [-1, 1]"""
    g = _g(sd, dtype)
    feat8, feat16, feat32 = resnet(g, preprocess(x, dtype))
    avg = conv_bn_relu(feat32.mean((2, 3), keepdim=True), g, "cp.conv_avg")
    s32 = arm(feat32, g, "cp.arm32") + avg
    up32 = conv_bn_relu(F.interpolate(s32, feat16.shape[2:], mode="nearest"), g, "cp.conv_head32")
    s16 = arm(feat16, g, "cp.arm16") + up32
    up16 = conv_bn_relu(F.interpolate(s16, feat8.shape[2:], mode="nearest"), g, "cp.conv_head16")
    f = conv_bn_relu(torch.cat([feat8, up16], 1), g, "ffm.convblk")
    a = torch.sigmoid(F.conv2d(torch.relu(F.conv2d(f.mean((2, 3), keepdim=True), g["ffm.conv1.weight"])),
                               g["ffm.conv2.weight"]))
    f = f * a + f
    return F.conv2d(conv_bn_relu(f, g, "conv_out.conv"), g["conv_out.conv_out.weight"])


def upsample(lg):
    """the logits at 512 x 512 (bilinear, align_corners=True)"""
    return F.interpolate(lg, (SIZE, SIZE), mode="bilinear", align_corners=True)


def labels(sd, x, dtype=torch.float64):
    return upsample(logits(sd, x, dtype)).argmax(1)


def top2_margin(lg):
    """per 512^2 pixel: the upsampled top-1 minus top-2 logit"""
    top = upsample(lg).topk(2, dim=1).values
    return top[:, 0] - top[:, 1]


def seg_consistency(sd, src, edited, dtype=torch.float64):
    """SC of edited row j against source row j % B: the fraction of pixels with equal labels"""
    B = src.shape[0]
    ls, le = labels(sd, src, dtype), labels(sd, edited, dtype)
    return (le == ls.repeat(edited.shape[0] // B, 1, 1)).double().mean((1, 2))
