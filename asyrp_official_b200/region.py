"""Region-restricted edits (`--edit_region`): a soft mask per image from the face parser's labels of the origin pass,
and what the edit pass blends with it.  `--region_compose` builds one such mask per attribute and composes the
attributes' edit passes into one image (UNetEngine.sample's compose).

Asyrp edits the 8x8 bottleneck h, and the decoder spreads the change over the whole image.  With a region, every step
of the edit pass ends with x <- m x + (1 - m) x_orig, where x_orig is the origin pass (the unedited trajectory of the
same x_T) after the same step: outside the region the edit pass follows the origin pass exactly.

    select   output pixel (y, x) of an S x S mask is 1 if any label of its footprint in the 512 x 512 label map is one
             of the chosen classes: rows [ceil(y 512 / S), ceil((y + 1) 512 / S)), columns likewise (S <= 512)
    dilate   a (2r + 1)^2 square max filter clipped at the image border, 0 <= r <= 32
    feather  a separable Gaussian, horizontal pass then vertical pass, sigma 0..16 (0: none): R = ceil(3 sigma), taps
             exp(-i^2 / 2 sigma^2) for |i| <= R normalised in fp64 and stored as fp32, indices clamped at the edges,
             fp32 accumulation in tap order -R..R; a window whose inputs are all equal returns that value, so flat
             regions stay exactly 0 or 1

Every step is a kernel of libasyrp_b200.so (csrc/region.cu); oracle/region.py restates them in numpy fp64.

The class names are the 19 labels of the public face-parsing BiSeNet, in index order.  No real 79999_iter.pth has been
loaded by this project's tests, so the order follows the public model and has not been checked against a real
checkpoint.
"""
import math

import numpy as np
import torch

from . import ops

CLASSES = ("background", "skin", "l_brow", "r_brow", "l_eye", "r_eye", "eye_g", "l_ear", "r_ear", "ear_r", "nose",
           "mouth", "u_lip", "l_lip", "neck", "neck_l", "cloth", "hair", "hat")
MAX_DILATE = 32
MAX_FEATHER = 16.0
MAX_SIZE = 512  # the parser's label maps
MAX_COMPOSE = 8  # attributes of one --region_compose composite (asyrp_compose_rows)


def parse_classes(text, flag="--edit_region"):
    """'hair hat' -> the class indices in the order given; ValueError for an unknown, repeated or missing name, naming
    `flag`"""
    names = str(text).split()
    if not names:
        raise ValueError(f"{flag} names no class; valid names: {' '.join(CLASSES)}")
    out = []
    for name in names:
        if name not in CLASSES:
            raise ValueError(f"{flag}: unknown class {name!r}; valid names: {' '.join(CLASSES)}")
        if CLASSES.index(name) in out:
            raise ValueError(f"{flag}: class {name!r} given twice; valid names: {' '.join(CLASSES)}")
        out.append(CLASSES.index(name))
    return out


def parse_compose(text):
    """--region_compose 'smiling=mouth,u_lip,l_lip grey_hair=hair' -> [(attribute, class indices)] in the order
    given; ValueError for a malformed item, an attribute named twice, an empty, unknown or repeated class, a class
    given to two attributes, or more than MAX_COMPOSE attributes"""
    flag = "--region_compose"
    out = []
    for item in str(text).split():
        attr, sep, names = item.partition("=")
        if not sep or not attr or "=" in names:
            raise ValueError(f"{flag}: {item!r} is not attribute=class,class,..")
        if attr in [a for a, _ in out]:
            raise ValueError(f"{flag} names attribute {attr!r} twice")
        if not names or "" in names.split(","):
            raise ValueError(f"{flag}: attribute {attr!r} has an empty class list or an empty class name "
                             f"({names!r}); valid names: {' '.join(CLASSES)}")
        classes = parse_classes(names.replace(",", " "), f"{flag} ({attr})")
        for a, other in out:
            shared = [CLASSES[c] for c in classes if c in other]
            if shared:
                raise ValueError(f"{flag}: class(es) {' '.join(shared)} given to both {a!r} and {attr!r}")
        out.append((attr, classes))
    if not out:
        raise ValueError(f"{flag} names no attribute")
    if len(out) > MAX_COMPOSE:
        raise ValueError(f"{flag} composes at most {MAX_COMPOSE} attributes, got {len(out)}")
    return out


def class_bits(classes):
    """class indices -> the u32 bit set the select kernel takes"""
    return sum(1 << int(c) for c in set(classes))


def check_options(r, sigma, size):
    """ValueError unless 0 <= r <= 32, 0 <= sigma <= 16 and the image size is at most 512"""
    if not (isinstance(r, int) and 0 <= r <= MAX_DILATE):
        raise ValueError(f"--edit_region_dilate must be an integer in 0..{MAX_DILATE}, got {r!r}")
    if not (math.isfinite(float(sigma)) and 0.0 <= float(sigma) <= MAX_FEATHER):
        raise ValueError(f"--edit_region_feather must be in 0..{MAX_FEATHER:g}, got {sigma!r}")
    if not 1 <= int(size) <= MAX_SIZE:
        raise ValueError(f"--edit_region: the image size {size} is above the parser's {MAX_SIZE} x {MAX_SIZE} labels")


def taps(sigma):
    """the feather taps, fp32 [2R + 1] with R = ceil(3 sigma): exp(-i^2 / 2 sigma^2) normalised in fp64; None for
    sigma = 0 (no feathering)"""
    sigma = float(sigma)
    if sigma == 0.0:
        return None
    R = math.ceil(3.0 * sigma)
    i = np.arange(-R, R + 1, dtype=np.float64)
    w = np.exp(-i * i / (2.0 * sigma * sigma))
    return torch.from_numpy((w / w.sum()).astype(np.float32))


@torch.no_grad()
def masks_from_labels(labels, classes, size, r=0, sigma=0.0):
    """labels u8 [N][512][512] on the device -> soft masks fp32 [N][size][size] on the same device"""
    N = labels.shape[0]
    dev = labels.device
    mask = torch.empty(N, size, size, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ops.region_mask(labels.contiguous(), class_bits(classes), mask)
        tmp = torch.empty_like(mask)
        if r:
            ops.mask_dilate(mask, tmp, r, 0)
            ops.mask_dilate(tmp, mask, r, 1)
        w = taps(sigma)
        if w is not None:
            w = w.to(dev)
            ops.mask_blur(mask, w, tmp, 0)
            ops.mask_blur(tmp, w, mask, 1)
    return mask


@torch.no_grad()
def region_masks(parser, origin, classes, r=0, sigma=0.0):
    """the masks of a batch: parse the origin pass's x0 (fp32 [B][3][S][S], [-1, 1]) with parser
    (face_parsing.FaceParser) and build one S x S soft mask per image, fp32 [B][S][S] on the parser's device"""
    S = origin.shape[-1]
    check_options(r, sigma, S)
    return masks_from_labels(parser.labels(origin), classes, S, r, sigma)


@torch.no_grad()
def compose_masks(parser, origin, class_lists, r=0, sigma=0.0):
    """--region_compose's masks of a batch: the origin pass's x0 (fp32 [B][3][S][S]) parsed once, then one soft mask
    per attribute and image from that attribute's classes, fp32 [K][B][S][S] on the parser's device.  Attribute k's
    masks are region_masks(parser, origin, class_lists[k], r, sigma)."""
    S = origin.shape[-1]
    check_options(r, sigma, S)
    labels = parser.labels(origin)
    return torch.stack([masks_from_labels(labels, classes, S, r, sigma) for classes in class_lists])
