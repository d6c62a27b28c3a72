"""numpy fp64 restatement of the region masks of `--edit_region` (asyrp_official_b200/region.py) and of the blended
edit trajectory — TEST INFRASTRUCTURE ONLY.

    select   mask[y][x] = 1 if any label in rows [ceil(y 512 / S), ceil((y + 1) 512 / S)) x (columns likewise) is chosen
    dilate   (2r + 1)^2 max filter, the window clipped at the border
    feather  Gaussian taps exp(-i^2 / 2 sigma^2), |i| <= ceil(3 sigma), normalised; horizontal then vertical pass with
             clamped indices; a window whose inputs are all equal returns that value
    blend    after every step's update x <- m x + (1 - m) x_orig,k
"""
import math

import numpy as np
import torch

from . import sampler

LABEL_SIZE = 512


def select(labels, classes, S):
    """labels int [N][512][512] -> fp64 [N][S][S]"""
    labels = np.asarray(labels)
    hit = np.isin(labels, list(classes)).astype(np.uint8)
    lo = [-(-y * LABEL_SIZE // S) for y in range(S)]  # ceil(y 512 / S): every footprint is at least one pixel
    out = np.maximum.reduceat(np.maximum.reduceat(hit, lo, axis=1), lo, axis=2)
    return out.astype(np.float64)


def dilate(m, r):
    """square max filter of radius r, clipped at the border"""
    m = np.asarray(m, dtype=np.float64)
    if r == 0:
        return m.copy()
    S = m.shape[-1]
    h = np.stack([m[..., :, max(0, x - r):min(S, x + r + 1)].max(axis=-1) for x in range(S)], axis=-1)
    return np.stack([h[..., max(0, y - r):min(S, y + r + 1), :].max(axis=-2) for y in range(S)], axis=-2)


def taps(sigma):
    R = math.ceil(3.0 * sigma)
    i = np.arange(-R, R + 1, dtype=np.float64)
    w = np.exp(-i * i / (2.0 * sigma * sigma))
    return w / w.sum()


def _blur_axis(m, w, axis):
    R = len(w) // 2
    S = m.shape[axis]
    idx = np.clip(np.arange(S)[:, None] + np.arange(-R, R + 1)[None, :], 0, S - 1)  # [S][2R + 1]
    win = np.take(np.moveaxis(m, axis, -1), idx, axis=-1)                          # [..][S][2R + 1]
    flat = (win == win[..., :1]).all(axis=-1)
    out = np.where(flat, win[..., 0], win @ w)
    return np.moveaxis(out, -1, axis)


def feather(m, sigma):
    m = np.asarray(m, dtype=np.float64)
    if sigma == 0:
        return m.copy()
    w = taps(sigma)
    return _blur_axis(_blur_axis(m, w, -1), w, -2)


def masks(labels, classes, S, r=0, sigma=0.0):
    return feather(dilate(select(labels, classes, S), r), sigma)


@torch.no_grad()
def run_blended_trajectory(model, x_T, mask, x_orig, *, betas, seq, seq_next, t_edit, t_addnoise=0, index=0,
                           hs_coeff=(1.0, 1.0), learn_sigma=False, noises=None, logvars=None):
    """run_trajectory's edit loop with the blend after every step: x_orig[k] is the origin pass's x after step k
    ([steps][B][C][S][S]), mask [B][S][S]; row n blends with image n % B"""
    x = x_T.clone()
    n = x.shape[0]
    B = mask.shape[0]
    m = torch.as_tensor(mask, dtype=torch.float32)[torch.arange(n) % B][:, None]
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t = torch.ones(n) * i
        t_next = torch.ones(n) * j
        eta = 1.0 if i < t_addnoise else 0.0
        x, _, _, _ = sampler.denoising_step(x, t, t_next, model=model, logvars=logvars, b=betas, eta=eta,
                                            learn_sigma=learn_sigma, index=index, t_edit=t_edit, hs_coeff=hs_coeff,
                                            noise=None if noises is None else noises.get(i))
        ref = torch.as_tensor(x_orig[k], dtype=torch.float32)[torch.arange(n) % B]
        x = m * x + (1 - m) * ref
    return x
