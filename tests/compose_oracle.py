"""Restatement of `--region_compose` (several attribute edits composed into one image, each in its own region) for
the tests: the weights and the composite in numpy fp64, the kernel's exact fp32 operation order, and the composed
edit trajectory on oracle/sampler.py's denoising_step.

    weights  s = M_1 + .. + M_K; w_k = M_k and w_0 = 1 - s where s <= 1, else w_k = M_k / s and w_0 = 0
    compose  x_j <- w_0 x_orig,j + sum_k w_k x_{k, j}, written to all K rows of image j
"""
import numpy as np
import torch

from oracle import sampler


def compose_weights(masks):
    """masks [K][...] -> (w_0 [...], w [K][...]) in fp64"""
    m = np.asarray(masks, dtype=np.float64)
    s = m.sum(axis=0)
    over = s > 1
    w = np.where(over, m / np.where(over, s, 1.0), m)
    return np.where(over, 0.0, 1.0 - s), w


def compose(x, ref, masks):
    """x [K][B][C][H][W], ref [B][C][H][W], masks [K][B][H][W] -> the composite [B][C][H][W] in fp64"""
    w0, w = compose_weights(masks)
    x = np.asarray(x, dtype=np.float64)
    return w0[:, None] * np.asarray(ref, dtype=np.float64) + (w[:, :, None] * x).sum(axis=0)


def fma32(a, b, c):
    """a * b + c of fp32 arrays rounded once to fp32, as fmaf: the product is exact in fp64, a two-sum gives the exact
    sum as s + err, and rounding s to odd with err makes the rounding to fp32 the single correct one"""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    prod = a * b
    s = prod + c
    bb = s - prod
    err = (prod - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    odd = np.nextafter(s, np.where(err > 0, np.inf, -np.inf))
    return np.where((err != 0) & even, odd, s).astype(np.float32)


def compose_fp32(x, ref, masks):
    """the composite as asyrp_compose_rows computes it, every fp32 rounding in its order: s = M_1, s = s + M_k;
    w_0 = 1 - s (or w_k = M_k / s, w_0 = 0 where s > 1); acc = w_0 r, then acc = fmaf(w_k, x_k, acc) for k = 1..K.
    x [K][B][C][H][W], ref [B][C][H][W], masks [K][B][H][W] (float32) -> [B][C][H][W] float32"""
    m = np.asarray(masks, dtype=np.float32)
    x = np.asarray(x, dtype=np.float32)
    r = np.asarray(ref, dtype=np.float32)
    s = m[0].copy()
    for k in range(1, m.shape[0]):
        s = (s + m[k]).astype(np.float32)  # fp32 + fp32 in numpy rounds once to nearest even
    over = s > np.float32(1)
    w0 = np.where(over, np.float32(0), (np.float32(1) - s).astype(np.float32)).astype(np.float32)
    w = np.where(over[None], (m / np.where(over, s, np.float32(1))[None]).astype(np.float32), m).astype(np.float32)
    acc = (w0[:, None] * r).astype(np.float32)
    for k in range(m.shape[0]):
        acc = fma32(np.broadcast_to(w[k][:, None], acc.shape), x[k], acc)
    return acc


def blend_fp32(x, ref, mask):
    """asyrp_blend_rows of one row per image: fmaf(m, x, (1 - m) * r), fp32"""
    m = np.asarray(mask, dtype=np.float32)[:, None]
    rest = ((np.float32(1) - m).astype(np.float32) * np.asarray(ref, dtype=np.float32)).astype(np.float32)
    return fma32(np.broadcast_to(m, rest.shape), x, rest)


@torch.no_grad()
def run_composed_trajectory(models, x_T, masks, x_orig, *, betas, seq, seq_next, t_edit, t_addnoise, hs_coeff,
                            learn_sigma=False, noises=None, logvars=None):
    """the edit loop of every attribute k (its forward models[k], t_edit[k], t_addnoise[k], hs_coeff[k]) from the same
    images x_T [b][C][S][S], with the composite after every step: x_orig[k] is the origin pass's x after step k
    ([steps][b][C][S][S]), masks [K][b][S][S].  noises: {t: [b][C][S][S]}, shared by the attributes.  The composite
    is taken in fp64 and stored in x_T's dtype; returns the last one, [b][C][S][S]."""
    K = len(models)
    x = x_T.clone()
    n = x.shape[0]
    for k_step, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        t, t_nx = torch.ones(n) * i, torch.ones(n) * j
        rows = []
        for k in range(K):
            eta = 1.0 if i < t_addnoise[k] else 0.0
            xk, _, _, _ = sampler.denoising_step(x, t, t_nx, model=models[k], logvars=logvars, b=betas, eta=eta,
                                                 learn_sigma=learn_sigma, index=0, t_edit=t_edit[k],
                                                 hs_coeff=hs_coeff[k], noise=None if noises is None else noises.get(i))
            rows.append(xk.double().numpy())
        x = torch.from_numpy(compose(np.stack(rows), torch.as_tensor(x_orig[k_step]).double().numpy(),
                                     np.asarray(masks))).to(x_T.dtype)
    return x
