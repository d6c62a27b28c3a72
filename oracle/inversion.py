"""numpy fp64 restatement of exact inversion (asyrp_official_b200/inversion.py, ops.ddim_update_anchored) — TEST
INFRASTRUCTURE ONLY.

    anchored step   y  = Phi_k(x, eps_mod, eps),  yr = Phi_k(A[k], E[k], E[k]),  x' = A[k+1] + (y - yr)
                    Phi_k the oracle's denoising_step without its noise term (the same c1 z in both would cancel)

The anchors A / E are inputs: the engine's recorded inversion, as oracle/region.py takes the recorded origin pass.
"""
import numpy as np
import torch

from . import sampler


def anchored_step(x, em, et, a, ea, a_next, at, an, c2):
    """one anchored update in fp64: x, em, et for the rows, a, ea, a_next for their images (broadcast to the rows)"""
    x, em, et, a, ea, a_next = (np.asarray(v, dtype=np.float64) for v in (x, em, et, a, ea, a_next))
    at, an, c2 = float(at), float(an), float(c2)

    def phi(xx, m, e):
        return np.sqrt(an) * ((xx - m * np.sqrt(1.0 - at)) / np.sqrt(at)) + c2 * e

    return a_next + (phi(x, em, et) - phi(a, ea, ea))


def _phi(model, x, t, t_next, betas, eta, learn_sigma, **kw):
    """denoising_step in fp64 with zero noise: sqrt(an) x0 + c2 eps"""
    zeros = torch.zeros(x.shape, dtype=torch.float64)
    y, _, _, _ = sampler.denoising_step(x, t, t_next, model=model, b=betas, eta=eta, learn_sigma=learn_sigma,
                                        noise=zeros if eta else None, **kw)
    return y.double()


@torch.no_grad()
def run_anchored_trajectory(model, A, E, *, betas, seq, seq_next, t_edit, t_addnoise=0, index=0, hs_coeff=(1.0, 1.0),
                            learn_sigma=False, xs=None):
    """run_trajectory's edit loop, every step anchored: starts from A[0] (rows n on image n % B), A [n + 1][B][C][S][S],
    E [n][B][C][S][S] (the engine's recorded anchors); returns the final x in fp64.  `model` has the reference forward
    signature (the oracle's UNets).
    xs: the engine's x after every step ([n][N][C][S][S], its record_process "x").  Step k then starts from the engine's
    x (A[0], then xs[k - 1]) rather than from the oracle's own, and the list of (x after step k, max |eps| of the
    oracle's UNet at step k) is returned: a per-step comparison in which UNet errors do not compound."""
    seen = {}

    def fp64(fwd):  # the oracle UNets take fp32 inputs; their outputs are carried on in fp64
        def f(xx, t, **k):
            out = tuple(v.double() if torch.is_tensor(v) else v for v in fwd(xx.float(), t, **k))
            seen["eps"] = max(float(v.abs().max()) for v in out[:2] if torch.is_tensor(v))
            return out
        return f

    model = fp64(model)
    A = torch.as_tensor(A, dtype=torch.float64)
    E = torch.as_tensor(E, dtype=torch.float64)
    B = A.shape[1]
    x = A[0].clone()
    n = x.shape[0]
    idx = torch.arange(n) % B

    def anchor_model(e):
        def fwd(xx, t, **k):
            return e, e, None, None
        return fwd

    steps = []
    for k, (i, j) in enumerate(zip(reversed(seq), reversed(seq_next))):
        if xs is not None and k:
            x = torch.as_tensor(xs[k - 1], dtype=torch.float64)
        t, t_next = torch.ones(n) * i, torch.ones(n) * j
        eta = 1.0 if i < t_addnoise else 0.0
        y = _phi(model, x, t, t_next, betas, eta, learn_sigma, index=index, t_edit=t_edit, hs_coeff=hs_coeff)
        e = E[k][idx]
        if learn_sigma:  # denoising_step splits [eps | variance]; the anchor's eps carries no variance half
            e = torch.cat([e, torch.zeros_like(e)], dim=1)
        yr = _phi(anchor_model(e), A[k][idx], t, t_next, betas, eta, learn_sigma, index=0, t_edit=0)
        x = A[k + 1][idx] + (y - yr)
        steps.append((x, seen["eps"]))
    return steps if xs is not None else x
