"""Drop-in for the reference's utils/diffusion_utils.py (get_beta_schedule :5-9, extract :12-20,
denoising_step :24-109) on the CUDA engine: same names, argument meaning and return values.

`denoising_step` keeps the reference's per-call semantics (one UNet forward + one update, new tensors returned).
The fast path for whole trajectories is UNetEngine.sample() (engine.py), which `Asyrp.run_test` uses.
"""
import numpy as np
import torch

from .. import ops


def get_beta_schedule(*, beta_start, beta_end, num_diffusion_timesteps):
    betas = np.linspace(beta_start, beta_end, num_diffusion_timesteps, dtype=np.float64)
    assert betas.shape == (num_diffusion_timesteps,)
    return betas


def extract(a, t, x_shape):
    """a[t] as fp32, shaped to broadcast against x (host-side table lookup)."""
    bs, = t.shape
    assert x_shape[0] == bs, f"{x_shape[0]}, {t.shape}"
    out = torch.gather(torch.as_tensor(a, dtype=torch.float, device=t.device), 0, t.long())
    assert out.shape == (bs,)
    return out.reshape((bs,) + (1,) * (len(x_shape) - 1))


def denoising_step(xt, t, t_next, *, models, logvars=None, b, sampling_type='ddim', eta=0.0, learn_sigma=False,
                   index=None, t_edit=0, hs_coeff=(1.0), delta_h=None, use_mask=False, dt_lambda=1,
                   ignore_timestep=False, image_space_noise=0, dt_end=999, warigari=False, noise=None):
    """One reverse (or inversion, t < t_next) step.  Returns (xt_next, x0_t, delta_h, middle_h).

    `models` is an asyrp_official_b200 UNet module (DDPM / UNetModel mirror).  All samples of a batch share the
    timestep, as in every call site of the reference (diffusion_latent.py:504-505).  `noise` optionally supplies the
    N(0,1) draw the reference takes from torch.randn_like (:97)."""
    if type(image_space_noise) != int:
        raise NotImplementedError("image_space_noise optimisation is a training-side experiment (out of scope)")
    if sampling_type not in ('ddim', 'ddpm'):
        raise ValueError(f"unknown sampling_type {sampling_type!r}")
    model = models.module if hasattr(models, "module") and not hasattr(models, "engine") else models
    et, et_modified, delta_h, middle_h = model(xt, t, index=index, t_edit=t_edit, hs_coeff=hs_coeff, delta_h=delta_h,
                                               ignore_timestep=ignore_timestep, use_mask=use_mask)
    # alpha-bar lookups on the host, fp32 cumprod as the reference (:66-71)
    ti, tn = int(t[0].item()), int(t_next[0].item())
    bf = torch.as_tensor(b, dtype=torch.float32).cpu()
    ac = (1.0 - bf).cumprod(dim=0)
    at = ac[ti]
    if sampling_type == 'ddpm':  # ancestral step (:74-82); x0_t is not produced on this branch
        xt = xt.to(et.device, torch.float32).contiguous()
        z = (noise if noise is not None else torch.randn_like(xt)).to(et.device, torch.float32).contiguous()
        lv = 0.0 if learn_sigma else float(torch.as_tensor(logvars, dtype=torch.float32)[ti])
        xt_next = torch.empty_like(xt)
        with torch.cuda.device(et.device):
            ops.ddpm_update(xt, et, z, xt_next, float(at), float(bf[ti]), lv, learn_sigma, 0.0 if ti == 0 else 1.0)
        return xt_next, None, delta_h, middle_h
    an = torch.ones_like(at) if tn == -1 else ac[tn]
    if eta == 0:
        c1, c2 = torch.zeros_like(at), (1 - an).sqrt()
    else:
        c1 = eta * ((1 - at / an) * (1 - an) / (1 - at)).sqrt()
        c2 = ((1 - an) - c1 ** 2).sqrt()
    if dt_lambda != 1 and ti >= dt_end:  # :99-100
        c1, c2 = torch.zeros_like(at), (1 - an).sqrt() * dt_lambda
    xt = xt.to(et.device, torch.float32).contiguous()
    z = None
    if float(c1) != 0.0:
        z = noise if noise is not None else torch.randn_like(xt)
        z = z.to(et.device, torch.float32).contiguous()
    xt_next, x0_t = torch.empty_like(xt), torch.empty_like(xt)
    em = et_modified if index is not None else et
    with torch.cuda.device(et.device):
        ops.ddim_update(xt, et, em, z, xt_next, x0_t, float(at), float(an), float(c1), float(c2))
    return xt_next, x0_t, delta_h, middle_h
