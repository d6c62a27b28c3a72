"""Generate tests/golden/diff_style_mini.npz by running the REFERENCE'S OWN modules and denoising_step (imported through
make_golden.py) on the reduced DDPM and ADM configurations with the synthetic weights of oracle/synth.py.

    python tests/golden/make_diff_style_golden.py

DiffStyle as --diff_style runs it (asyrp_official_b200.diffusion_latent.Asyrp.run_diff_style):
  * inversion with h (precompute_pairs_with_h, diffusion_latent.py:877-947): DDIM, eta 0, plain UNet over
    zip(seq_inv_next[1:], seq_inv[1:]), h_dic[t] = the middle_h of the step that ran the UNet at t;
  * the content h at t_0 = middle_h of the content's x_T at t_0 (the inversion never evaluates t_0);
  * generation from the style's x_T over zip(reversed(seq_inv), reversed(seq_inv_next)), each step
    denoising_step(..., index=0, t_edit, hs_coeff=(gamma,), delta_h=h_c[t], use_mask, eta = 1 below t_noise,
    dt_lambda, dt_end), the eta = 1 draws pre-drawn (seeded) instead of torch.randn_like.
Two contents x two styles, gamma in GAMMAS, use_mask off and on; the four pairs of one (gamma, use_mask) run as one
batch of 4.  The oracle restatement (tests/test_diff_style_host.py) must reproduce every tensor bit for bit.

The input images are regenerated from their seeds (test_diff_style_host.style_images), so only their sums are kept.
Every other tensor is kept as its fp64 sum and its max |.| (per image / row and step), which pin every element, plus a
sparse sample (SUB) of its elements; the file stays about 100 KB.

Keys per family f (ddpm, adm):
  f_x0_sum [4] (contents then styles); f_xT_sum / f_xT_absmax [4], f_xT_sub [4][3][S/8][S/8];
  h_dic: f_h_t (the keys), f_h_sum / f_h_absmax [4][steps], f_h_c0 [steps][C/4][h/4][w/4] (content 0's entries);
  f_h0_sum / f_h0_absmax [2], f_h0_sub [2][C/4][h/4][w/4] (content h at t_0);
  f_traj_g<k>_m<0|1>_sum / _absmax [steps][4] (x after every generation step) and f_traj_g<k>_m<0|1>_sub
  [steps][4][3][S/8][S/8], rows = pairs (c0,s0) (c0,s1) (c1,s0) (c1,s1);
shared: seq, t_edit, t_noise, dt_lambda, dt_end, gammas, noise_seed.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402  (puts the repository and the reference on sys.path)
from make_golden import o_adm, o_ddpm, o_smp, ref_du, synth  # noqa: E402

from test_diff_style_host import (DT_END, DT_LAMBDA, GAMMAS, N_STEP, NOISE_SEED, T_EDIT, T_NOISE,  # noqa: E402
                                  golden_noises, oracle_diff_style, oracle_invert_with_h, oracle_model, pair_rows,
                                  style_images)


def sub_x(t):
    """the sparse sample of an image tensor [..][3][S][S]: every 8th pixel"""
    return t[..., ::8, ::8].contiguous().numpy()


def sub_h(t):
    """the sparse sample of a bottleneck tensor [..][C][h][w]: every 4th channel, every 4th pixel"""
    return t[..., ::4, ::4, ::4].contiguous().numpy()


def stats(t, dims):
    """(fp64 sum, max |.|) over `dims`"""
    return t.double().sum(dim=dims).numpy(), t.abs().amax(dim=dims).numpy()


def ref_step(model, x, i, j, logv, betas, learn_sigma, **kw):
    n = x.shape[0]
    return ref_du.denoising_step(x, t=torch.ones(n) * i, t_next=torch.ones(n) * j, models=model, logvars=logv,
                                 sampling_type="ddim", b=betas, learn_sigma=learn_sigma, **kw)


@torch.no_grad()
def family_fixture(family, out):
    if family == "ddpm":
        cfg, shapes, model = o_ddpm.MINI_CFG, o_ddpm.ddpm_param_shapes(o_ddpm.MINI_CFG, 0), mg.ref_ddpm(o_ddpm.MINI_CFG, 0)
        learn_sigma = False
    else:
        cfg, shapes, model = o_adm.MINI_HP, o_adm.adm_param_shapes(o_adm.MINI_HP, 0), mg.ref_adm(o_adm.MINI_HP, 0)
        learn_sigma = True
    sd = synth.synth_state_dict(shapes, seed=1234, style="jittered")
    mg.load_checked(model, shapes, sd)
    betas = o_smp.make_betas()
    logv = None if learn_sigma else o_smp.make_logvar(o_smp.get_beta_schedule(beta_start=1e-4, beta_end=0.02,
                                                                             num_diffusion_timesteps=1000))
    seq, seq_next = o_smp.make_sequences(999, N_STEP)
    x0 = style_images(cfg["image_size"])
    # inversion with h, one image at a time as precompute_pairs_with_h runs it
    xT, hs = [], []
    for k in range(x0.shape[0]):
        x, h_dic = x0[k:k + 1].clone(), {}
        for i, j in zip(seq_next[1:], seq[1:]):
            x, _, _, h = ref_step(model, x, i, j, logv, betas, learn_sigma, eta=0)
            h_dic[i] = h.detach().clone()
        xT.append(x)
        hs.append(torch.cat([h_dic[t] for t in seq[:-1]]))
    xT = torch.cat(xT)
    _, fwd, _, _ = oracle_model(family)
    for k in range(x0.shape[0]):  # the oracle restatement reproduces the reference bit for bit
        xo, ho = oracle_invert_with_h(fwd, x0[k:k + 1], seq, seq_next, learn_sigma)
        assert torch.equal(xo, xT[k:k + 1]) and torch.equal(torch.cat([ho[t] for t in seq[:-1]]), hs[k])
    h0 = torch.cat([model(xT[c:c + 1], torch.ones(1) * seq[-1])[3] for c in range(2)])
    out[f"{family}_x0_sum"] = stats(x0, (1, 2, 3))[0]
    out[f"{family}_xT_sum"], out[f"{family}_xT_absmax"] = stats(xT, (1, 2, 3))
    out[f"{family}_xT_sub"] = sub_x(xT)
    hs = torch.stack(hs)
    out[f"{family}_h_t"] = np.array(seq[:-1])
    out[f"{family}_h_sum"], out[f"{family}_h_absmax"] = stats(hs, (2, 3, 4))
    out[f"{family}_h_c0"] = sub_h(hs[0])
    out[f"{family}_h0_sum"], out[f"{family}_h0_absmax"] = stats(h0, (1, 2, 3))
    out[f"{family}_h0_sub"] = sub_h(h0)
    h_c = [{**{t: hs[c, k:k + 1] for k, t in enumerate(seq[:-1])}, seq[-1]: h0[c:c + 1]} for c in range(2)]
    rows = pair_rows()
    for gi, gamma in enumerate(GAMMAS):
        for use_mask in (False, True):
            noises = golden_noises(gi, use_mask, len(rows), cfg["image_size"], seq)
            x = x_T_rows = torch.cat([xT[2 + s:3 + s] for _, s in rows])
            traj = []
            for i, j in zip(reversed(seq), reversed(seq_next)):
                dh = torch.cat([h_c[c][i] for c, _ in rows])
                orig = torch.randn_like
                ref_du.torch.randn_like = lambda ten, _i=i: noises[_i]
                try:
                    x = ref_step(model, x, i, j, logv, betas, learn_sigma, eta=1.0 if i < T_NOISE else 0.0, index=0,
                                 t_edit=T_EDIT, hs_coeff=(gamma,), delta_h=dh, use_mask=use_mask,
                                 dt_lambda=DT_LAMBDA, dt_end=DT_END)[0]
                finally:
                    ref_du.torch.randn_like = orig
                traj.append(x.clone())
            traj = torch.stack(traj)
            assert torch.equal(traj, oracle_diff_style(fwd, x_T_rows, [h_c[c] for c, _ in rows], seq, seq_next, gamma,
                                                       use_mask, learn_sigma, noises))
            key = f"{family}_traj_g{gi}_m{int(use_mask)}"
            out[key + "_sum"], out[key + "_absmax"] = stats(traj, (2, 3, 4))
            out[key + "_sub"] = sub_x(traj)
    print(f"{family}: |x_0 out| max {out[f'{family}_traj_g0_m0_absmax'][-1].max():.3f}")


if __name__ == "__main__":
    out = {}
    for fam in ("ddpm", "adm"):
        family_fixture(fam, out)
    seq, _ = o_smp.make_sequences(999, N_STEP)
    np.savez_compressed(os.path.join(HERE, "diff_style_mini.npz"), seq=np.array(seq), t_edit=np.array(T_EDIT),
                        t_noise=np.array(T_NOISE), dt_lambda=np.array(DT_LAMBDA), dt_end=np.array(DT_END),
                        gammas=np.array(GAMMAS), noise_seed=np.array(NOISE_SEED), **out)
    print("diff_style_mini.npz written")
