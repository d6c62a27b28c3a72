"""Host-side schedule of one Asyrp reverse trajectory.

Everything the reference decides per step with device->host synchronisations — `t[0] >= t_edit`
(models/ddpm/diffusion.py:510), `t[0] < t_addnoise` (diffusion_latent.py:513), `t_next.sum() == -bs`
(utils/diffusion_utils.py:68) and the alpha-bar lookups (:66-71) — is an integer/float decision made here, once,
before the trajectory graph is captured.
"""
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np
import torch


@dataclass(frozen=True)
class Step:
    t: int
    t_next: int
    edit: bool     # t >= t_edit: DeltaBlock injection + second decoder pass
    at: float      # alpha-bar_t       (fp32 value)
    an: float      # alpha-bar_t_next  (1.0 when t_next == -1)
    c1: float      # coefficient of the injected noise (0 for eta = 0)
    c2: float      # coefficient of e_t: sqrt(1-an) for eta = 0
    kind: str = "ddim"     # 'ddpm': ancestral step (utils/diffusion_utils.py:74-82), uses bt / logvar / mask below
    bt: float = 0.0
    logvar: float = 0.0    # fixed-variance table entry (ignored when the UNet predicts the variance)
    mask: float = 1.0      # 0 at t == 0: no noise on the last ancestral step

    @property
    def stochastic(self):
        return self.kind == "ddpm" or self.c1 != 0.0


def make_sequences(t_0=999, n_step=40):
    """seq_test, seq_test_next  (diffusion_latent.py:570-574)"""
    seq = [int(s + 1e-6) for s in list(np.linspace(0, 1, n_step) * t_0)]
    return seq, [-1] + list(seq[:-1])


class Schedule:
    def __init__(self, betas, seq, seq_next, t_edit, t_addnoise=0, hs_coeff=(1.0, 1.0), edit=True, pairs=None,
                 sample_type="ddim", dt_lambda=1.0, dt_end=999, ignore_timestep=False, logvars=None):
        """betas: fp32 tensor (Asyrp.betas).  Coefficients are evaluated with the same fp32 torch expressions as
        utils/diffusion_utils.py:66-100 (cumprod in fp32 on the host) so that they are bit-identical to the CPU oracle.

        sample_type / dt_lambda / dt_end / ignore_timestep: what save_image forwards to denoising_step on every step
        (diffusion_latent.py:507-520; it never passes dt_end, i.e. 999).  logvars: Asyrp.logvar, needed by 'ddpm'
        sampling with a fixed-variance model."""
        if sample_type not in ("ddim", "ddpm"):
            raise ValueError(f"unknown sample_type {sample_type!r}")
        b = torch.as_tensor(betas, dtype=torch.float32).cpu()
        ac = (1.0 - b).cumprod(dim=0)
        lv = None if logvars is None else torch.as_tensor(logvars, dtype=torch.float32)
        steps: List[Step] = []
        for i, j in (pairs if pairs is not None else zip(reversed(seq), reversed(seq_next))):
            at = ac[i]
            an = torch.ones_like(at) if j == -1 else ac[j]
            eta = 1.0 if i < t_addnoise else 0.0
            if eta == 0.0:
                c1 = torch.zeros_like(at)
                c2 = (1 - an).sqrt()
            else:
                c1 = eta * ((1 - at / an) * (1 - an) / (1 - at)).sqrt()
                c2 = ((1 - an) - c1 ** 2).sqrt()
            if sample_type == "ddpm":
                if dt_lambda != 1 and i >= dt_end:
                    raise ValueError("sample_type='ddpm' with dt_lambda != 1 at t >= dt_end is undefined in the "
                                     "reference (x0_t is not computed on that branch, utils/diffusion_utils.py:99)")
                steps.append(Step(int(i), int(j), bool(edit and i >= t_edit), float(at), float(an), 0.0, 0.0, "ddpm",
                                  float(b[i]), 0.0 if lv is None else float(lv[i]), 0.0 if i == 0 else 1.0))
                continue
            if dt_lambda != 1 and i >= dt_end:  # :99-100 overrides whatever the eta branch produced
                c1 = torch.zeros_like(at)
                c2 = (1 - an).sqrt() * dt_lambda
            steps.append(Step(int(i), int(j), bool(edit and i >= t_edit), float(at), float(an), float(c1), float(c2)))
        self.steps = steps
        self.hs_coeff: Tuple[float, ...] = tuple(float(c) for c in hs_coeff)
        self.t_edit, self.t_addnoise = t_edit, t_addnoise
        self.ignore_timestep = bool(ignore_timestep)

    @classmethod
    def inversion(cls, betas, seq, seq_next):
        """DDIM inversion x_0 -> x_T: the deterministic step applied with t < t_next, plain UNet (index=None)
        (precompute_pairs, diffusion_latent.py:1032-1044: zip(seq_inv_next[1:], seq_inv[1:]))"""
        return cls(betas, None, None, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False,
                   pairs=list(zip(seq_next[1:], seq[1:])))

    def key(self):
        """identifies the captured graph: the DeltaBlock coefficients are device-side parameters, not part of it"""
        return (tuple(self.steps), self.ignore_timestep, len(self.hs_coeff))

    @property
    def n_stochastic(self):
        return sum(1 for s in self.steps if s.stochastic)

    @property
    def n_edit(self):
        return sum(1 for s in self.steps if s.edit)


@dataclass(frozen=True)
class RowStep:
    """one step of a RowSchedule: what the whole batch shares, and which rows edit"""
    t: int
    t_next: int
    at: float
    an: float
    edit_rows: Tuple[bool, ...]   # row n edits at this step: t >= t_edit[n] and its coefficients are not (1, 0, ..)
    stochastic: bool              # any row has eta = 1 at this step (c1 != 0)
    kind: str = "ddim"

    @property
    def edit(self):
        return any(self.edit_rows)


class RowSchedule:
    """A trajectory whose rows follow their own schedules: row n is the single-row
    Schedule(betas, seq, seq_next, t_edit[n], t_addnoise[n], hs_coeffs[n], ...).  The step list (t, t_next, alpha-bars)
    is the same for every row; what differs per row lives in tables:

      c         fp32 [steps][N][2]        (c1, c2) of each row, the values of its own Schedule
      coeffs    fp32 [steps][N][1 + K]    DeltaBlock coefficients: hs_coeffs[n] while the row edits, (1, 0, .., 0)
                                          below its t_edit (h2 = h, the reference's t[0] < t_edit branch)

    A step edits when any row edits and is stochastic when any row has eta = 1.  'ddpm' sampling is refused: its
    ancestral step has no per-row form here."""

    def __init__(self, betas, seq, seq_next, t_edit, t_addnoise, hs_coeffs, sample_type="ddim", dt_lambda=1.0,
                 dt_end=999, ignore_timestep=False, logvars=None):
        if sample_type != "ddim":
            raise ValueError(f"a per-row schedule needs sample_type 'ddim', got {sample_type!r}")
        t_edit, t_addnoise = [int(v) for v in t_edit], [int(v) for v in t_addnoise]
        coeffs = [tuple(float(c) for c in row) for row in hs_coeffs]
        N = len(t_edit)
        if not N or len(t_addnoise) != N or len(coeffs) != N:
            raise ValueError(f"t_edit, t_addnoise and hs_coeffs need one entry per row, got {len(t_edit)}, "
                             f"{len(t_addnoise)} and {len(coeffs)}")
        if len({len(r) for r in coeffs}) != 1 or len(coeffs[0]) < 1:
            raise ValueError("every row of hs_coeffs needs the same length 1 + K")
        self.rows = [Schedule(betas, seq, seq_next, t_edit=t_edit[n], t_addnoise=t_addnoise[n], hs_coeff=coeffs[n],
                              sample_type="ddim", dt_lambda=dt_lambda, dt_end=dt_end, ignore_timestep=ignore_timestep,
                              logvars=logvars) for n in range(N)]
        K1 = len(coeffs[0])
        gate = (1.0,) + (0.0,) * (K1 - 1)
        steps: List[RowStep] = []
        c = torch.zeros(len(self.rows[0].steps), N, 2, dtype=torch.float32)
        co = torch.zeros(len(self.rows[0].steps), N, K1, dtype=torch.float32)
        for k, row_steps in enumerate(zip(*(r.steps for r in self.rows))):
            s0 = row_steps[0]
            edit_rows = []
            for n, s in enumerate(row_steps):
                c[k, n, 0], c[k, n, 1] = s.c1, s.c2
                co[k, n] = torch.tensor(coeffs[n] if s.edit else gate, dtype=torch.float32)
                edit_rows.append(bool(s.edit) and tuple(co[k, n].tolist()) != gate)
            steps.append(RowStep(s0.t, s0.t_next, s0.at, s0.an, tuple(edit_rows), any(s.stochastic for s in row_steps)))
        self.steps = steps
        self.c, self.coeffs = c, co
        self.t_edit, self.t_addnoise, self.hs_coeffs = t_edit, t_addnoise, coeffs
        self.ignore_timestep = bool(ignore_timestep)

    @property
    def N(self):
        return len(self.rows)

    @property
    def n_delta(self):
        return self.coeffs.shape[2] - 1

    def key(self):
        """identifies the captured graph: the step list and which rows edit where; (c1, c2) and the DeltaBlock
        coefficients are device-side tables, filled before every replay"""
        return ("rows", tuple(self.steps), self.ignore_timestep, self.n_delta)

    @property
    def n_stochastic(self):
        return sum(1 for s in self.steps if s.stochastic)

    @property
    def n_edit(self):
        return sum(1 for s in self.steps if s.edit)

    def noise_rows(self, n, noise):
        """the noise a row's own Schedule consumes, [its n_stochastic][1][...], taken from a RowSchedule noise tensor
        [n_stochastic][N][...]: the entries of the steps at which row n is stochastic"""
        ks = [k for k, s in enumerate(self.steps) if s.stochastic]
        return noise[[zi for zi, k in enumerate(ks) if self.rows[n].steps[k].stochastic], n:n + 1]
