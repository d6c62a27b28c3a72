"""Exact inversion (--exact_inversion): the anchors of a batch of input images.

A DDIM inversion of x0 followed by the unedited reverse pass from its x_T does not return x0: the reverse steps are not
the inverse of the inversion steps.  The anchored reverse step (ops.ddim_update_anchored) removes that drift.  It moves
each row from the inversion's own state at the next timestep by the difference between the row's update and the same
update applied to the inversion's state at this timestep (Direct Inversion, Ju et al., ICLR 2024, written as a
difference so that an unedited row is exact):

    x_{k+1} = A[k+1] + (Phi_k(x_k, eps_mod, eps) - Phi_k(A[k], E[k], E[k]))

With the reverse grid t_0 > t_1 > .. > t_{n-1} = 0 (t_n = -1) of make_sequences(t_0, n):
  A  fp32 [n + 1][B][C][S][S]  A[k] the inversion's state at t_k, A[0] = x_T, A[n - 1] = A[n] = x0 (the input)
  E  fp32 [n][B][C][S][S]      E[k] the plain UNet's eps (channels [0, C)) at (A[k], t_k)
A row that does not edit therefore reproduces A step by step and ends on x0, bit for bit.
"""
from dataclasses import dataclass
from typing import Tuple

import torch

from . import ops


@dataclass
class Anchors:
    """the anchors of B images (UNetEngine.anchors): x = A, eps = E, grid = the (t, t_next) of every reverse step"""
    x: torch.Tensor
    eps: torch.Tensor
    grid: Tuple[Tuple[int, int], ...]

    @property
    def B(self):
        return self.x.shape[1]

    @property
    def x_T(self):
        return self.x[0]

    @property
    def x0(self):
        return self.x[-1]

    @property
    def ref(self):
        """the anchored pass's x after every step, [n][B][C][S][S]: the reference of blend= and compose="""
        return self.x[1:]

    def check(self, schedule, N):
        """AsyrpError unless schedule (a Schedule or RowSchedule of N rows) can be anchored to these anchors: the
        same step grid, DDIM steps only, N a multiple of B"""
        grid = tuple((int(s.t), int(s.t_next)) for s in schedule.steps)
        if grid != tuple(self.grid):
            raise ops._lib.AsyrpError(f"anchors: the schedule's step grid {list(grid)} is not the anchors' grid "
                                      f"{list(self.grid)}")
        if any(s.kind != "ddim" for s in schedule.steps):
            raise ops._lib.AsyrpError("anchors: every step must be a DDIM step ('ddpm' sampling has no anchored form)")
        n = len(grid)
        if self.x.dim() != 5 or self.x.shape[0] != n + 1 or tuple(self.eps.shape) != (n, *self.x.shape[1:]):
            raise ops._lib.AsyrpError(f"anchors: x must be [{n + 1}][B][C][S][S] and eps [{n}][B][C][S][S], got "
                                      f"{tuple(self.x.shape)} and {tuple(self.eps.shape)}")
        if N % self.B:
            raise ops._lib.AsyrpError(f"anchors: the batch of {N} rows is not a multiple of the {self.B} anchored images")

    def images(self, j0, j1, b):
        """the anchors of images [j0, j1), padded to b images by repeating the last one (as pad_rows pads rows)"""
        def pad(t):
            t = t[:, j0:j1]
            if t.shape[1] < b:
                t = torch.cat([t, t[:, -1:].expand(t.shape[0], b - t.shape[1], *t.shape[2:])], dim=1)
            return t
        return Anchors(pad(self.x), pad(self.eps), self.grid)


def reverse_grid(seq, seq_next):
    """the (t, t_next) of every reverse step of make_sequences' grid, in the order the steps run"""
    return tuple((int(i), int(j)) for i, j in zip(reversed(seq), reversed(seq_next)))
