"""--exact_inversion on the GPU: the anchored DDIM update (bit for bit against an fp32 restatement on both forms, B in
{1, 2, 3}, HW % 4 zero and not, Ce in {Cx, 2 Cx}, x0_out, in place, the no-edit identity, refusals, a launch past 2^31
elements), the anchors of mini DDPM / mini ADM / CelebA 256² (A[0] = the plain inversion, A = its recorded states,
E = forward()), anchored passes that do not edit (they record A[1:] and return x0), edits (graph = eager, rows = batch-1
runs, the fp64 oracle), regions, and `--run_test --exact_inversion` end to end."""
import csv
import ctypes
import math
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, face_parsing, main as cli, modules, ops, region, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.inversion import Anchors, reverse_grid
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import adm as oa, ddpm as od, inversion as oi, sampler as osmp

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------------------------
def _f32(v, dev):
    return torch.tensor(v, dtype=torch.float32, device=dev)


def _restated(x, et, em, a_cur, a_next, e_cur, at, an, c2):
    """the three lines in fp32, one torch op per rounding: y, yr, A_next + (y - yr); c2 a scalar or a [N] column"""
    dev = x.device
    N, Cx, B = x.shape[0], x.shape[1], a_cur.shape[0]
    idx = torch.arange(N, device=dev) % B
    one = _f32(1.0, dev)
    sq1, sqa, sqn = (one - _f32(at, dev)).sqrt(), _f32(at, dev).sqrt(), _f32(an, dev).sqrt()
    c2 = c2.view(N, 1, 1, 1) if torch.is_tensor(c2) else _f32(c2, dev)

    def phi(xx, m, e):
        x0 = (xx - m * sq1) / sqa
        return sqn * x0 + c2 * e, x0

    y, x0 = phi(x, em[:, :Cx], et[:, :Cx])
    yr, _ = phi(a_cur[idx], e_cur[idx], e_cur[idx])
    return a_next[idx] + (y - yr), x0


STEP = (0.35, 0.52, 0.61)  # at, an, c2 (fp32 values of a schedule step)


@pytest.mark.parametrize("rows", [False, True])
@pytest.mark.parametrize("B,k", [(1, 3), (2, 2), (3, 2)])
@pytest.mark.parametrize("H,W", [(16, 16), (5, 7)])
@pytest.mark.parametrize("ce2", [False, True])
def test_anchored_update(cuda_device, rows, B, k, H, W, ce2):
    dev = cuda_device
    Cx = 3
    Ce, N = (2 * Cx if ce2 else Cx), B * k
    g = torch.Generator().manual_seed(B * 100 + H + 7 * int(rows) + int(ce2))
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev)  # noqa: E731
    x, et, em = rnd(N, Cx, H, W), rnd(N, Ce, H, W), rnd(N, Ce, H, W)
    a_cur, a_next, e_cur = rnd(B, Cx, H, W), rnd(B, Cx, H, W), rnd(B, Cx, H, W)
    at, an, c2 = (float(np.float32(v)) for v in STEP)
    c12 = None
    if rows:
        c12 = torch.stack([torch.rand(N, generator=g), torch.rand(N, generator=g)], 1).to(dev)
        c2 = c12[:, 1].clone()
    want, want_x0 = _restated(x, et, em, a_cur, a_next, e_cur, at, an, c2)
    out, x0 = torch.empty_like(x), torch.empty_like(x)
    ops.ddim_update_anchored(x, et, em, out, x0, a_cur, a_next, e_cur, at, an, 0.0 if rows else c2, c12=c12)
    assert torch.equal(out, want) and torch.equal(x0, want_x0)
    inplace = x.clone()  # x_next aliasing x, without x0_out
    ops.ddim_update_anchored(inplace, et, em, inplace, None, a_cur, a_next, e_cur, at, an, 0.0 if rows else c2,
                             c12=c12)
    assert torch.equal(inplace, want)
    # a row that does not edit lands on A_next exactly
    idx = torch.arange(N, device=dev) % B
    xs = a_cur[idx].clone()
    es = torch.cat([e_cur[idx], rnd(N, Ce - Cx, H, W)], 1) if ce2 else e_cur[idx].clone()
    ops.ddim_update_anchored(xs, es, es, xs, None, a_cur, a_next, e_cur, at, an, 0.0 if rows else c2, c12=c12)
    assert torch.equal(xs, a_next[idx])
    if rows:  # row n equals the scalar form with its own c2; c1 is not read
        c12[:, 0] = 7.0
        for n in range(N):
            one = torch.empty_like(x[n:n + 1])
            ops.ddim_update_anchored(x[n:n + 1], et[n:n + 1], em[n:n + 1], one, None, a_cur[n % B:n % B + 1],
                                     a_next[n % B:n % B + 1], e_cur[n % B:n % B + 1], at, an, float(c2[n]))
            assert torch.equal(one, out[n:n + 1]), f"row {n}"
        ops.ddim_update_anchored(x, et, em, inplace, None, a_cur, a_next, e_cur, at, an, c12=c12)
        assert torch.equal(inplace, want)


def test_anchored_update_refusals(cuda_device):
    dev = cuda_device
    N, B, C, H, W = 4, 2, 3, 8, 8
    x, e = torch.randn(N, C, H, W, device=dev), torch.randn(N, C, H, W, device=dev)
    a = torch.randn(B, C, H, W, device=dev)
    at, an, c2 = STEP
    call = lambda **kw: ops.ddim_update_anchored(**{**dict(x=x, et=e, em=e, x_next=x.clone(), x0_out=None, a_cur=a,  # noqa: E731
                                                             a_next=a, e_cur=a, at=at, an=an, c2=c2), **kw})
    for kw in ({"a_cur": a[:1].expand(3, C, H, W).contiguous()}, {"e_cur": a.cpu()}, {"et": e.half()},
               {"et": e[:, :2].contiguous()}, {"x_next": x[:2].clone()}, {"c12": torch.zeros(N, 3, device=dev)},
               {"a_next": a[:, :, :4].contiguous()}):
        with pytest.raises(_lib.AsyrpError):
            call(**kw)
    buf = torch.randn(N * C * H * W + 1, device=dev)
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        call(x=buf[1:].view(N, C, H, W))
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        call(x0_out=buf[1:].view(N, C, H, W))
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    out = x.clone()
    before = out.clone()

    def raw(ptrs=None, shape=(N, B, C, C, H * W)):
        p = ptrs or [P(x), P(e), P(e), P(a), P(a), P(a), P(out), None]
        return lib.asyrp_ddim_update_anchored(*p, *shape, at, an, c2, None, s)

    for shape in ((N, 3, C, C, H * W), (0, B, C, C, H * W), (N, 0, C, C, H * W), (N, B, 0, C, H * W),
                  (N, B, C, 2, H * W), (N, B, C, C, 0), (N, B, C, C, -4)):
        assert raw(shape=shape) == -1, shape
    for i in range(7):
        p = [P(x), P(e), P(e), P(a), P(a), P(a), P(out), None]
        p[i] = None
        assert raw(p) == -1, i
    mis = ctypes.c_void_p(a.data_ptr() + 4)
    for i in range(8):
        p = [P(x), P(e), P(e), P(a), P(a), P(a), P(out), P(out)]
        p[i] = mis
        assert raw(p) == -1, i
    torch.cuda.synchronize()
    assert torch.equal(out, before)
    assert raw() == 0
    torch.cuda.synchronize()
    assert torch.equal(out, _restated(x, e, e, a, a, a, at, an, c2)[0])


def test_anchored_update_past_2_31_elements(cuda_device):
    """N Cx HW > 2^31 on the one-element-per-thread path, B = 1: every row but the last does not edit and must give
    A_next; the last row, whose elements lie past 2^31, equals the restatement"""
    dev = cuda_device
    H = W = 255
    Cx, B = 3, 1
    N = (2 ** 31) // (Cx * H * W) + 1
    assert N * Cx * H * W > 2 ** 31
    g = torch.Generator().manual_seed(5)
    a_cur, a_next, e_cur = (torch.randn(B, Cx, H, W, generator=g).to(dev) for _ in range(3))
    x = a_cur.expand(N, Cx, H, W).contiguous()
    e = e_cur.expand(N, Cx, H, W).contiguous()
    x[-1] += torch.randn(Cx, H, W, generator=g).to(dev)
    e[-1] = torch.randn(Cx, H, W, generator=g).to(dev)
    at, an, c2 = STEP
    want, _ = _restated(x[-1:], e[-1:], e[-1:], a_cur, a_next, e_cur, at, an, c2)
    ops.ddim_update_anchored(x, e, e, x, None, a_cur, a_next, e_cur, at, an, c2)
    torch.cuda.synchronize()
    assert torch.equal(x[-1:], want)
    assert torch.equal(x[:-1], a_next.expand(N - 1, Cx, H, W))
    del x, e
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# anchors
# ------------------------------------------------------------------------------------------------------------------
TOL_EPS = 5e-3  # the UNet's eps against the fp64 oracle, relative to max |eps| (as smoke() bounds forward())


def _check_steps(tag, sch, out, rec, want):
    """the engine's anchored steps against the oracle's, each started from the engine's x: an anchored step is linear in
    the UNet's eps with gain sqrt(an) sqrt(1 - at) / sqrt(at) (eps_mod) + c2 (eps), so each step is bounded by that gain
    times the eps tolerance.  Without restarting, the random-weight UNets amplify each step's fp16 error in the next
    evaluation, which no anchoring removes."""
    got = list(rec.cpu().double()) + [out.cpu().double()]
    for k, (s, (w, eps)) in enumerate(zip(sch.steps, want)):
        gain = math.sqrt(s.an) * math.sqrt(1 - s.at) / math.sqrt(s.at) + s.c2
        e = (got[k] - w).abs().max().item()
        print(f"\n{tag} step {k}: max-abs {e:.3e}, bound {gain * TOL_EPS * max(1.0, eps):.3e}")
        assert e <= gain * TOL_EPS * max(1.0, eps), f"{tag} step {k}: {e:.3e}"


def _module(family, cfg=None, style="jittered", n_delta=1):
    if family == "ddpm":
        cfg = cfg or od.MINI_CFG
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
    else:
        m = modules._create_adm(cfg or oa.MINI_HP)
    if n_delta:
        m.setattr_layers(n_delta)
    synthetic.randomize_(m, 1234, style)
    return m


def _anchors_case(eng, x0, n):
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, n)
    inv = Schedule.inversion(betas, seq, seq_next)
    anc = eng.anchors(x0, inv)
    return betas, seq, seq_next, inv, anc


def _check_anchors(eng, x0, n):
    betas, seq, seq_next, inv, anc = _anchors_case(eng, x0, n)
    C = x0.shape[1]
    assert anc.x.shape == (n + 1, *x0.shape) and anc.eps.shape == (n, *x0.shape)
    assert anc.grid == reverse_grid(seq, seq_next)
    assert torch.equal(anc.x[n], x0) and torch.equal(anc.x[n - 1], x0)
    plain = eng.sample(x0, inv, record_process=True)
    rec = eng.last_records["x"].clone()
    assert torch.equal(anc.x[0], plain), "A[0] must be the plain inversion's x_T"
    assert torch.equal(anc.x[:n - 1], rec.flip(0)), "A[0..n-2] must be its recorded states, reversed"
    for k, (t, _) in enumerate(anc.grid):
        et = eng.forward(anc.x[k], torch.full((x0.shape[0],), float(t), device=x0.device))[0]
        assert torch.equal(anc.eps[k], et[:, :C]), f"E[{k}] (t = {t})"
    # a second call replays the same graph and returns copies
    n_graphs = len(eng.graphs)
    again = eng.anchors(x0, inv)
    assert len(eng.graphs) == n_graphs and torch.equal(again.x, anc.x) and torch.equal(again.eps, anc.eps)
    assert again.x.data_ptr() != anc.x.data_ptr()
    assert eng.last_launches == n * len(eng.plan(x0.shape[0]).launches(False, temb=False)) + n - 1
    return betas, seq, seq_next, anc


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_mini_anchors(cuda_device, family):
    m = _module(family).to(cuda_device)
    S = m.engine.arch.image_size
    x0 = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(2)).clamp(-1, 1).to(cuda_device)
    _check_anchors(m.engine, x0, 6)


def _identity(eng, anc, betas, seq, seq_next, B, learn_sigma):
    """anchored passes that do not edit record A[1:] and return x0: edit=False with t_addnoise > 0, a DeltaBlock
    (1, 0), and a per-row schedule whose rows have different t_addnoise"""
    n = len(anc.grid)
    x0 = anc.x0
    for sch in (Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=400, hs_coeff=(1.0,), edit=False),
                Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0,), edit=False)):
        out = eng.sample(anc.x_T, sch, anchors=anc, record_process=True)
        assert torch.equal(out, x0)
        assert torch.equal(eng.last_records["x"], anc.ref)
    rows = RowSchedule(betas, seq, seq_next, t_edit=[500] * (2 * B), t_addnoise=[0, 400, 700, 300, 200, 0][:2 * B],
                       hs_coeffs=[(1.0, 0.0)] * (2 * B))
    assert len({s.stochastic for s in rows.steps}) == 2
    out = eng.sample(anc.x_T.repeat(2, 1, 1, 1), rows, anchors=anc, record_process=True)
    assert torch.equal(out, x0.repeat(2, 1, 1, 1))
    assert torch.equal(eng.last_records["x"], anc.ref.repeat(1, 2, 1, 1, 1))
    # a DeltaBlock (1, 0) edits with h2 = 1 h + 0 delta = h bit for bit, but the edited decoder's GroupNorm sums come
    # from the DeltaBlock epilogue (over the fp16 h2) rather than from h's producer (over its fp32 values before
    # rounding): eps_mod differs from eps in the last bits, so such a row is close to the anchors, not equal
    P = eng.plan(B)
    for k, (t, _) in enumerate(anc.grid):
        et, em, _, _ = eng.forward(anc.x[k], torch.full((B,), float(t), device=x0.device), index=0, t_edit=0,
                                   hs_coeff=(1.0, 0.0))
        assert torch.equal(P.h2.t, P.middle_h.t), f"step {k}: h2 must be h"
        e, mx = (em - et).abs().max().item(), et.abs().max().item()
        print(f"\nDeltaBlock (1, 0) step {k}: |eps_mod - eps| {e:.3e} of {mx:.3e}, GroupNorm sums equal: "
              f"{torch.equal(P.h2.stats, P.middle_h.stats)}")
        assert e <= 5e-3 * max(1.0, mx)
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 0.0))
    out = eng.sample(anc.x_T, sch, anchors=anc)
    print(f"DeltaBlock (1, 0) trajectory: max-abs {(out - x0).abs().max().item():.3e} from x0 (n = {n})")
    return out


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_mini_identity_and_edits(cuda_device, family):
    dev = cuda_device
    m = _module(family)
    sd = {k_: v.cpu() for k_, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    learn_sigma = family == "adm"
    S, B, n = eng.arch.image_size, 2, 6
    x0 = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(4)).clamp(-1, 1).to(dev)
    betas, seq, seq_next, inv, anc = _anchors_case(eng, x0, n)
    _identity(eng, anc, betas, seq, seq_next, B, learn_sigma)  # the mini UNets amplify the (1, 0) row's last bits
    # edits: graph = eager, rows = batch-1 runs, not x0, the launch count of the plain pass, the fp64 oracle
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(1.0, 1.0))
    out = eng.sample(anc.x_T, sch, anchors=anc)
    launches = eng.last_launches
    eng.sample(anc.x_T, sch, noise=torch.zeros(sch.n_stochastic, *x0.shape, device=dev))
    assert eng.last_launches == launches, "anchoring must not change the launch count"
    assert not torch.equal(out, x0)
    assert torch.equal(eng.sample(anc.x_T, sch, anchors=anc, use_graph=False), out), "graph vs eager"
    coefs = [(1.0, 1.0), (1.0, 0.5), (0.9, 1.5)]
    table = torch.tensor([c for c in coefs for _ in range(B)])
    rows = eng.sample(anc.x_T.repeat(3, 1, 1, 1), sch, anchors=anc, hs_coeffs=table)
    for r in range(3 * B):
        b = r % B
        one = eng.sample(anc.x_T[b:b + 1], sch, anchors=anc.images(b, b + 1, 1), hs_coeffs=table[r:r + 1])
        assert torch.equal(rows[r:r + 1], one), f"row {r}"
    fwd = (lambda *a, **k: od.ddpm_forward(sd, od.MINI_CFG, *a, **k)) if family == "ddpm" else \
        (lambda *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k))
    eng.sample(anc.x_T, sch, anchors=anc, record_process=True)
    rec = eng.last_records["x"][:-1].clone()
    want = oi.run_anchored_trajectory(fwd, anc.x.cpu(), anc.eps.cpu(), betas=betas, seq=seq, seq_next=seq_next,
                                      t_edit=500, t_addnoise=300, index=0, hs_coeff=(1.0, 1.0),
                                      learn_sigma=learn_sigma, xs=rec.cpu())
    _check_steps(family, sch, out, rec, want)
    # per-row schedules, h directions and regions
    rs = RowSchedule(betas, seq, seq_next, t_edit=[500, 400, 500, 400], t_addnoise=[0, 300, 200, 0],
                     hs_coeffs=[(1.0, 1.0)] * 4)
    ro = eng.sample(anc.x_T.repeat(2, 1, 1, 1), rs, anchors=anc)
    assert torch.equal(eng.sample(anc.x_T.repeat(2, 1, 1, 1), rs, anchors=anc, use_graph=False), ro)
    mask = (torch.rand(B, S, S, generator=torch.Generator().manual_seed(8)) > 0.5).float().to(dev)
    bl = eng.sample(anc.x_T, sch, anchors=anc, blend=(mask, anc.ref))
    keep = (mask == 0)[:, None].expand_as(bl)
    assert torch.equal(bl[keep], x0[keep]) and not torch.equal(bl, x0)
    masks = torch.stack([mask, 1 - mask]) * 0.5
    masks[0] = mask
    masks[1] = (1 - mask) * (torch.arange(S, device=dev) < S // 2).float()
    co = eng.sample(anc.x_T.repeat(2, 1, 1, 1), rs, anchors=anc, compose=(masks, anc.ref))
    zero = (masks.sum(0) == 0)[:, None].expand(B, 3, S, S)
    for k_ in range(2):
        assert torch.equal(co[k_ * B:(k_ + 1) * B][zero], x0[zero])
    # refusals
    with pytest.raises(_lib.AsyrpError, match="noise"):
        eng.sample(anc.x_T, sch, anchors=anc, noise=torch.zeros(sch.n_stochastic, *x0.shape, device=dev))
    with pytest.raises(_lib.AsyrpError, match="grid"):
        eng.sample(anc.x_T, Schedule(betas, *make_sequences(999, 5), t_edit=500), anchors=anc)
    with pytest.raises(_lib.AsyrpError, match="multiple"):
        eng.sample(anc.x_T[:1].repeat(3, 1, 1, 1), sch, anchors=anc)
    with pytest.raises(_lib.AsyrpError, match="DDIM"):
        eng.sample(anc.x_T, Schedule(betas, seq, seq_next, t_edit=500, sample_type="ddpm",
                                     logvars=None if learn_sigma else torch.ones(1000)), anchors=anc)
    with pytest.raises(_lib.AsyrpError, match="lpips"):
        eng.sample(anc.x_T, sch, anchors=anc, lpips=object())
    with pytest.raises(_lib.AsyrpError):
        eng.sample(anc.x_T, sch, anchors=Anchors(anc.x.cpu(), anc.eps.cpu(), anc.grid))


def test_mini_h_direction_identity(cuda_device):
    """an --h_direction α = 0 row (h2 = 1 h + 0 d) anchored: report its distance from x0; α != 0 edits; graph = eager"""
    dev = cuda_device
    m = _module("ddpm", n_delta=0).to(dev)
    eng = m.engine
    S, B, n = eng.arch.image_size, 2, 6
    x0 = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(6)).clamp(-1, 1).to(dev)
    betas, seq, seq_next, inv, anc = _anchors_case(eng, x0, n)
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 0.0))
    n_edit = sum(1 for s in sch.steps if s.edit)
    D = torch.randn(n_edit, *eng.plan(B).dh_user.shape[1:], generator=torch.Generator().manual_seed(1)).to(dev)
    # h2 = fmaf(0, d, 1 h) = h, with add_h_rows' own GroupNorm sums: close to the anchors, as a DeltaBlock (1, 0)
    out = eng.sample(anc.x_T, sch, anchors=anc, h_direction=D, hs_coeffs=torch.tensor([[1.0, 0.0]] * B))
    print(f"\nh_direction α = 0: max-abs {(out - x0).abs().max().item():.3e} from x0")
    moved = eng.sample(anc.x_T, sch, anchors=anc, h_direction=D, hs_coeffs=torch.tensor([[1.0, 2.0]] * B))
    assert not torch.equal(moved, x0)
    assert torch.equal(eng.sample(anc.x_T, sch, anchors=anc, h_direction=D, hs_coeffs=torch.tensor([[1.0, 2.0]] * B),
                                  use_graph=False), moved)


def test_celeba256_anchors_and_edits(cuda_device):
    dev = cuda_device
    m = _module("ddpm", od.CELEBA_CFG, style="torch_default")
    sd = {k_: v.cpu() for k_, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    S, B, n = 256, 2, 4
    x0 = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(12)).clamp(-1, 1).to(dev)
    betas, seq, seq_next, anc = _check_anchors(eng, x0, n)
    _identity(eng, anc, betas, seq, seq_next, B, False)
    sch = Schedule(betas, seq, seq_next, t_edit=400, t_addnoise=0, hs_coeff=(1.0, 1.0))
    out = eng.sample(anc.x_T, sch, anchors=anc)
    assert not torch.equal(out, x0)
    assert torch.equal(eng.sample(anc.x_T, sch, anchors=anc, use_graph=False), out)
    mask = region.masks_from_labels(torch.randint(0, 19, (B, 512, 512), dtype=torch.uint8).to(dev), [17, 1], S, 0,
                                    0.0)
    bl = eng.sample(anc.x_T, sch, anchors=anc, blend=(mask, anc.ref))
    keep = (mask == 0)[:, None].expand_as(bl)
    assert torch.equal(bl[keep], x0[keep])
    eng.sample(anc.x_T, sch, anchors=anc, record_process=True)
    rec, A, E = eng.last_records["x"][:-1].cpu(), anc.x.cpu(), anc.eps.cpu()
    del m, eng, anc
    torch.cuda.empty_cache()
    fwd = lambda *a, **k: od.ddpm_forward(sd, od.CELEBA_CFG, *a, **k)  # noqa: E731
    want = oi.run_anchored_trajectory(fwd, A, E, betas=betas, seq=seq, seq_next=seq_next, t_edit=400, index=0,
                                      hs_coeff=(1.0, 1.0), xs=rec)
    _check_steps("celeba256", sch, out, rec, want)


# ------------------------------------------------------------------------------------------------------------------
# end to end (DDPM CelebA-HQ 256², synthetic weights, generated PNGs)
# ------------------------------------------------------------------------------------------------------------------
BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/ei", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--user_defined_t_edit", "500", "--user_defined_t_addnoise",
        "300", "--synthetic_weights", "--seed", "1234", "--train_delta_block", "--get_h_num", "1",
        "--custom_test_dataset_dir", "faces", "--custom_train_dataset_dir", "faces", "--exact_inversion",
        "--save_x_origin", "--max_rows_per_replay", "4"]
EDIT = ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]


def _faces(n, S):
    from PIL import Image
    os.makedirs("faces")
    g = torch.Generator().manual_seed(21)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, S), torch.linspace(0, 1, S), indexing="ij")
    for i in range(n):
        base = torch.stack([torch.sin(5 * xx + 3 * c * yy + i) * torch.cos(4 * yy + c) for c in range(3)])
        x = (0.7 * base + 0.2 * torch.randn(3, S, S, generator=g)).clamp(-1, 1)
        Image.fromarray(((x + 1) * 127.5).round().byte().permute(1, 2, 0).numpy()).save(f"faces/{i}.png")


def _setup(tmp_path, monkeypatch):
    from test_seg_consistency_gpu import _delta_block_ckpt
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)
    torch.save(synthetic.face_parsing_state_dict(seed=5), "79999_iter.pth")
    _faces(2, 256)


def _run(argv, dev):
    args, cfg = cli.parse_args_and_config(argv)
    r = Asyrp(args, cfg, device=dev)
    return r, r.run_test()


def test_run_test_exact_inversion_end_to_end(cuda_device, tmp_path, monkeypatch):
    from asyrp_official_b200.diffusion_latent import _load_image_folder
    _setup(tmp_path, monkeypatch)
    x0 = torch.cat(_load_image_folder("faces", 256, 2))
    r, res = _run(BASE + EDIT + ["--content_preservation", "--delta_interpolation", "--num_delta", "3", "--min_delta",
                                 "0.5", "--max_delta", "1.5"], cuda_device)
    rows = res[("test", 1)]
    assert len(rows) == 4 and torch.equal(rows[0], x0), "the origin row is the input image"
    assert all(not torch.equal(e, x0) for e in rows[1:])
    rec = r.reconstruction["test_1_0"]
    print(f"\norigin vs input: {rec.tolist()}")
    assert bool(torch.isinf(rec[:, 0]).all()) and bool((rec[:, 1] == 1).all()) and bool((rec[:, 2] == 1).all()) \
        and bool((rec[:, 3] == 0).all())
    with open(os.path.join(r.args.test_image_folder, "test_1_0_ngen4_content_preservation.tsv")) as f:
        table = list(csv.reader(f, delimiter="\t"))
    assert [t[1] for t in table[1:3]] == ["origin", "origin"] and len(table) == 1 + 2 + 3 * 2
    # the anchors the run used: rows equal the engine's anchored pass on them
    seg = ["--seg_weights", "79999_iter.pth"]
    parser = face_parsing.FaceParser(torch.load("79999_iter.pth", weights_only=True), device=cuda_device)
    mask = region.region_masks(parser, x0, [17], 1, 0.0).cpu()
    print(f"\nmask covers {mask.mean().item():.3f} of the image")
    out = (mask == 0)[:, None].expand(2, 3, 256, 256)
    _, res = _run(BASE + EDIT + ["--edit_region", "hair", "--edit_region_dilate", "1"] + seg, cuda_device)
    for e in res[("test", 1)][1:]:
        assert torch.equal(e[out], x0[out])
    _, res = _run(BASE + ["--attr_sweep", "smiling angry", "--manual_checkpoint_name", "attribute_0.pth"],
                  cuda_device)
    sweep = res[("test", 1)]
    assert len(sweep) == 3 and torch.equal(sweep[0], x0) and all(not torch.equal(e, x0) for e in sweep[1:])
    _, res = _run(BASE + ["--region_compose", "smiling=mouth,u_lip,l_lip angry=hair", "--manual_checkpoint_name",
                          "attribute_0.pth"] + seg, cuda_device)
    comp = res[("test", 1)]
    masks = region.compose_masks(parser, x0, [[11, 12, 13], [17]], 0, 0.0).cpu()
    zero = (masks.sum(0) == 0)[:, None].expand(2, 3, 256, 256)
    assert torch.equal(comp[0], x0) and torch.equal(comp[-1][zero], x0[zero])
