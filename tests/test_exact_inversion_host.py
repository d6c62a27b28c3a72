"""--exact_inversion on the host: every refusal before a model loads, the exported C-ABI symbol, oracle/inversion.py's
anchored step on hand cases, the Anchors grid check, and save_image's wiring with a stub engine: without the flag it
makes the calls it made before, with it no origin pass runs and every edit pass is anchored.  No GPU needed."""
import ctypes
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, main as cli, region
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.inversion import Anchors, reverse_grid
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import inversion as oi, sampler as osmp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = ["--config", "celeba.yml", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0"]


# ------------------------------------------------------------------------------------------------------------------
# refusals before any model loads
# ------------------------------------------------------------------------------------------------------------------
def _no_model(monkeypatch):
    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)


def test_flag_refusals(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    _no_model(monkeypatch)
    ok = BASE + ["--run_test", "--exact_inversion"]
    cases = [(ok + ["--load_random_noise"], "with --load_random_noise"),
             (ok + ["--saved_random_noise"], "with --saved_random_noise"),
             (ok + ["--n_test_step", "20"], "--n_test_step equal to --n_inv_step"),
             (ok + ["--n_inv_step", "20"], "--n_test_step equal to --n_inv_step"),
             (ok + ["--sample_type", "ddpm"], "with --sample_type ddpm"),
             (ok + ["--origin_process_addnoise"], "with --origin_process_addnoise"),
             (ok + ["--save_process_origin"], "with --save_process_origin"),
             (ok + ["--lpips"], "with --lpips"),
             (ok + ["--num_mean_of_delta_hs", "2"], "with --num_mean_of_delta_hs"),
             (ok + ["--attr_sweep", "smiling young", "--load_random_noise"], "with --load_random_noise")]
    for argv, match in cases:
        args, cfg = cli.parse_args_and_config(argv)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    # outside --run_test, and in the other modes
    args, cfg = cli.parse_args_and_config(BASE + ["--lpips", "--exact_inversion"])
    with pytest.raises(ValueError, match="add --run_test"):
        Asyrp(args, cfg, device="cpu").compute_lpips_distance()
    for flag, run in (("--diff_style", "run_diff_style"), ("--h_directions", "run_h_directions"),
                      ("--lpips", "compute_lpips_distance")):
        args, cfg = cli.parse_args_and_config(ok + [flag])
        with pytest.raises(ValueError, match=f"with {flag}"):
            getattr(Asyrp(args, cfg, device="cpu"), run)()
        assert cli.main(ok + [flag]) == 1
    # accepted, and off without the flag
    args, cfg = cli.parse_args_and_config(ok + ["--user_defined_t_addnoise", "300"])
    assert Asyrp(args, cfg, device="cpu").exact_inversion_setup() is True
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test", "--load_random_noise"])
    assert Asyrp(args, cfg, device="cpu").exact_inversion_setup() is False


# ------------------------------------------------------------------------------------------------------------------
# symbol
# ------------------------------------------------------------------------------------------------------------------
def test_symbol_is_declared_and_exported():
    name = "asyrp_ddim_update_anchored"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "asyrp_b200.h")).read()
    assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert f"int {name}(" in header


# ------------------------------------------------------------------------------------------------------------------
# the oracle on hand cases
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_anchored_step_by_hand():
    g = np.random.default_rng(0)
    a, ea, a_next = g.normal(size=(2, 3, 4, 4)), g.normal(size=(2, 3, 4, 4)), g.normal(size=(2, 3, 4, 4))
    at, an, c2 = 0.3, 0.6, 0.5
    # a row that does not edit lands on A[k+1]
    assert np.array_equal(oi.anchored_step(a, ea, ea, a, ea, a_next, at, an, c2), a_next)
    # an edit moves by the difference of the two updates: eps_mod shifted by d moves x by -sqrt(an (1 - at) / at) d
    d = 0.25
    out = oi.anchored_step(a, ea + d, ea, a, ea, a_next, at, an, c2)
    np.testing.assert_allclose(out - a_next, -np.sqrt(an) * np.sqrt(1 - at) / np.sqrt(at) * d, rtol=1e-12)
    out = oi.anchored_step(a + d, ea, ea, a, ea, a_next, at, an, c2)  # x shifted: sqrt(an / at) d
    np.testing.assert_allclose(out - a_next, np.sqrt(an / at) * d, rtol=1e-12)
    out = oi.anchored_step(a, ea, ea + d, a, ea, a_next, at, an, c2)  # eps shifted: c2 d
    np.testing.assert_allclose(out - a_next, c2 * d, rtol=1e-12)


def test_oracle_trajectory_that_does_not_edit_returns_x0():
    """with E the stand-in model's eps along A, an unedited anchored loop ends on A[n] whatever A is"""
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 4)
    grid = reverse_grid(seq, seq_next)

    def model(x, t, **k):
        e = 0.1 * x + 0.01 * t.view(-1, 1, 1, 1) / 1000
        return e, e, None, None

    g = torch.Generator().manual_seed(0)
    A = torch.randn(5, 2, 3, 4, 4, generator=g)
    A[4] = A[3]
    E = torch.stack([model(A[k], torch.full((2,), float(t)))[0] for k, (t, _) in enumerate(grid)])
    for t_addnoise in (0, 700):
        x = oi.run_anchored_trajectory(model, A, E, betas=betas, seq=seq, seq_next=seq_next, t_edit=10 ** 9,
                                       t_addnoise=t_addnoise, index=None)
        torch.testing.assert_close(x, A[4].double(), rtol=0, atol=1e-12)
        steps = oi.run_anchored_trajectory(model, A, E, betas=betas, seq=seq, seq_next=seq_next, t_edit=10 ** 9,
                                           t_addnoise=t_addnoise, index=None, xs=A[1:4])
        assert len(steps) == 4
        for k, (xk, eps) in enumerate(steps):
            torch.testing.assert_close(xk, A[k + 1].double(), rtol=0, atol=1e-12)
            assert eps > 0


# ------------------------------------------------------------------------------------------------------------------
# the Anchors type
# ------------------------------------------------------------------------------------------------------------------
def test_anchors_grid_check():
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 5)
    grid = reverse_grid(seq, seq_next)
    assert grid[0] == (999, 749) and grid[-1] == (0, -1) and len(grid) == 5
    B, n = 2, 5
    anc = Anchors(torch.zeros(n + 1, B, 3, 4, 4), torch.zeros(n, B, 3, 4, 4), grid)
    assert anc.B == 2 and anc.x_T.shape == (B, 3, 4, 4) and anc.ref.shape == (n, B, 3, 4, 4)
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=500)
    anc.check(sch, 4)
    anc.check(RowSchedule(betas, seq, seq_next, [500] * 4, [0, 300, 0, 200], [(1.0, 1.0)] * 4), 4)
    with pytest.raises(_lib.AsyrpError, match="multiple"):
        anc.check(sch, 3)
    with pytest.raises(_lib.AsyrpError, match="grid"):
        anc.check(Schedule(betas, *make_sequences(999, 6), t_edit=500), 4)
    with pytest.raises(_lib.AsyrpError, match="grid"):
        anc.check(Schedule(betas, *make_sequences(900, 5), t_edit=500), 4)
    with pytest.raises(_lib.AsyrpError, match="DDIM"):
        anc.check(Schedule(betas, seq, seq_next, t_edit=500, sample_type="ddpm", logvars=torch.zeros(1000)), 4)
    with pytest.raises(_lib.AsyrpError, match="eps"):
        Anchors(torch.zeros(n + 1, B, 3, 4, 4), torch.zeros(n - 1, B, 3, 4, 4), grid).check(sch, 4)
    # images [j0, j1) padded by the last one, as pad_rows pads latents
    x = torch.arange(n + 1)[:, None, None, None, None] * 10 + torch.arange(3)[None, :, None, None, None]
    a3 = Anchors(x.expand(n + 1, 3, 3, 4, 4).float(), x[:-1].expand(n, 3, 3, 4, 4).float(), grid)
    sub = a3.images(1, 3, 4)
    assert sub.x.shape == (n + 1, 4, 3, 4, 4) and sub.grid == grid
    assert [int(v) for v in sub.x[2, :, 0, 0, 0]] == [21, 22, 22, 22]
    assert torch.equal(sub.eps[:, 3], a3.eps[:, 2])


# ------------------------------------------------------------------------------------------------------------------
# save_image's wiring, with a stub engine
# ------------------------------------------------------------------------------------------------------------------
def _stub_run(tmp_path, monkeypatch, anchored, edit_region=None, bs=2, tuples=3, max_rows=4, addnoise=0):
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test", "--exp", "./runs/r", "--bs_train", str(bs),
                                                  "--n_test_step", "4", "--n_inv_step", "4",
                                                  "--max_rows_per_replay", str(max_rows)])
    r = Asyrp(args, cfg, device="cpu")
    r.t_edit, r.t_addnoise = 500, addnoise
    S, steps = 8, 4
    calls = []
    rec_x = torch.randn(steps, bs, 3, S, S)
    eng = NS(device=torch.device("cpu"), n_delta=1, last_records={"x": rec_x})

    def edit_batch(self, model, x_lat, schedule, noise=None, out=None, **kw):
        calls.append((x_lat.shape[0], schedule.steps[0].edit, noise is not None, kw))
        return torch.zeros(x_lat.shape[0], 3, S, S)
    monkeypatch.setattr(Asyrp, "edit_batch", edit_batch)
    masks = []

    def fake_masks(parser, origin, classes, rr, sigma):
        masks.append(origin.clone())
        return torch.ones(origin.shape[0], S, S)
    monkeypatch.setattr(region, "region_masks", fake_masks)
    seq, seq_next = make_sequences(999, steps)
    coeffs = [(1.0, 0.5 * k) for k in range(tuples)]
    anc = None
    if anchored:
        anc = Anchors(torch.randn(steps + 1, bs, 3, S, S), torch.randn(steps, bs, 3, S, S), reverse_grid(seq, seq_next))
    kw = {"anchors": anc} if anchored else {}
    xs = r.save_image(NS(engine=eng), anc.x_T if anchored else torch.zeros(bs, 3, S, S), seq, seq_next,
                      save_x_origin=True, folder_dir="out", file_name="f", hs_coeff=coeffs, edit_region=edit_region,
                      **kw)
    return calls, masks, anc, rec_x, xs


def test_save_image_without_the_flag_makes_the_same_calls(tmp_path, monkeypatch):
    calls, masks, _, _, xs = _stub_run(tmp_path, monkeypatch, False, addnoise=500)
    assert not masks and len(xs) == 4
    assert calls[0] == (2, False, False, {"record_process": False})  # the origin pass, as before
    for n, edit, noise, kw in calls[1:]:
        assert edit and noise and n == 4 and set(kw) == {"record_process", "hs_coeffs"}


def test_save_image_anchored(tmp_path, monkeypatch):
    calls, masks, anc, _, xs = _stub_run(tmp_path, monkeypatch, True, addnoise=500)
    assert len(calls) == 2, "no origin pass: 3 tuples of 2 images in chunks of 4 rows"
    for n, edit, noise, kw in calls:
        assert edit and not noise and n == 4 and kw["anchors"] is anc
    assert torch.equal(xs[0], anc.x0), "the origin row is the input image"
    parser = object()
    calls, masks, anc, rec_x, xs = _stub_run(tmp_path, monkeypatch, True, edit_region=(parser, [17], 1, 0.0))
    assert len(masks) == 1 and torch.equal(masks[0], anc.x0), "the mask parses the input image"
    for n, edit, noise, kw in calls:
        mask, ref = kw["blend"]
        assert kw["anchors"] is anc and torch.equal(ref, anc.ref) and not torch.equal(ref, rec_x)


def test_run_test_batches_without_the_flag(monkeypatch):
    """_edit_batches without the flag yields _batches' batches, unchanged, and no anchors"""
    r = Asyrp.__new__(Asyrp)
    seen = []

    def batches(self, pairs, keep_source):
        seen.append(keep_source)
        yield ("test", 1, "x_T", "x0", [0, 1], None)
    monkeypatch.setattr(Asyrp, "_batches", batches)

    def no_anchors(*a, **k):
        raise AssertionError("anchors without the flag")
    monkeypatch.setattr(Asyrp, "anchor_batch", no_anchors)
    out = list(r._edit_batches(None, None, NS(keeps_source=False), False))
    assert out == [("test", 1, "x_T", "x0", [0, 1], None, None)] and seen == [False]
