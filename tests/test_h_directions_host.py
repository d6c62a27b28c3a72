"""h-space directions on the host: hspace.py's math (run through numpy restatements of the two statistics kernels)
against oracle/hspace.py's independent SVD route, the direction file and its refusals, the flag refusals of
--h_directions / --h_direction, the hs_coeff tuples of --run_test --h_direction, and the exported C-ABI symbols."""
import ctypes
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, hspace
from oracle import hspace as oh


def _data(n, d, steps=3, seed=0):
    g = np.random.default_rng(seed + 7 * n + d)
    # a few dominant directions so that the leading eigenvalues are well separated
    scale = np.linspace(3.0, 0.2, d)
    X = g.standard_normal((steps, n, d)) * scale[None, None] + g.standard_normal((1, 1, d))
    return X.astype(np.float32)


@pytest.mark.parametrize("n", [2, 5, 64])
@pytest.mark.parametrize("d", [1, 300])
def test_pca_matches_the_svd_oracle(n, d):
    """components are unit and orthogonal before scaling, stored as v sqrt(λ / (n - 1)), with the oracle's signs"""
    X = _data(n, d)
    K = min(n - 1, d, 3)
    ts = [999, 500, 0]
    dirs, rows = hspace.discover(X, ts, K=K, gram=oh.gram, combine=oh.combine)
    ref = oh.pca(X, K)
    for k, t in enumerate(ts):
        V, lam, tr = hspace.pca_step(X[k], K, oh.gram, oh.combine)
        np.testing.assert_allclose(V @ V.T, np.eye(K), atol=1e-10)
        Vr, var, ratio, stored = ref[k]
        for c in range(K):
            got = dirs[c][2][t]
            np.testing.assert_allclose(np.linalg.norm(got), np.sqrt(lam[c] / (n - 1)), rtol=1e-10)
            np.testing.assert_allclose(got, stored[c], rtol=1e-8, atol=1e-9 * np.abs(stored[c]).max())
            assert dirs[c][3][t] == pytest.approx((var[c], ratio[c]), rel=1e-9)
    assert hspace.tsv_text("pca", rows, K).splitlines()[0] == oh.tsv("pca", ts, ref).splitlines()[0]
    got_tsv = np.array([[float(v) for v in r.split("\t")] for r in hspace.tsv_text("pca", rows, K).splitlines()[1:]])
    ref_tsv = np.array([[float(v) for v in r.split("\t")] for r in oh.tsv("pca", ts, ref).splitlines()[1:]])
    np.testing.assert_allclose(got_tsv, ref_tsv, rtol=1e-7, equal_nan=True)


@pytest.mark.parametrize("n", [5, 64])
def test_sign_rule_is_deterministic_under_row_permutation(n):
    X = _data(n, 300, seed=3)
    K = 3
    perm = np.random.default_rng(1).permutation(n)
    a, _ = hspace.discover(X, [999, 500, 0], K=K, gram=oh.gram, combine=oh.combine)
    b, _ = hspace.discover(X[:, perm], [999, 500, 0], K=K, gram=oh.gram, combine=oh.combine)
    for c in range(K):
        for t in (999, 500, 0):
            np.testing.assert_allclose(a[c][2][t], b[c][2][t], rtol=1e-8, atol=1e-10)
            assert np.sign(a[c][2][t] @ b[c][2][t]) > 0


def test_sign_rule_against_the_oracle():
    V = np.array([[0.1, -0.9, 0.2], [0.5, 0.5, -0.5]])
    np.testing.assert_array_equal(hspace.fix_signs(V), oh.sign_rule(V))
    assert hspace.fix_signs(V)[0, 1] > 0 and hspace.fix_signs(V)[1, 0] > 0  # a tie takes the first entry
    prev = np.array([[0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
    np.testing.assert_array_equal(hspace.fix_signs(V, prev), oh.sign_rule(V, prev))


@pytest.mark.parametrize("n", [2, 5, 64])
@pytest.mark.parametrize("d", [1, 300])
def test_mean_difference(n, d):
    X = _data(n, d)
    n_pos = max(1, n // 3)
    ts = [999, 500, 0]
    dirs, rows = hspace.discover(X, ts, n_pos=n_pos, combine=oh.combine)
    ref = oh.mean_diff(X, n_pos)
    for k, t in enumerate(ts):
        np.testing.assert_allclose(dirs[0][2][t], ref[k][0], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(np.array(rows)[:, 1:], np.array([r[1:] for r in ref]), rtol=1e-9)
    # a set against itself: exactly zero
    same = np.concatenate([X, X], axis=1)
    dirs, rows = hspace.discover(same, ts, n_pos=n, combine=oh.combine)
    for t in ts:
        assert not np.any(dirs[0][2][t])
    assert all(r[1] == 0.0 for r in rows)


def test_refusals_of_the_math():
    X = _data(5, 10)
    with pytest.raises(ValueError, match="K=5"):
        hspace.pca_step(X[0], 5, oh.gram, oh.combine)
    with pytest.raises(ValueError, match="K=0"):
        hspace.pca_step(X[0], 0, oh.gram, oh.combine)
    with pytest.raises(ValueError, match="variance"):  # rank-1 data has one direction
        hspace.pca_step(np.ones((4, 6), np.float32) * np.arange(4)[:, None], 2, oh.gram, oh.combine)
    with pytest.raises(ValueError, match="each set"):
        hspace.mean_diff_step(X[0], 5, oh.combine)
    with pytest.raises(ValueError):
        hspace.discover(X, [1, 2, 3])


# ------------------------------------------------------------------------------------------------------------------
# the file
# ------------------------------------------------------------------------------------------------------------------
def _meta():
    return {"category": "CelebA_HQ", "mid_ch": 512, "t_0": 999, "n_test_step": 3, "n": 5}


def _run(**kw):
    return NS(**{"t_0": 999, "n_test_step": 3, **kw})


def _cfg(category="CelebA_HQ"):
    return NS(data=NS(category=category))


def test_file_round_trip_and_refusals(tmp_path):
    X = _data(5, 512 * 4)
    ts = [999, 499, 0]
    dirs, rows = hspace.discover(X, ts, K=2, gram=oh.gram, combine=oh.combine)
    paths = hspace.write_directions(str(tmp_path), dirs, rows, (512, 2, 2), _meta())
    assert [os.path.basename(p) for p in paths] == ["pc0.pth", "pc1.pth"]
    assert (tmp_path / "h_directions.tsv").read_text() == hspace.tsv_text("pca", rows, 2)
    obj = hspace.load_direction(paths[1], _cfg(), _run(), 512)
    assert obj["kind"] == "pca" and obj["component"] == 1 and obj["n"] == 5
    assert sorted(obj["delta_h"]) == sorted(ts) and set(obj["explained_variance"]) == set(ts)
    for t in ts:
        assert obj["delta_h"][t].dtype == torch.float32 and obj["delta_h"][t].shape == (512, 2, 2)
        np.testing.assert_array_equal(obj["delta_h"][t].numpy().ravel(), dirs[1][2][t].astype(np.float32))
    rows_t = hspace.direction_rows(obj, [999, 499])
    assert rows_t.shape == (2, 512, 2, 2) and torch.equal(rows_t[1], obj["delta_h"][499])
    assert hspace.direction_rows(obj, []) is None
    with pytest.raises(KeyError, match="t=500"):
        hspace.direction_rows(obj, [999, 500])
    # every field the run checks
    with pytest.raises(ValueError, match="'category'"):
        hspace.load_direction(paths[0], _cfg("AFHQ"), _run(), 512)
    with pytest.raises(ValueError, match="'mid_ch'"):
        hspace.load_direction(paths[0], _cfg(), _run(), 1024)
    with pytest.raises(ValueError, match="'t_0'"):
        hspace.load_direction(paths[0], _cfg(), _run(t_0=500), 512)
    with pytest.raises(ValueError, match="'n_test_step'"):
        hspace.load_direction(paths[0], _cfg(), _run(n_test_step=40), 512)
    bad = {**torch.load(paths[0], weights_only=True), "format": "something_else"}
    torch.save(bad, tmp_path / "bad.pth")
    with pytest.raises(ValueError, match="'format'"):
        hspace.load_direction(str(tmp_path / "bad.pth"), _cfg(), _run(), 512)
    torch.save({999: torch.zeros(512, 2, 2)}, tmp_path / "raw.pth")  # a raw Δh dict stays on the slerp path
    with pytest.raises(ValueError, match="'format'"):
        hspace.load_direction(str(tmp_path / "raw.pth"), _cfg(), _run(), 512)
    # the mean difference file
    dirs, rows = hspace.discover(X, ts, n_pos=2, combine=oh.combine)
    (p,) = hspace.write_directions(str(tmp_path / "md"), dirs, rows, (512, 2, 2), {**_meta(), "n": {"pos": 2, "neg": 3}})
    obj = hspace.load_direction(p, _cfg(), _run(), 512)
    assert os.path.basename(p) == "mean_diff.pth" and obj["kind"] == "mean_diff" and "explained_variance" not in obj
    assert (tmp_path / "md" / "h_directions.tsv").read_text().splitlines()[0] == "t\tnorm_d\tnorm_mu_pos\tnorm_mu_neg"


# ------------------------------------------------------------------------------------------------------------------
# the run
# ------------------------------------------------------------------------------------------------------------------
def _no_model(monkeypatch):
    from asyrp_official_b200.diffusion_latent import Asyrp

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    return Asyrp


def test_discovery_flag_refusals(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    monkeypatch.chdir(tmp_path)
    Asyrp = _no_model(monkeypatch)
    os.makedirs("imgs")
    from PIL import Image
    Image.new("RGB", (8, 8)).save("imgs/a.png")
    base = ["--config", "celeba.yml", "--h_directions", "--h_direction_out", "out", "--n_train_img", "8"]
    cases = [([], "exactly one mode"),
             (["--h_pca", "3", "--h_pos_dir", "imgs", "--h_neg_dir", "imgs"], "exactly one mode"),
             (["--h_pca", "8"], "n_train_img - 1 = 7"),
             (["--h_pca", "0"], "between 1"),
             (["--h_pos_dir", "imgs"], "go together"),
             (["--h_pos_dir", "imgs", "--h_neg_dir", "missing"], "--h_neg_dir 'missing'")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_h_directions()
    args, cfg = cli.parse_args_and_config(["--config", "celeba.yml", "--h_directions", "--h_pca", "2"])
    with pytest.raises(ValueError, match="--h_direction_out"):
        Asyrp(args, cfg, device="cpu").run_h_directions()
    args, cfg = cli.parse_args_and_config(base + ["--h_pca", "7"])
    r = Asyrp(args, cfg, device="cpu")
    assert r.h_directions_setup() == ("pca", 7)
    r.world = 2
    with pytest.raises(ValueError, match="single-process"):
        r.h_directions_setup()
    monkeypatch.setenv("WORLD_SIZE", "2")
    assert cli.main(base + ["--h_pca", "3"]) == 1


def test_edit_flag_refusals(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    monkeypatch.chdir(tmp_path)
    Asyrp = _no_model(monkeypatch)
    torch.save({"format": hspace.FORMAT}, "pc0.pth")
    base = ["--config", "celeba.yml", "--run_test", "--h_direction", "pc0.pth", "--user_defined_t_edit", "500",
            "--user_defined_t_addnoise", "200"]

    def no_sweep(self):
        raise AssertionError("--attr_sweep was dispatched before --h_direction was checked")
    monkeypatch.setattr(Asyrp, "run_attr_sweep", no_sweep)
    for extra, flag in ((["--train_delta_block"], "--train_delta_block"), (["--train_delta_h"], "--train_delta_h"),
                        (["--multiple_attr", "smiling young"], "--multiple_attr"),
                        (["--num_mean_of_delta_hs", "4"], "--num_mean_of_delta_hs"),
                        (["--attr_sweep", "smiling young"], "--attr_sweep")):
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=f"--h_direction replaces the Δh checkpoint: it does not combine with {flag}"):
            Asyrp(args, cfg, device="cpu").run_test()
    args, cfg = cli.parse_args_and_config(base[:4] + ["missing.pth"] + base[5:])
    with pytest.raises(FileNotFoundError, match="missing.pth"):
        Asyrp(args, cfg, device="cpu").run_test()
    args, cfg = cli.parse_args_and_config(base)
    assert Asyrp(args, cfg, device="cpu").h_direction_setup() == "pc0.pth"


def test_run_test_tuples():
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import h_direction_coeffs
    a = cli.build_parser().parse_args(["--config", "celeba.yml", "--hs_coeff_delta_h", "2.5",
                                       "--hs_coeff_origin_h", "0.9", "--n_train_step", "6", "--n_test_step", "40"])
    assert h_direction_coeffs(a) == (0.9, 2.5)  # no n_train_step / n_test_step scaling
    a.delta_interpolation, a.min_delta, a.max_delta, a.num_delta = True, -1.0, 1.0, 5
    assert h_direction_coeffs(a) == [(1.0, v * 2.5) for v in (-1.0, -0.5, 0.0, 0.5, 1.0)]


def test_symbols_are_exported():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("asyrp_add_h_rows", "asyrp_h_gram", "asyrp_h_combine"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
