"""Precision / recall / density / coverage (`--prdc`) on the host: a numpy fp64 restatement of the definition, checked
on the two worked examples and against a pure-Python double loop; the nan rule, the CLI refusals and the TSV layouts.

Definition: D(u, v) = sum_c (u_c - v_c)^2 in fp64; r_k(i) = the (k + 1)-th smallest D(x_i, x_j) over every j, j = i
included; with R the real rows (n) and F the fake rows (m), every comparison strict:
    precision = #{j : exists i, D(r_i, f_j) < r_k^R(i)} / m
    recall    = #{i : exists j, D(r_i, f_j) < r_k^F(j)} / n
    density   = sum_j #{i : D(r_i, f_j) < r_k^R(i)} / (k m)
    coverage  = #{i : exists j, D(r_i, f_j) < r_k^R(i)} / n
and all four nan when n <= k or m <= k."""
import math
import random

import numpy as np
import pytest
import torch

from asyrp_official_b200 import fid

NAN4 = (math.nan,) * 4


# ---- the numpy fp64 restatement ----
def sqdist(a, b):
    """D [n][m] fp64 of a [n][d] and b [m][d]: differences in fp64, squared and summed"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    out = np.empty((a.shape[0], b.shape[0]))
    for i in range(a.shape[0]):
        out[i] = ((a[i] - b) ** 2).sum(axis=1)
    return out


def radii_oracle(x, k):
    """the (k + 1)-th smallest D of each row of x over all rows of x, itself included"""
    return np.sort(sqdist(x, x), axis=1)[:, k]


def counts_oracle(a, ra, b, rb, dist=None):
    """(b_in_a [m], a_in_b [n], a_covered [n]) int64"""
    D = sqdist(a, b) if dist is None else dist
    ra, rb = np.asarray(ra, dtype=np.float64), np.asarray(rb, dtype=np.float64)
    return (D < ra[:, None]).sum(0), (D < rb[None, :]).sum(1), (D < ra[:, None]).sum(1)


def prdc_oracle(real, fake, k):
    n, m = len(real), len(fake)
    if n <= k or m <= k:
        return NAN4
    b_in_a, a_in_b, a_covered = counts_oracle(real, radii_oracle(real, k), fake, radii_oracle(fake, k))
    return (int((b_in_a > 0).sum()) / m, int((a_in_b > 0).sum()) / n, int(b_in_a.sum()) / (k * m),
            int((a_covered > 0).sum()) / n)


def prdc_loop(real, fake, k):
    """the definition as a pure-Python double loop over Python floats"""
    if len(real) <= k or len(fake) <= k:
        return NAN4
    real = [[float(v) for v in r] for r in np.asarray(real, dtype=np.float32)]
    fake = [[float(v) for v in f] for f in np.asarray(fake, dtype=np.float32)]

    def dist(u, v):
        s = 0.0
        for a, b in zip(u, v):
            s += (a - b) * (a - b)
        return s

    def radius(x, i):
        return sorted(dist(x[i], x[j]) for j in range(len(x)))[k]

    n, m = len(real), len(fake)
    rr = [radius(real, i) for i in range(n)]
    rf = [radius(fake, j) for j in range(m)]
    D = [[dist(real[i], fake[j]) for j in range(m)] for i in range(n)]
    precision = sum(any(D[i][j] < rr[i] for i in range(n)) for j in range(m)) / m
    recall = sum(any(D[i][j] < rf[j] for j in range(m)) for i in range(n)) / n
    density = sum(D[i][j] < rr[i] for i in range(n) for j in range(m)) / (k * m)
    coverage = sum(any(D[i][j] < rr[i] for j in range(m)) for i in range(n)) / n
    return precision, recall, density, coverage


def _col(v):
    return np.asarray(v, dtype=np.float32)[:, None]


# ---- tests ----
def test_worked_examples():
    assert prdc_oracle(_col([0, 1, 2, 3]), _col([0.5, 10]), 1) == (0.5, 1.0, 1.0, 0.5)
    real = _col([0, 0, 0, 5])
    assert list(radii_oracle(real, 1)) == [0.0, 0.0, 0.0, 25.0]
    # strict <: the fake at 0 lies in no zero-radius ball, only in the ball of 5 (radius 25)
    assert prdc_oracle(real, _col([0, 7]), 1) == (0.5, 1.0, 0.5, 0.25)
    for real, fake in ((_col([0, 1, 2, 3]), _col([0.5, 10])), (real, _col([0, 7]))):
        assert prdc_loop(real, fake, 1) == prdc_oracle(real, fake, 1)


@pytest.mark.parametrize("seed,n,m,d,k", [(0, 9, 7, 3, 1), (1, 12, 15, 5, 3), (2, 20, 11, 4, 5), (3, 6, 6, 2, 5),
                                          (4, 40, 33, 2, 32)])
def test_oracle_equals_the_double_loop(seed, n, m, d, k):
    g = np.random.default_rng(seed)
    real = g.standard_normal((n, d)).astype(np.float32)
    fake = (g.standard_normal((m, d)) * 1.3 + 0.2).astype(np.float32)
    fake[0] = real[0]  # a shared row
    assert prdc_oracle(real, fake, k) == prdc_loop(real, fake, k)
    ints = g.integers(-3, 4, (n, d)).astype(np.float32)  # many ties
    assert prdc_oracle(ints, ints[::-1] + 1, k) == prdc_loop(ints, ints[::-1] + 1, k)


def test_radii_count_duplicates():
    x = _col([1, 1, 1, 4, 9])
    assert list(radii_oracle(x, 1)) == [0.0, 0.0, 0.0, 9.0, 25.0]
    assert list(radii_oracle(x, 2)) == [0.0, 0.0, 0.0, 9.0, 64.0]


def test_nan_and_a_warning_for_sets_of_k_rows_or_fewer():
    real, fake = torch.zeros(6, 8), torch.ones(3, 8)  # host tensors: the rule applies before any kernel
    for k, r, f in ((3, real, fake), (6, real, torch.ones(9, 8)), (5, real[:2], fake)):
        with pytest.warns(RuntimeWarning, match="nan"):
            got = fid.prdc(r, f, k)
        assert len(got) == 4 and all(math.isnan(v) for v in got)
        assert all(math.isnan(v) for v in prdc_oracle(r.numpy(), f.numpy(), k))


def test_cli_refusals_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli, scoring
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    monkeypatch.setattr(scoring, "fid_setup", fail_load)  # --prdc is checked before --fid's own requirements
    base = ["--run_test", "--config", "celeba.yml"]
    fid_argv = ["--fid", "--fid_weights", "missing.pth"]
    cases = [(["--prdc"], "add --fid"),
             (["--prdc", "--attr_sweep", "smiling angry"], "add --fid"),
             (fid_argv + ["--prdc", "--prdc_k", "0"], r"--prdc_k must be in 1\.\.32, got 0"),
             (fid_argv + ["--prdc", "--prdc_k", "33"], r"--prdc_k must be in 1\.\.32, got 33"),
             (fid_argv + ["--prdc", "--prdc_k", "-5", "--attr_sweep", "smiling angry"], "got -5")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, cfg = cli.parse_args_and_config(["--diff_style", "--config", "celeba.yml", "--prdc"])
    with pytest.raises(ValueError, match="add --fid"):
        Asyrp(args, cfg, device="cpu").run_diff_style()
    args, _ = cli.parse_args_and_config(base)
    assert args.prdc is False and args.prdc_k == 5
    for k in (1, 32):  # the bounds themselves pass the check
        args, cfg = cli.parse_args_and_config(base + fid_argv + ["--prdc", "--prdc_k", str(k)])
        scoring.prdc_check(Asyrp(args, cfg, device="cpu"))


def test_prdc_table_layout(tmp_path, capsys):
    from asyrp_official_b200.scoring import write_prdc
    nan = float("nan")
    rows = [(0.5, 1.0, 1.0, 0.5), (0.1 + 0.2, nan, 1e-17, 0.0)]
    write_prdc(str(tmp_path / "t.tsv"), [(1.0, 0.5), (1.0, 1.5)], rows, 40, None, "test")
    lines = (tmp_path / "t.tsv").read_text().splitlines()
    assert lines == ["tuple\ths_coeff\tn\tprecision\trecall\tdensity\tcoverage",
                     "0\t1,0.5\t40\t0.5\t1.0\t1.0\t0.5",
                     f"1\t1,1.5\t40\t{0.1 + 0.2!r}\tnan\t1e-17\t0.0"]
    out = capsys.readouterr().out
    assert "(test, 40 images), hs_coeff (1,0.5): P 0.500000, R 1.000000, D 1.000000, C 0.500000" in out
    write_prdc(str(tmp_path / "s.tsv"), [(1.0, 1.0, 0.0), (1.0, 0.0, 1.0)], rows, 3, None, "train",
               attrs=["smiling", "angry"])
    lines = (tmp_path / "s.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tprecision\trecall\tdensity\tcoverage\tattr"
    assert lines[1] == "0\t1,1,0\t3\t0.5\t1.0\t1.0\t0.5\tsmiling" and lines[2].endswith("\tangry")
    assert "attribute angry" in capsys.readouterr().out


def test_prdc_real_table_layout(tmp_path, capsys):
    from asyrp_official_b200.scoring import write_prdc
    rows = [(0.25, 0.5, 0.75, 1.0), (0.5, 1.0, 1.0, 0.5), (0.0, 0.0, 0.0, 0.0)]
    write_prdc(str(tmp_path / "r.tsv"), [(1.0, 0.5), (1.0, 1.5)], rows, 40, 30000, "test", real=True)
    lines = (tmp_path / "r.tsv").read_text().splitlines()
    assert lines == ["tuple\ths_coeff\tn\tn_ref\tprecision\trecall\tdensity\tcoverage",
                     "origin\t-\t40\t30000\t0.25\t0.5\t0.75\t1.0",
                     "0\t1,0.5\t40\t30000\t0.5\t1.0\t1.0\t0.5",
                     "1\t1,1.5\t40\t30000\t0.0\t0.0\t0.0\t0.0"]
    assert "against the real images (test, 40 images, 30000 reference), origin: P 0.250000" in capsys.readouterr().out
    # a file without features (pytorch-fid's own): n_ref '-', the four columns nan; the attr column under a sweep
    write_prdc(str(tmp_path / "f.tsv"), [(1.0, 1.0, 0.0), (1.0, 0.0, 1.0)], [NAN4] * 3, 3, None, "train",
               attrs=["smiling", "angry"], real=True)
    lines = (tmp_path / "f.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tn_ref\tprecision\trecall\tdensity\tcoverage\tattr"
    assert lines[1] == "origin\t-\t3\t-\tnan\tnan\tnan\tnan\t-"
    assert [ln.split("\t")[-1] for ln in lines[1:]] == ["-", "smiling", "angry"]


def test_loop_restatement_on_random_small_sets():
    rnd = random.Random(7)
    for _ in range(5):
        n, m, d, k = rnd.randint(2, 9), rnd.randint(2, 9), rnd.randint(1, 4), rnd.randint(1, 3)
        g = np.random.default_rng(rnd.randint(0, 1 << 30))
        real, fake = g.random((n, d)).astype(np.float32), g.random((m, d)).astype(np.float32)
        got, ref = prdc_oracle(real, fake, k), prdc_loop(real, fake, k)
        assert got == ref or (all(map(math.isnan, got)) and all(map(math.isnan, ref)))
