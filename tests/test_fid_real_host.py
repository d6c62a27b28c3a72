"""FID / KID against real images' statistics (`--fid_ref`, `python -m asyrp_official_b200.fid --save-stats`) on the
host: a numpy fp64 restatement of torch-fidelity's subset KID and its index draws, the .npz statistics file and its
validator, the CLI refusals and the _fid_real.tsv layout."""
import numpy as np
import pytest
import torch

from asyrp_official_b200 import fid, synthetic
from oracle import fid as ofid


# ---- torch-fidelity's kid_features_to_metric (polynomial_kernel, mmd2 'unbiased', the subset loop), fp64 ----
def polynomial_kernel(X, Y, degree=3, coef0=1):
    gamma = 1.0 / X.shape[1]
    return (np.matmul(X, Y.T) * gamma + coef0) ** degree


def mmd2(K_XX, K_XY, K_YY):
    m = K_XX.shape[0]
    diag_X, diag_Y = np.diagonal(K_XX), np.diagonal(K_YY)
    Kt_XX_sums = K_XX.sum(axis=1) - diag_X
    Kt_YY_sums = K_YY.sum(axis=1) - diag_Y
    K_XY_sums_0 = K_XY.sum(axis=0)
    mmd = (Kt_XX_sums.sum() + Kt_YY_sums.sum()) / (m * (m - 1))
    return mmd - 2 * K_XY_sums_0.sum() / (m * m)


def kid_subsets_oracle(f1, f2, subsets, size, seed=2020, record=None):
    """(mean, std) of the subset MMD^2s; record: a list that receives each subset's (i1, i2)"""
    f1, f2 = np.asarray(f1, dtype=np.float64), np.asarray(f2, dtype=np.float64)
    mmds = np.zeros(subsets)
    rng = np.random.RandomState(seed)
    for i in range(subsets):
        i1 = rng.choice(len(f1), size, replace=False)
        i2 = rng.choice(len(f2), size, replace=False)
        if record is not None:
            record.append((i1, i2))
        a, b = f1[i1], f2[i2]
        mmds[i] = mmd2(polynomial_kernel(a, a), polynomial_kernel(a, b), polynomial_kernel(b, b))
    return float(np.mean(mmds)), float(np.std(mmds))


def _feats(n, d, seed, shift=0.0):
    g = np.random.default_rng(seed)
    return (g.random((n, d)) + shift).astype(np.float32)


def test_oracle_on_full_size_subsets_is_the_full_kid():
    f1, f2 = _feats(12, 16, 1), _feats(12, 16, 2, shift=0.3)
    mean, std = kid_subsets_oracle(f1, f2, 3, 12)
    ref = ofid.kid_loop(f1, f2)
    assert abs(mean - ref) <= 1e-10 * abs(ref) and std <= 1e-10 * abs(ref)


def test_index_draws_follow_randomstate_in_order():
    rec = []
    kid_subsets_oracle(_feats(30, 16, 3), _feats(25, 16, 4), 4, 7, record=rec)
    rng = np.random.RandomState(2020)
    for i1, i2 in rec:
        assert np.array_equal(i1, rng.choice(30, 7, replace=False))
        assert np.array_equal(i2, rng.choice(25, 7, replace=False))
    got1, got2 = fid.kid_subset_indices(30, 25, 4, 7)
    assert got1.dtype == np.int32 and got1.shape == (4, 7)
    assert np.array_equal(got1, np.stack([r[0] for r in rec])) and np.array_equal(got2, np.stack([r[1] for r in rec]))
    other = fid.kid_subset_indices(30, 25, 4, 7, seed=1)
    assert not np.array_equal(other[0], got1)


def _arrays(n=5, seed=0):
    g = np.random.default_rng(seed)
    f = g.random((n, fid.DIMS)).astype(np.float32)
    return {"mu": f.mean(0, dtype=np.float64), "sigma": np.cov(f.astype(np.float64), rowvar=False),
            "features": f, "kid_kxx": np.float64(123.25)}


def test_stats_file_round_trip(tmp_path):
    a = _arrays()
    p = str(tmp_path / "ref.npz")
    fid.write_stats(p, a)
    first = open(p, "rb").read()
    fid.write_stats(p, a)
    assert open(p, "rb").read() == first  # fixed member time stamps: the same arrays, the same bytes
    assert np.array_equal(np.load(p)["mu"], a["mu"]) and np.array_equal(np.load(p)["sigma"], a["sigma"])
    assert fid.validate_stats(p) == (5, True)
    got = fid.load_stats(p)
    assert set(got) == {"mu", "sigma", "features", "kid_kxx"} and got["kid_kxx"] == 123.25
    assert all(np.array_equal(got[k], a[k]) for k in ("mu", "sigma", "features"))
    assert set(fid.load_stats(p, with_features=False)) == {"mu", "sigma"}
    # pytorch-fid's --save-stats file: np.savez_compressed of mu / sigma only; FID only
    q = str(tmp_path / "pytorch_fid.npz")
    np.savez_compressed(q, mu=a["mu"], sigma=a["sigma"])
    assert fid.validate_stats(q) == (None, False)
    got = fid.load_stats(q)
    assert set(got) == {"mu", "sigma"} and np.array_equal(got["sigma"], a["sigma"])


@pytest.mark.parametrize("change,match", [
    (dict(mu=np.zeros(2047)), "'mu' has shape"),
    (dict(sigma=np.zeros((fid.DIMS, fid.DIMS), np.float32)), "'sigma' has dtype float32"),
    (dict(mu=None), "missing key 'mu'"),
    (dict(kid_kxx=None), "missing key 'kid_kxx'"),
    (dict(features=None), "missing key 'features'"),
    (dict(features=np.zeros((1, fid.DIMS), np.float32)), "'features' has shape"),
    (dict(features=np.zeros((4, fid.DIMS), np.float64)), "'features' has dtype float64"),
    (dict(kid_kxx=np.zeros(1)), "'kid_kxx' has shape"),
    (dict(extra=np.zeros(1)), "unexpected keys \\['extra'\\]"),
])
def test_validator_names_the_bad_key(tmp_path, change, match):
    a = {**_arrays(), **change}
    p = str(tmp_path / "bad.npz")
    np.savez(p, **{k: v for k, v in a.items() if v is not None})
    with pytest.raises(ValueError, match=match):
        fid.validate_stats(p)


def test_validator_refuses_other_files(tmp_path):
    with pytest.raises(ValueError, match="is a directory.*--save-stats"):
        fid.validate_stats(str(tmp_path))
    with pytest.raises(ValueError, match="no such file"):
        fid.validate_stats(str(tmp_path / "missing.npz"))
    (tmp_path / "junk.npz").write_bytes(b"\x00" * 64)
    with pytest.raises(ValueError, match="not an .npz"):
        fid.validate_stats(str(tmp_path / "junk.npz"))
    np.save(str(tmp_path / "plain.npy"), np.zeros(3))
    with pytest.raises(ValueError, match="not an .npz"):
        fid.validate_stats(str(tmp_path / "plain.npy"))


def test_cli_refusals_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    torch.save(synthetic.inception_state_dict(seed=1, fc=False), "pt_inception.pth")
    fid.write_stats("ref.npz", _arrays())
    np.savez("bad.npz", mu=np.zeros(3), sigma=np.zeros((fid.DIMS, fid.DIMS)))
    (tmp_path / "real").mkdir()

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    base = ["--run_test", "--config", "celeba.yml"]
    fid_argv = ["--fid", "--fid_weights", "pt_inception.pth"]
    cases = [(["--fid_ref", "ref.npz"], "add --fid"),
             (["--fid_ref", "ref.npz", "--attr_sweep", "smiling angry"], "add --fid"),
             (fid_argv + ["--fid_ref", "missing.npz"], "no such file"),
             (fid_argv + ["--fid_ref", "real"], "is a directory.*--save-stats"),
             (fid_argv + ["--fid_ref", "bad.npz"], "'mu' has shape"),
             (fid_argv + ["--fid_ref", "ref.npz", "--kid_subsets", "-1"], "--kid_subsets must be >= 0"),
             (fid_argv + ["--fid_ref", "ref.npz", "--kid_subset_size", "1"], "--kid_subset_size >= 2")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, _ = cli.parse_args_and_config(base)
    assert args.fid_ref is None and args.kid_subsets == 100 and args.kid_subset_size == 1000


def test_stats_command_refusals(tmp_path, monkeypatch):
    (tmp_path / "real").mkdir()
    for i in range(2):
        (tmp_path / "real" / f"{i}.png").write_bytes(b"")
    argv = ["--save-stats", str(tmp_path / "real"), str(tmp_path / "out.npz"), "--fid_weights",
            str(tmp_path / "missing.pth")]
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="single-process"):
        fid.main(argv)
    monkeypatch.setenv("WORLD_SIZE", "1")
    with pytest.raises(ValueError, match="is not a file"):  # the weights are checked before any model load
        fid.main(argv)
    with pytest.raises(ValueError, match="not a directory"):
        fid.main(["--save-stats", str(tmp_path / "none"), "o.npz", "--fid_weights", "w"])
    with pytest.raises(ValueError, match="--batch_size"):
        fid.main(argv + ["--batch_size", "0"])
    assert not (tmp_path / "out.npz").exists()


def test_image_files_are_pytorch_fids(tmp_path):
    names = ["b.png", "a.jpg", "c.JPG", "d.webp", "e.txt", "f.tiff", "g", "h.pgm"]
    for nm in names:
        (tmp_path / nm).write_bytes(b"")
    (tmp_path / "sub.png").mkdir()
    (tmp_path / "sub.png" / "x.png").write_bytes(b"")
    got = [p.split("/")[-1] for p in fid.image_files(str(tmp_path))]
    assert got == ["a.jpg", "b.png", "d.webp", "f.tiff", "h.pgm"]


def test_fid_real_table_layout(tmp_path, capsys):
    from asyrp_official_b200.scoring import write_fid_real
    nan = float("nan")
    rows = [(1.5, 0.25, 0.125, 0.01), (12.5, 0.5, nan, nan), (0.1 + 0.2, 1e-17, 2.0, 0.0)]
    write_fid_real(str(tmp_path / "t.tsv"), [(1.0, 0.5), (1.0, 1.5)], rows, 40, 30000, "test")
    lines = (tmp_path / "t.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tn_ref\tFID\tKID\tKID_mean\tKID_std"
    assert lines[1] == "origin\t-\t40\t30000\t1.5\t0.25\t0.125\t0.01"
    assert lines[2] == "0\t1,0.5\t40\t30000\t12.5\t0.5\tnan\tnan"
    assert lines[3] == f"1\t1,1.5\t40\t30000\t{0.1 + 0.2!r}\t1e-17\t2.0\t0.0"
    out = capsys.readouterr().out
    assert "origin: FID 1.500000" in out and "hs_coeff (1.0, 1.5): FID 0.300000" in out
    write_fid_real(str(tmp_path / "s.tsv"), [(1.0, 1.0, 0.0), (1.0, 0.0, 1.0)], rows, 3, None, "train",
                   attrs=["smiling", "angry"])
    lines = (tmp_path / "s.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tn_ref\tFID\tKID\tKID_mean\tKID_std\tattr"
    assert [ln.split("\t")[0] for ln in lines[1:]] == ["origin", "0", "1"]
    assert [ln.split("\t")[8] for ln in lines[1:]] == ["-", "smiling", "angry"]
    assert all(ln.split("\t")[3] == "-" for ln in lines[1:]) and lines[2].split("\t")[1] == "1,1,0"
