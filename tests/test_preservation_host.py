"""Content preservation, host side (no GPU): the fp64 oracle's SSIM against scipy's Gaussian filter and a direct 2-D
definition, its MS-SSIM pooling against torch's avg_pool2d, the relu clamp, exact scores of identical images, the
quantisation against a PNG written by torchvision, the host combination of the statistics, the
--content_preservation CLI refusals (which come before any model loads) and the score table."""
import numpy as np
import pytest
import scipy.ndimage as nd
import torch
import torch.nn.functional as F

from asyrp_official_b200 import preservation as pv, synthetic
from oracle import lpips as olp, preservation as op


def _planes(shape, seed):
    """u8-valued fp64 planes and an edit of them: noise over a smooth image, so that the maps are not trivial"""
    rng = np.random.default_rng(seed)
    H, W = shape[-2:]
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    base = 0.5 + 0.4 * np.sin(6 * xx + 3 * yy) * np.cos(4 * yy)
    x = np.clip(base + 0.1 * rng.standard_normal(shape), 0, 1)
    y = np.clip(x + 0.08 * rng.standard_normal(shape), 0, 1)
    return np.round(x * 255) / 255, np.round(y * 255) / 255


def _skimage_ssim(x, y):
    """scikit-image's structural_similarity(gaussian_weights=True, sigma=1.5, use_sample_covariance=False,
    data_range=1) of one plane: scipy's gaussian_filter (truncate 3.5: the same 11 taps), 5 pixels cropped per border"""
    f = lambda t: nd.gaussian_filter(t, sigma=1.5, truncate=3.5)[5:-5, 5:-5]  # noqa: E731
    ux, uy = f(x), f(y)
    vx, vy, vxy = f(x * x) - ux * ux, f(y * y) - uy * uy, f(x * y) - ux * uy
    s = ((2 * ux * uy + op.C1) * (2 * vxy + op.C2)) / ((ux * ux + uy * uy + op.C1) * (vx + vy + op.C2))
    return s.mean()


def _direct_stats(x, y):
    """(mean ssim, mean cs) of one plane from the 2-D window g g^T, summed tap by tap over every valid pixel"""
    g = op.window()
    H, W = x.shape
    Ho, Wo = H - 10, W - 10
    m = {k: np.zeros((Ho, Wo)) for k in ("x", "y", "xx", "yy", "xy")}
    for dy in range(11):
        for dx in range(11):
            w = g[dy] * g[dx]
            a, b = x[dy:dy + Ho, dx:dx + Wo], y[dy:dy + Ho, dx:dx + Wo]
            for k, v in (("x", a), ("y", b), ("xx", a * a), ("yy", b * b), ("xy", a * b)):
                m[k] += w * v
    sxx, syy, sxy = m["xx"] - m["x"] ** 2, m["yy"] - m["y"] ** 2, m["xy"] - m["x"] * m["y"]
    cs = (2 * sxy + op.C2) / (sxx + syy + op.C2)
    s = (2 * m["x"] * m["y"] + op.C1) / (m["x"] ** 2 + m["y"] ** 2 + op.C1) * cs
    return s.mean(), cs.mean()


def test_window_is_scipys_gaussian():
    g = op.window()
    delta = np.zeros(21)
    delta[10] = 1.0
    assert np.abs(nd.gaussian_filter1d(delta, 1.5, truncate=3.5)[5:16] - g).max() <= 1e-16
    assert abs(g.sum() - 1) <= 1e-15


@pytest.mark.parametrize("H,W", [(256, 256), (37, 53), (161, 162), (11, 11), (12, 13)])
def test_oracle_ssim_equals_scipy_and_the_direct_definition(H, W):
    x, y = _planes((3, H, W), H + W)
    st = op.ssim_stats(x, y)
    for c in range(3):
        assert abs(st[c, 0] - _skimage_ssim(x[c], y[c])) <= 1e-12
        s, cs = _direct_stats(x[c], y[c])
        assert abs(st[c, 0] - s) <= 1e-12 and abs(st[c, 1] - cs) <= 1e-12
    assert (st[:, 0] < 0.99).all()  # the edit is visible: the comparison is not trivial


@pytest.mark.parametrize("H,W", [(256, 256), (161, 161), (21, 20), (11, 12), (1, 1), (3, 2)])
def test_pool2_equals_torch_avg_pool2d(H, W):
    x = np.random.default_rng(H * W).random((2, 3, H, W))
    ref = F.avg_pool2d(torch.from_numpy(x), 2, stride=2, padding=(H % 2, W % 2)).numpy()
    got = op.pool2(x)
    assert got.shape == ref.shape == (2, 3, (H + 1) // 2, (W + 1) // 2)
    assert np.abs(got - ref).max() <= 1e-15
    assert [s for s in pv.level_shapes(H, W)][1] == got.shape[2:]


def test_relu_clamp_gives_ms_ssim_zero_for_anti_correlated_images():
    x, _ = _planes((1, 3, 256, 256), 5)
    src = torch.from_numpy(x * 2 - 1).float()
    neg = -src  # q_neg = 255 - q_src up to the rounding of .5: anti-correlated at every level
    st = op.level_stats(op.quantize(src.numpy()) / 255.0, op.quantize(neg.numpy()) / 255.0)
    assert (st[0, ..., 1] < 0).all()  # cs of level 0 is negative: relu makes the product 0
    s = op.scores(src.numpy(), neg.numpy())
    assert s[0, 2] == 0.0 and s[0, 1] < 0
    # the host combination clamps the same way
    sse = np.array([1], dtype=np.int64)
    assert pv.combine(sse, st, np.zeros(1), 256, 256)[0, 2] == 0.0


def test_identical_images_score_exactly():
    rng = np.random.default_rng(3)
    x = (rng.random((2, 3, 256, 256)) * 2.4 - 1.2).astype(np.float32)  # partly outside [-1, 1]
    s = op.scores(x, np.concatenate([x, x]))
    assert (s[:, 0] == np.inf).all() and (s[:, 1] == 1.0).all() and (s[:, 2] == 1.0).all()
    q = op.quantize(x)
    st = op.level_stats(q / 255.0, q / 255.0)
    assert (st == 1.0).all()
    out = pv.combine(np.zeros(2, dtype=np.int64), st, np.zeros(2, dtype=np.float32), 256, 256)
    assert out.tolist() == [[np.inf, 1.0, 1.0, 0.0]] * 2
    sd = synthetic.lpips_state_dict(seed=3)
    xq = torch.from_numpy((2.0 * q.astype(np.float32) - 255.0) / 255.0)
    assert (olp.lpips(sd, xq.double(), xq.double()) == 0).all()


def test_quantisation_equals_a_png_written_by_torchvision(tmp_path):
    import torchvision.utils as tvu
    from PIL import Image
    g = torch.Generator().manual_seed(4)
    x = torch.rand(1, 3, 64, 80, generator=g) * 2.4 - 1.2
    # values whose save_image value (x + 1) * 0.5 * 255 + 0.5 lands exactly on an integer (the truncation boundary)
    k = torch.arange(64 * 80, dtype=torch.float32).remainder(256)
    x[0, 1] = ((k / 255.0) * 2 - 1).view(64, 80)
    x[0, 2, :4] = torch.tensor([-1.0, 1.0, -3.0, 5.0]).view(4, 1)
    tvu.save_image((x + 1) * 0.5, str(tmp_path / "x.png"))  # what Asyrp.save_image writes
    png = np.asarray(Image.open(tmp_path / "x.png").convert("RGB")).transpose(2, 0, 1)
    assert np.array_equal(op.quantize(x.numpy())[0], png)


def test_psnr_and_the_host_combination():
    rng = np.random.default_rng(6)
    x = (rng.random((2, 3, 161, 170)) * 2 - 1).astype(np.float32)
    e = np.clip(np.concatenate([x, x]) + 0.05 * rng.standard_normal((4, 3, 161, 170)), -1, 1).astype(np.float32)
    qs, qe = op.quantize(x), op.quantize(e)
    qs = qs[np.arange(4) % 2]
    sse = ((qs.astype(np.int64) - qe) ** 2).reshape(4, -1).sum(1)
    assert np.array_equal(op.psnr(qs, qe), 10 * np.log10(255.0 ** 2 * 3 * 161 * 170 / sse))
    st = op.level_stats(qs / 255.0, qe / 255.0)
    lp = np.array([0.1, 0.2, 0.3, 0.4], dtype=np.float32)
    got = pv.combine(sse, st, lp, 161, 170)
    ref = op.scores(x, e)
    assert np.array_equal(got[:, :3], ref) and np.array_equal(got[:, 3], lp.astype(np.float64))
    assert pv.row_bytes(256, 256) > 3 * 256 * 256 * 8 and pv.ACTIVATION_BUDGET // pv.row_bytes(256, 256) >= 16


def test_image_size_limit():
    pv.check_image_size(161, 161)
    for H, W in ((160, 256), (256, 160), (64, 64)):
        with pytest.raises(ValueError, match="larger than 160"):
            pv.check_image_size(H, W)


def test_cli_rejections_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200 import scoring
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    sd = synthetic.lpips_state_dict(seed=1)
    torch.save(sd, "alex.pth")
    torch.save({k: v for k, v in sd.items() if k != "lin2.model.1.weight"}, "partial.pth")
    (tmp_path / "junk.pth").write_bytes(b"\x00" * 64)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    monkeypatch.setattr(Asyrp, "attr_sweep_setup", lambda self: (["smiling"], ["checkpoint/smiling_0.pth"]))
    base = ["--config", "celeba.yml", "--content_preservation"]
    cases = [(["--run_test", "--lpips_weights", "alex.pth", "--pass_editing"], "--pass_editing"),
             (["--run_test"], "needs --lpips_weights"),
             (["--run_test", "--lpips_weights", "missing.pth"], "is not a file"),
             (["--run_test", "--lpips_weights", "partial.pth"], "missing key 'lin2.model.1.weight'"),
             (["--run_test", "--lpips_weights", "junk.pth", "--synthetic_weights"], "junk.pth"),
             (["--run_test", "--synthetic_weights", "--attr_sweep", "smiling", "--lpips_weights", "partial.pth",
               "--manual_checkpoint_name", "attribute_0.pth"], "missing key"),
             (["--lpips", "--lpips_weights", "alex.pth"], "scores the edits of --run_test")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        r = Asyrp(args, cfg, device="cpu")
        with pytest.raises(ValueError, match=match):
            r.compute_lpips_distance() if args.lpips else r.run_test()
    args, cfg = cli.parse_args_and_config(base + ["--lpips_weights", "alex.pth"])  # no --run_test
    with pytest.raises(ValueError, match="scores the edits of --run_test"):
        scoring.content_preservation_setup(Asyrp(args, cfg, device="cpu"))
    args, cfg = cli.parse_args_and_config(base + ["--run_test", "--lpips_weights", "alex.pth"])
    cfg.data.image_size = 160
    with pytest.raises(ValueError, match="larger than 160"):
        scoring.content_preservation_setup(Asyrp(args, cfg, device="cpu"))
    cfg.data.image_size = 256
    assert scoring.content_preservation_setup(Asyrp(args, cfg, device="cpu")) == "alex.pth"
    args, cfg = cli.parse_args_and_config(base + ["--run_test", "--synthetic_weights"])
    got = scoring.content_preservation_setup(Asyrp(args, cfg, device="cpu"))
    assert set(got) == set(sd) and all(torch.equal(got[k], synthetic.lpips_state_dict(seed=1234)[k]) for k in got)
    args, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml"])
    assert not args.content_preservation and args.lpips_weights is None


def test_diff_style_refuses_the_flag(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    args, cfg = cli.parse_args_and_config(["--config", "celeba.yml", "--diff_style", "--content_preservation",
                                           "--synthetic_weights", "--user_defined_t_edit", "500"])
    with pytest.raises(ValueError, match="scores the edits of --run_test"):
        Asyrp(args, cfg, device="cpu").run_diff_style()


def test_score_table_layout(tmp_path, capsys):
    from asyrp_official_b200.scoring import write_scores
    g = torch.Generator().manual_seed(2)
    cp = torch.rand(3, 2, 4, generator=g, dtype=torch.float64)
    cp[0, 1, 0] = float("inf")
    rec = torch.rand(2, 4, generator=g, dtype=torch.float64)
    coeffs = [(1.0, 0.5), (1.0, 1.0), (1.0, 1.5)]
    cells = lambda v: "\t".join(repr(x) for x in v.tolist())  # noqa: E731
    for origin in (None, rec):
        write_scores(str(tmp_path / "t.tsv"), coeffs, cp, pv.COLUMNS, "content preservation", origin=origin)
        lines = (tmp_path / "t.tsv").read_text().splitlines()
        assert lines[0] == "image\ttuple\ths_coeff\tPSNR\tSSIM\tMS_SSIM\tLPIPS"
        head = [] if origin is None else [f"{i}\torigin\t-\t{cells(rec[i])}" for i in range(2)]
        assert lines[1:] == head + [f"{i}\t{k}\t1,{c}\t{cells(cp[k][i])}" for k, c in enumerate(("0.5", "1", "1.5"))
                                    for i in range(2)]
    assert "inf" in (tmp_path / "t.tsv").read_text()
    out = capsys.readouterr().out
    assert "content preservation, origin: mean PSNR" in out and "hs_coeff (1.0, 1.5): mean PSNR" in out
    attrs = ["smiling", "angry", "young"]  # --attr_sweep: tuple k is attribute k
    sweep = [(1.0, 1.0, 0.0, 0.0), (1.0, 0.0, 1.0, 0.0), (1.0, 0.0, 0.0, 1.0)]
    for origin in (None, rec):
        write_scores(str(tmp_path / "s.tsv"), sweep, cp, pv.COLUMNS, "content preservation", attrs=attrs,
                     origin=origin)
        lines = (tmp_path / "s.tsv").read_text().splitlines()
        assert lines[0] == "image\ttuple\ths_coeff\tPSNR\tSSIM\tMS_SSIM\tLPIPS\tattr"
        head = [] if origin is None else [f"{i}\torigin\t-\t{cells(rec[i])}\t-" for i in range(2)]
        assert lines[1:] == head + [f"{i}\t{k}\t{','.join('1' if j in (0, k + 1) else '0' for j in range(4))}\t"
                                    f"{cells(cp[k][i])}\t{attrs[k]}" for k in range(3) for i in range(2)]
    # one column: the layout of the other score files
    write_scores(str(tmp_path / "one.tsv"), coeffs, cp[..., 1], "SC", "segmentation consistency")
    lines = (tmp_path / "one.tsv").read_text().splitlines()
    assert lines[0] == "image\ttuple\ths_coeff\tSC"
    assert lines[1:] == [f"{i}\t{k}\t1,{c}\t{cp[k][i][1].item()!r}" for k, c in enumerate(("0.5", "1", "1.5"))
                         for i in range(2)]
