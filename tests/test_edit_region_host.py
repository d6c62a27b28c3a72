"""--edit_region on the host: class names, feather taps, oracle/region.py on hand-computed masks (edges, r = 0,
sigma = 0, flat windows), every refusal before a model loads, the exported C-ABI symbols, and save_image's wiring with
a stub engine: without the flag it makes the calls it made before, with it the origin pass records its trajectory and
the edit pass gets the blend.  No GPU needed."""
import ctypes
import math
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, main as cli, region, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import region as orr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# classes and taps
# ------------------------------------------------------------------------------------------------------------------
def test_class_names():
    assert len(region.CLASSES) == 19
    assert region.CLASSES[0] == "background" and region.CLASSES[17] == "hair" and region.CLASSES[18] == "hat"
    assert region.parse_classes("hair hat") == [17, 18]
    assert region.parse_classes("  skin\tnose ") == [1, 10]
    assert region.class_bits([17, 18]) == (1 << 17) | (1 << 18)
    for text, match in (("hair beard", "unknown class 'beard'"), ("hair hair", "given twice"), ("", "names no class"),
                        ("Hair", "unknown class")):
        with pytest.raises(ValueError, match=match) as e:
            region.parse_classes(text)
        assert "background skin l_brow" in str(e.value) and "cloth hair hat" in str(e.value)


@pytest.mark.parametrize("sigma", [0.2, 0.7, 1.0, 2.5, 16.0])
def test_taps(sigma):
    w = region.taps(sigma)
    R = math.ceil(3 * sigma)
    assert w.dtype == torch.float32 and w.shape == (2 * R + 1,)
    assert torch.equal(w, w.flip(0)) and int(w.argmax()) == R
    i = np.arange(-R, R + 1)
    ref = np.exp(-i * i / (2 * sigma * sigma))
    assert np.array_equal(w.numpy(), (ref / ref.sum()).astype(np.float32))  # normalised in fp64, then rounded
    assert np.array_equal(orr.taps(sigma).astype(np.float32), w.numpy())
    assert region.taps(0) is None and region.taps(0.0) is None


def test_option_refusals():
    region.check_options(0, 0.0, 256)
    region.check_options(32, 16.0, 512)
    for r, s, size, match in ((-1, 0, 256, "dilate"), (33, 0, 256, "dilate"), (1.5, 0, 256, "dilate"),
                              (0, -0.1, 256, "feather"), (0, 16.01, 256, "feather"), (0, float("nan"), 256, "feather"),
                              (0, 0, 513, "above"), (0, 0, 1024, "above")):
        with pytest.raises(ValueError, match=match):
            region.check_options(r, s, size)


# ------------------------------------------------------------------------------------------------------------------
# the oracle on hand-computed masks
# ------------------------------------------------------------------------------------------------------------------
def test_select_footprints():
    lab = np.zeros((2, 512, 512), dtype=np.uint8)
    lab[0, 0, 0] = 17                 # one parser pixel in the top-left corner
    lab[0, 511, 300] = 18
    lab[1, 100:102, 200:204] = 17
    lab[1, 5, 5] = 16                 # not chosen
    m = orr.select(lab, [17, 18], 256)  # footprints of 2 x 2
    want = np.zeros((2, 256, 256))
    want[0, 0, 0] = want[0, 255, 150] = 1
    want[1, 50, 100:102] = 1
    assert np.array_equal(m, want)
    assert np.array_equal(orr.select(lab, [17, 18], 512), np.isin(lab, [17, 18]).astype(np.float64))
    # S = 3: rows / columns [0, 171), [171, 342), [342, 512)
    lab = np.zeros((1, 512, 512), dtype=np.uint8)
    lab[0, 170, 341] = 17
    lab[0, 342, 511] = 17
    m = orr.select(lab, [17], 3)
    assert np.array_equal(m[0], np.array([[0, 1, 0], [0, 0, 0], [0, 0, 1]], dtype=np.float64))
    assert not orr.select(lab, [18], 3).any()


def test_dilate_by_hand():
    m = np.zeros((1, 5, 5))
    m[0, 0, 0] = 1
    m[0, 3, 2] = 1
    assert np.array_equal(orr.dilate(m, 0), m)
    want = np.array([[1, 1, 0, 0, 0],
                     [1, 1, 0, 0, 0],
                     [0, 1, 1, 1, 0],
                     [0, 1, 1, 1, 0],
                     [0, 1, 1, 1, 0]], dtype=np.float64)  # clipped at the border
    assert np.array_equal(orr.dilate(m, 1)[0], want)
    assert np.array_equal(orr.dilate(m, 32)[0], np.ones((5, 5)))


def test_feather_by_hand():
    m = np.zeros((1, 6, 6))
    m[0, :, 3:] = 1                    # a vertical edge: every column constant
    assert np.array_equal(orr.feather(m, 0), m)
    sigma = 0.7
    w = orr.taps(sigma)                # R = 3
    f = orr.feather(m, sigma)[0]
    # horizontal pass at column x, clamped indices: sum of the taps that land on columns >= 3
    for x in range(6):
        cols = np.clip(np.arange(x - 3, x + 4), 0, 5)
        vals = (cols >= 3).astype(np.float64)
        want = vals[0] if (vals == vals[0]).all() else float(w @ vals)
        assert np.all(f[:, x] == want), x  # the vertical pass sees flat columns and keeps them exactly
    # flat windows are exact: far from the edge 0 and 1, not the sum of the taps
    big = np.zeros((1, 40, 40))
    big[0, 10:30, 10:30] = 1
    f = orr.feather(big, 2.5)
    assert f[0, 0, 0] == 0.0 and f[0, 20, 20] == 1.0 and 0 < f[0, 10, 20] < 1
    assert np.array_equal(orr.feather(np.ones((1, 7, 7)), 16.0), np.ones((1, 7, 7)))
    assert np.array_equal(orr.feather(np.full((1, 7, 7), 0.3), 1.0), np.full((1, 7, 7), 0.3))


def test_blended_trajectory_loop():
    """mask ones -> the unblended loop; zeros -> the reference's last step; row n blends with image n % B"""
    from oracle import sampler as osmp
    betas = osmp.make_betas()
    seq, seq_next = osmp.make_sequences(999, 4)

    def model(x, t, **k):  # an affine stand-in for a UNet
        e = 0.1 * x + 0.01 * t.view(-1, 1, 1, 1) / 1000
        return e, e * 1.5, None, None

    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 3, 8, 8, generator=g)
    ref = torch.randn(4, 2, 3, 8, 8, generator=g)
    kw = dict(betas=betas, seq=seq, seq_next=seq_next, t_edit=500)
    plain = osmp.run_trajectory(model, x, **kw)
    assert torch.equal(orr.run_blended_trajectory(model, x, torch.ones(2, 8, 8), ref, **kw), plain)
    zero = orr.run_blended_trajectory(model, x, torch.zeros(2, 8, 8), ref, **kw)
    assert torch.equal(zero, ref[-1][[0, 1, 0, 1]])


# ------------------------------------------------------------------------------------------------------------------
# refusals before any model loads
# ------------------------------------------------------------------------------------------------------------------
def _no_model(monkeypatch):
    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)


BASE = ["--config", "celeba.yml", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0"]


def test_flag_refusals(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    _no_model(monkeypatch)
    torch.save(synthetic.face_parsing_state_dict(seed=1), "fp.pth")
    torch.save({"not": torch.zeros(1)}, "bad.pth")
    with open("junk.pth", "wb") as f:
        f.write(b"not a checkpoint")
    ok = BASE + ["--run_test", "--edit_region", "hair", "--seg_weights", "fp.pth"]

    def no_sweep(self):
        raise AssertionError("--attr_sweep was dispatched before --edit_region was checked")
    monkeypatch.setattr(Asyrp, "run_attr_sweep", no_sweep)
    cases = [(ok + ["--attr_sweep", "smiling young"], "with --attr_sweep"),
             (ok + ["--pass_editing"], "with --pass_editing"),
             (ok + ["--num_mean_of_delta_hs", "2"], "with --num_mean_of_delta_hs"),
             (ok + ["--lpips"], "with --lpips"),
             (ok[:-4] + ["--edit_region", "hair beard", "--seg_weights", "fp.pth"], "unknown class 'beard'"),
             (ok[:-2] + ["--seg_weights", "missing.pth"], "--edit_region: --seg_weights 'missing.pth' is not a file"),
             (ok[:-2] + ["--seg_weights", "bad.pth"], "--edit_region: "),
             (ok[:-2] + ["--seg_weights", "junk.pth"], "--edit_region: "),
             (ok + ["--edit_region_dilate", "33"], "--edit_region_dilate"),
             (ok + ["--edit_region_dilate", "-1"], "--edit_region_dilate"),
             (ok + ["--edit_region_feather", "16.5"], "--edit_region_feather"),
             (ok + ["--edit_region_feather", "-1"], "--edit_region_feather")]
    for argv, match in cases:
        args, cfg = cli.parse_args_and_config(argv)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    # outside --run_test, and in the other modes
    args, cfg = cli.parse_args_and_config(BASE + ["--lpips", "--edit_region", "hair", "--seg_weights", "fp.pth"])
    with pytest.raises(ValueError, match="add --run_test"):
        Asyrp(args, cfg, device="cpu").compute_lpips_distance()
    for flag, run in (("--diff_style", "run_diff_style"), ("--h_directions", "run_h_directions"),
                      ("--lpips", "compute_lpips_distance")):
        args, cfg = cli.parse_args_and_config(ok + [flag])
        with pytest.raises(ValueError, match=f"with {flag}"):
            getattr(Asyrp(args, cfg, device="cpu"), run)()
        assert cli.main(ok + [flag]) == 1
    # an image size above the parser's labels
    args, cfg = cli.parse_args_and_config(ok)
    r = Asyrp(args, cfg, device="cpu")
    r.config.data.image_size = 1024
    with pytest.raises(ValueError, match="above the parser's 512"):
        r.run_test()
    # accepted
    args, cfg = cli.parse_args_and_config(ok + ["--edit_region", "hair hat", "--edit_region_dilate", "32",
                                                "--edit_region_feather", "16"])
    classes, rr, sigma, sd = Asyrp(args, cfg, device="cpu").edit_region_setup()
    assert classes == [17, 18] and rr == 32 and sigma == 16.0 and "conv_out.conv_out.weight" in sd
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test"])
    assert Asyrp(args, cfg, device="cpu").edit_region_setup() is None


# ------------------------------------------------------------------------------------------------------------------
# symbols
# ------------------------------------------------------------------------------------------------------------------
NAMES = ("asyrp_blend_rows", "asyrp_region_mask", "asyrp_mask_dilate", "asyrp_mask_blur")


def test_symbols_are_declared_and_exported():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "asyrp_b200.h")).read()
    for name in NAMES:
        assert hasattr(lib, name) and name in _lib.SIGNATURES
        assert f"int {name}(" in header


# ------------------------------------------------------------------------------------------------------------------
# save_image's wiring, with a stub engine
# ------------------------------------------------------------------------------------------------------------------
def _stub_run(tmp_path, monkeypatch, edit_region, bs=2, tuples=3, max_rows=4):
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test", "--exp", "./runs/r", "--bs_train", str(bs),
                                                  "--n_test_step", "4", "--max_rows_per_replay", str(max_rows)])
    r = Asyrp(args, cfg, device="cpu")
    r.t_edit, r.t_addnoise = 500, 0
    S = 8
    steps = 4
    calls = []
    rec_x = torch.randn(steps, bs, 3, S, S)
    eng = NS(device=torch.device("cpu"), n_delta=1, last_records={"x": rec_x})

    def edit_batch(self, model, x_lat, schedule, noise=None, out=None, **kw):
        calls.append((x_lat.shape[0], schedule.steps[0].edit, kw))
        return torch.zeros(x_lat.shape[0], 3, S, S)
    monkeypatch.setattr(Asyrp, "edit_batch", edit_batch)
    masks = []

    def fake_masks(parser, origin, classes, rr, sigma):
        masks.append((parser, origin.shape, classes, rr, sigma))
        return torch.ones(origin.shape[0], S, S)
    monkeypatch.setattr(region, "region_masks", fake_masks)
    seq = [int(s + 1e-6) for s in np.linspace(0, 1, steps) * 999]
    coeffs = [(1.0, 0.5 * k) for k in range(tuples)]
    xs = r.save_image(NS(engine=eng), torch.zeros(bs, 3, S, S), seq, [-1] + seq[:-1], save_x_origin=True,
                      folder_dir="out", file_name="f", hs_coeff=coeffs, edit_region=edit_region)
    return r, calls, masks, rec_x, xs


def test_save_image_without_the_flag_makes_the_same_calls(tmp_path, monkeypatch):
    _, calls, masks, _, xs = _stub_run(tmp_path, monkeypatch, None)
    assert not masks and len(xs) == 4
    assert calls[0] == (2, False, {"record_process": False})  # the origin pass, as before
    for n, edit, kw in calls[1:]:
        assert edit and "blend" not in kw and n == 4 and set(kw) == {"record_process", "hs_coeffs"}
    assert not os.path.exists("out/f_ngen6_region_mask.png")


def test_save_image_with_a_region_blends_every_chunk(tmp_path, monkeypatch):
    parser = object()
    _, calls, masks, rec_x, xs = _stub_run(tmp_path, monkeypatch, (parser, [17], 2, 0.7))
    assert masks == [(parser, (2, 3, 8, 8), [17], 2, 0.7)]
    assert calls[0] == (2, False, {"record_process": True})   # the origin pass records its trajectory
    assert len(calls) == 3                                      # 3 tuples of 2 images in chunks of 4 rows (2 tuples)
    for n, edit, kw in calls[1:]:
        mask, ref = kw["blend"]
        assert n == 4 and edit and torch.equal(ref, rec_x) and ref is not rec_x  # a copy, not the graph's buffer
        assert mask.shape == (2, 8, 8)
    assert os.path.isfile("out/f_ngen6_region_mask.png") and len(xs) == 4
