"""--region_compose on the host: the flag's parsing, every refusal before a model loads, the chunk plan and the noise
layout, the composite's fp32 restatement against its fp64 form (overlaps, all-zero masks, K = 1 equal to the blend),
the exported C-ABI symbol, and the wiring of run_test and save_image with a stub engine: without the flag they make the
calls they made before.  No GPU needed."""
import ctypes
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import compose_oracle as oc
from asyrp_official_b200 import _lib, main as cli, region, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp, compose_noise, plan_compose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# parsing
# ------------------------------------------------------------------------------------------------------------------
def test_parse_compose():
    assert region.parse_compose("smiling=mouth,u_lip,l_lip grey_hair=hair") == [("smiling", [11, 12, 13]),
                                                                                ("grey_hair", [17])]
    assert region.parse_compose("  smiling=hair\t") == [("smiling", [17])]
    eight = " ".join(f"a{k}={region.CLASSES[k]}" for k in range(8))
    assert len(region.parse_compose(eight)) == 8
    for text, match in (("smiling", "is not attribute=class"), ("=hair", "is not attribute=class"),
                        ("smiling=hair=hat", "is not attribute=class"),
                        ("smiling=hair smiling=mouth", "names attribute 'smiling' twice"),
                        ("smiling=hair grey_hair=hat,hair", "hair given to both 'smiling' and 'grey_hair'"),
                        ("smiling=beard", "unknown class 'beard'"), ("smiling=hair,hair", "given twice"),
                        ("smiling=", "empty class list"), ("smiling=hair,,mouth", "empty class"),
                        ("smiling=hair,", "empty class"), ("", "names no attribute"),
                        (" ".join(f"a{k}={region.CLASSES[k]}" for k in range(9)), "at most 8")):
        with pytest.raises(ValueError, match=match) as e:
            region.parse_compose(text)
        assert "--region_compose" in str(e.value)
    args, _ = cli.parse_args_and_config(["--config", "celeba.yml", "--region_compose", "smiling=mouth grey_hair=hair"])
    assert args.region_compose == "smiling=mouth grey_hair=hair"
    args, _ = cli.parse_args_and_config(["--config", "celeba.yml"])
    assert args.region_compose is None


# ------------------------------------------------------------------------------------------------------------------
# refusals before any model loads
# ------------------------------------------------------------------------------------------------------------------
BASE = ["--config", "celeba.yml", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0", "--get_h_num", "1"]


def _scratch(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    os.makedirs("checkpoint", exist_ok=True)
    for attr in ("smiling", "grey_hair"):
        open(f"checkpoint/{attr}_0.pth", "wb").close()  # only their existence is checked here
    torch.save(synthetic.face_parsing_state_dict(seed=1), "fp.pth")
    torch.save({"not": torch.zeros(1)}, "bad.pth")
    with open("junk.pth", "wb") as f:
        f.write(b"not a checkpoint")
    return BASE + ["--run_test", "--manual_checkpoint_name", "attribute_0.pth", "--seg_weights", "fp.pth",
                   "--region_compose", "smiling=mouth,u_lip grey_hair=hair"]


def test_flag_refusals(tmp_path, monkeypatch):
    ok = _scratch(tmp_path, monkeypatch)

    def no_dispatch(self, *a):
        raise AssertionError("a mode was dispatched before --region_compose was checked")
    monkeypatch.setattr(Asyrp, "run_attr_sweep", no_dispatch)
    monkeypatch.setattr(Asyrp, "run_region_compose", no_dispatch)
    torch.save({}, "dir.pth")
    with_flag = [("--attr_sweep", ["smiling young"]), ("--edit_region", ["hair"]), ("--multiple_attr", ["a b"]),
                 ("--delta_interpolation", []), ("--num_mean_of_delta_hs", ["2"]), ("--train_delta_h", []),
                 ("--h_direction", ["dir.pth"]), ("--pass_editing", []), ("--lpips", []),
                 ("--DirectionalClipSmilarity", []), ("--save_process_delta_h", [])]
    cases = [(ok + [flag] + val, f"--region_compose does not combine with {flag}") for flag, val in with_flag]
    cases += [(ok + ["--sample_type", "ddpm"], "--region_compose needs --sample_type ddim"),
              (ok + ["--get_h_num", "2"], "--region_compose loads one DeltaBlock per attribute"),
              (ok + ["--region_compose", "smiling=hair smiling=mouth"], "twice"),
              (ok + ["--region_compose", "smiling=hair grey_hair=hair"], "given to both"),
              (ok + ["--region_compose", "smiling=beard"], "unknown class 'beard'"),
              (ok + ["--region_compose", "smiling= grey_hair=hair"], "empty class list"),
              (ok + ["--region_compose", " ".join(f"a{k}={region.CLASSES[k]}" for k in range(9))], "at most 8"),
              (ok + ["--max_rows_per_replay", "1"], "2 attributes need 2 rows per image, above --max_rows_per_replay 1"),
              (ok + ["--region_compose", "smiling=mouth young=hat"], "--region_compose: checkpoint"),
              (ok + ["--manual_checkpoint_name", "smiling_0.pth"], "has no 'attribute'"),
              (ok + ["--seg_weights", "missing.pth"], "--region_compose: --seg_weights 'missing.pth' is not a file"),
              (ok + ["--seg_weights", "bad.pth"], "--region_compose: "),
              (ok + ["--seg_weights", "junk.pth"], "--region_compose: "),
              (ok + ["--edit_region_dilate", "33"], "--edit_region_dilate"),
              (ok + ["--edit_region_dilate", "-1"], "--edit_region_dilate"),
              (ok + ["--edit_region_feather", "16.5"], "--edit_region_feather"),
              (ok + ["--edit_region_feather", "-1"], "--edit_region_feather")]
    for argv, match in cases:
        args, cfg = cli.parse_args_and_config(argv)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    # outside --run_test, and in the other modes
    args, cfg = cli.parse_args_and_config([a for a in ok if a != "--run_test"] + ["--lpips"])
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


def test_accepted_spec_and_dispatch(tmp_path, monkeypatch):
    ok = _scratch(tmp_path, monkeypatch)
    args, cfg = cli.parse_args_and_config(ok + ["--edit_region_dilate", "32", "--edit_region_feather", "16"])
    attrs, classes, r, sigma, sd, paths = Asyrp(args, cfg, device="cpu").region_compose_setup()
    assert attrs == ["smiling", "grey_hair"] and classes == [[11, 12], [17]] and r == 32 and sigma == 16.0
    assert "conv_out.conv_out.weight" in sd
    assert paths == [os.path.join("checkpoint", "smiling_0.pth"), os.path.join("checkpoint", "grey_hair_0.pth")]
    seen = []
    monkeypatch.setattr(Asyrp, "run_region_compose", lambda self, spec: seen.append(spec) or "composed")
    monkeypatch.setattr(Asyrp, "run_attr_sweep", lambda self: "swept")
    args, cfg = cli.parse_args_and_config(ok)
    assert Asyrp(args, cfg, device="cpu").run_test() == "composed" and seen[0][0] == attrs
    # without the flag: nothing to set up, and --attr_sweep is dispatched as before
    plain = [a for a in ok if a not in ("--region_compose", "smiling=mouth,u_lip grey_hair=hair")]
    args, cfg = cli.parse_args_and_config(plain)
    assert Asyrp(args, cfg, device="cpu").region_compose_setup() is None
    args, cfg = cli.parse_args_and_config(plain + ["--attr_sweep", "smiling grey_hair"])
    assert Asyrp(args, cfg, device="cpu").run_test() == "swept" and len(seen) == 1


# ------------------------------------------------------------------------------------------------------------------
# chunks and noise
# ------------------------------------------------------------------------------------------------------------------
def test_plan_compose():
    assert plan_compose(4, 2, 16) == (4, [(0, 4)])
    assert plan_compose(4, 2, 4) == (2, [(0, 2), (2, 4)])
    assert plan_compose(5, 2, 4) == (2, [(0, 2), (2, 4), (4, 5)])   # the last chunk padded to 2 images
    assert plan_compose(3, 3, 3) == (1, [(0, 1), (1, 2), (2, 3)])
    assert plan_compose(3, 3, 8) == (2, [(0, 2), (2, 3)])
    assert plan_compose(1, 8, 8) == (1, [(0, 1)])
    for bs in range(1, 7):
        for K in range(1, 9):
            for max_rows in range(K, 20):
                b, chunks = plan_compose(bs, K, max_rows)
                assert 1 <= b <= bs and K * b <= max_rows
                assert [j for j0, j1 in chunks for j in range(j0, j1)] == list(range(bs))
                assert all(j1 - j0 <= b for j0, j1 in chunks)


def test_compose_noise_layout():
    z = torch.arange(2 * 3 * 2, dtype=torch.float32).view(2, 3, 2)   # [n_stochastic][images][..]
    out = compose_noise(z, 3, 4)
    assert out.shape == (2, 12, 2)
    for k in range(4):
        assert torch.equal(out[:, k * 3:(k + 1) * 3], z), f"attribute {k} rows share the images' draw"
    short = compose_noise(z[:, 1:], 3, 2)   # two images padded to three: the last image repeated
    assert torch.equal(short, torch.cat([z[:, 1:], z[:, 2:], z[:, 1:], z[:, 2:]], dim=1))
    assert torch.equal(compose_noise(z, 3, 1), z)


# ------------------------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------------------------
def test_weights_by_hand():
    m = np.array([[0.0, 0.25, 1.0, 0.75, 0.5], [0.0, 0.5, 0.0, 0.75, 1.0]])
    w0, w = oc.compose_weights(m)
    assert np.array_equal(w0, [1.0, 0.25, 0.0, 0.0, 0.0])
    assert np.array_equal(w, [[0.0, 0.25, 1.0, 0.5, 1 / 3], [0.0, 0.5, 0.0, 0.5, 2 / 3]])   # overlaps normalised
    assert np.allclose(w0 + w.sum(axis=0), 1.0)


def _case(K, B, C, H, W, seed, kind):
    g = np.random.default_rng(seed)
    x = g.standard_normal((K, B, C, H, W)).astype(np.float32)
    ref = g.standard_normal((B, C, H, W)).astype(np.float32)
    if kind == "soft":
        m = g.random((K, B, H, W)).astype(np.float32) / K
    elif kind == "hard":   # one attribute or none per pixel
        own = g.integers(0, K + 1, (B, H, W))
        m = np.stack([(own == k + 1) for k in range(K)]).astype(np.float32)
    else:                  # overlapping: sums above 1 in most pixels
        m = g.random((K, B, H, W)).astype(np.float32)
        m[:, :, 0] = 1.0
    return x, ref, m


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("kind", ["soft", "hard", "overlap"])
def test_fp32_restatement_against_fp64(K, kind):
    x, ref, m = _case(K, 2, 3, 5, 7, K * 7 + len(kind), kind)
    got = oc.compose_fp32(x, ref, m)
    want = oc.compose(x, ref, m)
    assert got.dtype == np.float32
    scale = np.abs(ref).max() + np.abs(x).max()
    assert np.abs(got - want).max() <= (K + 3) * 2.0 ** -23 * scale
    if kind == "hard":   # weights 0 or 1: the composite selects one row or the origin exactly
        own = (m * np.arange(1, K + 1)[:, None, None, None]).sum(axis=0).astype(int)
        sel = np.where(own[:, None] == 0, ref, np.take_along_axis(x, np.maximum(own - 1, 0)[None, :, None]
                                                                   .repeat(3, axis=2), axis=0)[0])
        assert np.array_equal(got, sel)
    if kind == "overlap" and K > 1:
        assert (m.sum(axis=0) > 1).mean() > 0.2


def test_all_zero_masks_keep_the_origin():
    for K in (1, 3, 8):
        x, ref, _ = _case(K, 2, 3, 4, 4, K, "soft")
        zero = np.zeros((K, 2, 4, 4), dtype=np.float32)
        assert np.array_equal(oc.compose_fp32(x, ref, zero), ref)
        assert np.array_equal(oc.compose(x, ref, zero), ref)


def test_k1_is_the_blend():
    x, ref, m = _case(1, 3, 3, 6, 6, 3, "soft")
    m[0, 0, 0, :3] = (0.0, 1.0, 0.5)
    assert np.array_equal(oc.compose_fp32(x, ref, m), oc.blend_fp32(x[0], ref, m[0]))


def test_fma32_rounds_once():
    a = np.float32(1 + 2.0 ** -12)
    c = np.float32(-(1 + 2.0 ** -11))
    # a * a = 1 + 2^-11 + 2^-24: fmaf keeps the 2^-24, a product rounded to fp32 first would lose it
    assert oc.fma32(a, a, c) == np.float32(2.0 ** -24)
    assert (np.float32(a * a) + c) == 0
    # random operands against exact rational arithmetic: the result is the fp32 value nearest a * b + c
    from fractions import Fraction
    g = np.random.default_rng(0)
    p, q, r = (g.standard_normal(300).astype(np.float32) for _ in range(3))
    got = oc.fma32(p, q, r)
    for i in range(300):
        exact = Fraction(float(p[i])) * Fraction(float(q[i])) + Fraction(float(r[i]))
        y = got[i]
        lo, hi = np.nextafter(y, np.float32(-np.inf)), np.nextafter(y, np.float32(np.inf))
        d = abs(Fraction(float(y)) - exact)
        assert d <= abs(Fraction(float(lo)) - exact) and d <= abs(Fraction(float(hi)) - exact), i


# ------------------------------------------------------------------------------------------------------------------
# symbols
# ------------------------------------------------------------------------------------------------------------------
def test_symbol_is_declared_and_exported():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "asyrp_b200.h")).read()
    assert hasattr(lib, "asyrp_compose_rows") and "asyrp_compose_rows" in _lib.SIGNATURES
    assert "int asyrp_compose_rows(float* x, const float* ref, const float* masks, int K, int B, int C, int HW, " \
           "void* stream);" in header


# ------------------------------------------------------------------------------------------------------------------
# save_image's wiring, with a stub engine
# ------------------------------------------------------------------------------------------------------------------
def _stub_run(tmp_path, monkeypatch, region_compose, bs=3, max_rows=4, t_addnoise=0):
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test", "--exp", "./runs/r", "--bs_train", str(bs),
                                                  "--n_test_step", "4", "--max_rows_per_replay", str(max_rows)])
    r = Asyrp(args, cfg, device="cpu")
    r.t_edit, r.t_addnoise = 500, 0
    S, steps = 8, 4
    calls = []
    rec_x = torch.randn(steps, bs, 3, S, S)
    eng = NS(device=torch.device("cpu"), n_delta=2, last_records={"x": rec_x})

    def edit_batch(self, model, x_lat, schedule, noise=None, out=None, **kw):
        calls.append((x_lat.clone(), schedule, noise, kw))
        return torch.arange(x_lat.shape[0], dtype=torch.float32).view(-1, 1, 1, 1).expand(-1, 3, S, S).clone()
    monkeypatch.setattr(Asyrp, "edit_batch", edit_batch)
    built = []

    def fake_masks(parser, origin, classes, rr, sigma):
        built.append((parser, origin.shape, classes, rr, sigma))
        return torch.rand(len(classes), origin.shape[0], S, S)
    monkeypatch.setattr(region, "compose_masks", fake_masks)
    seq = [int(s + 1e-6) for s in np.linspace(0, 1, steps) * 999]
    x_lat = torch.randn(bs, 3, S, S)
    kw = {}
    if region_compose is not None:
        kw = dict(region_compose=region_compose, hs_coeff=[(1.0, 0.5, 0.5)])
    else:
        kw = dict(hs_coeff=[(1.0, 0.5 * k, 0.0) for k in range(2)])
    xs = r.save_image(NS(engine=eng), x_lat, seq, [-1] + seq[:-1], save_x_origin=True, folder_dir="out",
                      file_name="f", **kw)
    return calls, built, rec_x, x_lat, xs


def test_save_image_without_the_flag_makes_the_same_calls(tmp_path, monkeypatch):
    calls, built, _, _, xs = _stub_run(tmp_path, monkeypatch, None, bs=2)
    assert not built and len(xs) == 3
    assert calls[0][0].shape[0] == 2 and calls[0][3] == {"record_process": False}   # the origin pass, as before
    for x, sch, noise, kw in calls[1:]:
        assert "compose" not in kw and x.shape[0] == 4 and set(kw) == {"record_process", "hs_coeffs"}
    assert not os.path.exists("out/f_ngen6_region_compose.png")


@pytest.mark.parametrize("t_addnoise", [0, 600])
def test_save_image_composes_every_chunk(tmp_path, monkeypatch, t_addnoise):
    parser = object()
    times = [(500, t_addnoise), (700, 0)]
    coeffs = [(1.0, 0.5, 0.0), (1.0, 0.0, 0.5)]
    calls, built, rec_x, x_lat, xs = _stub_run(tmp_path, monkeypatch, (parser, [[11], [17]], 2, 0.7, times, coeffs))
    assert built == [(parser, (3, 3, 8, 8), [[11], [17]], 2, 0.7)]
    assert calls[0][3] == {"record_process": True}                 # the origin pass records its trajectory
    assert len(calls) == 3                                          # 3 images, 2 attributes, 4 rows: chunks of 2
    noises = []
    for c, (x, sch, noise, kw) in enumerate(calls[1:]):
        j0 = 2 * c
        real = min(2, 3 - j0)
        assert set(kw) == {"compose"} and x.shape[0] == 4
        assert sch.t_edit == [500, 500, 700, 700] and sch.t_addnoise == [t_addnoise] * 2 + [0] * 2
        assert sch.hs_coeffs == [coeffs[0]] * 2 + [coeffs[1]] * 2
        masks, ref = kw["compose"]
        assert masks.shape == (2, 2, 8, 8) and ref.shape == (4, 2, 3, 8, 8)
        for j in range(2):
            src = j0 + min(j, real - 1)                              # padding repeats the chunk's last image
            assert torch.equal(ref[:, j], rec_x[:, src]) and torch.equal(x[j], x_lat[src])
            assert torch.equal(x[2 + j], x_lat[src])
        if t_addnoise:
            assert noise.shape[:2] == (sch.n_stochastic, 4) and torch.equal(noise[:, :2], noise[:, 2:])
            noises.append(noise[:, :real])
        else:
            assert noise is None
    if t_addnoise:   # one draw for the batch, independent of the chunking
        assert torch.cat(noises, dim=1).shape[1] == 3
    assert os.path.isfile("out/f_ngen6_region_compose.png") and len(xs) == 2
    # the composite of image j is row j of its chunk
    assert torch.equal(xs[1][:, 0, 0, 0], torch.tensor([0.0, 1.0, 0.0]))
