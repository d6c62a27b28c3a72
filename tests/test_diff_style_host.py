"""DiffStyle content injection (`--diff_style`) without a GPU: the flags, the cache name and format, the image
transform, the schedule, the content h of every step, the refusals, and the CPU oracle of the whole loop against the
reference's golden (tests/golden/diff_style_mini.npz, written by tests/golden/make_diff_style_golden.py).

The oracle here restates the loop Asyrp.run_diff_style composes from the reference's functions, on the oracle's
UNets and denoising_step (oracle/sampler.py); tests/test_diff_style_gpu.py compares the engine with it."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import diffusion_latent as dl, main as cli
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.schedule import make_sequences
from oracle import adm as oa, ddpm as od, sampler as osmp, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")

# the golden's run: 10 steps from t_0 = 999, edit from 500, eta = 1 below 300, dt_lambda from 950 on
N_STEP, T_EDIT, T_NOISE, DT_LAMBDA, DT_END = 10, 500, 300, 0.9985, 950
GAMMAS = (0.9, 0.6)
NOISE_SEED = 4321


# ------------------------------------------------------------------------------------------------------------------
# the CPU oracle of the loop
# ------------------------------------------------------------------------------------------------------------------
def style_images(S):
    """two contents then two styles: synthetic images in [-1, 1]"""
    return torch.cat([synth.synth_image((1, 3, S, S), seed=77 + k) for k in range(4)])


def pair_rows():
    """(content, style) of the four pairs, content-major"""
    return [(c, s) for c in range(2) for s in range(2)]


def oracle_model(family):
    if family == "ddpm":
        sd = synth.synth_state_dict(od.ddpm_param_shapes(od.MINI_CFG, 0), seed=1234, style="jittered")
        return sd, (lambda *a, **k: od.ddpm_forward(sd, od.MINI_CFG, *a, **k)), False, od.MINI_CFG["image_size"]
    sd = synth.synth_state_dict(oa.adm_param_shapes(oa.MINI_HP, 0), seed=1234, style="jittered")
    return sd, (lambda *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k)), True, oa.MINI_HP["image_size"]


def mini_logvar(learn_sigma):
    return None if learn_sigma else osmp.make_logvar(osmp.get_beta_schedule(beta_start=1e-4, beta_end=0.02,
                                                                           num_diffusion_timesteps=1000))


@torch.no_grad()
def oracle_invert_with_h(fwd, x0, seq, seq_next, learn_sigma):
    """precompute_pairs_with_h's loop (diffusion_latent.py:928-939): (x_T, {t: middle_h at t})"""
    betas, logv = osmp.make_betas(), mini_logvar(learn_sigma)
    x, h_dic, n = x0.clone(), {}, x0.shape[0]
    for i, j in zip(seq_next[1:], seq[1:]):
        x, _, _, h = osmp.denoising_step(x, torch.ones(n) * i, torch.ones(n) * j, model=fwd, logvars=logv, b=betas,
                                         eta=0.0, learn_sigma=learn_sigma)
        h_dic[i] = h.clone()
    return x, h_dic


@torch.no_grad()
def oracle_diff_style(fwd, x_T, h_c, seq, seq_next, gamma, use_mask, learn_sigma, noises, t_edit=T_EDIT,
                      t_noise=T_NOISE, dt_lambda=DT_LAMBDA, dt_end=DT_END):
    """the generation loop of one batch of rows: x_T [R] style latents, h_c[r] = {t: content h [1,C,h,w]} of row r;
    noises {t: [R][3][S][S]} for the eta = 1 steps.  Returns x after every step, [steps][R][3][S][S]."""
    betas, logv = osmp.make_betas(), mini_logvar(learn_sigma)
    x, n, traj = x_T.clone(), x_T.shape[0], []
    for i, j in zip(reversed(seq), reversed(seq_next)):
        dh = torch.cat([d[i] for d in h_c])
        x = osmp.denoising_step(x, torch.ones(n) * i, torch.ones(n) * j, model=fwd, logvars=logv, b=betas,
                                eta=1.0 if i < t_noise else 0.0, learn_sigma=learn_sigma, index=0, t_edit=t_edit,
                                hs_coeff=(gamma,), delta_h=dh, use_mask=use_mask, dt_lambda=dt_lambda, dt_end=dt_end,
                                noise=noises.get(i))[0]
        traj.append(x.clone())
    return torch.stack(traj)


def golden_noises(gi, use_mask, R, S, seq):
    g = torch.Generator().manual_seed(NOISE_SEED + 10 * gi + int(use_mask))
    return {i: torch.randn(R, 3, S, S, generator=g) for i in seq if i < T_NOISE}


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_oracle_matches_the_reference_golden(family):
    """inversion with h, the content h at t_0 and every generation step of 2 contents x 2 styles x 2 gamma x
    use_mask off / on, against the reference's own modules"""
    gold = np.load(os.path.join(G, "diff_style_mini.npz"))
    seq = gold["seq"].tolist()
    assert (seq, int(gold["t_edit"]), int(gold["t_noise"]), float(gold["dt_end"])) == \
        (make_sequences(999, N_STEP)[0], T_EDIT, T_NOISE, DT_END)
    assert float(gold["dt_lambda"]) == DT_LAMBDA and tuple(gold["gammas"].tolist()) == GAMMAS
    seq_next = [-1] + seq[:-1]
    _, fwd, learn_sigma, S = oracle_model(family)
    x0 = style_images(S)
    assert np.array_equal(x0.double().sum(dim=(1, 2, 3)).numpy(), gold[f"{family}_x0_sum"])
    tol = 2e-5  # the golden equals the oracle bit for bit on the machine that wrote it; other CPUs may round convs

    def close(a, b, what):
        b = torch.as_tensor(b)
        err = (a.double() - b.double()).abs().max().item()
        assert err <= tol * max(1.0, b.abs().max().item()), f"{family} {what}: max-abs err {err:.3e}"

    def pinned(t, key, dims, sub, what):
        """the golden keeps every tensor as per-entry fp64 sums and max |.| plus a sparse sample of its elements"""
        close(t.abs().amax(dim=dims), gold[key + "_absmax"], what + " max |.|")
        err = (t.double().sum(dim=dims) - torch.from_numpy(gold[key + "_sum"])).abs().max().item()
        assert err <= tol * t.double().abs().sum(dim=dims).max().item(), f"{family} {what} sums: {err:.3e}"
        close(sub(t), gold[key + "_sub"], what + " elements")

    def sub_x(t):
        return t[..., ::8, ::8]

    def sub_h(t):
        return t[..., ::4, ::4, ::4]

    xT, hs = [], []
    for k in range(4):
        x, h_dic = oracle_invert_with_h(fwd, x0[k:k + 1], seq, seq_next, learn_sigma)
        assert sorted(h_dic) == sorted(seq[:-1]) and seq[-1] not in h_dic
        xT.append(x)
        hs.append(h_dic)
    xT = torch.cat(xT)
    pinned(xT, f"{family}_xT", (1, 2, 3), sub_x, "x_T")
    assert gold[f"{family}_h_t"].tolist() == seq[:-1]
    H = torch.stack([torch.cat([hs[k][t] for t in seq[:-1]]) for k in range(4)])  # [image][step][C][h][w]
    close(H.abs().amax(dim=(2, 3, 4)), gold[f"{family}_h_absmax"], "h_dic max |h|")
    err = (H.double().sum(dim=(2, 3, 4)) - torch.from_numpy(gold[f"{family}_h_sum"])).abs().max().item()
    assert err <= tol * H.double().abs().sum(dim=(2, 3, 4)).max().item(), f"{family} h_dic sums: {err:.3e}"
    close(sub_h(H[0]), gold[f"{family}_h_c0"], "h_dic of content 0")
    h0 = torch.cat([fwd(xT[c:c + 1], torch.ones(1) * seq[-1])[3] for c in range(2)])
    pinned(h0, f"{family}_h0", (1, 2, 3), sub_h, "content h at t_0")
    h_c = [{**hs[c], seq[-1]: h0[c:c + 1]} for c in range(2)]
    rows = pair_rows()
    x_rows = xT[[2 + s for _, s in rows]]
    for gi, gamma in enumerate(GAMMAS):
        for use_mask in (False, True):
            traj = oracle_diff_style(fwd, x_rows, [h_c[c] for c, _ in rows], seq, seq_next, gamma, use_mask,
                                     learn_sigma, golden_noises(gi, use_mask, 4, S, seq))
            pinned(traj, f"{family}_traj_g{gi}_m{int(use_mask)}", (2, 3, 4), sub_x,
                   f"gamma {gamma} use_mask {use_mask}")


# ------------------------------------------------------------------------------------------------------------------
# host logic
# ------------------------------------------------------------------------------------------------------------------
def test_parser_flags_and_defaults():
    a = cli.build_parser().parse_args(["--config", "celeba.yml"])
    assert (a.diff_style, a.content_dir, a.style_dir, a.save_dir) == \
        (False, "./source_images/content", "./source_images/style", "./results")
    assert (a.hs_coeff, a.use_mask, a.dt_lambda, a.dt_end, a.t_noise, a.hs_coeff_list) == (0.9, False, 1.0, 950, 0, "")
    a = cli.build_parser().parse_args(["--config", "c.yml", "--diff_style", "--content_dir", "C", "--style_dir", "S",
                                       "--save_dir", "R", "--hs_coeff_list", "0.9 0.7", "--use_mask", "--t_noise",
                                       "200", "--dt_lambda", "0.9985", "--dt_end", "900"])
    assert (a.diff_style, a.content_dir, a.style_dir, a.save_dir, a.use_mask, a.t_noise, a.dt_lambda, a.dt_end) == \
        (True, "C", "S", "R", True, 200, 0.9985, 900)
    assert dl.diff_style_gammas(a.hs_coeff, a.hs_coeff_list) == [0.9, 0.7]
    assert dl.diff_style_gammas(0.5, "") == [0.5]


def test_cache_name_is_the_reference_expression():
    p = lambda path: dl.diff_style_cache_path("CelebA_HQ", 40, path)  # noqa: E731
    assert p("./source_images/content/face.png") == os.path.join("precomputed", "CelebA_HQ_inv40_content_face.pt")
    assert p("style/a.jpg") == os.path.join("precomputed", "CelebA_HQ_inv40_style_a.pt")
    assert p("a.png") == os.path.join("precomputed", "CelebA_HQ_inv40_a.pt")
    # the quirks of splitting at dots: a dotted directory cuts what lies before it, a dotted stem keeps its last part
    assert p("/data/v1.2/content/face.png") == os.path.join("precomputed", "CelebA_HQ_inv40_content_face.pt")
    assert p("/data/content/face.v2.png") == os.path.join("precomputed", "CelebA_HQ_inv40_v2.pt")
    assert p("/data.x/face.png") == os.path.join("precomputed", "CelebA_HQ_inv40_x_face.pt")


def _runner(tmp_path, **over):
    a = dict(t_0=999, n_inv_step=N_STEP, bs_train=2, re_precompute=False, user_defined_t_edit=T_EDIT, t_noise=T_NOISE,
             dt_lambda=DT_LAMBDA, dt_end=DT_END, sample_type="ddim", run_test=False, lpips=False, hs_coeff=0.9,
             hs_coeff_list="", content_dir=str(tmp_path / "C"), style_dir=str(tmp_path / "S"), use_mask=False,
             max_rows_per_replay=16, save_dir=str(tmp_path / "R"))
    a.update(over)
    cfg = NS(model=NS(var_type="fixedsmall"), data=NS(category="CelebA_HQ", image_size=32, channels=3),
             diffusion=NS(beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000))
    return Asyrp(NS(**a), cfg, device="cpu")


def _write_pngs(folder, names, sizes):
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    g = np.random.default_rng(len(names))
    for n, (w, h) in zip(names, sizes):
        Image.fromarray(g.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(os.path.join(folder, n))


def test_cache_round_trip_and_reference_format(tmp_path, monkeypatch):
    """an existing cache is read as is (a list in the reference's format, x0 saved on any device), so nothing is
    inverted; the file stays the reference's [x0, 0, x_T, {int t: h}]"""
    monkeypatch.chdir(tmp_path)
    _write_pngs("C", ["a.png"], [(40, 32)])
    r = _runner(tmp_path)
    os.makedirs("precomputed")
    path = dl.diff_style_cache_path("CelebA_HQ", N_STEP, "C/a.png")
    g = torch.Generator().manual_seed(0)
    ref = [torch.randn(1, 3, 32, 32, generator=g), 0, torch.randn(1, 3, 32, 32, generator=g),
           {t: torch.randn(1, 256, 8, 8, generator=g) for t in make_sequences(999, N_STEP)[0][:-1]}]
    torch.save(ref, path)
    out = r.precompute_pairs_with_h(model=None, img_paths=["C/a.png", "C/a.png"])
    assert r.n_inverted == 0 and list(out) == ["C/a.png"]
    got = out["C/a.png"]
    assert isinstance(got, list) and len(got) == 4 and got[1] == 0
    assert torch.equal(got[0], ref[0]) and torch.equal(got[2], ref[2])
    assert sorted(got[3]) == sorted(ref[3]) and all(torch.equal(got[3][t], ref[3][t]) for t in ref[3])
    # what the runner writes loads back the same way (temp file + rename)
    dl._atomic_save(got, path + ".copy")
    again = torch.load(path + ".copy", map_location="cpu", weights_only=True)
    assert torch.equal(again[2], ref[2]) and sorted(again[3]) == sorted(ref[3])
    assert not [f for f in os.listdir("precomputed") if ".tmp." in f]


def test_image_transform_matches_torchvision(tmp_path):
    """centre crop to the shorter side, Resize((S, S)), ToTensor, Normalize(0.5, 0.5), as the reference composes it
    (landscape and portrait images)"""
    from PIL import Image
    from torchvision import transforms
    _write_pngs(str(tmp_path), ["wide.png", "tall.png", "sq.jpg"], [(50, 30), (20, 44), (33, 33)])
    for name in ("wide.png", "tall.png", "sq.jpg"):
        path = os.path.join(str(tmp_path), name)
        got = dl.diff_style_image(path, 16)
        im = Image.open(path).convert("RGB")
        w, h = im.size
        im = transforms.CenterCrop(h)(im) if w > h else transforms.CenterCrop(w)(im)
        ref = transforms.Compose([transforms.Resize((16, 16)), transforms.ToTensor(),
                                  transforms.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])(im)
        assert got.shape == (1, 3, 16, 16) and torch.equal(got[0], ref)
        # the crop by hand: the central square of the array
        arr = np.asarray(Image.open(path).convert("RGB"))
        s = min(arr.shape[:2])
        y, x = int(round((arr.shape[0] - s) / 2.0)), int(round((arr.shape[1] - s) / 2.0))
        sq = Image.fromarray(arr[y:y + s, x:x + s]).resize((16, 16), Image.BILINEAR)
        hand = torch.from_numpy(np.asarray(sq).copy()).permute(2, 0, 1).float() / 255.0 * 2.0 - 1.0
        assert (got[0] - hand).abs().max().item() <= 2.0 / 255 + 1e-6


def test_schedule_steps(tmp_path):
    """the generation grid is the inversion grid reversed; edit from t_edit, eta = 1 below t_noise, dt_lambda from
    dt_end on (--dt_end, not save_image's 999)"""
    r = _runner(tmp_path)
    sch = r.diff_style_schedule(0.7)
    seq, seq_next = make_sequences(999, N_STEP)
    assert [(s.t, s.t_next) for s in sch.steps] == list(zip(reversed(seq), reversed(seq_next)))
    assert sch.hs_coeff == (0.7,)
    assert [s.t for s in sch.steps if s.edit] == [t for t in reversed(seq) if t >= T_EDIT]
    # eta = 1 below t_noise; the last step (t_next = -1) has c1 = 0 and draws nothing
    assert [s.t for s in sch.steps if s.stochastic] == [t for t in reversed(seq) if 0 < t < T_NOISE]
    ac = (1.0 - osmp.make_betas()).cumprod(0)
    for s in sch.steps:
        an = torch.tensor(1.0) if s.t_next == -1 else ac[s.t_next]
        if s.t >= DT_END:
            assert s.c1 == 0.0 and s.c2 == float((1 - an).sqrt() * DT_LAMBDA)
        elif s.t >= T_NOISE:
            assert s.c1 == 0.0 and s.c2 == float((1 - an).sqrt())
    assert any(s.t >= DT_END for s in sch.steps)
    late = _runner(tmp_path, dt_end=999).diff_style_schedule(0.7)
    assert late.steps[0].c2 == float((1 - ac[late.steps[0].t_next]).sqrt() * DT_LAMBDA)
    assert _runner(tmp_path, dt_lambda=1.0).diff_style_schedule(0.7).steps[0].c2 == \
        float((1 - ac[sch.steps[0].t_next]).sqrt())


@pytest.mark.parametrize("n_step,t_edit", [(N_STEP, T_EDIT), (40, 400), (40, 0), (7, 999), (1000, 1)])
def test_every_edit_step_has_a_content_h(n_step, t_edit):
    """the inversion's keys seq_inv[:-1] plus t_0 cover every generation step: delta_hs has one row per edit step,
    in step order; a missing t is an error"""
    seq, seq_next = make_sequences(999, n_step)
    inv_keys = [i for i, _ in zip(seq_next[1:], seq[1:])]
    assert inv_keys == seq[:-1]
    h = [{**{t: torch.full((1, 2, 1, 1), float(t) + 0.5 * r) for t in inv_keys}, seq[-1]: torch.zeros(1, 2, 1, 1)}
         for r in range(3)]
    gen = [i for i, _ in zip(reversed(seq), reversed(seq_next))]
    edit_ts = [t for t in gen if t >= t_edit]
    assert all(t in h[0] for t in gen)
    dh = dl.diff_style_delta_hs(h, edit_ts)
    assert dh.shape == (len(edit_ts), 3, 2, 1, 1)
    for k, t in enumerate(edit_ts):
        for r in range(3):
            assert torch.equal(dh[k, r], h[r][t][0])
    del h[1][seq[0]]
    if seq[0] in edit_ts:
        with pytest.raises(KeyError):
            dl.diff_style_delta_hs(h, edit_ts)


def test_refusals(tmp_path, monkeypatch):
    """every refusal is a ValueError raised before any model is loaded"""
    monkeypatch.chdir(tmp_path)
    _write_pngs("C", ["a.png", "b.png"], [(32, 32)] * 2)
    _write_pngs("S", ["x.jpg"], [(32, 32)])
    os.makedirs("E")
    with open("E/notes.txt", "w") as f:
        f.write("no image\n")

    def load(*a, **k):
        raise AssertionError("a model was loaded")

    monkeypatch.setattr(Asyrp, "load_pretrained_model", load)
    ok = _runner(tmp_path)
    c, s, g = ok.diff_style_setup()
    assert (c, s, g) == ([str(tmp_path / "C" / "a.png"), str(tmp_path / "C" / "b.png")], [str(tmp_path / "S" / "x.jpg")],
                         [0.9])
    assert _runner(tmp_path, hs_coeff_list="0.9 0.5").diff_style_setup()[2] == [0.9, 0.5]
    bad = [dict(user_defined_t_edit=None), dict(content_dir=str(tmp_path / "missing")), dict(style_dir="E"),
           dict(style_dir=None), dict(sample_type="ddpm"), dict(run_test=True), dict(lpips=True),
           dict(hs_coeff=0.5, hs_coeff_list="0.9 0.7"), dict(hs_coeff_list="0.9 x"), dict(hs_coeff_list=" ")]
    for over in bad:
        with pytest.raises(ValueError):
            _runner(tmp_path, **over).run_diff_style()
    # two images that would share one inversion cache
    _write_pngs("S", ["a.png"], [(32, 32)])
    _write_pngs("C2/S", ["a.jpg"], [(32, 32)])
    with pytest.raises(ValueError, match="share the inversion cache"):
        _runner(tmp_path, content_dir="C2/S", style_dir="S").run_diff_style()


def test_main_dispatch_refuses_before_loading(tmp_path, monkeypatch):
    """`main --diff_style` with --run_test returns 1 and loads nothing"""
    monkeypatch.chdir(tmp_path)
    name = "celeba.yml"  # one of the reference's configs, built in

    def load(*a, **k):
        raise AssertionError("a model was loaded")

    monkeypatch.setattr(Asyrp, "load_pretrained_model", load)
    assert cli.main(["--diff_style", "--run_test", "--config", name, "--user_defined_t_edit", "400"]) == 1
    assert cli.main(["--diff_style", "--config", name]) == 1  # no --user_defined_t_edit


def test_chunks_hold_whole_pairs():
    """rows are (pair, gamma), pair-major; a replay holds whole pairs, every replay the same row count"""
    ppc, chunks = dl.plan_sweep(6, 3, 16)
    assert ppc == 5 and chunks == [[0, 1, 2, 3, 4], [5]]
    ppc, chunks = dl.plan_sweep(4, 3, 2)
    assert ppc == 1 and len(chunks) == 4
