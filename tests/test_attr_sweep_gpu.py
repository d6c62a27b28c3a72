"""Attribute sweeps on the GPU: the per-row DDIM update against the scalar kernel, UNetEngine.sample() with a
RowSchedule against one single-block run per row (bit for bit) on the reduced DDPM / ADM UNets and at 256² CelebA with
the shipped 'smiling' DeltaBlock, a never-edited row against the origin pass, and `--run_test --attr_sweep` against
one `--run_test --edit_attr` per attribute."""
import csv
import os
import shutil
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import yaml

from asyrp_official_b200 import _lib, main as cli, modules, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp, _read_tsv
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import adm as oa, clip_text as oct, ddpm as od, sampler as osmp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


# ------------------------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 3, 16])
@pytest.mark.parametrize("Ce", [3, 6])
def test_ddim_update_rows_equals_the_scalar_kernel(cuda_device, N, Ce):
    """rows mixing eta = 0 and eta = 1 (and c1 = 0 at t_next = -1): row n == ddim_update with row n's scalars, z passed
    only for c1 != 0; x0_out and in-place x_next too"""
    dev = cuda_device
    g = torch.Generator().manual_seed(100 + N)
    S = 13
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 8)
    for k in (7, 3, 0):  # steps run from t = 999: the last (t_next = -1), a middle one, the first
        scheds = [Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=(1000 if n % 2 else 0)) for n in range(N)]
        st = [s.steps[k] for s in scheds]
        c12 = torch.tensor([[s.c1, s.c2] for s in st], dtype=torch.float32, device=dev)
        x = torch.randn(N, 3, S, S, generator=g).to(dev)
        et = torch.randn(N, Ce, S, S, generator=g).to(dev)
        em = torch.randn(N, Ce, S, S, generator=g).to(dev)
        z = torch.randn(N, 3, S, S, generator=g).to(dev)
        out, x0 = torch.empty_like(x), torch.empty_like(x)
        ops.ddim_update_rows(x, et, em, z, out, x0, st[0].at, st[0].an, c12)
        inplace = x.clone()
        ops.ddim_update_rows(inplace, et, em, z, inplace, None, st[0].at, st[0].an, c12)
        torch.cuda.synchronize()
        assert torch.equal(inplace, out)
        for n, s in enumerate(st):
            o1, x01 = torch.empty_like(x[n:n + 1]), torch.empty_like(x[n:n + 1])
            ops.ddim_update(x[n:n + 1], et[n:n + 1], em[n:n + 1], z[n:n + 1] if s.c1 != 0.0 else None, o1, x01,
                            s.at, s.an, s.c1, s.c2)
            assert torch.equal(out[n:n + 1], o1), f"N={N} step {k} row {n} (c1={s.c1})"
            assert torch.equal(x0[n:n + 1], x01)
        assert any(s.c1 != 0.0 for s in st) == (k != 7 and N > 1)
    with pytest.raises(_lib.AsyrpError):
        ops.ddim_update_rows(x, et, em, z, out, None, 0.5, 0.6, c12[:-1] if N > 1 else c12.cpu())


# ------------------------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------------------------
def _module(family, n_delta, cfg=None):
    if family == "ddpm":
        cfg = cfg or od.MINI_CFG
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
    else:
        m = modules._create_adm(cfg or oa.MINI_HP)
    m.setattr_layers(n_delta)
    return m


def _single(family, sd, k, dev, cfg=None):
    """the UNet of `sd` with only DeltaBlock k packed (as layer_0)"""
    m = _module(family, 1, cfg)
    one = {n: v for n, v in sd.items() if not n.startswith("layer_")}
    one.update({"layer_0." + n[len(f"layer_{k}."):]: v for n, v in sd.items() if n.startswith(f"layer_{k}.")})
    m.load_state_dict(one)
    return m.to(dev)


def _check_rows(eng, singles, x, rs, nz, dev, what):
    """every row of the sweep == its own Schedule on the engine with only its block packed, bit for bit"""
    out = eng.sample(x.to(dev), rs, noise=nz.to(dev) if nz is not None else None)
    n_graphs = len(eng.graphs)
    again = eng.sample(x.to(dev), rs, noise=nz.to(dev) if nz is not None else None)
    assert torch.equal(out, again) and len(eng.graphs) == n_graphs, f"{what}: the replay must reuse the graph"
    for n, row in enumerate(rs.rows):
        k = max(range(rs.n_delta), key=lambda i: abs(rs.hs_coeffs[n][1 + i]))
        c0, s = rs.hs_coeffs[n][0], rs.hs_coeffs[n][1 + k]
        single = _single_schedule(rs, n, c0, s)
        zr = rs.noise_rows(n, nz).contiguous().to(dev) if single.n_stochastic else None
        one = singles[k].engine.sample(x[n:n + 1].to(dev), single, noise=zr)
        assert torch.equal(out[n:n + 1], one), f"{what}: row {n} (block {k}, t_edit {rs.t_edit[n]}, t_addnoise " \
                                               f"{rs.t_addnoise[n]}) != its single-block run"
    return out


def _single_schedule(rs, n, c0, s):
    return Schedule(osmp.make_betas(), None, None, t_edit=rs.t_edit[n], t_addnoise=rs.t_addnoise[n], hs_coeff=(c0, s),
                    pairs=[(st.t, st.t_next) for st in rs.steps])


def _noise(rs, R, S, g):
    return torch.randn(rs.n_stochastic, R, 3, S, S, generator=g) if rs.n_stochastic else None


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_sweep_rows_equal_single_block_runs(cuda_device, family):
    """K = 3 seeded DeltaBlocks, three t_edit / t_addnoise pairs, two images, one row with another c0, and a row
    whose t_edit lies above every step, which equals the origin pass"""
    dev = cuda_device
    m = _module(family, 3)
    synthetic.randomize_(m, 1234, "jittered")
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    singles = [_single(family, sd, k, dev) for k in range(3)]
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 6)
    te, ta = [700, 500, 300], [0, 450, 650]
    rows = []   # (block, image, t_edit, t_addnoise, c0, scale)
    for k in range(3):
        for i in range(2):
            rows.append((k, i, te[k], ta[k], 1.0, 1.0 + 0.25 * k))
    rows.append((1, 0, 500, 450, 0.9, -0.7))   # its own c0
    rows.append((2, 1, 10 ** 9, 0, 1.0, 1.0))  # never edits
    g = torch.Generator().manual_seed(5)
    imgs = torch.randn(2, 3, 32, 32, generator=g)
    x = torch.stack([imgs[r[1]] for r in rows])
    coeffs = [tuple([r[4]] + [r[5] if j == r[0] else 0.0 for j in range(3)]) for r in rows]
    rs = RowSchedule(betas, seq, seq_next, [r[2] for r in rows], [r[3] for r in rows], coeffs)
    assert len({tuple(s.edit_rows) for s in rs.steps}) >= 3 and rs.n_stochastic
    assert not any(s.edit_rows[-1] for s in rs.steps)
    nz = _noise(rs, len(rows), 32, g)
    out = _check_rows(m.engine, singles, x, rs, nz, dev, family)
    origin = m.engine.sample(x[-1:].to(dev), Schedule(betas, seq, seq_next, t_edit=10 ** 9, t_addnoise=0,
                                                      hs_coeff=(1.0,), edit=False))
    assert torch.equal(out[-1:], origin), f"{family}: the never-edited row != the origin pass"
    # oracle: one row within the trajectory bound
    fwd = (lambda *a, **k: od.ddpm_forward(sd1, od.MINI_CFG, *a, **k)) if family == "ddpm" else \
        (lambda *a, **k: oa.adm_forward(sd1, oa.MINI_HP, *a, **k))
    n = 2  # block 1, t_edit 500, t_addnoise 450
    sd1 = {k: v.cpu() for k, v in singles[1].state_dict().items()}
    noises = {s.t: nz[zi, n:n + 1] for zi, s in enumerate([s for s in rs.steps if s.stochastic])}
    ref = osmp.run_trajectory(fwd, x[n:n + 1], betas=betas, seq=seq, seq_next=seq_next, t_edit=500, t_addnoise=450,
                              index=0, hs_coeff=(1.0, 1.25), learn_sigma=family == "adm", noises=noises)
    e, mx = (out[n:n + 1].double().cpu() - ref.double()).abs().max().item(), ref.abs().max().item()
    print(f"\n{family}: sweep row vs the oracle: max-abs {e:.3e} of {mx:.3e}")
    assert e <= 2e-3 * max(1.0, mx), f"{family}: row {n} vs the oracle: max-abs {e:.3e} of {mx:.3e}"
    # malformed
    with pytest.raises(_lib.AsyrpError):
        m.engine.sample(x[:2].to(dev), rs, noise=nz.to(dev))
    two = RowSchedule(betas, seq, seq_next, [500], [0], [(1.0, 1.0, 0.5, 0.0)])
    with pytest.raises(_lib.AsyrpError):
        m.engine.sample(x[:1].to(dev), two)
    with pytest.raises(_lib.AsyrpError):
        singles[0].engine.sample(x[:1].to(dev), RowSchedule(betas, seq, seq_next, [500], [0], [(1.0, 1.0, 0.0, 0.0)]))


def test_sweep_at_256_with_the_shipped_block(cuda_device):
    """DDPM CelebA-HQ 256²: the shipped 'smiling' DeltaBlock and two seeded ones, one image, 40 steps, each row its
    own t_edit / t_addnoise; the smiling row also against the reference's own trajectory of that image"""
    dev = cuda_device
    gold = np.load(os.path.join(G, "ddpm_celeba_smiling_traj40_b16.npz"))
    m = _module("ddpm", 3, od.CELEBA_CFG)
    synthetic.randomize_(m, 1234, "torch_default")
    seeded = _module("ddpm", 3, od.CELEBA_CFG)
    synthetic.randomize_(seeded, 99, "jittered")
    m.layer_0.load_state_dict(torch.load(os.path.join(G, "checkpoint", "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth"),
                                         map_location="cpu", weights_only=True)["0"])
    for k in (1, 2):
        getattr(m, f"layer_{k}").load_state_dict(getattr(seeded, f"layer_{k}").state_dict())
    del seeded
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    seq = gold["seq"].tolist()
    seq_next = [-1] + seq[:-1]
    B = int(gold["batch"])
    x = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(int(gold["x_seed"])))[:1]
    gn = torch.Generator().manual_seed(int(gold["noise_seed"]))
    noises = {i: torch.randn(B, 3, 256, 256, generator=gn)[:1] for i in seq}
    te, ta = [int(gold["t_edit"]), 700, 300], [int(gold["t_addnoise"]), 0, 400]
    rs = RowSchedule(osmp.make_betas(), seq, seq_next, te, ta, [(1.0, 1.0, 0.0, 0.0), (1.0, 0.0, 0.8, 0.0),
                                                                (1.0, 0.0, 0.0, 1.2)])
    nz = torch.stack([torch.cat([noises[s.t]] * 3) for s in rs.steps if s.stochastic])
    singles = [_single("ddpm", sd, k, dev, od.CELEBA_CFG) for k in range(3)]
    out = _check_rows(m.engine, singles, x.expand(3, -1, -1, -1).contiguous(), rs, nz, dev, "celeba256")
    ref = torch.from_numpy(gold["x0_sub"][:1]).double()
    e = (out[:1, :, ::4, ::4].double().cpu() - ref).abs().max().item()
    mx = float(gold["x0_absmax_per_sample"][0])
    print(f"\nceleba256: smiling row vs the reference: max-abs {e:.4f} of {mx:.2f} -> {e / mx:.2e}")
    assert e <= 1e-3 * max(1.0, mx)
    del m, singles
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# runner
# ------------------------------------------------------------------------------------------------------------------
CFG = od.MINI_CFG
DIC = {"smiling": (["face"], ["smiling face"]), "car": (["face"], ["a photo of a red sports car on the street"]),
       "gogh": (["photo"], ["painting by gogh"])}
TEMPLATES = ["a photo of a {}.", "a rendering of a {}."]


def _scratch(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    os.makedirs("utils")
    with open("utils/text_dic.py", "w") as f:
        f.write(f"SRC_TRG_TXT_DIC = {DIC!r}\n")
    with open("templates.py", "w") as f:
        f.write(f"imagenet_templates = {TEMPLATES!r}\n")
    shutil.copy(os.path.join(G, "lpips", "celeba_LPIPS_distance_x0_t.tsv"), "utils/mini_LPIPS_distance_x0_t.tsv")
    texts = [t for src, trg in DIC.values() for t in src + trg]
    n = synthetic.write_clip_vocab("bpe.txt.gz", synthetic.clip_bpe_merges(
        texts + [t.format(c) for t in TEMPLATES for c in texts]))
    sd = synthetic.clip_text_state_dict(seed=7, width=128, layers=2, vocab=n, embed_dim=128)
    sd.update(synthetic.clip_image_state_dict(seed=7, width=128, layers=2, patch=16, grid=14, embed_dim=128))
    torch.save(sd, "clip.pt")
    tok = oct.SimpleTokenizer("bpe.txt.gz")
    table = _read_tsv("utils/mini_LPIPS_distance_x0_t.tsv")
    t_edit = {}
    for k, (s, t) in DIC.items():
        cos = oct.cosine(oct.encode_text(sd, tok.tokenize(s)), oct.encode_text(sd, tok.tokenize(t))).item()
        t_edit[k] = next(tt for tt, v in table if v >= 0.33 * cos)
    for i, a in enumerate(DIC):
        m = _module("ddpm", 1)
        synthetic.randomize_(m, seed=11 + i, style="jittered")
        torch.save({"0": {k: v.clone() for k, v in m.layer_0.state_dict().items()}}, f"checkpoint/{a}_0.pth")
    cfg = {"data": dict(dataset="CelebA_HQ", category="CelebA_HQ", image_size=CFG["image_size"], channels=3,
                        rescaled=True, num_workers=0),
           "model": dict(type="simple", in_channels=3, out_ch=3, ch=CFG["ch"], ch_mult=list(CFG["ch_mult"]),
                         num_res_blocks=CFG["num_res_blocks"], attn_resolutions=list(CFG["attn_resolutions"]),
                         dropout=0.0, var_type="fixedsmall", ema_rate=0.999, ema=True, resamp_with_conv=True),
           "diffusion": dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
           "sampling": dict(batch_size=4, last_only=True)}
    with open("mini.yml", "w") as f:
        yaml.safe_dump(cfg, f)
    argv = ["--run_test", "--config", os.path.join(str(tmp_path), "mini.yml"), "--exp", "./runs/sweep", "--do_train",
            "0", "--do_test", "1", "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999",
            "--n_inv_step", "6", "--n_train_step", "6", "--n_test_step", "6", "--load_random_noise",
            "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
            "--get_h_num", "1", "--save_x_origin"]
    return argv, t_edit


def _run(argv, dev):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config, device=dev)
    return r, r.run_test()


@pytest.mark.parametrize("max_rows", [16, 4])
def test_run_test_attr_sweep_equals_one_run_per_attribute(cuda_device, tmp_path, monkeypatch, max_rows):
    """three attributes whose CLIP cosines pick three t_edit values: every row of the sweep's grid equals the
    --edit_attr run of that attribute with --user_defined_t_edit set to the t_edit the sweep chose; the S_dir table
    scores each row with its own texts and names its attribute"""
    argv, t_edit = _scratch(tmp_path, monkeypatch)
    assert len(set(t_edit.values())) == 3, t_edit
    attrs = list(DIC)
    r, res = _run(argv + ["--attr_sweep", " ".join(attrs), "--manual_checkpoint_name", "attribute_0.pth",
                          "--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz", "--DirectionalClipSmilarity",
                          "--text_templates", "templates.py", "--max_rows_per_replay", str(max_rows)], cuda_device)
    rows = res[("test", 1)]
    assert len(rows) == 1 + len(attrs)
    assert r.sweep_times == {a: (t_edit[a], 0) for a in attrs}
    for k, a in enumerate(attrs):
        _, one = _run(argv + ["--edit_attr", a, "--manual_checkpoint_name", f"{a}_0.pth", "--user_defined_t_edit",
                              str(t_edit[a])], cuda_device)
        origin, edit = one[("test", 1)]
        assert torch.equal(rows[0], origin)
        assert torch.equal(rows[1 + k], edit), f"attribute {a} (t_edit {t_edit[a]})"
    path = os.path.join(r.args.test_image_folder, "test_1_0_ngen6_directional_clip.tsv")
    with open(path) as f:
        table = list(csv.reader(f, delimiter="\t"))
    assert table[0] == ["image", "tuple", "hs_coeff", "S_dir", "attr"]
    assert [(int(t[1]), int(t[0]), t[4]) for t in table[1:]] == [(k, i, a) for k, a in enumerate(attrs)
                                                                  for i in range(2)]
    assert r.directional_clip["test_1_0"].shape == (3, 2)
