"""Host-side logic and the C-ABI surface (no GPU): library loads and exports every declared symbol, state-dict /
checkpoint compatibility of the module mirrors, schedule coefficients, config / CLI surface, loud failure without
a CUDA device."""
import argparse
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from asyrp_official_b200 import _lib
    from asyrp_official_b200.build import build_library
    build_library()
    hdr = open(os.path.join(ROOT, "include", "asyrp_b200.h")).read()
    declared = set(re.findall(r"\b(asyrp_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 15
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/asyrp_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert lib.asyrp_last_error() is not None
    # pure host helper (no device): tile bookkeeping for the GroupNorm partial sums
    assert lib.asyrp_conv_stats_tiles(256, 256, 256, 0) == 512  # 16x8-pixel tiles, 128 channels each
    assert lib.asyrp_conv_stats_tiles(256, 256, 128, 1) == 512  # 8x16-pixel halo tiles, one slot each
    assert lib.asyrp_conv_tile_config(256, 256, 128, 1) == 128 * 16 + 1
    assert lib.asyrp_conv_tile_config(16, 16, 128, 1) == 64 * 16 + 1   # small layer: more, narrower tiles
    assert lib.asyrp_conv_stats_tiles(8, 8, 512, 1) == 4        # 2 samples per tile, one slot per lane quarter


_UNTILEABLE_PROBE = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from asyrp_official_b200 import _lib
lib = _lib.load()
for H, W in ((4, 12), (3, 3), (1, 96)):
    for has3 in (0, 1):
        print("stats_tiles", H, W, has3, lib.asyrp_conv_stats_tiles(H, W, 64, has3), flush=True)
        print("tile_config", H, W, has3, lib.asyrp_conv_tile_config(H, W, 64, has3), flush=True)
        d = _lib.AsyrpConvDesc()
        d.N, d.H, d.W, d.Cout, d.nseg = 2, H, W, 64, 1
        d.seg[0].src, d.seg[0].C, d.seg[0].mode = None, 64, has3
        h = C.c_void_p()
        rc = lib.asyrp_conv_create(C.byref(d), C.byref(h))
        print("create", H, W, has3, rc, bool(h.value), lib.asyrp_last_error().decode(), flush=True)
for H, W in ((2, 0), (0, 0)):  # empty images
    print("stats_tiles", H, W, 0, lib.asyrp_conv_stats_tiles(H, W, 64, 0), flush=True)
    print("tile_config", H, W, 0, lib.asyrp_conv_tile_config(H, W, 64, 0), flush=True)
"""


def test_untileable_conv_geometry_is_reported_not_fatal():
    """A width that no 128-pixel tile fits (W = 12 for H = 4, 3x3 images, a T = 96 GEMM row) or an empty image is
    unsupported: the tile queries return 0 and asyrp_conv_create returns ASYRP_ERR_INVALID before touching a device,
    instead of dividing by zero in the tiler.  Run in a subprocess so that a crash is reported as a failure of this
    test."""
    import subprocess
    import sys
    from asyrp_official_b200.build import build_library
    build_library()
    r = subprocess.run([sys.executable, "-c", _UNTILEABLE_PROBE, ROOT], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, f"probe exited with {r.returncode}\n{r.stdout}\n{r.stderr}"
    lines = [ln.split(" ", 4) for ln in r.stdout.splitlines()]
    assert len(lines) == 22, r.stdout
    for ln in lines:
        if ln[0] == "create":
            rc, made, msg = ln[4].split(" ", 2)
            assert rc == "-1" and made == "False" and "cannot tile" in msg, ln
        else:
            assert ln[4] == "0", ln
    # geometries that tile still do
    from asyrp_official_b200 import _lib
    lib = _lib.load()
    for H, W in ((16, 16), (24, 24), (1, 200)):
        assert lib.asyrp_conv_stats_tiles(H, W, 64, 0) > 0 and lib.asyrp_conv_tile_config(H, W, 64, 0) > 0


def test_no_cpu_fallback():
    from asyrp_official_b200 import modules
    from asyrp_official_b200._lib import AsyrpError
    from asyrp_official_b200.configs import load_config
    cfg = load_config("celeba")
    cfg.model.ch, cfg.model.ch_mult, cfg.data.image_size = 64, [1, 2], 32
    m = modules.DDPM(cfg)
    if not torch.cuda.is_available():
        with pytest.raises(AsyrpError):
            m(torch.zeros(1, 3, 32, 32), torch.zeros(1))


def test_param_inventory_matches_oracle_inventory():
    from asyrp_official_b200 import arch
    from oracle import adm as oa, ddpm as od
    pairs = [(arch.ddpm_arch(**od.CELEBA_CFG), od.ddpm_param_shapes(od.CELEBA_CFG, 2)),
             (arch.ddpm_arch(**od.MINI_CFG), od.ddpm_param_shapes(od.MINI_CFG, 2)),
             (arch.adm_arch(**oa.AFHQ_HP), oa.adm_param_shapes(oa.AFHQ_HP, 2)),
             (arch.adm_arch(**oa.IMAGENET_HP), oa.adm_param_shapes(oa.IMAGENET_HP, 2)),
             (arch.adm_arch(**oa.MINI_HP), oa.adm_param_shapes(oa.MINI_HP, 2))]
    for a, o in pairs:
        mine = {k: tuple(v) for k, v in arch.param_shapes(a, 2).items()}
        assert mine == {k: tuple(v) for k, v in o.items()}


def test_module_state_dict_and_delta_checkpoint_format():
    """same keys as the reference modules; a Δh checkpoint {"0": layer_0.state_dict()} loads with all keys matched
    (diffusion_latent.py:674-676), on the reference's shipped 'smiling' checkpoint (tests/golden/checkpoint/)."""
    from asyrp_official_b200 import modules, synthetic
    from asyrp_official_b200.configs import load_config
    m = modules.DDPM(load_config("celeba.yml"))
    m.setattr_layers(1)
    keys = set(m.layer_0.state_dict())
    assert keys == {"conv1.weight", "conv1.bias", "temb_proj.weight", "temb_proj.bias", "norm2.weight", "norm2.bias",
                    "conv2.weight", "conv2.bias"}
    v0 = m._version
    ck = os.path.join(ROOT, "tests", "golden", "checkpoint", "smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth")
    sd = torch.load(ck, map_location="cpu", weights_only=True)["0"]
    res = m.layer_0.load_state_dict(sd)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(m.layer_0.conv1.weight, sd["conv1.weight"])
    assert m._version > v0  # engine weights are re-packed after any load_state_dict
    a = modules.i_DDPM("AFHQ")
    a.setattr_layers(1)
    assert set(a.layer_0.state_dict()) == {"in_layers.0.weight", "in_layers.0.bias", "in_layers.2.weight",
                                           "in_layers.2.bias", "emb_layers.1.weight", "emb_layers.1.bias",
                                           "out_layers.0.weight", "out_layers.0.bias", "out_layers.3.weight",
                                           "out_layers.3.bias"}
    # zero_module() layers of the ADM family start at zero like the reference's (unet.py:252-254,336,657)
    assert a.state_dict()["out.2.weight"].abs().max() == 0 and a.state_dict()["input_blocks.1.0.out_layers.3.weight"].abs().max() == 0
    synthetic.randomize_(a, 7)
    assert a.state_dict()["out.2.weight"].abs().max() > 0
    with pytest.raises(ValueError):
        modules.i_DDPM("LSUN")
    assert modules.guided_Diffusion("MetFACE").arch.mid_ch == 512 and modules.i_DDPM("IMAGENET").arch.mid_ch == 1024


def test_schedule_coefficients_match_oracle_step():
    """Schedule's host-side coefficients reproduce the oracle's denoising_step update bit-for-bit (fp32)"""
    from asyrp_official_b200.schedule import Schedule, make_sequences
    from oracle import sampler as osmp
    betas = osmp.make_betas()
    seq, nxt = make_sequences(999, 40)
    assert (seq, nxt) == osmp.make_sequences(999, 40)
    sch = Schedule(betas, seq, nxt, t_edit=500, t_addnoise=200, hs_coeff=(1.0, 0.5))
    # 8 steps have t < t_addnoise, but the last one (t_next = -1, alpha-bar_next = 1) has a zero noise coefficient
    assert sch.n_edit == 20 and sch.n_stochastic == 7 and len(sch.steps) == 40
    assert sch.steps[0].t == 999 and sch.steps[-1].t_next == -1 and sch.steps[-1].an == 1.0
    g = torch.Generator().manual_seed(0)
    x, e, em, z = (torch.randn(1, 3, 4, 4, generator=g) for _ in range(4))
    for s in (sch.steps[0], sch.steps[25], sch.steps[-1]):
        model = lambda xt, t, **k: (e, em, None, None)  # noqa: E731
        eta = 1.0 if s.c1 != 0.0 else 0.0
        ref, x0, _, _ = osmp.denoising_step(x, torch.ones(1) * s.t, torch.ones(1) * s.t_next, model=model, b=betas,
                                            eta=eta, index=0, t_edit=500, hs_coeff=(1.0, 0.5), noise=z)
        at, an = torch.tensor(s.at), torch.tensor(s.an)
        x0_mine = (x - em * (1 - at).sqrt()) / at.sqrt()
        mine = an.sqrt() * x0_mine + torch.tensor(s.c2) * e
        if s.c1 != 0.0:
            mine = mine + torch.tensor(s.c1) * z
        assert torch.equal(x0, x0_mine) and torch.allclose(ref, mine, rtol=0, atol=1e-6)


def test_config_and_cli_surface(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.configs import load_config
    c = load_config("afhq.yml")
    assert c.data.dataset == "AFHQ" and c.model.ch_mult == [1, 1, 2, 2, 4, 4] and c.diffusion.beta_end == 0.02
    y = tmp_path / "my.yml"
    y.write_text("data:\n  dataset: LSUN\n  category: church_outdoor\n  image_size: 256\n  channels: 3\n"
                 "model:\n  ch: 128\n  var_type: fixedsmall\ndiffusion:\n  beta_start: 0.0001\n  beta_end: 0.02\n"
                 "  num_diffusion_timesteps: 1000\n")
    assert load_config(str(y)).data.category == "church_outdoor"
    with pytest.raises(FileNotFoundError):
        load_config("nope.yml")
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml", "--exp", "./runs/smiling",
                                           "--n_train_step", "40", "--user_defined_t_edit", "500"])
    assert args.exp == "./runs/smiling_LC_CelebA_HQ_t999_ninv40_ngen40"  # main.py:235
    assert args.lpips_edit_th == 0.33 and args.n_test_step == 40 and args.bs_train == 1 and args.seed == 1234
    assert os.path.isdir(args.test_image_folder)


def test_runner_host_logic():
    """sequences, hs_coeff scaling (diffusion_latent.py:626,654,659) and LPIPS-table t_edit lookup (the reference's
    CelebA tables, tests/golden/lpips/)"""
    from asyrp_official_b200.configs import load_config
    from asyrp_official_b200.diffusion_latent import Asyrp
    a = argparse.Namespace(user_defined_t_edit=None, user_defined_t_addnoise=None, clip_cosine=0.8, config="celeba.yml",
                           lpips_table_dir=os.path.join(ROOT, "tests", "golden", "lpips"), add_noise_from_xt=True)
    r = Asyrp(a, load_config("celeba"), device="cpu")
    assert r.betas.dtype == torch.float32 and r.logvar.shape == (1000,)
    r.set_t_edit_t_addnoise(LPIPS_th=0.33, LPIPS_addnoise_th=1.2)
    assert 400 <= r.t_edit <= 560 and r.t_addnoise == 167  # SURVEY.md Appendix D
    a2 = argparse.Namespace(user_defined_t_edit=500, user_defined_t_addnoise=200)
    r2 = Asyrp(a2, load_config("celeba"), device="cpu")
    r2.set_t_edit_t_addnoise()
    sch = r2.make_schedule(*__import__("asyrp_official_b200.schedule", fromlist=["x"]).make_sequences(999, 40),
                           hs_coeff=(1.0, 1.0))
    assert (r2.t_edit, r2.t_addnoise, sch.n_edit, sch.n_stochastic) == (500, 200, 20, 7)
    with pytest.raises(ValueError):
        Asyrp(argparse.Namespace(user_defined_t_edit=None, user_defined_t_addnoise=None), load_config("celeba"),
              device="cpu").set_t_edit_t_addnoise()


def test_weight_packing_layout():
    """pack_weights is pure tensor reshuffling: check the K layouts the kernels rely on, on the CPU"""
    from asyrp_official_b200 import arch, modules, synthetic
    from asyrp_official_b200.engine import pack_weights
    from oracle import adm as oa, ddpm as od
    for a, make in ((arch.ddpm_arch(**od.MINI_CFG), None), (arch.adm_arch(**oa.MINI_HP), None)):
        shapes = arch.param_shapes(a, 1)
        from oracle import synth
        sd = synth.synth_state_dict(shapes, 1234, "jittered")
        W, emb_off, emb_total = pack_weights(a, sd, "cpu", 1)
        assert emb_total == W["emb_cat.w"].shape[0] == W["emb_cat.b"].shape[0] and emb_total % 64 == 0
        for stage in a.enc + [a.mid] + a.dec:
            for layer in stage:
                if isinstance(layer, arch.Res):
                    p = layer.name
                    assert W[p + ".w1"].shape == (layer.cout, 9 * layer.cin) and W[p + ".w1"].dtype == torch.float16
                    # conv2: 9*cout columns, then the 1x1 shortcut (cin columns) or the identity skip (cout columns)
                    assert W[p + ".w2"].shape == (layer.cout, 9 * layer.cout + layer.cin)
                    if layer.cin == layer.cout:
                        assert torch.equal(W[p + ".w2"][:, 9 * layer.cout:].float(), torch.eye(layer.cout))
                    if layer.split:  # decoder: segment-major K (h columns of every tap, then skip columns of every tap)
                        c0 = layer.split[0]
                        key = p + (".conv1.weight" if a.family == "ddpm" else ".in_layers.2.weight")
                        w = sd[key]
                        assert torch.equal(W[p + ".w1"][:, :9 * c0].float().reshape(layer.cout, 3, 3, c0),
                                           w[:, :c0].permute(0, 2, 3, 1).to(torch.float16).float())
        assert W["conv_in.w"].shape[1] == 9 * 64 and W["conv_out.w"].shape[0] == 16


def test_upconv_subpixel_weights():
    """pack_upconv_weight: conv3x3(nearest-x2(x)) == four 2x2 phase convs on x (reference: Upsample.forward,
    models/ddpm/diffusion.py:77-87).  Checked in fp64 with the packed layout the kernel consumes."""
    import torch.nn.functional as F
    from asyrp_official_b200 import ops
    torch.manual_seed(0)
    n, ci, co, h, w = 2, 5, 3, 6, 4
    x = torch.randn(n, ci, h, w, dtype=torch.float64)
    wt = torch.randn(co, ci, 3, 3, dtype=torch.float64)
    ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), wt, padding=1)
    # packed rows: (a*2+b)*co + o ; columns: (dy*2+dx)*ci + i ; source pixel (y-1+a+dy, x-1+b+dx)
    # (computed in fp32 by the packer; compare against an fp64 re-evaluation with a matching tolerance)
    pk = ops.pack_upconv_weight(wt.float()).double().reshape(2, 2, co, 2, 2, ci)
    xp = F.pad(x, (1, 1, 1, 1))
    out = torch.zeros(n, co, 2 * h, 2 * w, dtype=torch.float64)
    for a in (0, 1):
        for b in (0, 1):
            acc = torch.zeros(n, co, h, w, dtype=torch.float64)
            for dy in (0, 1):
                for dx in (0, 1):
                    patch = xp[:, :, a + dy:a + dy + h, b + dx:b + dx + w]
                    acc += torch.einsum("oi,nihw->nohw", pk[a, b, :, dy, dx, :], patch)
            out[:, :, a::2, b::2] = acc
    assert (out - ref).abs().max() < 2e-2 * ref.abs().max()  # fp16 rounding of the packed weights
    pk32 = ops.pack_upconv_weight(wt.float())
    assert pk32.shape == (4 * co, 4 * ci) and pk32.dtype == torch.float16


@pytest.mark.parametrize("mode", ["ddpm", "dt_lambda", "ignore"])
def test_schedule_sample_type_dt_lambda_and_key(mode):
    """Schedule carries what save_image forwards to denoising_step on every step (diffusion_latent.py:507-520):
    'ddpm' ancestral coefficients, the dt_lambda override at t >= 999, ignore_timestep; the coefficients reproduce the
    oracle's step; hs_coeff VALUES are not part of the graph key (they are device-side parameters)"""
    from asyrp_official_b200.schedule import Schedule, make_sequences
    from oracle import sampler as osmp
    betas = osmp.make_betas()
    logvar = osmp.make_logvar(osmp.get_beta_schedule(beta_start=1e-4, beta_end=0.02, num_diffusion_timesteps=1000))
    seq, nxt = make_sequences(999, 10)
    base = Schedule(betas, seq, nxt, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0))
    assert base.key() == Schedule(betas, seq, nxt, t_edit=500, t_addnoise=0, hs_coeff=(0.3, 2.0)).key()
    g = torch.Generator().manual_seed(0)
    x, e, z = (torch.randn(1, 3, 4, 4, generator=g) for _ in range(3))
    model = lambda xt, t, **k: (e, e, None, None)  # noqa: E731
    if mode == "ignore":
        s2 = Schedule(betas, seq, nxt, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0), ignore_timestep=True)
        assert s2.key() != base.key() and s2.ignore_timestep
        return
    if mode == "ddpm":
        sch = Schedule(betas, seq, nxt, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0), sample_type="ddpm", logvars=logvar)
        assert sch.n_stochastic == 10 and sch.key() != base.key() and sch.steps[-1].mask == 0.0
        for s in (sch.steps[0], sch.steps[-1]):
            ref = osmp.denoising_step(x, torch.ones(1) * s.t, torch.ones(1) * s.t_next, model=model, b=betas,
                                      logvars=logvar, sampling_type="ddpm", noise=z)[0]
            at, bt = torch.tensor(s.at), torch.tensor(s.bt)
            mine = 1 / torch.sqrt(1.0 - bt) * (x - bt / torch.sqrt(1 - at) * e) + s.mask * torch.exp(
                torch.tensor(0.5 * s.logvar)) * z
            assert torch.allclose(ref, mine, rtol=0, atol=1e-6)
        with pytest.raises(ValueError):
            Schedule(betas, seq, nxt, t_edit=500, sample_type="ddpm", dt_lambda=0.5, logvars=logvar)
        return
    sch = Schedule(betas, seq, nxt, t_edit=500, t_addnoise=0, hs_coeff=(1.0, 1.0), dt_lambda=0.7)
    assert sch.key() != base.key() and sch.steps[1] == base.steps[1]  # only t >= dt_end = 999 is affected
    s = sch.steps[0]
    ref = osmp.denoising_step(x, torch.ones(1) * s.t, torch.ones(1) * s.t_next, model=model, b=betas, dt_lambda=0.7)[0]
    at, an = torch.tensor(s.at), torch.tensor(s.an)
    mine = an.sqrt() * ((x - e * (1 - at).sqrt()) / at.sqrt()) + torch.tensor(s.c2) * e
    assert torch.allclose(ref, mine, rtol=0, atol=1e-6) and s.c1 == 0.0


def test_reference_staging_script(tmp_path):
    """oracle/stage_reference.py copies the reference's hot-path sources verbatim into a git-ignored directory, and
    does nothing where no reference tree exists.  Runs on a stand-in tree with the reference's layout."""
    from oracle import stage_reference as mod
    assert os.path.relpath(mod.DST, ROOT) == os.path.join("oracle", "_ref")
    assert "oracle/_ref/" in open(os.path.join(ROOT, ".gitignore")).read()
    src = tmp_path / "reference"
    assert mod.stage(str(src), str(tmp_path / "x"), quiet=True) is False
    rels = ["utils/diffusion_utils.py", "models/ddpm/diffusion.py", "models/improved_ddpm/unet.py",
            "models/guided_diffusion/unet.py", "configs/celeba.yml"] + ["checkpoint/" + c for c in mod.CKPTS]
    for i, rel in enumerate(rels):
        (src / rel).parent.mkdir(parents=True, exist_ok=True)
        (src / rel).write_bytes(bytes([i]) * (100 + i))
    (src / "utils" / "__pycache__").mkdir()
    (src / "utils" / "__pycache__" / "x.pyc").write_bytes(b"0")
    assert mod.stage(str(src), str(tmp_path / "ref"), quiet=True)
    for rel in rels:
        assert (src / rel).read_bytes() == (tmp_path / "ref" / rel).read_bytes(), rel
    assert not (tmp_path / "ref" / "utils" / "__pycache__").exists()


def test_engine_numerics_emulation_switches():
    """oracle/emulate.py with every rounding switched off is the fp32 oracle; switched on it differs at the fp16 level"""
    from oracle import ddpm as od, emulate as em, synth
    cfg = od.MINI_CFG
    sd = synth.synth_state_dict(od.ddpm_param_shapes(cfg, 1), 1234, "jittered")
    x, t = synth.synth_noise((1, 3, 32, 32), 1234), torch.ones(1) * 700
    ref = od.ddpm_forward(sd, cfg, x, t, index=0, t_edit=500, hs_coeff=(1.0, 0.7))
    off = em.ddpm_forward(sd, cfg, x, t, index=0, t_edit=500, hs_coeff=(1.0, 0.7), flags=em.NONE)
    on = em.ddpm_forward(sd, cfg, x, t, index=0, t_edit=500, hs_coeff=(1.0, 0.7), flags=em.ALL)
    for a, b, c in zip(ref, off, on):
        scale = a.abs().max().item()
        assert (a - b).abs().max().item() <= 2e-5 * scale
        assert 1e-5 * scale < (a - c).abs().max().item() < 1e-2 * scale


def test_shipped_delta_block_fixtures_load():
    """tests/golden/checkpoint/*.pth: the DeltaBlocks SURVEY §8(d) names, in the {"0": state_dict} format run_test loads"""
    from asyrp_official_b200 import modules
    from asyrp_official_b200.configs import load_config
    d = os.path.join(ROOT, "tests", "golden", "checkpoint")
    m = modules.DDPM(load_config("celeba"))
    m.setattr_layers(1)
    for name in ("smiling_LC_CelebA_HQ_t999_ninv40_ngen40_0.pth", "church_gothic_LC_church_outdoor_t999_ninv40_ngen40_0.pth"):
        ck = torch.load(os.path.join(d, name), map_location="cpu", weights_only=True)
        res = m.layer_0.load_state_dict(ck["0"])
        assert not res.missing_keys and not res.unexpected_keys
    a = modules.i_DDPM("AFHQ")
    a.setattr_layers(1)
    ck = torch.load(os.path.join(d, "dog_happy_LC_dog_t999_ninv40_ngen40_0.pth"), map_location="cpu", weights_only=True)
    res = a.layer_0.load_state_dict(ck["0"])
    assert not res.missing_keys and not res.unexpected_keys


def test_bench_dump_outputs_is_capped_and_seeded(tmp_path):
    """bench.py --dump-outputs: a batch over 64 MB becomes a fixed, seeded sample of whole images (indices written next
    to it), the same on every run; a smaller batch is written whole; --steps below 1, and a dump of the reference arm
    (which computes no x_0 batch), are rejected"""
    import subprocess
    import sys
    import numpy as np
    import bench
    x = torch.randn(100, 3, 256, 256, generator=torch.Generator().manual_seed(0))  # 78.6 MB of float32
    n = bench.dump_outputs(x, str(tmp_path / "a"))
    a, idx = np.load(tmp_path / "a" / "x0.npy"), np.load(tmp_path / "a" / "x0_indices.npy")
    assert a.dtype == np.float32 and a.nbytes <= 64 << 20 and a.shape == (n, 3, 256, 256) and n == 85
    assert len(set(idx.tolist())) == n and np.array_equal(a, x.numpy()[idx])
    bench.dump_outputs(x, str(tmp_path / "b"))
    assert np.array_equal(np.load(tmp_path / "b" / "x0_indices.npy"), idx)
    assert bench.dump_outputs(x[:4], str(tmp_path / "c")) == 4
    assert np.array_equal(np.load(tmp_path / "c" / "x0.npy"), x[:4].numpy())
    assert not (tmp_path / "c" / "x0_indices.npy").exists()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "0"], capture_output=True, text=True)
    assert r.returncode == 2 and "--steps must be at least 1" in r.stderr
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs",
                        str(tmp_path / "d")], capture_output=True, text=True)
    assert r.returncode == 2 and "engine arm only" in r.stderr and not (tmp_path / "d").exists()
