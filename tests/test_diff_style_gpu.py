"""DiffStyle on the GPU: the per-row slerp kernel against the scalar one, h recorded inside the inversion graph
against the step API's middle_h, a mixed-hs_coeff batch against batch-1 runs (bit for bit), engine trajectories against
the CPU oracle (reduced DDPM / ADM, 256² DDPM), and `main --diff_style` end to end."""
import os
from types import SimpleNamespace as NS

import pytest
import torch
import yaml

from asyrp_official_b200 import _lib, diffusion_latent as dl, main as cli, modules, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.schedule import Schedule, make_sequences
from oracle import adm as oa, ddpm as od, sampler as osmp
from test_diff_style_host import _write_pngs, oracle_diff_style, oracle_invert_with_h

pytestmark = pytest.mark.gpu
# engine vs oracle after a whole DiffStyle generation, relative to max(1, max |ref|): the bound test_model_gpu.py holds
# one explicit-Δh forward to (the fp16 h2 of the slerp feeds the edited decoder); measured 2.0e-3 .. 2.8e-3 on an H100
TOL_TRAJ = 4e-3
TOL_INV = 2e-2   # DDIM inversion x_T (and its h), as tests/test_model_gpu.py bounds the inversion


# ------------------------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [256, 512, 1024])  # bottlenecks: reduced UNets, DDPM 256² / ADM AFHQ, ADM ImageNet
@pytest.mark.parametrize("N", [1, 3, 17])
def test_slerp_h_rows_equals_slerp_h(cuda_device, C, N):
    """row n of slerp_h_rows == slerp_h with t = t_rows[n], bit for bit: h2, every GroupNorm tile slot (slot 0 the
    sums, the others zeroed) in both mask modes, per-sample and shared dh; t includes 0 and 1"""
    dev = cuda_device
    g = torch.Generator().manual_seed(C + N)
    H = W = 8
    T = 3
    h = (torch.randn(N, H, W, C, generator=g) * 3).half().to(dev)
    dh = torch.randn(N, C, H, W, generator=g).to(dev)
    base = [0.0, 1.0, 0.1, 0.35, 0.5, 0.999]
    t_rows = torch.tensor([base[n % len(base)] if n < len(base) else float(torch.rand(1, generator=g))
                           for n in range(N)], dtype=torch.float32, device=dev)
    for use_mask in (False, True):
        for d in (dh, dh[0]):
            h2 = torch.full((N, H, W, C), float("nan"), dtype=torch.float16, device=dev)
            st = torch.full((N, T, C // 2, 2), float("nan"), device=dev)
            ops.slerp_h_rows(h, d, h2, st, t_rows, use_mask)
            again = h2.clone()
            ops.slerp_h_rows(h, d, again, st.clone(), t_rows, use_mask)
            for n in range(N):
                r2 = torch.full_like(h2, float("nan"))
                rs = torch.full_like(st, float("nan"))
                ops.slerp_h(h, d, r2, rs, float(t_rows[n]), use_mask)
                torch.cuda.synchronize()
                what = f"C={C} N={N} row {n} t={float(t_rows[n])} mask={use_mask} shared={d.dim() == 3}"
                assert torch.equal(h2[n], r2[n]), what
                assert torch.equal(st[n], rs[n]), what + " (GroupNorm sums)"
            assert not torch.isnan(h2).any() and torch.equal(h2, again)
            assert torch.equal(st[:, 1:], torch.zeros_like(st[:, 1:]))
    with pytest.raises(_lib.AsyrpError):
        ops.slerp_h_rows(h, dh, h2, st, t_rows[:-1] if N > 1 else t_rows.cpu())


# ------------------------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------------------------
def _module(family, cfg=None, style="jittered"):
    if family == "ddpm":
        cfg = cfg or od.MINI_CFG
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
    else:
        m = modules._create_adm(cfg or oa.MINI_HP)
    synthetic.randomize_(m, 1234, style)
    return m


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_record_h_equals_the_step_api(cuda_device, family):
    """the h recorded inside the inversion graph == forward()'s middle_h at every step, and recording leaves x_T
    unchanged"""
    dev = cuda_device
    m = _module(family).to(dev)
    eng = m.engine
    seq, seq_next = make_sequences(999, 8)
    sch = Schedule.inversion(osmp.make_betas(), seq, seq_next)
    x0 = torch.tanh(torch.randn(3, 3, 32, 32, generator=torch.Generator().manual_seed(2))).to(dev)
    plain = eng.sample(x0, sch)
    rec = eng.sample(x0, sch, record_h=True)
    assert torch.equal(plain, rec), f"{family}: recording h changed x_T"
    hs = eng.last_records["h"].clone()
    assert hs.shape == (len(sch.steps), 3, 256, 8, 8)
    eng.sample(x0, sch, record_h=True, record_process=True)
    xs = eng.last_records["x"].clone()
    assert torch.equal(xs[-1], plain)
    for k, s in enumerate(sch.steps):
        x_in = x0 if k == 0 else xs[k - 1]
        mid = eng.forward(x_in, torch.full((3,), float(s.t), device=dev))[3]
        assert torch.equal(hs[k], mid), f"{family}: step {k} (t={s.t})"


def _rows_setup(dev, R, n_step=8):
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, n_step)
    mk = lambda gamma: Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(gamma,),  # noqa: E731
                                dt_lambda=0.9985, dt_end=950)
    sch = mk(0.9)
    g = torch.Generator().manual_seed(R)
    x = torch.randn(R, 3, 32, 32, generator=g).to(dev)
    dh = torch.randn(sch.n_edit, R, 256, 8, 8, generator=g).to(dev)
    nz = torch.randn(sch.n_stochastic, R, 3, 32, 32, generator=g).to(dev)
    return mk, sch, x, dh, nz


def test_mixed_gamma_batch_equals_batch_one_runs(cuda_device):
    """rows with their own hs_coeff (slerp weight 1 - γ read per row) == batch-1 runs with that γ, bit for bit, with
    use_mask off and on; another γ list of the same row count replays the same graph"""
    dev = cuda_device
    m = _module("ddpm").to(dev)
    eng = m.engine
    gammas = [0.9, 0.6, 0.9, 0.3, 1.0]
    mk, sch, x, dh, nz = _rows_setup(dev, len(gammas))
    assert sch.n_stochastic and sch.n_edit and any(s.t >= 950 and s.c2 != 0 for s in sch.steps)
    for use_mask in (False, True):
        table = torch.tensor([[gm] for gm in gammas])
        out = eng.sample(x, sch, noise=nz, delta_hs=dh, hs_coeffs=table, use_mask=use_mask)
        rec, n_graphs = eng.last_records, len(eng.graphs)
        other = eng.sample(x, sch, noise=nz, delta_hs=dh, hs_coeffs=torch.tensor([[0.5], [0.7], [0.9], [0.2], [0.8]]),
                           use_mask=use_mask)
        assert eng.last_records is rec and len(eng.graphs) == n_graphs, "a second γ list must replay the same graph"
        for n, gm in enumerate(gammas):
            one = eng.sample(x[n:n + 1], mk(gm), noise=nz[:, n:n + 1].contiguous(), delta_hs=dh[:, n:n + 1].contiguous(),
                             hs_coeffs=torch.tensor([[gm]]), use_mask=use_mask)
            assert torch.equal(out[n:n + 1], one), f"row {n} (γ {gm}, use_mask {use_mask})"
        one = eng.sample(x[1:2], mk(0.7), noise=nz[:, 1:2].contiguous(), delta_hs=dh[:, 1:2].contiguous(),
                         hs_coeffs=torch.tensor([[0.7]]), use_mask=use_mask)
        assert torch.equal(other[1:2], one)
    # a shared Δh still takes one c0
    with pytest.raises(_lib.AsyrpError):
        eng.sample(x, sch, noise=nz, delta_hs=dh[:, 0], hs_coeffs=torch.tensor([[gm] for gm in gammas]))


def _engine_diff_style(eng, x0_c, x0_s, seq, seq_next, gammas, use_mask, noises_rows, betas):
    """the engine's DiffStyle of 2 contents x 2 styles (rows content-major, gammas[r] per row): x_T, h_dic per image,
    the content h at t_0, and the results"""
    dev = eng.device
    inv = Schedule.inversion(betas, seq, seq_next)
    imgs = torch.cat([x0_c, x0_s]).to(dev)
    x_T = eng.sample(imgs, inv, record_h=True)
    hs = eng.last_records["h"].cpu().clone()
    h_dic = [{int(s.t): hs[k][i:i + 1] for k, s in enumerate(inv.steps)} for i in range(imgs.shape[0])]
    mid = eng.forward(x_T[:2], torch.full((2,), float(seq[-1]), device=dev))[3].cpu()
    h_c = [{**h_dic[c], seq[-1]: mid[c:c + 1]} for c in range(2)]
    rows = [(c, s) for c in range(2) for s in range(2)]
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(gammas[0],), dt_lambda=0.9985,
                   dt_end=950)
    dh = dl.diff_style_delta_hs([h_c[c] for c, _ in rows], [s.t for s in sch.steps if s.edit])
    nz = torch.stack([noises_rows[s.t] for s in sch.steps if s.stochastic]).to(dev)
    out = eng.sample(torch.stack([x_T[2 + s] for _, s in rows]), sch, noise=nz, delta_hs=dh,
                     hs_coeffs=torch.tensor([[gm] for gm in gammas]), use_mask=use_mask).cpu()
    return x_T.cpu(), h_dic, h_c, rows, out


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_mini_trajectories_against_the_oracle(cuda_device, family):
    """inversion x_T and h, then the generation of every (pair, γ) row, against the CPU oracle fed the same inputs"""
    dev = cuda_device
    m = _module(family)
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    fwd = (lambda *a, **k: od.ddpm_forward(sd, od.MINI_CFG, *a, **k)) if family == "ddpm" else \
        (lambda *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k))
    learn_sigma = family == "adm"
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 10)
    g = torch.Generator().manual_seed(9)
    x0 = torch.tanh(torch.randn(4, 3, 32, 32, generator=g))
    noises = {t: torch.randn(4, 3, 32, 32, generator=g) for t in seq}
    gammas = [0.9, 0.6, 0.6, 0.9]
    for use_mask in (False, True):
        x_T, h_dic, h_c, rows, out = _engine_diff_style(m.engine, x0[:2], x0[2:], seq, seq_next, gammas, use_mask,
                                                        noises, betas)
        if not use_mask:
            for i in range(4):
                rx, rh = oracle_invert_with_h(fwd, x0[i:i + 1], seq, seq_next, learn_sigma)
                e = (x_T[i:i + 1] - rx).abs().max().item()
                assert e <= TOL_INV * max(1.0, rx.abs().max().item()), f"{family} image {i}: x_T err {e:.3e}"
                for t in rh:
                    e = (h_dic[i][t] - rh[t]).abs().max().item()
                    assert e <= TOL_INV * max(1.0, rh[t].abs().max().item()), f"{family} image {i} h[{t}]: {e:.3e}"
        for r, ((c, s), gm) in enumerate(zip(rows, gammas)):
            ref = oracle_diff_style(fwd, x_T[2 + s:3 + s], [h_c[c]], seq, seq_next, gm, use_mask, learn_sigma,
                                    {t: v[r:r + 1] for t, v in noises.items()})[-1]
            e, mx = (out[r:r + 1] - ref).abs().max().item(), ref.abs().max().item()
            print(f"\n{family} row {r} γ {gm} mask {use_mask}: max-abs {e:.3e} of {mx:.3e}")
            assert e <= TOL_TRAJ * max(1.0, mx), f"{family} row {r} (γ {gm}, use_mask {use_mask}): {e:.3e} of {mx:.3e}"


def test_celeba256_trajectory_against_the_oracle(cuda_device):
    """DDPM CelebA-HQ 256², synthetic weights, 6 steps: one content injected into one style with two γ as one batch,
    against the oracle's generation from the engine's x_T and content h"""
    dev = cuda_device
    m = _module("ddpm", od.CELEBA_CFG, style="torch_default")
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 6)
    g = torch.Generator().manual_seed(11)
    x0 = torch.tanh(torch.randn(2, 3, 256, 256, generator=g))
    inv = Schedule.inversion(betas, seq, seq_next)
    x_T = eng.sample(x0.to(dev), inv, record_h=True)
    hs = eng.last_records["h"].cpu().clone()
    mid = eng.forward(x_T[:1], torch.full((1,), float(seq[-1]), device=dev))[3].cpu()
    h_c = {**{int(s.t): hs[k][:1] for k, s in enumerate(inv.steps)}, seq[-1]: mid}
    gammas = [0.9, 0.5]
    sch = Schedule(betas, seq, seq_next, t_edit=400, t_addnoise=300, hs_coeff=(0.9,), dt_lambda=0.9985, dt_end=950)
    noises = {t: torch.randn(2, 3, 256, 256, generator=g) for t in seq}
    dh = dl.diff_style_delta_hs([h_c, h_c], [s.t for s in sch.steps if s.edit])
    nz = torch.stack([noises[s.t] for s in sch.steps if s.stochastic]).to(dev)
    out = eng.sample(x_T[1:2].expand(2, -1, -1, -1).contiguous(), sch, noise=nz, delta_hs=dh,
                     hs_coeffs=torch.tensor([[gm] for gm in gammas])).cpu()
    del m, eng
    torch.cuda.empty_cache()
    fwd = lambda *a, **k: od.ddpm_forward(sd, od.CELEBA_CFG, *a, **k)  # noqa: E731
    ref = torch.cat([oracle_diff_style(fwd, x_T[1:2].cpu(), [h_c], seq, seq_next, gm, False, False,
                                       {t: v[r:r + 1] for t, v in noises.items()}, t_edit=400)[-1]
                     for r, gm in enumerate(gammas)])
    for r in range(2):
        e, mx = (out[r] - ref[r]).abs().max().item(), ref[r].abs().max().item()
        print(f"\nceleba256 γ {gammas[r]}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"γ {gammas[r]}: {e:.3e} of {mx:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# runner
# ------------------------------------------------------------------------------------------------------------------
def test_main_diff_style_end_to_end(cuda_device, tmp_path, monkeypatch):
    """2 contents x 2 styles of tiny PNGs, two γ, synthetic weights: a PNG per pair and a cache per image; a second
    run inverts nothing and gives the same results, as does a run with one pair per replay"""
    monkeypatch.chdir(tmp_path)
    cfg = od.MINI_CFG
    _write_pngs("content", ["c0.png", "c1.jpg"], [(40, 32), (32, 48)])
    _write_pngs("style", ["s0.png", "s1.png"], [(32, 32), (64, 40)])
    conf = {"data": dict(dataset="CelebA_HQ", category="CelebA_HQ", image_size=cfg["image_size"], channels=3,
                         rescaled=True, num_workers=0),
            "model": dict(type="simple", in_channels=3, out_ch=3, ch=cfg["ch"], ch_mult=list(cfg["ch_mult"]),
                          num_res_blocks=cfg["num_res_blocks"], attn_resolutions=list(cfg["attn_resolutions"]),
                          dropout=0.0, var_type="fixedsmall", ema_rate=0.999, ema=True, resamp_with_conv=True),
            "diffusion": dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
            "sampling": dict(batch_size=4, last_only=True)}
    with open("mini.yml", "w") as f:
        yaml.safe_dump(conf, f)
    argv = ["--diff_style", "--config", os.path.join(str(tmp_path), "mini.yml"), "--content_dir", "content",
            "--style_dir", "style", "--save_dir", "out", "--user_defined_t_edit", "500", "--hs_coeff_list", "0.9 0.6",
            "--t_noise", "300", "--dt_lambda", "0.9985", "--n_inv_step", "8", "--bs_train", "3",
            "--max_rows_per_replay", "4", "--synthetic_weights", "--seed", "1234"]

    def run(*extra):
        args, config = cli.parse_args_and_config(argv + list(extra))
        r = Asyrp(args, config, device=cuda_device)
        return r, r.run_diff_style()

    r, res = run()
    assert r.n_inverted == 4
    pngs = sorted(os.listdir("out"))
    assert pngs == ["c0__s0.png", "c0__s1.png", "c1__s0.png", "c1__s1.png"]
    caches = sorted(os.listdir("precomputed"))
    assert caches == [f"CelebA_HQ_inv8_{d}_{n}.pt" for d, n in (("content", "c0"), ("content", "c1"),
                                                                 ("style", "s0"), ("style", "s1"))]
    from PIL import Image
    assert Image.open(os.path.join("out", "c0__s1.png")).size == (4 * 32 + 5, 32 + 2)
    pair = torch.load(os.path.join("precomputed", caches[0]), map_location="cpu", weights_only=True)
    assert pair[1] == 0 and sorted(pair[3]) == make_sequences(999, 8)[0][:-1]
    assert pair[3][0].shape == (1, 256, 8, 8) and pair[3][0].dtype == torch.float32 and not pair[2].is_cuda
    assert len(res) == 4 and all(v.shape == (2, 3, 32, 32) and torch.isfinite(v).all() for v in res.values())
    r2, res2 = run()
    assert r2.n_inverted == 0
    for k in res:
        assert torch.equal(res[k], res2[k]), k
    r3, res3 = run("--max_rows_per_replay", "2")  # each row draws its own noise: chunking does not change a result
    assert r3.n_inverted == 0
    for k in res:
        assert torch.equal(res[k], res3[k]), k
