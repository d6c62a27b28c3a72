"""Per-sample DeltaBlock coefficients on the GPU: the conv epilogue reading one (acc_scale, res_scale) pair per batch
row, UNetEngine.sample(hs_coeffs=table) against one batch-1 trajectory per row (bit for bit) and against the CPU
oracle and the reference's goldens, and save_image's batched hs_coeff sweep against the one-replay-per-tuple loop
(--max_rows_per_replay 1), byte for byte on every PNG."""
import math
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import yaml

from asyrp_official_b200 import _lib, modules, ops, synthetic
from asyrp_official_b200.schedule import Schedule, make_sequences
from oracle import adm as oa, ddpm as od, sampler as osmp

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
TOL_RAW, TOL_STATS = 1.5e-3, 2e-3  # those of test_conv_coverage_gpu.py (raw fp16 operands)
TOL_TRAJ = 2e-3                    # short trajectories of the reduced UNets (test_features_gpu.py)

# distinct (acc_scale, res_scale) per row, including the pure residual (0, 1) and the identity-scale (1, 1) rows
PAIRS = [(0.0, 1.0), (1.0, 1.0), (0.75, -0.5), (-1.25, 0.25), (1.5, 2.0), (0.3, 0.0), (-0.6, 1.7)]


def _h(x):
    return x.to(torch.float16).double()


def _nhwc(x, dev):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.float16).to(dev)


def _from_nhwc(t):
    return t.double().cpu().permute(0, 3, 1, 2)


# (H, W, Cin, Cout, mode, N, NB): the DeltaBlock h2 convs (1x1 at 8x8, C = 512 / 1024, two samples per tile), tiles of
# eight samples (4x4), and a 16x16 3x3 conv with tiles inside one sample; every N leaves the last tile part empty
GEOMETRIES = {"delta_8x8_c512": (8, 8, 512, 512, ops.MODE_1x1, 5, 2),
              "delta_8x8_c1024": (8, 8, 1024, 1024, ops.MODE_1x1, 7, 2),
              "nb8_4x4_c512": (4, 4, 512, 512, ops.MODE_1x1, 5, 8),
              "halo_16x16_c128": (16, 16, 128, 128, ops.MODE_3x3, 3, 1)}


@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_conv_reads_one_coefficient_pair_per_row(cuda_device, geom):
    dev = cuda_device
    H, W, Cin, Cout, mode, N, NB = GEOMETRIES[geom]
    has3 = mode == ops.MODE_3x3
    g = torch.Generator().manual_seed(17)
    taps = 9 if has3 else 1
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin) if has3 else \
        torch.randn(Cout, Cin, generator=g) / math.sqrt(Cin)
    eb = torch.randn(Cout, generator=g)
    res = torch.randn(N, Cout, H, W, generator=g)
    pairs = PAIRS[:N]
    # the engine's layout: [N][n_delta][2] with the op reading block 1 of 2 -> row stride 4 floats; one NaN row behind
    table = torch.full((N + 1, 2, 2), float("nan"), dtype=torch.float32)
    table[:N, 1] = torch.tensor(pairs)
    table = table.to(dev)
    slots = ops.conv_stats_tiles(H, W, Cout, has3)
    args = ([(_nhwc(x, dev), mode)], ops.pack_conv_weight(w).to(dev))
    kw = dict(ebias=eb.to(dev), residual=_nhwc(res, dev))

    def run(**scale_kw):
        out_full = torch.full((N + 1, H, W, Cout), float("nan"), dtype=torch.float16, device=dev)
        st_full = torch.full((N + 1, slots, Cout // 2, 2), float("nan"), dtype=torch.float32, device=dev)
        op = ops.ConvOp(*args, out=out_full[:N], stats=st_full[:N], **kw, **scale_kw)
        assert ops.conv_tile_config(H, W, Cout, has3)[0] > 0
        op.launch()
        torch.cuda.synchronize()
        for name, full in (("out", out_full), ("stats", st_full)):
            assert torch.isfinite(full[:N]).all(), f"{geom}: {name} not fully written"
            assert torch.isnan(full[N]).all(), f"{geom}: {name} guard sample overwritten"
        return out_full[:N], st_full[:N]

    out, st = run(scales=table[0, 1], scales_stride=table.stride(0))
    assert torch.isnan(table[N]).all()
    conv = (F.conv2d(_h(x), _h(w), padding=1) if has3 else F.conv2d(_h(x), _h(w)[:, :, None, None])) \
        + eb.double()[None, :, None, None]
    a = torch.tensor([p[0] for p in pairs], dtype=torch.float32).double()[:, None, None, None]
    b = torch.tensor([p[1] for p in pairs], dtype=torch.float32).double()[:, None, None, None]
    ref = a * conv + b * _h(res)
    err, mag = (_from_nhwc(out) - ref).abs().max().item(), ref.abs().max().item()
    assert err <= TOL_RAW * mag, f"{geom}: output max-abs err {err:.3e} of {mag:.3e}"
    r = ref.reshape(N, Cout // 2, 2, H * W)
    st_ref = torch.stack([r.sum(dim=(2, 3)), (r * r).sum(dim=(2, 3))], dim=-1)
    st_err = (st.double().cpu().sum(1) - st_ref).abs().max().item()
    assert st_err <= TOL_STATS * st_ref.abs().max().item() + 1e-3, f"{geom}: statistics max-abs err {st_err:.3e}"
    # every row is bit-identical to a launch that gives the whole batch that row's pair
    for n, (an, bn) in enumerate(pairs):
        o1, s1 = run(scales=torch.tensor([an, bn], dtype=torch.float32, device=dev))
        assert torch.equal(out[n], o1[n]) and torch.equal(st[n], s1[n]), f"{geom}: row {n} ({an}, {bn})"
    # malformed descriptors
    with pytest.raises(_lib.AsyrpError):
        ops.ConvOp(*args, out=out, scales=table[0, 1], scales_stride=-4, **kw)
    with pytest.raises(_lib.AsyrpError):
        ops.ConvOp(*args, out=out, scales_stride=4, **kw)


# ------------------------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------------------------
def _mini(family, n_delta, dev):
    if family == "ddpm":
        cfg = od.MINI_CFG
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
        fwd = lambda sd, *a, **k: od.ddpm_forward(sd, cfg, *a, **k)  # noqa: E731
    else:
        m = modules._create_adm(oa.MINI_HP)
        fwd = lambda sd, *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k)  # noqa: E731
    m.setattr_layers(n_delta)
    m = synthetic.randomize_(m, 1234, "jittered").to(dev)
    return m, fwd


@pytest.mark.parametrize("family,n_delta", [("ddpm", 1), ("ddpm", 2), ("adm", 1), ("adm", 2)])
def test_sample_with_a_coefficient_table_equals_one_run_per_row(cuda_device, family, n_delta):
    """K rows with K different tuples in one batch == K batch-1 trajectories, bit for bit; each row against the CPU
    oracle; several tables replay one captured graph"""
    dev = cuda_device
    m, fwd = _mini(family, n_delta, dev)
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 6)
    base = (1.0,) + (1.0,) * n_delta
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=400, hs_coeff=base)
    assert sch.n_stochastic and any(s.edit for s in sch.steps) and not all(s.edit for s in sch.steps)
    rows = [(1.0, 1.0, 1.0), (0.8, 1.5, -0.5), (1.2, -0.7, 0.9)]
    rows = [r[:1 + n_delta] for r in rows]
    K = len(rows)
    g = torch.Generator().manual_seed(21)
    x = torch.randn(1, 3, 32, 32, generator=g).expand(K, -1, -1, -1).contiguous()
    x[1:] += 0.1 * torch.randn(K - 1, 3, 32, 32, generator=g)  # not only the same x_T
    nz = torch.randn(sch.n_stochastic, K, 3, 32, 32, generator=g)
    eng = m.engine
    table = torch.tensor(rows, dtype=torch.float32)
    batch = eng.sample(x.to(dev), sch, noise=nz.to(dev), hs_coeffs=table)
    n_graphs = len(eng.graphs)
    again = eng.sample(x.to(dev), sch, noise=nz.to(dev), hs_coeffs=table.flip(0).to(dev))
    assert len(eng.graphs) == n_graphs, "a new table must replay the captured graph"
    assert torch.equal(again, eng.sample(x.to(dev), sch, noise=nz.to(dev), hs_coeffs=table.flip(0)))
    for k, row in enumerate(rows):
        s_k = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=400, hs_coeff=row)
        one = eng.sample(x[k:k + 1].to(dev), s_k, noise=nz[:, k:k + 1].contiguous().to(dev))
        assert torch.equal(batch[k:k + 1], one), f"{family} n_delta={n_delta}: row {k} {row} != its batch-1 run"
        noises = {s.t: nz[zi, k:k + 1] for zi, s in enumerate([s for s in sch.steps if s.stochastic])}
        ref = osmp.run_trajectory(lambda *a, **kk: fwd(sd, *a, **kk), x[k:k + 1], betas=betas, seq=seq,
                                  seq_next=seq_next, t_edit=500, t_addnoise=400, index=n_delta - 1, hs_coeff=row,
                                  learn_sigma=family == "adm", noises=noises)
        e, mx = (one.double().cpu() - ref.double()).abs().max().item(), ref.abs().max().item()
        assert e <= TOL_TRAJ * max(1.0, mx), f"{family} row {k}: max-abs err {e:.3e} of {mx:.3e}"
    # a flipped table flips the rows (each row keeps its own result)
    assert torch.equal(again[0], eng.sample(x[:1].to(dev), Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=400,
                                                                     hs_coeff=rows[-1]),
                                            noise=nz[:, :1].contiguous().to(dev))[0])
    with pytest.raises(_lib.AsyrpError):
        eng.sample(x.to(dev), sch, noise=nz.to(dev), hs_coeffs=table[:, :n_delta])
    with pytest.raises(_lib.AsyrpError):
        eng.sample(x.to(dev), sch, noise=nz.to(dev), hs_coeffs=table[:2])
    # step API: forward() takes the same table
    t = torch.ones(K, device=dev) * 700
    et, et_mod, _, _ = m(x.to(dev), t, index=n_delta - 1, t_edit=500, hs_coeff=table.to(dev))
    for k, row in enumerate(rows):
        _, em1, _, _ = m(x[k:k + 1].to(dev), t[:1], index=n_delta - 1, t_edit=500, hs_coeff=row)
        assert torch.equal(et_mod[k:k + 1], em1)


def test_explicit_delta_h_takes_one_c0(cuda_device):
    dev = cuda_device
    m, _ = _mini("ddpm", 0, dev)
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 4)
    sch = Schedule(betas, seq, seq_next, t_edit=500, hs_coeff=(0.7,))
    n_edit = sum(1 for s in sch.steps if s.edit)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 32, 32, generator=g).to(dev)
    dh = torch.randn(n_edit, 256, 8, 8, generator=g).to(dev)
    ref = m.engine.sample(x, sch, delta_hs=dh)
    same = m.engine.sample(x, Schedule(betas, seq, seq_next, t_edit=500, hs_coeff=(1.0,)), delta_hs=dh,
                           hs_coeffs=torch.tensor([[0.7], [0.7]]))
    assert torch.equal(same, m.engine.sample(x, sch, delta_hs=dh, hs_coeffs=torch.full((2, 1), 0.7)))
    assert (same - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()  # 1 - c0 from fp32 c0
    with pytest.raises(_lib.AsyrpError):
        m.engine.sample(x, sch, delta_hs=dh, hs_coeffs=torch.tensor([[0.7], [0.9]]))


# ------------------------------------------------------------------------------------------------------------------
# reference goldens (B = 1 fixtures) inside a batch of per-row coefficients
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,family,cfg,ckpt", [
    ("ddpm_church_gothic_traj40", "ddpm", od.CELEBA_CFG, "church_gothic_LC_church_outdoor_t999_ninv40_ngen40_0.pth"),
    ("adm_afhq_happy_traj40", "adm", oa.AFHQ_HP, "dog_happy_LC_dog_t999_ninv40_ngen40_0.pth")])
def test_golden_sample_in_a_batch_of_coefficient_rows(cuda_device, name, family, cfg, ckpt):
    dev = cuda_device
    gold = np.load(os.path.join(G, name + ".npz"))
    assert int(gold["batch"]) == 1
    if family == "ddpm":
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
    else:
        m = modules._create_adm(cfg)
    m.setattr_layers(1)
    m = synthetic.randomize_(m, 1234, "torch_default").to(dev)
    m.layer_0.load_state_dict(torch.load(os.path.join(G, "checkpoint", ckpt), map_location="cpu", weights_only=True)["0"])
    m.refresh_weights()
    seq = gold["seq"].tolist()
    seq_next = [-1] + seq[:-1]
    x = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(int(gold["x_seed"])))
    gn = torch.Generator().manual_seed(int(gold["noise_seed"]))
    noises = {i: torch.randn(x.shape, generator=gn) for i in seq}

    def schedule(c):
        return Schedule(osmp.make_betas(), seq, seq_next, t_edit=int(gold["t_edit"]),
                        t_addnoise=int(gold["t_addnoise"]), hs_coeff=c)

    nz = torch.stack([noises[s.t] for s in schedule((1.0, 1.0)).steps if s.stochastic]).to(dev)
    rows = [(1.0, 0.5), (0.9, 1.2), (1.0, 1.0), (1.1, -0.4)]
    R = len(rows)
    eng = m.engine
    batch = eng.sample(x.expand(R, -1, -1, -1).contiguous().to(dev), schedule((1.0, 1.0)),
                       noise=nz.expand(-1, R, -1, -1, -1).contiguous(), hs_coeffs=torch.tensor(rows))
    for k, row in enumerate(rows):
        one = eng.sample(x.to(dev), schedule(row), noise=nz)
        assert torch.equal(batch[k:k + 1], one), f"{name}: row {k} {row} != its batch-1 run"
        if row == (1.0, 1.0):
            e = (one[..., ::4, ::4].double().cpu() - torch.from_numpy(gold["x0_sub"]).double()).abs().max().item()
            mx = float(np.abs(gold["x0_sub"]).max())
            print(f"\n{name}: (1, 1) row of {R} vs the reference: max-abs {e:.4f} of {mx:.2f} -> {e / mx:.2e}")
            assert e <= 1e-3 * mx
    del eng, m
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# runner: batched sweep == one replay per tuple
# ------------------------------------------------------------------------------------------------------------------
def _write_cfg(path):
    cfg = od.MINI_CFG
    d = {"data": dict(dataset="CelebA_HQ", category="CelebA_HQ", image_size=cfg["image_size"], channels=3,
                      rescaled=True, num_workers=0),
         "model": dict(type="simple", in_channels=3, out_ch=3, ch=cfg["ch"], ch_mult=list(cfg["ch_mult"]),
                       num_res_blocks=cfg["num_res_blocks"], attn_resolutions=list(cfg["attn_resolutions"]),
                       dropout=0.0, var_type="fixedsmall", ema_rate=0.999, ema=True, resamp_with_conv=True),
         "diffusion": dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
         "sampling": dict(batch_size=4, last_only=True)}
    with open(path, "w") as f:
        yaml.safe_dump(d, f)
    return path


def _block(path, seed):
    cfg = od.MINI_CFG
    ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
    m = modules.DDPM(ns)
    m.setattr_layers(1)
    synthetic.randomize_(m, seed=seed, style="jittered")
    torch.save({"0": {k: v.clone() for k, v in m.layer_0.state_dict().items()}}, path)


def _run(root, dev, extra, max_rows, n_test_img=2, n_train_img=0, bs=2):
    """one run_test in its own directory; returns (results, {relative path: bytes} of every file it wrote)"""
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    d = os.path.join(root, f"rows{max_rows}")
    os.makedirs(os.path.join(d, "checkpoint"), exist_ok=True)
    cwd = os.getcwd()
    os.chdir(d)
    try:
        _block("checkpoint/a_0.pth", 11)
        _block("checkpoint/b_0.pth", 12)
        argv = ["--run_test", "--config", _write_cfg(os.path.join(d, "mini.yml")), "--exp", "./runs/attr",
                "--do_train", "1" if n_train_img else "0", "--do_test", "1" if n_test_img else "0",
                "--n_test_img", str(n_test_img), "--n_train_img", str(n_train_img), "--bs_train", str(bs),
                "--t_0", "999", "--n_inv_step", "5", "--n_train_step", "5", "--n_test_step", "5",
                "--load_random_noise", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "400",
                "--synthetic_weights", "--seed", "1234", "--max_rows_per_replay", str(max_rows)] + extra
        args, config = cli.parse_args_and_config(argv)
        res = Asyrp(args, config, device=dev).run_test()
        files = {}
        for top in ("runs", "checkpoint_latent"):
            for dp, _, fs in os.walk(top):
                for f in fs:
                    with open(os.path.join(dp, f), "rb") as fh:
                        files[os.path.join(dp, f)] = fh.read()
        return res, files
    finally:
        os.chdir(cwd)


def _same(a, b, what):
    (ra, fa), (rb, fb) = a, b
    assert ra.keys() == rb.keys()
    for k in ra:
        assert len(ra[k]) == len(rb[k]) and all(torch.equal(u, v) for u, v in zip(ra[k], rb[k])), f"{what}: rows of {k}"
    pngs = sorted(p for p in fa if p.endswith(".png"))
    assert pngs and pngs == sorted(p for p in fb if p.endswith(".png")), what
    for p in pngs:
        assert fa[p] == fb[p], f"{what}: {p} differs"


SWEEPS = {
    # 3 tuples x 2 images: 6 rows = one chunk; 4 -> chunks of 2 tuples, the last padded; 2 -> one tuple per chunk
    "interpolation": (["--train_delta_block", "--get_h_num", "1", "--manual_checkpoint_name", "a_0.pth",
                       "--delta_interpolation", "--num_delta", "3", "--min_delta", "0.0", "--max_delta", "1.5"],
                      (6, 4, 2)),
    # two attributes, 2 x 2 interpolated tuples x 2 images: 8 rows = one chunk; 6 -> 3 + 1 tuple (padded); 4 -> 2 + 2
    "two_attributes": (["--train_delta_block", "--get_h_num", "2", "--manual_checkpoint_name", "attribute_0.pth",
                        "--multiple_attr", "a b", "--multiple_hs_coeff", "1.0 0.5", "--delta_interpolation",
                        "--num_delta", "2", "--min_delta", "0.5", "--max_delta", "1.5"],
                       (8, 6, 4)),
}


@pytest.mark.parametrize("sweep", list(SWEEPS))
def test_batched_sweep_equals_one_replay_per_tuple(cuda_device, tmp_path, sweep):
    extra, sizes = SWEEPS[sweep]
    extra = extra + ["--save_x_origin", "--save_process_delta_h"]
    seq = _run(str(tmp_path), cuda_device, extra, 1)
    n_rows = len(next(iter(seq[0].values())))
    assert n_rows == 1 + (3 if sweep == "interpolation" else 4)
    assert any("delta_h_" in p for p in seq[1])
    for r in sizes:
        _same(seq, _run(str(tmp_path), cuda_device, extra, r), f"{sweep} at --max_rows_per_replay {r}")


def test_mean_delta_h_extraction_through_the_batched_sweep(cuda_device, tmp_path):
    """--num_mean_of_delta_hs with an interpolation sweep: the Δh rows of every tuple are added in tuple order, so the
    cached mean and the images edited with it are those of the per-tuple loop"""
    extra = ["--train_delta_block", "--get_h_num", "1", "--manual_checkpoint_name", "a_0.pth",
             "--num_mean_of_delta_hs", "2", "--delta_interpolation", "--num_delta", "3"]
    kw = dict(n_test_img=0, n_train_img=3, bs=1)
    a = _run(str(tmp_path), cuda_device, extra, 1, **kw)
    b = _run(str(tmp_path), cuda_device, extra, 16, **kw)
    _same(a, b, "mean-Δh sweep")
    (latent,) = [p for p in a[1] if p.startswith("checkpoint_latent")]
    la = torch.load(os.path.join(str(tmp_path), "rows1", latent), weights_only=True)
    lb = torch.load(os.path.join(str(tmp_path), "rows16", latent), weights_only=True)
    assert la.keys() == lb.keys()
    assert all((la[k] is None and lb[k] is None) or torch.equal(la[k], lb[k]) for k in la)
