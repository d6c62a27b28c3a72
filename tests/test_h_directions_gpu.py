"""h-space directions on the GPU: the additive kernel (add_h_rows) against a one-row call, a restatement of its
operation order and fp64; the statistics kernels (h_gram, h_combine) against numpy fp64; additive trajectories (mixed-α
batch against batch-1 runs, graph against eager, the CPU oracle with its DeltaBlock replaced by the direction, α = 0
against the origin pass); and `--h_directions` / `--run_test --h_direction` end to end."""
import ctypes
import os

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, main as cli, ops
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.schedule import Schedule, make_sequences
from oracle import adm as oa, ddpm as od, hspace as oh, sampler as osmp
from test_diff_style_gpu import TOL_TRAJ, _module
from test_diff_style_host import _write_pngs, mini_logvar

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# add_h_rows
# ------------------------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    """a * b + c of fp32 tensors rounded once to fp32, as fmaf does: the product is exact in fp64, a two-sum gives the
    exact sum as s + err, rounding s to odd with err makes the later rounding to fp32 the single correct one (53 bits
    >= 24 + 2)"""
    a, b, c = a.double(), b.double(), c.double()
    prod = a * b
    s = prod + c
    bb = s - prod
    err = (prod - (s - bb)) + (c - bb)
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(err > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))
    return torch.where((err != 0) & even, torch.nextafter(s, toward), s).float()


def _restated(h, d, coef):
    """h2 as the kernel computes it: v = fmaf(α, d, c0 * h) with c0 * h rounded to fp32, stored as fp16"""
    N = h.shape[0]
    p = coef[:, 0].view(N, 1, 1, 1) * h.float()
    v = _fma32(coef[:, 1].view(N, 1, 1, 1).expand_as(p), d.permute(1, 2, 0)[None].expand_as(p), p)
    return v.half(), v


def _fp16_ulp(y):
    """the spacing of fp16 values at |y| (subnormal spacing below 2^-14)"""
    e = torch.floor(torch.log2(y.double().abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


@pytest.mark.parametrize("C", [256, 512, 1024])
@pytest.mark.parametrize("N", [1, 3, 17])
def test_add_h_rows(cuda_device, C, N):
    dev = cuda_device
    g = torch.Generator().manual_seed(C + N)
    H = W = 8
    T = 3
    h = (torch.randn(N, H, W, C, generator=g) * 3).half()
    h[h == 0] = 1.0  # -0 + 0 is +0: keep the (1, 0) identity check about values
    h = h.to(dev)
    d = torch.randn(C, H, W, generator=g).to(dev)
    base = [(1.0, 0.0), (1.0, 1.0), (0.9, -2.5), (0.0, 1.0), (1.0, 0.37)]
    coef = torch.tensor([base[n % len(base)] if n < len(base) else (float(torch.rand(1, generator=g)),
                                                                     float(torch.randn(1, generator=g)))
                         for n in range(N)], dtype=torch.float32, device=dev)
    h2 = torch.full_like(h, float("nan"))
    st = torch.full((N, T, C // 2, 2), float("nan"), device=dev)
    ops.add_h_rows(h, d, h2, st, coef)
    torch.cuda.synchronize()
    ref16, v = _restated(h, d, coef)
    assert torch.equal(h2, ref16), "h2 differs from fmaf(α, d, c0 * h)"
    assert torch.equal(st[:, 1:], torch.zeros_like(st[:, 1:]))
    for n in range(N):
        r2, rs = torch.full_like(h2[:1], float("nan")), torch.full_like(st[:1], float("nan"))
        ops.add_h_rows(h[n:n + 1].contiguous(), d, r2, rs, coef[n:n + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(h2[n:n + 1], r2) and torch.equal(st[n:n + 1], rs), f"row {n}"
        if tuple(coef[n].tolist()) == (1.0, 0.0):
            assert torch.equal(h2[n], h[n]), f"row {n}: (1, 0) must return h"
    # against fp64: h2 within one fp16 ulp, the sums within 1e-6 of the sum of magnitudes
    exact = coef[:, 0].double().view(N, 1, 1, 1) * h.double() + coef[:, 1].double().view(N, 1, 1, 1) * \
        d.permute(1, 2, 0)[None].double()
    assert ((h2.double() - exact).abs() <= _fp16_ulp(h2)).all()
    pairs = exact.view(N, H * W, C // 2, 2)
    s_ref, ss_ref = pairs.sum(dim=(1, 3)), (pairs ** 2).sum(dim=(1, 3))
    assert ((st[:, 0, :, 0].double() - s_ref).abs() <= 1e-6 * pairs.abs().sum(dim=(1, 3)) + 1e-30).all()
    assert ((st[:, 0, :, 1].double() - ss_ref).abs() <= 1e-6 * ss_ref + 1e-30).all()
    # bad arguments
    with pytest.raises(_lib.AsyrpError):
        ops.add_h_rows(h, d, h2, st, coef[:1] if N > 1 else coef.view(2, 1))
    with pytest.raises(_lib.AsyrpError):
        ops.add_h_rows(h, d[:, :4], h2, st, coef)
    with pytest.raises(_lib.AsyrpError):
        ops.add_h_rows(h, d, h, st, coef)
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    for args in ((N, 3, H, W, T), (0, C, H, W, T), (N, C, H, W, 0), (N, C, 1 << 16, 1 << 16, T)):
        n_, c_, hh, ww, tt = args
        rc = lib.asyrp_add_h_rows(P(h), P(d), P(h2), P(st), tt, n_, c_, hh, ww, P(coef), s)
        assert rc == -1, args
    assert lib.asyrp_add_h_rows(P(h), P(d), P(h2), P(st), T, N, C, H, W, None, s) == -1


# ------------------------------------------------------------------------------------------------------------------
# statistics
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [16384, 32768, 65536])
def test_gram_and_combine_against_fp64(cuda_device, d):
    dev = cuda_device
    for n in (2, 63, 64, 65, 257):
        g = torch.Generator().manual_seed(n * 7 + d)
        x = (torch.randn(n, d, generator=g) * torch.linspace(0.1, 3.0, d) + torch.randn(1, d, generator=g)).float()
        xn = x.double().numpy()
        mu_ref = xn.mean(axis=0)
        mu = ops.h_combine(x.to(dev), torch.full((1, n), 1.0 / n, dtype=torch.float64, device=dev))[0]
        assert np.allclose(mu.cpu().numpy(), mu_ref, rtol=0, atol=1e-12 * np.abs(xn).max())
        G = ops.h_gram(x.to(dev), mu).cpu().numpy()
        xc = xn - mu.cpu().numpy()[None]
        ref = xc @ xc.T
        scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
        assert (np.abs(G - ref) <= 1e-12 * scale).all(), f"n={n} d={d}: Gram"
        assert np.array_equal(G, G.T)
        K = 10
        w = torch.randn(K, n, generator=g, dtype=torch.float64)
        for m in (mu, None):
            out = ops.h_combine(x.to(dev), w.to(dev), m).cpu().numpy()
            xcm = xn - (m.cpu().numpy()[None] if m is not None else 0.0)
            ref = w.numpy() @ xcm
            bound = np.abs(w.numpy()) @ np.abs(xcm)
            assert (np.abs(out - ref) <= 1e-12 * bound + 1e-300).all(), f"n={n} d={d}: combine"
            assert np.allclose(out, oh.combine(xn, w.numpy(), None if m is None else m.cpu().numpy()), rtol=1e-12,
                               atol=1e-12 * bound.max())


def test_statistics_refusals(cuda_device):
    dev = cuda_device
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(1024, dtype=torch.float64, device=dev)
    p = ctypes.c_void_p(buf.data_ptr())
    # the Gram: n < 2, d <= 0, n d at 2^31
    for n, d in ((1, 16), (0, 16), (2, 0), (1 << 15, 1 << 16), (2, 1 << 30)):
        assert lib.asyrp_h_gram(p, p, p, n, d, s) == -1, (n, d)
    assert lib.asyrp_h_gram(p, p, None, 2, 16, s) == -1
    # combine: K, n or d not positive, n d / K d / K n at 2^31
    for n, d, K in ((1, 16, 0), (0, 16, 1), (1, 0, 1), (1 << 15, 1 << 16, 1), (1, 1 << 16, 1 << 15),
                    (1 << 16, 1, 1 << 15)):
        assert lib.asyrp_h_combine(p, p, None, p, n, d, K, s) == -1, (n, d, K)
    assert lib.asyrp_h_combine(p, None, None, p, 2, 16, 1, s) == -1
    # the nearest accepted neighbours run
    x = torch.randn(2, 64, device=dev)
    G = ops.h_gram(x, x.double().mean(0))
    assert torch.allclose(G, G.T) and G.shape == (2, 2)
    assert ops.h_combine(x, torch.ones(1, 2, dtype=torch.float64, device=dev)).shape == (1, 64)
    with pytest.raises(_lib.AsyrpError):
        ops.h_gram(x[:1].contiguous(), x.double().mean(0))
    with pytest.raises(_lib.AsyrpError):
        ops.h_combine(x, torch.ones(1, 3, dtype=torch.float64, device=dev))


# ------------------------------------------------------------------------------------------------------------------
# trajectories
# ------------------------------------------------------------------------------------------------------------------
COEFS = [(1.0, 0.0), (1.0, 1.0), (0.9, 2.0), (1.0, -1.5), (1.0, 1.0)]


def _setup(dev, C, S, n_step=8, seed=5, t_edit=500):
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, n_step)
    mk = lambda edit=True: Schedule(betas, seq, seq_next, t_edit=t_edit, t_addnoise=300, hs_coeff=(1.0,),  # noqa: E731
                                    edit=edit, logvars=mini_logvar(False))
    sch = mk()
    g = torch.Generator().manual_seed(seed)
    R = len(COEFS)
    x = torch.randn(R, 3, S, S, generator=g)
    D = torch.randn(sch.n_edit, C, 8, 8, generator=g) * 0.5
    noises = {t: torch.randn(R, 3, S, S, generator=g) for t in seq if t < 300}
    assert sch.n_stochastic and sch.n_edit
    nz = torch.stack([noises[s.t] for s in sch.steps if s.stochastic])
    return betas, seq, seq_next, mk, sch, x.to(dev), D.to(dev), noises, nz.to(dev)


def test_mixed_alpha_batch_graph_and_origin(cuda_device):
    """rows with their own (c0, α) == batch-1 runs bit for bit; eager == graph; another table replays the same graph;
    α = 0 rows match the origin pass within TOL_TRAJ"""
    dev = cuda_device
    m = _module("ddpm").to(dev)
    eng = m.engine
    _, _, _, mk, sch, x, D, _, nz = _setup(dev, 256, 32)
    table = torch.tensor(COEFS)
    out = eng.sample(x, sch, noise=nz, h_direction=D, hs_coeffs=table)
    rec, n_graphs = eng.last_records, len(eng.graphs)
    eng.sample(x, sch, noise=nz, h_direction=D, hs_coeffs=table * 0.5)
    assert eng.last_records is rec and len(eng.graphs) == n_graphs, "a second table must replay the same graph"
    eager = eng.sample(x, sch, noise=nz, h_direction=D, hs_coeffs=table, use_graph=False)
    assert torch.equal(out, eager)
    for n, c in enumerate(COEFS):
        one = eng.sample(x[n:n + 1], sch, noise=nz[:, n:n + 1].contiguous(), h_direction=D,
                         hs_coeffs=torch.tensor([c]))
        assert torch.equal(out[n:n + 1], one), f"row {n} {c}"
    origin = eng.sample(x, mk(edit=False), noise=nz)
    for n, c in enumerate(COEFS):
        if c == (1.0, 0.0):
            e, mx = (out[n] - origin[n]).abs().max().item(), origin[n].abs().max().item()
            assert e <= TOL_TRAJ * max(1.0, mx), f"α = 0 row {n}: {e:.3e}"
    # refusals
    for kw in ({"hs_coeffs": None}, {"hs_coeffs": torch.ones(5, 3)}, {"delta_hs": D}, {"record_dh": True}):
        with pytest.raises(_lib.AsyrpError):
            eng.sample(x, sch, noise=nz, h_direction=D, **{"hs_coeffs": table, **kw})
    with pytest.raises(_lib.AsyrpError):
        eng.sample(x, sch, noise=nz, h_direction=D[1:], hs_coeffs=table)


def _oracle_rows(fwd_base, monkeypatch, module, x, D, sch, seq, seq_next, noises, learn_sigma, t_edit):
    """the oracle's edit loop one row at a time, its DeltaBlock replaced by the direction of the current step: the
    DeltaBlock branch h2 = h c0 + delta_block(...) α then computes h c0 + α d_t"""
    edit_ts = [s.t for s in sch.steps if s.edit]
    dirs = {t: D[k:k + 1].cpu() for k, t in enumerate(edit_ts)}
    cur = {}
    monkeypatch.setattr(module, "delta_block", lambda sd, p, h, temb: dirs[cur["t"]].expand_as(h))

    def fwd(xt, t, **k):
        cur["t"] = int(t[0])
        return fwd_base(xt, t, **k)

    betas, logv = osmp.make_betas(), mini_logvar(learn_sigma)
    outs = []
    for r, c in enumerate(COEFS):
        xr = x[r:r + 1].cpu().clone()
        for i, j in zip(reversed(seq), reversed(seq_next)):
            xr = osmp.denoising_step(xr, torch.ones(1) * i, torch.ones(1) * j, model=fwd, logvars=logv, b=betas,
                                     eta=1.0 if i < 300 else 0.0, learn_sigma=learn_sigma, index=0, t_edit=t_edit,
                                     hs_coeff=c, noise=noises[i][r:r + 1] if i in noises else None)[0]
        outs.append(xr)
    return torch.cat(outs)


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_mini_trajectories_against_the_oracle(cuda_device, monkeypatch, family):
    dev = cuda_device
    m = _module(family)
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    learn_sigma = family == "adm"
    fwd = (lambda *a, **k: od.ddpm_forward(sd, od.MINI_CFG, *a, **k)) if family == "ddpm" else \
        (lambda *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k))
    betas, seq, seq_next, mk, sch, x, D, noises, nz = _setup(dev, m.arch.mid_ch, 32)
    if learn_sigma:
        sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(1.0,))
    out = m.engine.sample(x, sch, noise=nz, h_direction=D, hs_coeffs=torch.tensor(COEFS)).cpu()
    ref = _oracle_rows(fwd, monkeypatch, od if family == "ddpm" else oa, x, D, sch, seq, seq_next, noises,
                       learn_sigma, 500)
    for r in range(len(COEFS)):
        e, mx = (out[r] - ref[r]).abs().max().item(), ref[r].abs().max().item()
        print(f"\n{family} row {r} {COEFS[r]}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"{family} row {r}: {e:.3e} of {mx:.3e}"


def test_celeba256_trajectory_against_the_oracle(cuda_device, monkeypatch):
    dev = cuda_device
    m = _module("ddpm", od.CELEBA_CFG, style="torch_default")
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    betas, seq, seq_next, mk, sch, x, D, noises, nz = _setup(dev, 512, 256, n_step=6, t_edit=400)
    out = m.engine.sample(x, sch, noise=nz, h_direction=D, hs_coeffs=torch.tensor(COEFS)).cpu()
    del m
    torch.cuda.empty_cache()
    fwd = lambda *a, **k: od.ddpm_forward(sd, od.CELEBA_CFG, *a, **k)  # noqa: E731
    ref = _oracle_rows(fwd, monkeypatch, od, x, D, sch, seq, seq_next, noises, False, 400)
    for r in range(len(COEFS)):
        e, mx = (out[r] - ref[r]).abs().max().item(), ref[r].abs().max().item()
        print(f"\nceleba256 row {r} {COEFS[r]}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"row {r}: {e:.3e} of {mx:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# end to end (DDPM CelebA-HQ 256², synthetic weights)
# ------------------------------------------------------------------------------------------------------------------
BASE = ["--config", "celeba.yml", "--synthetic_weights", "--n_test_step", "8", "--seed", "1234"]


def test_discovery_and_editing_end_to_end(cuda_device, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    args, cfg = cli.parse_args_and_config(BASE + ["--h_directions", "--load_random_noise", "--n_train_img", "24",
                                                  "--bs_train", "8", "--h_pca", "3", "--h_direction_out", "dirs"])
    r = Asyrp(args, cfg, device=cuda_device)
    paths = r.run_h_directions(keep_h=True)
    assert sorted(os.listdir("dirs")) == ["h_directions.tsv", "pc0.pth", "pc1.pth", "pc2.pth"]
    X = r.h_directions_x.cpu().double().numpy()
    assert X.shape == (8, 24, 512 * 64)
    ref = oh.pca(X, 3)
    ts = [s for s in reversed(make_sequences(999, 8)[0])]
    for c, p in enumerate(paths):
        obj = torch.load(p, weights_only=True)
        assert obj["n"] == 24 and obj["mid_ch"] == 512 and sorted(obj["delta_h"]) == sorted(ts)
        for k, t in enumerate(ts):
            got, want = obj["delta_h"][t].double().numpy().ravel(), ref[k][3][c]
            e = np.abs(got - want).max() / np.abs(want).max()
            assert e <= 1e-6, f"pc{c} t={t}: {e:.3e}"
    tsv = open("dirs/h_directions.tsv").read().splitlines()
    assert tsv[0].split("\t")[:4] == ["t", "pc0_variance", "pc0_ratio", "pc0_cos_prev"] and len(tsv) == 9
    # editing with the first component, as an interpolation sweep, scored for content preservation
    edit = BASE + ["--run_test", "--h_direction", "dirs/pc0.pth", "--delta_interpolation", "--num_delta", "3",
                   "--min_delta", "-1", "--max_delta", "1", "--hs_coeff_delta_h", "2", "--user_defined_t_edit", "500",
                   "--user_defined_t_addnoise", "0", "--load_random_noise", "--n_train_img", "2", "--n_test_img",
                   "2", "--bs_train", "2", "--save_x_origin", "--content_preservation"]
    args, cfg = cli.parse_args_and_config(edit)
    r = Asyrp(args, cfg, device=cuda_device)
    res = r.run_test()
    files = os.listdir(args.test_image_folder)
    for mode in ("train", "test"):
        assert f"{mode}_1_0_ngen6.png" in files and f"{mode}_1_0_ngen6_content_preservation.tsv" in files
        xs = res[(mode, 1)]
        assert len(xs) == 4 and all(torch.isfinite(v).all() for v in xs)
        # v = 0 (the middle tuple) edits with α = 0
        e, mx = (xs[2] - xs[0]).abs().max().item(), xs[0].abs().max().item()
        assert e <= TOL_TRAJ * max(1.0, mx), f"{mode}: α = 0 against the origin pass {e:.3e}"
        assert r.content_preservation[f"{mode}_1_0"].shape == (3, 2, 4)


def test_mean_difference_of_a_set_against_itself(cuda_device, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    _write_pngs("imgs", ["a.png", "b.png", "c.png"], [(256, 256), (240, 256), (256, 200)])
    args, cfg = cli.parse_args_and_config(BASE + ["--h_directions", "--h_pos_dir", "imgs", "--h_neg_dir", "imgs",
                                                  "--n_inv_step", "8", "--bs_train", "3", "--n_train_img", "3",
                                                  "--h_direction_out", "md"])
    with monkeypatch.context() as mp:  # device memory is checked before any image is inverted
        def no_inversion(*a, **k):
            raise AssertionError("an image was inverted before the memory check")
        mp.setattr(Asyrp, "invert_batch", no_inversion)
        mp.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 80 << 30))
        with pytest.raises(MemoryError, match="6 samples"):
            Asyrp(args, cfg, device=cuda_device).run_h_directions()
    r = Asyrp(args, cfg, device=cuda_device)
    r.run_h_directions()
    assert not hasattr(r, "h_directions_x"), "the recorded h is kept only with keep_h"
    obj = torch.load("md/mean_diff.pth", weights_only=True)
    assert obj["n"] == {"pos": 3, "neg": 3}
    assert all(not v.any() for v in obj["delta_h"].values())
    args, cfg = cli.parse_args_and_config(BASE + ["--run_test", "--h_direction", "md/mean_diff.pth",
                                                  "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0",
                                                  "--load_random_noise", "--n_train_img", "2", "--do_test", "0",
                                                  "--bs_train", "2", "--save_x_origin"])
    xs = Asyrp(args, cfg, device=cuda_device).run_test()[("train", 1)]
    e, mx = (xs[1] - xs[0]).abs().max().item(), xs[0].abs().max().item()
    assert e <= TOL_TRAJ * max(1.0, mx), f"zero direction against the origin pass: {e:.3e}"


def test_pca_of_an_image_folder(cuda_device, tmp_path, monkeypatch):
    """--h_pca over --custom_train_dataset_dir: the images are inverted by precompute_pairs into run_test's train
    cache, and no test set is needed"""
    monkeypatch.chdir(tmp_path)
    _write_pngs("imgs", ["a.png", "b.png", "c.png"], [(256, 256), (240, 256), (256, 200)])
    args, cfg = cli.parse_args_and_config(BASE + ["--h_directions", "--h_pca", "2", "--custom_train_dataset_dir",
                                                  "imgs", "--custom_test_dataset_dir", "missing", "--n_inv_step", "8",
                                                  "--bs_train", "2", "--n_train_img", "3", "--h_direction_out", "pc"])
    Asyrp(args, cfg, device=cuda_device).run_h_directions()
    assert sorted(os.listdir("pc")) == ["h_directions.tsv", "pc0.pth", "pc1.pth"]
    assert os.listdir("precomputed") == ["CelebA_HQ_train_t999_nim3_ninv8_pairs.pth"]
    pairs = torch.load("precomputed/CelebA_HQ_train_t999_nim3_ninv8_pairs.pth", weights_only=True)
    assert len(pairs) == 3 and torch.load("pc/pc0.pth", weights_only=True)["n"] == 3
