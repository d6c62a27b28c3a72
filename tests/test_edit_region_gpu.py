"""--edit_region on the GPU: the blend kernel (exact for m in {0, 1}, the exact fmaf restatement and 1 ulp of fp64 for
random m, at the benchmark shape, odd HW and N = k B, refusals), the mask kernels against oracle/region.py, blended
trajectories on synthetic mini UNets and DDPM CelebA 256² (mask of ones = unblended edit, zeros = origin pass, m = 0
pixels = origin, graph = eager, rows = their batch-1 runs, the fp64 oracle), and `--run_test --edit_region` end to
end."""
import csv
import ctypes
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, face_parsing, main as cli, modules, ops, region, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import adm as oa, ddpm as od, region as orr, sampler as osmp
from test_diff_style_gpu import TOL_TRAJ
from test_diff_style_host import mini_logvar
from test_h_directions_gpu import _fma32

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# blend kernel
# ------------------------------------------------------------------------------------------------------------------
def _restated(x, ref, mask):
    """fmaf(m, x, (1 - m) * r) in fp32 with each rounding explicit, rows n against image n % B"""
    N, B = x.shape[0], ref.shape[0]
    idx = torch.arange(N, device=x.device) % B
    m = mask[idx][:, None].expand_as(x)
    r = ref[idx]
    return _fma32(m, x, (1 - m) * r)


def _ulp32(y):
    e = torch.floor(torch.log2(y.double().abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 23)


@pytest.mark.parametrize("N,B,C,H,W", [(16, 16, 3, 256, 256), (16, 4, 3, 256, 256), (6, 3, 3, 5, 7), (4, 1, 3, 9, 9),
                                       (12, 4, 2, 64, 64), (3, 3, 1, 1, 1)])
def test_blend_rows(cuda_device, N, B, C, H, W):
    dev = cuda_device
    g = torch.Generator().manual_seed(N * 31 + H * W)
    x = torch.randn(N, C, H, W, generator=g).to(dev)
    x[x == 0] = 0.5
    ref = torch.randn(B, C, H, W, generator=g).to(dev)
    hard = (torch.rand(B, H, W, generator=g) > 0.5).float().to(dev)
    out = x.clone()
    ops.blend_rows(out, ref, hard)
    torch.cuda.synchronize()
    idx = torch.arange(N) % B
    m = hard[idx][:, None].expand_as(x)
    assert torch.equal(out, torch.where(m == 1, x, ref[idx])), "m in {0, 1} must select x or r exactly"
    soft = torch.rand(B, H, W, generator=g).to(dev)
    soft.view(-1)[::7] = 0.0
    soft.view(-1)[1::7] = 1.0
    out = x.clone()
    ops.blend_rows(out, ref, soft)
    torch.cuda.synchronize()
    assert torch.equal(out, _restated(x, ref, soft)), "differs from fmaf(m, x, (1 - m) * r)"
    # against fp64: one rounding of the result, and the two roundings of (1 - m) * r, which the fma carries unchanged
    # where m x and (1 - m) r cancel: within 1 ulp of the result plus 2 ulp of the (1 - m) r term
    ms = soft[idx][:, None].double()
    rest = (1 - ms) * ref[idx].double()
    exact = ms * x.double() + rest
    assert ((out.double() - exact).abs() <= _ulp32(exact) + 2 * _ulp32(rest)).all(), "beyond the rounding bound"
    for n in range(0, N, max(1, N // 4)):  # a row alone is the same bits
        one = x[n:n + 1].clone()
        ops.blend_rows(one, ref[n % B:n % B + 1].contiguous(), soft[n % B:n % B + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(one, out[n:n + 1]), f"row {n}"


def test_blend_rows_refusals(cuda_device):
    dev = cuda_device
    N, B, C, H, W = 4, 2, 3, 8, 8
    x = torch.randn(N, C, H, W, device=dev)
    ref = torch.randn(B, C, H, W, device=dev)
    mask = torch.rand(B, H, W, device=dev)
    for bad in ((x, ref[:1].expand(3, C, H, W).contiguous(), mask), (x, ref, mask[:1]), (x.half(), ref, mask),
                (x, ref.cpu(), mask), (x, ref, mask.cpu()), (x[:, :, :, :4], ref, mask),
                (x, ref[:, :, :4].contiguous(), mask)):
        with pytest.raises(_lib.AsyrpError):
            ops.blend_rows(*bad)
    # float4 loads need 16-byte alignment: a tensor one element into its storage is refused
    buf = torch.randn(N * C * H * W + 1, device=dev)
    before = buf.clone()
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        ops.blend_rows(buf[1:].view(N, C, H, W), ref, mask)
    mbuf = torch.rand(B * H * W + 1, device=dev)
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        ops.blend_rows(x.clone(), ref, mbuf[1:].view(B, H, W))
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
    # odd HW takes one element per thread and only 4-byte alignment
    xo = torch.randn(N * C * 9 + 1, device=dev)
    ro, mo = torch.randn(B, C, 3, 3, device=dev), torch.rand(B, 3, 3, device=dev)
    tgt = xo[1:].view(N, C, 3, 3)
    want = _restated(tgt.clone(), ro, mo)
    ops.blend_rows(tgt, ro, mo)
    torch.cuda.synchronize()
    assert torch.equal(tgt, want)
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    HW = H * W
    for args in ((N, 3, C, HW), (0, B, C, HW), (N, 0, C, HW), (N, B, 0, HW), (N, B, C, 0), (N, B, C, -4)):
        assert lib.asyrp_blend_rows(P(x), P(ref), P(mask), *args, s) == -1, args
    assert lib.asyrp_blend_rows(None, P(ref), P(mask), N, B, C, HW, s) == -1
    assert lib.asyrp_blend_rows(P(x), None, P(mask), N, B, C, HW, s) == -1
    assert lib.asyrp_blend_rows(P(x), P(ref), None, N, B, C, HW, s) == -1


# ------------------------------------------------------------------------------------------------------------------
# mask kernels
# ------------------------------------------------------------------------------------------------------------------
def _labels(n, seed):
    """blobby label maps: a coarse random class map, nearest-upsampled, with scattered single pixels"""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randint(0, 19, (n, 1, 16, 16), generator=g).float()
    lab = torch.nn.functional.interpolate(coarse, size=(512, 512), mode="nearest")[:, 0].to(torch.uint8)
    pts = torch.randint(0, 512, (n, 2, 200), generator=g)
    for i in range(n):
        lab[i, pts[i, 0], pts[i, 1]] = 17
    return lab


@pytest.mark.parametrize("S", [32, 256, 512])
def test_mask_kernels_against_the_oracle(cuda_device, S):
    dev = cuda_device
    lab = _labels(3, S)
    classes = [17, 18]
    sel = torch.empty(3, S, S, device=dev)
    ops.region_mask(lab.to(dev), region.class_bits(classes), sel)
    ref_sel = orr.select(lab.numpy(), classes, S)
    assert np.array_equal(sel.cpu().numpy(), ref_sel)
    assert 0 < ref_sel.mean() < 1
    for r in (0, 1, 32):
        got = region.masks_from_labels(lab.to(dev), classes, S, r, 0.0).cpu().numpy()
        assert np.array_equal(got, orr.dilate(ref_sel, r)), f"dilate r={r}"
    for r, sigma in ((0, 0.7), (1, 16.0), (0, 0.0), (32, 0.7)):
        got = region.masks_from_labels(lab.to(dev), classes, S, r, sigma).cpu().double().numpy()
        want = orr.feather(orr.dilate(ref_sel, r), sigma)
        err = np.abs(got - want).max()
        assert err <= 1e-6, f"r={r} sigma={sigma}: {err:.3e}"
        flat = (want == 0) | (want == 1)
        assert np.array_equal(got[flat], want[flat]), f"r={r} sigma={sigma}: flat windows must stay exactly 0 or 1"
        assert got.min() >= 0 and got.max() <= 1 + 1e-6


def test_mask_kernel_refusals(cuda_device):
    dev = cuda_device
    lab = torch.zeros(2, 512, 512, dtype=torch.uint8, device=dev)
    m = torch.zeros(2, 64, 64, device=dev)
    tmp = torch.empty_like(m)
    w = region.taps(1.0).to(dev)
    with pytest.raises(_lib.AsyrpError):
        ops.region_mask(lab[:, :256].contiguous(), 1, m)
    with pytest.raises(_lib.AsyrpError):
        ops.region_mask(lab, 1, m[:1])
    with pytest.raises(_lib.AsyrpError):
        ops.region_mask(lab, 1 << 32, m)
    with pytest.raises(_lib.AsyrpError):
        ops.mask_dilate(m, m, 1, 0)
    with pytest.raises(_lib.AsyrpError):
        ops.mask_dilate(m, tmp, 33, 0)
    with pytest.raises(_lib.AsyrpError):
        ops.mask_dilate(m, tmp, 1, 2)
    with pytest.raises(_lib.AsyrpError):
        ops.mask_blur(m, w[:-1].contiguous(), tmp, 0)
    with pytest.raises(_lib.AsyrpError):
        ops.mask_blur(m, torch.ones(99, device=dev) / 99, tmp, 0)  # R = 49
    with pytest.raises(_lib.AsyrpError):
        ops.mask_blur(m, w.cpu(), tmp, 0)
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    for n, S in ((0, 64), (2, 0), (2, 513), (65536, 64)):
        assert lib.asyrp_region_mask(P(lab), 1, P(m), n, S, s) == -1, (n, S)
        assert lib.asyrp_mask_dilate(P(m), P(tmp), n, S, 1, 0, s) == -1, (n, S)
        assert lib.asyrp_mask_blur(P(m), P(w), P(tmp), n, S, 3, 0, s) == -1, (n, S)
    assert lib.asyrp_region_mask(None, 1, P(m), 2, 64, s) == -1
    assert lib.asyrp_mask_dilate(P(m), P(tmp), 2, 64, -1, 0, s) == -1
    assert lib.asyrp_mask_blur(P(m), None, P(tmp), 2, 64, 3, 0, s) == -1
    assert lib.asyrp_mask_blur(P(m), P(w), P(tmp), 2, 64, 49, 0, s) == -1
    mis = torch.zeros(2 * 64 * 64 + 1, device=dev)
    assert lib.asyrp_mask_dilate(ctypes.c_void_p(mis.data_ptr() + 2), P(tmp), 2, 64, 1, 0, s) == -1
    assert lib.asyrp_mask_blur(P(m), P(w), ctypes.c_void_p(mis.data_ptr() + 2), 2, 64, 3, 0, s) == -1


# ------------------------------------------------------------------------------------------------------------------
# trajectories
# ------------------------------------------------------------------------------------------------------------------
COEFS = [(1.0, 1.0), (1.0, 0.5), (0.9, 1.5)]


def _module(family, cfg=None, style="jittered"):
    if family == "ddpm":
        cfg = cfg or od.MINI_CFG
        ns = NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=cfg["image_size"]))
        m = modules.DDPM(ns)
    else:
        m = modules._create_adm(cfg or oa.MINI_HP)
    m.setattr_layers(1)
    synthetic.randomize_(m, 1234, style)
    return m


def _schedules(learn_sigma, n_step=6, t_edit=500, t_addnoise=300, sample_type="ddim"):
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, n_step)
    lv = None if learn_sigma else mini_logvar(False)
    edit = Schedule(betas, seq, seq_next, t_edit=t_edit, t_addnoise=t_addnoise, hs_coeff=(1.0, 1.0),
                    sample_type=sample_type, logvars=lv)
    origin = Schedule(betas, seq, seq_next, t_edit=t_edit, t_addnoise=0, hs_coeff=(1.0,), edit=False,
                      sample_type=sample_type, logvars=lv)
    return betas, seq, seq_next, edit, origin


def _case(eng, x, edit, origin, noise_e, noise_o):
    o = eng.sample(x, origin, noise=noise_o, record_process=True)
    return o, eng.last_records["x"].clone()


@pytest.mark.parametrize("family,sample_type", [("ddpm", "ddim"), ("adm", "ddim"), ("ddpm", "ddpm")])
def test_blended_trajectories(cuda_device, family, sample_type):
    dev = cuda_device
    m = _module(family).to(dev)
    eng = m.engine
    B, k = 2, len(COEFS)
    S = eng.arch.image_size
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 3, S, S, generator=g).to(dev)
    betas, seq, seq_next, edit, origin = _schedules(family == "adm", sample_type=sample_type)
    nz_o = torch.randn(origin.n_stochastic, B, 3, S, S, generator=g).to(dev) if origin.n_stochastic else None
    nz_e = torch.randn(edit.n_stochastic, B, 3, S, S, generator=g).to(dev) if edit.n_stochastic else None
    o, ref = _case(eng, x, edit, origin, nz_e, nz_o)
    assert torch.equal(ref[-1], o)
    plain = eng.sample(x, edit, noise=nz_e)
    launches = eng.last_launches
    ones, zeros = torch.ones(B, S, S, device=dev), torch.zeros(B, S, S, device=dev)
    assert torch.equal(eng.sample(x, edit, noise=nz_e, blend=(ones, ref)), plain), "mask of ones"
    assert eng.last_launches == launches + len(edit.steps)
    n_graphs = len(eng.graphs)
    assert torch.equal(eng.sample(x, edit, noise=nz_e, blend=(zeros, ref)), o), "mask of zeros"
    assert len(eng.graphs) == n_graphs, "another mask must replay the same graph"
    hard = (torch.rand(B, S, S, generator=g) > 0.5).float().to(dev)
    out = eng.sample(x, edit, noise=nz_e, blend=(hard, ref))
    keep = (hard == 0)[:, None].expand_as(out)
    assert torch.equal(out[keep], o[keep]), "m = 0 pixels must equal the origin pass"
    assert not torch.equal(out, o) and not torch.equal(out, plain)
    assert torch.equal(eng.sample(x, edit, noise=nz_e, blend=(hard, ref), use_graph=False), out), "graph vs eager"
    assert torch.equal(eng.sample(x, edit, noise=nz_e), plain), "without blend the trajectory is unchanged"
    # tuple-major rows of k tuples x B images: row n equals its batch-1 run
    xs = x.repeat(k, 1, 1, 1)
    nzs = nz_e.repeat(1, k, 1, 1, 1) if nz_e is not None else None
    table = torch.tensor([c for c in COEFS for _ in range(B)])
    soft = torch.rand(B, S, S, generator=g).to(dev)
    rows = eng.sample(xs, edit, noise=nzs, blend=(soft, ref), hs_coeffs=table)
    for n in range(k * B):
        b = n % B
        one = eng.sample(x[b:b + 1], edit, noise=nz_e[:, b:b + 1].contiguous() if nz_e is not None else None,
                         blend=(soft[b:b + 1].contiguous(), ref[:, b:b + 1].contiguous()), hs_coeffs=table[n:n + 1])
        assert torch.equal(rows[n:n + 1], one), f"row {n}"
    # refusals
    bad = [(ones[:1].expand(3, S, S).contiguous(), ref), (ones, ref[1:]), (ones.cpu(), ref), (ones, ref.cpu()),
           (ones.double(), ref), (ones[:, :4].contiguous(), ref), ones]
    for b in bad:
        with pytest.raises(_lib.AsyrpError):
            eng.sample(x, edit, noise=nz_e, blend=b)
    with pytest.raises(_lib.AsyrpError):
        eng.sample(x, edit, noise=nz_e, blend=(ones, ref), lpips=object())
    if sample_type == "ddim":
        rs = RowSchedule(betas, seq, seq_next, [500] * B, [0] * B, [(1.0, 1.0)] * B)
        with pytest.raises(_lib.AsyrpError):
            eng.sample(x, rs, blend=(ones, ref))


def _oracle_blended(fwd, x, mask, ref, betas, seq, seq_next, learn_sigma, noises, t_edit, t_addnoise):
    return orr.run_blended_trajectory(fwd, x.cpu(), mask.cpu(), ref.cpu(), betas=betas, seq=seq, seq_next=seq_next,
                                      t_edit=t_edit, t_addnoise=t_addnoise, index=0, hs_coeff=(1.0, 1.0),
                                      learn_sigma=learn_sigma, noises=noises,
                                      logvars=None if learn_sigma else mini_logvar(False))


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_mini_blended_trajectory_against_the_oracle(cuda_device, family):
    dev = cuda_device
    m = _module(family)
    sd = {k_: v.cpu() for k_, v in m.state_dict().items()}
    m = m.to(dev)
    learn_sigma = family == "adm"
    fwd = (lambda *a, **k: od.ddpm_forward(sd, od.MINI_CFG, *a, **k)) if family == "ddpm" else \
        (lambda *a, **k: oa.adm_forward(sd, oa.MINI_HP, *a, **k))
    S = 32
    betas, seq, seq_next, edit, origin = _schedules(learn_sigma)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 3, S, S, generator=g)
    noises = {t: torch.randn(2, 3, S, S, generator=g) for t in seq if t < 300}
    nz = torch.stack([noises[s.t] for s in edit.steps if s.stochastic]).to(dev)
    o, ref = _case(m.engine, x.to(dev), edit, origin, None, None)
    mask = orr.feather(orr.select(_labels(2, 4).numpy(), [17, 3], S), 1.5)
    mask = torch.from_numpy(mask).float()
    out = m.engine.sample(x.to(dev), edit, noise=nz, blend=(mask.to(dev), ref)).cpu()
    want = _oracle_blended(fwd, x, mask, ref, betas, seq, seq_next, learn_sigma, noises, 500, 300)
    for r in range(2):
        e, mx = (out[r] - want[r]).abs().max().item(), want[r].abs().max().item()
        print(f"\n{family} row {r}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"{family} row {r}: {e:.3e} of {mx:.3e}"


def test_celeba256_blended_trajectory(cuda_device):
    """DDPM CelebA 256²: ones = unblended edit, zeros = origin, m = 0 pixels = origin, rows = batch-1 runs, and the
    fp64 oracle within the trajectory tolerance"""
    dev = cuda_device
    m = _module("ddpm", od.CELEBA_CFG, style="torch_default")
    sd = {k_: v.cpu() for k_, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    S, B = 256, 2
    betas, seq, seq_next, edit, origin = _schedules(False, n_step=5, t_edit=400, t_addnoise=0)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, 3, S, S, generator=g)
    o, ref = _case(eng, x.to(dev), edit, origin, None, None)
    plain = eng.sample(x.to(dev), edit)
    assert torch.equal(eng.sample(x.to(dev), edit, blend=(torch.ones(B, S, S, device=dev), ref)), plain)
    assert torch.equal(eng.sample(x.to(dev), edit, blend=(torch.zeros(B, S, S, device=dev), ref)), o)
    mask = region.masks_from_labels(_labels(B, 8).to(dev), [17, 5, 6], S, 2, 0.0)
    out = eng.sample(x.to(dev), edit, blend=(mask, ref))
    keep = (mask == 0)[:, None].expand_as(out)
    assert torch.equal(out[keep], o[keep])
    table = torch.tensor([c for c in COEFS[:2] for _ in range(B)])
    rows = eng.sample(x.to(dev).repeat(2, 1, 1, 1), edit, blend=(mask, ref), hs_coeffs=table)
    assert torch.equal(rows[:B], out)
    for n in range(2 * B):
        one = eng.sample(x[n % B:n % B + 1].to(dev), edit, hs_coeffs=table[n:n + 1],
                         blend=(mask[n % B:n % B + 1].contiguous(), ref[:, n % B:n % B + 1].contiguous()))
        assert torch.equal(rows[n:n + 1], one), f"row {n}"
    out = out.cpu()
    del m, eng
    torch.cuda.empty_cache()
    fwd = lambda *a, **k: od.ddpm_forward(sd, od.CELEBA_CFG, *a, **k)  # noqa: E731
    want = _oracle_blended(fwd, x, mask, ref, betas, seq, seq_next, False, None, 400, 0)
    for r in range(B):
        e, mx = (out[r] - want[r]).abs().max().item(), want[r].abs().max().item()
        print(f"\nceleba256 row {r}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"row {r}: {e:.3e} of {mx:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# end to end (DDPM CelebA-HQ 256², synthetic weights)
# ------------------------------------------------------------------------------------------------------------------
BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/er", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500",
        "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
        "--get_h_num", "1", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling",
        "--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5",
        "--max_rows_per_replay", "4", "--save_x_origin"]


def _png(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"))


def test_run_test_edit_region_end_to_end(cuda_device, tmp_path, monkeypatch):
    from test_seg_consistency_gpu import _delta_block_ckpt
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    torch.save(synthetic.face_parsing_state_dict(seed=5), "79999_iter.pth")
    built = []

    class Counting(face_parsing.FaceParser):
        def __init__(self, *a, **k):
            built.append(1)
            super().__init__(*a, **k)
    monkeypatch.setattr(face_parsing, "FaceParser", Counting)
    argv = BASE + ["--edit_region", "hair", "--seg_weights", "79999_iter.pth", "--edit_region_dilate", "1",
                   "--seg_consistency"]
    args, cfg = cli.parse_args_and_config(argv)
    r = Asyrp(args, cfg, device=cuda_device)
    res = r.run_test()
    assert len(built) == 1, "--seg_consistency and --edit_region share one parser"
    folder = args.test_image_folder
    files = os.listdir(folder)
    for name in ("test_1_0_ngen4.png", "test_1_0_ngen4_region_mask.png", "test_1_0_ngen4_seg_consistency.tsv"):
        assert name in files, name
    with open(os.path.join(folder, "test_1_0_ngen4_seg_consistency.tsv")) as f:
        assert len(list(csv.reader(f, delimiter="\t"))) == 1 + 3 * 2
    rows = res[("test", 1)]
    assert len(rows) == 4  # the origin row and three tuples
    origin = rows[0]
    # the mask the run built, from the origin pass it saved
    parser = face_parsing.FaceParser(torch.load("79999_iter.pth", weights_only=True), device=cuda_device)
    mask = region.region_masks(parser, origin, [17], 1, 0.0).cpu()
    print(f"\nmask covers {mask.mean().item():.3f} of the image")
    grid_mask = _png(os.path.join(folder, "test_1_0_ngen4_region_mask.png"))
    S = 256
    for i in range(2):
        m_png = grid_mask[1:1 + S, 1 + i * (S + 1):1 + i * (S + 1) + S, 0]
        assert np.array_equal(m_png, (mask[i].numpy() * 255).astype(np.uint8))
    grid = _png(os.path.join(folder, "test_1_0_ngen4.png"))
    cell = lambda row, col: grid[1 + row * (S + 1):1 + row * (S + 1) + S, 1 + col * (S + 1):1 + col * (S + 1) + S]  # noqa: E731
    for k in range(1, 4):
        for i in range(2):
            out = (mask[i] == 0).numpy()
            assert np.array_equal(cell(k, i)[out], cell(0, i)[out]), f"tuple {k - 1} image {i}"
            keep = (mask[i] == 0)[None].expand(3, S, S)
            assert torch.equal(rows[k][i][keep], origin[i][keep])
    # without the flag the edits are the unrestricted ones
    args, cfg = cli.parse_args_and_config(BASE)
    plain = Asyrp(args, cfg, device=cuda_device).run_test()[("test", 1)]
    assert torch.equal(plain[0], origin)
    if bool((mask == 1).all()):
        assert all(torch.equal(a, b) for a, b in zip(plain[1:], rows[1:]))
