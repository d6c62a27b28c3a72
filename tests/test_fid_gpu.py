"""FID Inception-v3 and the FID / KID statistics on the GPU: each kernel against fp64 or torch at the shapes the network
launches and at odd sizes, the full synthetic network within the DESIGN.md §2 bound, batch and chunk independence of
the features, and `main --run_test --fid` end to end."""
import csv
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import fid, main as cli, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import fid as ofid

pytestmark = pytest.mark.gpu
# DESIGN.md §2, TF32 emulation of the full synthetic network (scripts/fid_emulate.py), about 3x its worst errors:
# features max-abs 2.9e-3, FID abs 2.5e-3.  KID abs 1.1e-5 emulated, 4.9e-5 measured on an H100 for the unrelated set
# (the GPU rounds the BN-folded weights, the emulation the raw ones): about 2x the measured error
FEAT_TOL, FID_TOL, KID_TOL = 1e-2, 1e-2, 1e-4


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _tf32(x):
    b = x.float().contiguous().view(torch.int32)
    b = (b + 0x1000) & ~0x1FFF  # round to nearest, ties away (cvt.rna)
    return b.view(torch.float32).double()


@pytest.mark.parametrize("B,H,W", [(2, 256, 256), (1, 64, 64), (3, 37, 45), (1, 1, 1), (1, 512, 300)])
def test_pack(cuda_device, B, H, W):
    x = torch.rand(B, 3, H, W, generator=_g(H)) * 2.4 - 1.2
    x.view(-1)[:6] = torch.tensor([-1.0, 1.0, -1 + 1 / 255, 0.0, 2 / 255 - 1, 1 - 0.5 / 255])[:x.numel()]
    out = torch.empty(B, 299, 299, 4, device=cuda_device)
    ops.fid_pack(x.to(cuda_device), out)
    ref = ofid.preprocess(x, dtype=torch.float32).permute(0, 2, 3, 1)
    assert (out[..., :3].cpu() - ref).abs().max().item() <= 2e-6  # the resize, within fp32 rounding
    assert torch.equal(out[..., 3].cpu(), torch.zeros(B, 299, 299))
    if H == W:  # at S = H the resize is the identity: the u8 values exactly
        same = torch.empty(B, H, H, 4, device=cuda_device)
        ops.fid_pack(x.to(cuda_device), same)
        q = ofid.quantise(x).float() / 255 * 2 - 1
        assert torch.equal(same[..., :3].cpu(), q.permute(0, 2, 3, 1))


# (cin, cout, kh, kw, stride, pad_h, pad_w, H, W): the stem, the 1x7 / 7x1 / 1x3 / 3x1 convs with their one-sided
# padding, the stride-2 convs of InceptionB / D, at the network's sizes 149 / 147 / 73 / 71 / 35 / 17 / 8
CONVS = [(4, 32, 3, 3, 2, 0, 0, 299, 299), (32, 64, 3, 3, 1, 1, 1, 147, 147), (64, 80, 1, 1, 1, 0, 0, 73, 73),
         (80, 192, 3, 3, 1, 0, 0, 73, 73), (48, 64, 5, 5, 1, 2, 2, 35, 35), (288, 384, 3, 3, 2, 0, 0, 35, 35),
         (160, 160, 1, 7, 1, 0, 3, 17, 17), (160, 192, 7, 1, 1, 3, 0, 17, 17), (192, 320, 3, 3, 2, 0, 0, 17, 17),
         (384, 384, 1, 3, 1, 0, 1, 8, 8), (384, 384, 3, 1, 1, 1, 0, 8, 8), (32, 32, 3, 3, 1, 0, 0, 149, 149),
         (8, 64, 1, 7, 2, 0, 3, 11, 13)]


def _conv_case(cuda_device, cin, cout, kh, kw, stride, ph, pw, H, W, ldo, c0, seed):
    x = torch.randn(2, H, W, cin, generator=_g(seed))
    w = torch.randn(cout, cin, kh, kw, generator=_g(seed + 1)) * (2 / (cin * kh * kw)) ** 0.5
    b = torch.randn(cout, generator=_g(seed + 2)) * 0.1
    rows = -(-cout // 64) * 64
    wp, bp = torch.zeros(rows, cin, kh, kw), torch.zeros(rows)
    wp[:cout], bp[:cout] = w, b
    packed = ops.pack_lpips_conv_weight(wp.to(cuda_device))
    Ho, Wo = (H + 2 * ph - kh) // stride + 1, (W + 2 * pw - kw) // stride + 1
    full = torch.full((2, Ho, Wo, ldo), 12345.0, device=cuda_device)  # sentinel around the slice
    ops.fid_conv(x.to(cuda_device), packed, bp.to(cuda_device), full[..., c0:c0 + cout], kh, kw, stride, (ph, pw),
                 cstore=cout)
    xt, wt = _tf32(x).permute(0, 3, 1, 2), _tf32(w)
    ref = F.conv2d(xt, wt, b.double(), stride=stride, padding=(ph, pw)).clamp_min(0).permute(0, 2, 3, 1)
    absc = F.conv2d(xt.abs(), wt.abs(), stride=stride, padding=(ph, pw)).permute(0, 2, 3, 1) + b.double().abs()
    got = full.cpu().double()
    assert ((got[..., c0:c0 + cout] - ref).abs() <= 2e-5 * absc + 1e-6).all()
    assert (got[..., :c0] == 12345.0).all() and (got[..., c0 + cout:] == 12345.0).all()


@pytest.mark.parametrize("cin,cout,kh,kw,stride,ph,pw,H,W", CONVS)
def test_conv_shapes(cuda_device, cin, cout, kh, kw, stride, ph, pw, H, W):
    _conv_case(cuda_device, cin, cout, kh, kw, stride, ph, pw, H, W, cout, 0, cin + H)


@pytest.mark.parametrize("cout,c0,ldo", [(32, 224, 256), (48, 0, 48), (96, 128, 288), (160, 8, 170), (320, 0, 2048),
                                         (448, 1600, 2048)])
def test_conv_channel_slices(cuda_device, cout, c0, ldo):
    _conv_case(cuda_device, 36, cout, 3, 1, 1, 1, 0, 17, 17, ldo, c0, cout)


def test_conv_refusals(cuda_device):
    x = torch.zeros(1, 8, 8, 8, device=cuda_device)
    w = ops.pack_lpips_conv_weight(torch.zeros(64, 8, 1, 1, device=cuda_device))
    b = torch.zeros(64, device=cuda_device)
    out = torch.zeros(1, 8, 8, 66, device=cuda_device)
    with pytest.raises(Exception, match="cstore"):
        ops.fid_conv(x, w, b, out[..., 1:66], 1, 1, cstore=65)
    with pytest.raises(Exception, match="aligned"):
        ops.fid_conv(x, w, b, out[..., 1:33], 1, 1)


@pytest.mark.parametrize("N,H,W,C", [(2, 147, 147, 64), (2, 71, 71, 192), (1, 35, 35, 288), (1, 17, 17, 768),
                                     (3, 8, 8, 2048), (2, 5, 7, 12), (1, 1, 1, 4), (1, 3, 3, 8)])
def test_pools_exact_against_torch(cuda_device, N, H, W, C):
    x = torch.randn(N, C, H, W, generator=_g(H * C)).to(cuda_device)
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    cases = [(ops.FID_POOL_AVG3S1, F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)),
             (ops.FID_POOL_MAX3S1, F.max_pool2d(x, 3, 1, 1))]
    if H >= 3 and W >= 3:
        cases.append((ops.FID_POOL_MAX3S2, F.max_pool2d(x, 3, 2)))
    for mode, ref in cases:
        Ho, Wo = ref.shape[2:]
        full = torch.full((N, Ho, Wo, C + 8), -7.0, device=cuda_device)  # a slice at channel 4 of a wider tensor
        ops.fid_pool(nhwc, full[..., 4:4 + C], mode)
        assert torch.equal(full[..., 4:4 + C], ref.permute(0, 2, 3, 1)), mode
        assert (full[..., :4] == -7).all() and (full[..., 4 + C:] == -7).all()


def test_global_mean(cuda_device):
    x = torch.randn(3, 8, 8, 2048, generator=_g(1)).to(cuda_device)
    out = torch.empty(3, 2048, device=cuda_device)
    ops.fid_mean(x, out)
    ref = x.cpu().double().mean((1, 2))
    assert (out.cpu().double() - ref).abs().max().item() <= 1e-6


@pytest.mark.parametrize("n,d", [(2, 64), (300, 2048), (1000, 128), (77, 192)])
def test_moments_match_numpy(cuda_device, n, d):
    g = np.random.default_rng(n + d)
    f = (g.standard_normal((n, d)) * g.uniform(0.1, 3, d) + g.uniform(0, 2, d)).astype(np.float32)
    mu, sigma = ops.fid_moments(torch.from_numpy(f).to(cuda_device))
    rmu, rs = ofid.moments(f)
    assert np.abs(mu.cpu().numpy() - rmu).max() <= 1e-12 * np.abs(rmu).max()
    assert np.abs(sigma.cpu().numpy() - rs).max() <= 1e-12 * np.abs(rs).max()
    assert torch.equal(ops.fid_moments(torch.from_numpy(f).to(cuda_device))[1], sigma)


@pytest.mark.parametrize("n,m,d", [(300, 257, 2048), (1, 1, 16), (65, 64, 48), (130, 200, 2048)])
def test_kernel_sum_matches_numpy(cuda_device, n, m, d):
    g = np.random.default_rng(n * m)
    x, y = (g.random((k, d)).astype(np.float32) for k in (n, m))
    kxy = (x.astype(np.float64) @ y.astype(np.float64).T / d + 1) ** 3
    for excl in (False, True):
        got = ops.fid_kernel_sum(torch.from_numpy(x).to(cuda_device), torch.from_numpy(y).to(cuda_device), excl).item()
        ref = kxy.sum() - (np.trace(kxy) if excl else 0.0)
        assert abs(got - ref) <= 1e-12 * abs(ref) or (excl and n == m == 1 and got == 0.0)


def test_kid_against_the_double_loop(cuda_device):
    g = np.random.default_rng(3)
    f1, f2 = (g.random((k, 64)).astype(np.float32) for k in (11, 9))
    got = fid.kid(torch.from_numpy(f1).to(cuda_device), torch.from_numpy(f2).to(cuda_device))
    assert abs(got - ofid.kid_loop(f1, f2)) <= 1e-12 * 50


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model(cuda_device):
    sd = synthetic.inception_state_dict(seed=7)
    return sd, fid.FIDInception(sd, device=cuda_device)


def _images(n, seed, S=64):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    from clip_image_emulate import smooth_images
    return smooth_images(n, S, seed)


def test_full_network_within_the_design_bound(model, cuda_device):
    sd, m = model
    src = _images(8, 7)
    sets = {"edit": (src + 0.1 * _images(8, 107)).clamp(-1, 1), "unrelated": _images(8, 207)}
    ref_net = ofid.fid_inception(sd)
    f64 = {k: ofid.features(ref_net, ofid.preprocess(v)) for k, v in {"src": src, **sets}.items()}
    gpu = {k: m.features(v) for k, v in {"src": src, **sets}.items()}
    for k in f64:
        assert gpu[k].shape == (8, 2048)
        assert (gpu[k].double().cpu() - f64[k]).abs().max().item() <= FEAT_TOL
    scores = {}
    for k in sets:
        fd, kd = fid.fid_kid(gpu["src"], gpu[k])
        rf = fid.frechet_distance(*ofid.moments(f64["src"]), *ofid.moments(f64[k]))
        rk = ofid.kid_loop(f64["src"].numpy(), f64[k].numpy())
        assert abs(fd - rf) <= FID_TOL and abs(kd - rk) <= KID_TOL, (k, fd, rf, kd, rk)
        scores[k] = fd, kd
    assert scores["unrelated"][0] > 10 * scores["edit"][0] and scores["unrelated"][1] > scores["edit"][1]
    fd, _ = fid.fid_kid(gpu["src"], gpu["src"])
    assert abs(fd) <= 1e-4
    assert all(np.isnan(v) for v in fid.fid_kid(gpu["src"][:1], gpu["edit"][:1]))


def test_features_bit_identical_in_any_batch(model, cuda_device):
    sd, m = model
    x = _images(7, 3, S=96)
    f = m.features(x)
    assert torch.equal(m.features(x), f)
    for i in (0, 4, 6):
        assert torch.equal(m.features(x[i:i + 1]), f[i:i + 1])
    chunked = fid.FIDInception(sd, device=cuda_device, max_rows=3)  # chunks (0-2), (3-5), (6)
    assert torch.equal(chunked.features(x), f)
    assert torch.equal(chunked.features(torch.cat([x[5:], x[:2]])), torch.cat([f[5:], f[:2]]))


# ---------------------------------------------------------------------------------------------------------------------
def _delta_block_ckpt(path, seed):
    from types import SimpleNamespace as NS
    from asyrp_official_b200 import configs, modules
    c = configs.builtin_config("celeba")
    ns = NS(model=NS(**c["model"]), data=NS(image_size=256))
    m = modules.DDPM(ns)
    m.setattr_layers(1)
    synthetic.randomize_(m, seed=seed, style="jittered")
    torch.save({"0": {k: v.clone() for k, v in m.layer_0.state_dict().items()}}, path)


def _run(argv, dev):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config, device=dev)
    return r, r.run_test()


def _table(path):
    with open(path) as f:
        return list(csv.reader(f, delimiter="\t"))


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/fid", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500",
        "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
        "--get_h_num", "1"]


@pytest.mark.parametrize("mode", ["single", "interp", "sweep"])
def test_run_test_fid(cuda_device, tmp_path, monkeypatch, mode):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    sd = synthetic.inception_state_dict(seed=5)
    torch.save(sd, "pt_inception.pth")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)
    argv = BASE + ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]
    tuples = 1
    if mode == "interp":
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
        tuples = 3
    elif mode == "sweep":
        argv = BASE + ["--attr_sweep", "smiling angry", "--manual_checkpoint_name", "attribute_0.pth"]
        tuples = 2
    fid_argv = ["--fid", "--fid_weights", "pt_inception.pth"]
    r, res = _run(argv + ["--bs_train", "2"] + fid_argv, cuda_device)
    folder = r.args.test_image_folder
    tsv = os.path.join(folder, "test_ngen4_fid.tsv")
    png = os.path.join(folder, "test_1_0_ngen4.png")
    with_fid = _bytes(png), _bytes(tsv)
    _, plain = _run(argv + ["--bs_train", "2"], cuda_device)  # without the flag: the same edits, the same PNG
    assert _bytes(png) == with_fid[0]
    assert all(torch.equal(a, b) for a, b in zip(res[("test", 1)], plain[("test", 1)]))
    table = _table(tsv)
    header = ["tuple", "hs_coeff", "n", "FID", "KID"] + (["attr"] if mode == "sweep" else [])
    assert table[0] == header and len(table) == 1 + tuples
    assert [int(t[0]) for t in table[1:]] == list(range(tuples)) and all(t[2] == "2" for t in table[1:])
    if mode == "sweep":
        assert [t[5] for t in table[1:]] == ["smiling", "angry"]
    vals = torch.tensor([[float(t[3]), float(t[4])] for t in table[1:]], dtype=torch.float64)
    assert torch.equal(vals, r.fid["test"]) and torch.isfinite(vals).all()
    # one image per batch: the same features, the same set order, the same bits
    _run(argv + ["--bs_train", "1"] + fid_argv, cuda_device)
    assert _bytes(tsv) == with_fid[1]
    if mode == "single":  # the scorer on the run's own origin and edited images gives the table's bits
        _, with_origin = _run(argv + ["--bs_train", "2", "--save_x_origin"], cuda_device)
        origin, edited = with_origin[("test", 1)]
        m = fid.FIDInception(sd, device=cuda_device)
        fd, kd = fid.fid_kid(m.features(origin), m.features(edited))
        assert (fd, kd) == tuple(vals[0].tolist())


def test_run_test_with_all_four_scores_shares_the_origin_pass(cuda_device, tmp_path, monkeypatch):
    from asyrp_official_b200 import diffusion_latent
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    os.makedirs("utils")
    templates = ["a photo of a {}.", "{}"]
    with open("utils/text_dic.py", "w") as f:
        f.write("SRC_TRG_TXT_DIC = {'smiling': (['face'], ['smiling face'])}\n")
    with open("utils/text_templates.py", "w") as f:
        f.write(f"imagenet_templates = {templates!r}\n")
    n = synthetic.write_clip_vocab("bpe.txt.gz", synthetic.clip_bpe_merges(["a photo of a smiling face."]))
    clip_sd = synthetic.clip_text_state_dict(seed=5, width=128, layers=2, vocab=n, embed_dim=128)
    clip_sd.update(synthetic.clip_image_state_dict(seed=5, width=128, layers=2, patch=16, grid=14, embed_dim=128))
    torch.save(clip_sd, "clip.pt")
    torch.save(synthetic.arcface_state_dict(seed=5), "ir_se50.pth")
    torch.save(synthetic.face_parsing_state_dict(seed=5), "79999_iter.pth")
    torch.save(synthetic.inception_state_dict(seed=5), "pt_inception.pth")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = BASE + ["--bs_train", "2", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling",
                   "--DirectionalClipSmilarity", "--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz",
                   "--id_similarity", "--id_weights", "ir_se50.pth", "--seg_consistency", "--seg_weights",
                   "79999_iter.pth"]
    r1, res1 = _run(argv, cuda_device)
    folder = r1.args.test_image_folder
    names = ["test_1_0_ngen4.png", "test_1_0_ngen4_directional_clip.tsv", "test_1_0_ngen4_id_similarity.tsv",
             "test_1_0_ngen4_seg_consistency.tsv"]
    before = [_bytes(os.path.join(folder, nm)) for nm in names]
    calls = []
    orig = diffusion_latent.Asyrp.edit_batch

    def counting(self, *a, **kw):
        calls.append(1)
        return orig(self, *a, **kw)
    monkeypatch.setattr(diffusion_latent.Asyrp, "edit_batch", counting)
    r2, res2 = _run(argv + ["--fid", "--fid_weights", "pt_inception.pth"], cuda_device)
    assert len(calls) == 2  # one origin pass, one edit pass, for all four scores
    assert [_bytes(os.path.join(folder, nm)) for nm in names] == before
    assert all(torch.equal(a, b) for a, b in zip(res1[("test", 1)], res2[("test", 1)]))
    assert r2.fid["test"].shape == (1, 2) and torch.isfinite(r2.fid["test"]).all()
