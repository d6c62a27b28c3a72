"""Content preservation on the GPU: the quantiser bit for bit against the fp64 oracle, the SSE exact, each SSIM level
and the pooling against fp64 at small, odd and 256^2 sizes, exact scores of identical images, batch and chunk
independence, LPIPS against lpips.LPIPS.forward bit for bit, every argument rule of the four entry points, and
`main --run_test --content_preservation` end to end."""
import csv
import ctypes
import os

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, lpips, main as cli, ops, preservation as pv, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp, _load_image_folder
from oracle import preservation as op

pytestmark = pytest.mark.gpu


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _images(n, H, W, seed, scale=1.0):
    """smooth images with noise in [-1, 1] (partly outside with scale > 1)"""
    g = _g(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    base = torch.stack([torch.sin(5 * xx + 3 * c * yy) * torch.cos(4 * yy + c) for c in range(3)])
    return (0.7 * base + 0.2 * torch.randn(n, 3, H, W, generator=g)).clamp(-1, 1) * scale


def _edit(x, seed, amount=0.1):
    return (x + amount * torch.randn(x.shape, generator=_g(seed))).clamp(-1, 1)


@pytest.mark.parametrize("B,H,W", [(2, 256, 256), (3, 11, 13), (1, 1, 1)])
def test_quantize_bit_exact(cuda_device, B, H, W):
    x = _images(B, H, W, H + W, scale=1.3)
    flat = x.view(-1)
    if flat.numel() > 600:
        # x = k / 255 - 1: (x + 1) * 0.5 * 255 + 0.5 on the truncation boundary (k odd) and half way (k even), up to
        # the fp32 rounding of x; then values far outside [-1, 1]
        flat[:511] = torch.arange(511, dtype=torch.float32) / 255.0 - 1
        flat[512:520] = torch.tensor([-1.0, 1.0, -7.0, 3.0, 1.0 / 255 - 1, 2.0 / 255 - 1, float("inf"), -float("inf")])
    else:
        flat[:] = torch.tensor([-1.0, 1.0, 5.0])
    d = x.to(cuda_device)
    q = torch.full((B, 3, H, W), 7, dtype=torch.uint8, device=cuda_device)
    lvl0 = torch.full((B, 3, H, W), float("nan"), dtype=torch.float64, device=cuda_device)
    xq = torch.full((B, 3, H, W), float("nan"), device=cuda_device)
    ops.png_quantize(d, q, lvl0, xq)
    ref = torch.from_numpy(op.quantize(x.numpy()))
    assert torch.equal(q.cpu(), ref)
    assert torch.equal(lvl0.cpu(), ref.double() / 255.0)
    assert torch.equal(xq.cpu(), (2.0 * ref.float() - 255.0) / 255.0)
    # xq is lpips.im2tensor's value of the PNG (q / 127.5 - 1 in fp64, then fp32) up to the last fp32 bit
    im2 = torch.from_numpy(ref.numpy() / 127.5 - 1.0).float()
    assert ((xq.cpu() - im2).abs() <= 6e-8).all()
    q2 = torch.zeros_like(q)
    ops.png_quantize(d, q2)  # lvl0 / xq skipped
    assert torch.equal(q2, q)


@pytest.mark.parametrize("n,B,H,W", [(5, 2, 256, 256), (3, 3, 11, 13), (4, 1, 1, 1)])
def test_sse_exact(cuda_device, n, B, H, W):
    g = _g(n + H)
    src = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    ed = torch.randint(0, 256, (n, 3, H, W), generator=g, dtype=torch.uint8)
    src[(n - 1) % B], ed[n - 1] = 0, 255  # every difference the largest: 65025 per value
    ed[0] = src[0]
    sse = torch.full((n,), -1, dtype=torch.int64, device=cuda_device)
    ops.preserve_sse(src.to(cuda_device), ed.to(cuda_device), sse)
    s, e = src.numpy().astype(np.int64), ed.numpy().astype(np.int64)
    ref = np.array([((e[j] - s[j % B]) ** 2).sum() for j in range(n)])
    assert np.array_equal(sse.cpu().numpy(), ref) and ref[0] == 0


@pytest.mark.parametrize("n,B,H,W", [(2, 1, 11, 11), (3, 3, 12, 13), (4, 2, 161, 161), (4, 2, 256, 256),
                                     (1, 1, 45, 300)])
def test_ssim_level_and_pool_against_fp64(cuda_device, n, B, H, W):
    src = torch.from_numpy(op.quantize(_images(B, H, W, H).numpy()) / 255.0)
    ed = torch.from_numpy(op.quantize(_edit(_images(B, H, W, H), W).repeat(n // B + 1, 1, 1, 1)[:n].numpy()) / 255.0)
    stats = torch.full((n, 3, 2), float("nan"), dtype=torch.float64, device=cuda_device)
    ds, de = src.to(cuda_device), ed.to(cuda_device)
    ops.ssim_level(ds, de, stats)
    ref = op.ssim_stats(src.numpy()[np.arange(n) % B], ed.numpy())
    assert np.abs(stats.cpu().numpy() - ref).max() <= 1e-12
    assert (ref[..., 0] < 0.999).all()
    # a row's statistics do not depend on the launch it is in
    one = torch.empty(1, 3, 2, dtype=torch.float64, device=cuda_device)
    ops.ssim_level(ds[(n - 1) % B:(n - 1) % B + 1], de[n - 1:], one)
    assert torch.equal(one, stats[n - 1:])
    pooled = torch.full((n, 3, (H + 1) // 2, (W + 1) // 2), float("nan"), dtype=torch.float64, device=cuda_device)
    ops.ssim_pool2(de, pooled)
    assert np.abs(pooled.cpu().numpy() - op.pool2(ed.numpy())).max() <= 1e-12


@pytest.fixture(scope="module")
def scorer(cuda_device):
    sd = synthetic.lpips_state_dict(seed=7)
    return sd, pv.ContentPreservation(sd, device=cuda_device)


def test_scores_against_the_oracle(scorer):
    _, m = scorer
    src = _images(2, 256, 256, 1)
    ed = torch.cat([_edit(src, 2, 0.05), _edit(src, 3, 0.2), src])
    s = m.scores(src, ed)
    ref = op.scores(src.numpy(), ed.numpy())
    assert s.dtype == torch.float64 and tuple(s.shape) == (6, 4)
    assert np.array_equal(s[:4, 0].numpy(), ref[:4, 0])  # the SSE is exact and the log the same expression
    assert np.abs(s[:, 1:3].numpy() - ref[:, 1:]).max() <= 1e-12
    assert (s[:2, :3] > s[2:4, :3]).all() and (s[:4, 3] > 0).all()  # the stronger edit preserves less
    assert s[4:].tolist() == [[float("inf"), 1.0, 1.0, 0.0]] * 2  # identical images


def test_lpips_equals_the_forward_bit_for_bit(scorer, cuda_device):
    sd, m = scorer
    src = _images(2, 256, 256, 4)
    ed = torch.cat([_edit(src, 5), _edit(src, 6, 0.3)])
    s = m.scores(src, ed)
    deq = lambda x: torch.from_numpy((2.0 * op.quantize(x.numpy()).astype(np.float32) - 255.0) / 255.0)  # noqa: E731
    net = lpips.LPIPS(sd, device=cuda_device)
    ref = net(deq(ed).to(cuda_device), deq(src).repeat(2, 1, 1, 1).to(cuda_device)).view(-1).cpu().double()
    assert torch.equal(s[:, 3], ref) and (ref > 0).all()


def test_rows_are_independent_of_batch_and_chunk(scorer, cuda_device):
    sd, m = scorer
    src = _images(3, 200, 176, 8)
    ed = torch.cat([_edit(src, 9 + k, 0.05 * (k + 1)) for k in range(3)])  # 9 rows, 3 tuples
    s = m.scores(src, ed)
    assert torch.equal(m.scores(src, ed), s)
    for j in (0, 4, 8):
        assert torch.equal(m.scores(src[j % 3:j % 3 + 1], ed[j:j + 1]), s[j:j + 1])  # alone
    assert torch.equal(m.scores(src, ed[3:6]), s[3:6])
    chunked = pv.ContentPreservation(sd, device=cuda_device, max_rows=1)  # one tuple (3 rows) per chunk
    assert torch.equal(chunked.scores(src, ed), s)
    assert torch.equal(pv.ContentPreservation(sd, device=cuda_device, max_rows=7).scores(src, ed), s)


def test_scorer_refusals(scorer):
    _, m = scorer
    with pytest.raises(ValueError, match="larger than 160"):
        m.scores(_images(1, 160, 256, 1), _images(1, 160, 256, 2))
    with pytest.raises(ValueError, match="whole multiple"):
        m.scores(_images(2, 256, 256, 1), _images(3, 256, 256, 2))
    with pytest.raises(ValueError, match="one size"):
        m.scores(_images(1, 256, 256, 1), _images(1, 256, 200, 2))


def _err():
    return _lib.load().asyrp_last_error().decode()


def test_argument_rules(cuda_device):
    lib = _lib.load()
    P, st = ops._ptr, ops._stream()
    dev = cuda_device
    f32 = torch.zeros(2, 3, 12, 12, device=dev)
    u8 = torch.zeros(2, 3, 12, 12, dtype=torch.uint8, device=dev)
    f64 = torch.zeros(2, 3, 12, 12, dtype=torch.float64, device=dev)
    sse = torch.zeros(4, dtype=torch.int64, device=dev)
    stats = torch.zeros(4, 3, 2, dtype=torch.float64, device=dev)
    pooled = torch.zeros(2, 3, 6, 6, dtype=torch.float64, device=dev)
    off = lambda t, b: ctypes.c_void_p(t.data_ptr() + b)  # noqa: E731

    def refused(rc, match):
        assert rc == -1 and match in _err(), (rc, _err())

    # asyrp_png_quantize
    q = lambda x, qq, l0, xq, B, H, W: lib.asyrp_png_quantize(x, qq, l0, xq, B, H, W, st)  # noqa: E731
    assert q(P(f32), P(u8), P(f64), P(f32.clone()), 2, 12, 12) == 0
    for B, H, W in ((0, 12, 12), (2, 0, 12), (2, 12, -1)):
        refused(q(P(f32), P(u8), None, None, B, H, W), "bad shape")
    refused(q(P(f32), P(u8), None, None, 1 << 30, 1 << 30, 1 << 4), "too large")
    refused(q(None, P(u8), None, None, 2, 12, 12), "null")
    refused(q(P(f32), None, None, None, 2, 12, 12), "null")
    refused(q(off(f32, 2), P(u8), None, None, 1, 1, 1), "aligned")
    refused(q(P(f32), P(u8), off(f64, 4), None, 1, 1, 1), "aligned")
    refused(q(P(f32), P(u8), None, off(f32, 2), 1, 1, 1), "aligned")
    assert q(off(f32, 4), off(u8, 1), off(f64, 8), off(f32, 4), 1, 1, 1) == 0  # the nearest aligned neighbours
    # asyrp_preserve_sse
    s = lambda a, b, o, n, B, plane: lib.asyrp_preserve_sse(a, b, o, n, B, plane, st)  # noqa: E731
    assert s(P(u8), P(u8), P(sse), 2, 2, 432) == 0
    for n, B, plane in ((0, 2, 432), (2, 0, 432), (2, 2, 0)):
        refused(s(P(u8), P(u8), P(sse), n, B, plane), "bad shape")
    refused(s(P(u8), P(u8), P(sse), 1, 1, (1 << 47) + 1), "above 2^47")
    refused(s(P(u8), P(u8), P(sse), 1 << 16, 1, 1 << 47), "too large")
    refused(s(None, P(u8), P(sse), 2, 2, 432), "null")
    refused(s(P(u8), P(u8), None, 2, 2, 432), "null")
    refused(s(P(u8), P(u8), off(sse, 4), 2, 2, 432), "aligned")
    assert s(off(u8, 1), off(u8, 3), off(sse, 8), 2, 2, 430) == 0  # u8 rows need no alignment
    # asyrp_ssim_level
    lv = lambda a, b, o, n, B, H, W: lib.asyrp_ssim_level(a, b, o, n, B, H, W, st)  # noqa: E731
    assert lv(P(f64), P(f64), P(stats), 2, 2, 12, 12) == 0
    assert lv(P(f64), P(f64), P(stats), 2, 2, 11, 11) == 0
    for n, B in ((0, 2), (2, 0)):
        refused(lv(P(f64), P(f64), P(stats), n, B, 12, 12), "bad shape")
    refused(lv(P(f64), P(f64), P(stats), 2, 2, 10, 12), "below the 11 x 11 window")
    refused(lv(P(f64), P(f64), P(stats), 2, 2, 12, 10), "below the 11 x 11 window")
    refused(lv(P(f64), P(f64), P(stats), 715827883, 1, 11, 11), "planes above")
    refused(lv(P(f64), P(f64), P(stats), 1, 1, 11, 2147483647 - 41), "too large")
    refused(lv(P(f64), P(f64), P(stats), 1, 1, 1 << 16, 1 << 30), "too many tiles")
    refused(lv(P(f64), P(f64), P(stats), 1 << 29, 1, 1 << 16, 1 << 16), "rows x 3 H W too large")
    refused(lv(None, P(f64), P(stats), 2, 2, 12, 12), "null")
    refused(lv(P(f64), P(f64), None, 2, 2, 12, 12), "null")
    for a, b, o in ((off(f64, 4), P(f64), P(stats)), (P(f64), off(f64, 4), P(stats)), (P(f64), P(f64), off(stats, 4))):
        refused(lv(a, b, o, 1, 1, 11, 11), "aligned")
    assert lv(P(f64), off(f64, 8), off(stats, 8), 1, 1, 11, 11) == 0
    # asyrp_ssim_pool2
    pl = lambda a, b, rows, H, W: lib.asyrp_ssim_pool2(a, b, rows, H, W, st)  # noqa: E731
    assert pl(P(f64), P(pooled), 2, 12, 12) == 0
    for rows, H, W in ((0, 12, 12), (2, 0, 12), (2, 12, 0)):
        refused(pl(P(f64), P(pooled), rows, H, W), "bad shape")
    refused(pl(P(f64), P(pooled), 1, 2147483647, 1), "too large")
    refused(pl(P(f64), P(pooled), 1 << 21, 1 << 21, 1 << 21), "rows x 3 H W too large")  # 3 * 2^63 elements
    refused(pl(P(f64), P(f64), 2, 12, 12), "aliased")
    refused(pl(None, P(pooled), 2, 12, 12), "null")
    refused(pl(off(f64, 4), P(pooled), 1, 1, 1), "aligned")
    refused(pl(P(f64), off(pooled, 4), 1, 1, 1), "aligned")
    assert pl(off(f64, 8), off(pooled, 8), 1, 1, 1) == 0
    torch.cuda.synchronize()


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


BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/cp", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0",
        "--synthetic_weights", "--seed", "1234", "--train_delta_block", "--get_h_num", "1"]
TSV = "test_1_0_ngen4_content_preservation.tsv"


def _setup(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)


@pytest.mark.parametrize("mode", ["single", "interp", "sweep"])
def test_run_test_scores_every_edit(cuda_device, tmp_path, monkeypatch, mode):
    _setup(tmp_path, monkeypatch)
    argv = BASE + ["--load_random_noise", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]
    tuples = 1
    if mode == "interp":
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
        tuples = 3
    elif mode == "sweep":
        argv = BASE + ["--load_random_noise", "--attr_sweep", "smiling angry", "--manual_checkpoint_name",
                       "attribute_0.pth"]
        tuples = 2
    r, res = _run(argv + ["--content_preservation"], cuda_device)
    _, plain = _run(argv, cuda_device)                              # without the flag
    _, with_origin = _run(argv + ["--save_x_origin"], cuda_device)  # the origin row the scores compare against
    rows = res[("test", 1)]
    assert len(rows) == tuples and len(with_origin[("test", 1)]) == tuples + 1
    for a, b, c in zip(rows, plain[("test", 1)], with_origin[("test", 1)][1:]):
        assert torch.equal(a, b) and torch.equal(a, c)  # the scores change no edited image
    origin = with_origin[("test", 1)][0]
    table = _table(os.path.join(r.args.test_image_folder, TSV))
    header = ["image", "tuple", "hs_coeff", "PSNR", "SSIM", "MS_SSIM", "LPIPS"] + (["attr"] if mode == "sweep" else [])
    assert table[0] == header and len(table) == 1 + tuples * 2  # random latents: no origin rows
    assert [(int(t[1]), int(t[0])) for t in table[1:]] == [(k, i) for k in range(tuples) for i in range(2)]
    if mode == "sweep":
        assert [t[7] for t in table[1:]] == ["smiling", "smiling", "angry", "angry"]
    vals = torch.tensor([[float(v) for v in t[3:7]] for t in table[1:]], dtype=torch.float64)
    assert torch.equal(vals.view(tuples, 2, 4), r.content_preservation["test_1_0"])
    assert r.reconstruction == {}
    # the scorer on the run's own origin and edited images gives the table's bits
    m = pv.ContentPreservation(synthetic.lpips_state_dict(seed=1234), device=cuda_device)
    assert torch.equal(m.scores(origin, torch.cat(rows)), vals)
    assert ((vals[:, 1] > -1) & (vals[:, 1] < 1) & (vals[:, 3] > 0)).all()


def test_run_test_shares_the_origin_pass(cuda_device, tmp_path, monkeypatch):
    from asyrp_official_b200 import diffusion_latent
    _setup(tmp_path, monkeypatch)
    torch.save(synthetic.arcface_state_dict(seed=5), "ir_se50.pth")
    torch.save(synthetic.face_parsing_state_dict(seed=5), "79999_iter.pth")
    argv = BASE + ["--load_random_noise", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling",
                   "--id_similarity", "--id_weights", "ir_se50.pth", "--seg_consistency", "--seg_weights",
                   "79999_iter.pth"]
    calls = []
    orig = diffusion_latent.Asyrp.edit_batch

    def counting(self, *a, **kw):
        calls.append(1)
        return orig(self, *a, **kw)
    r1, res1 = _run(argv, cuda_device)
    monkeypatch.setattr(diffusion_latent.Asyrp, "edit_batch", counting)
    r2, res2 = _run(argv + ["--content_preservation"], cuda_device)
    assert len(calls) == 2  # one origin pass, one edit pass, for all three scores
    assert all(torch.equal(a, b) for a, b in zip(res1[("test", 1)], res2[("test", 1)]))
    assert torch.equal(r1.id_similarity["test_1_0"], r2.id_similarity["test_1_0"])
    assert torch.equal(r1.seg_consistency["test_1_0"], r2.seg_consistency["test_1_0"])
    assert r2.content_preservation["test_1_0"].shape == (1, 2, 4)


def test_run_on_real_images_scores_the_reconstruction(cuda_device, tmp_path, monkeypatch):
    from PIL import Image
    _setup(tmp_path, monkeypatch)
    os.makedirs("faces")
    for i, x in enumerate(_images(2, 256, 256, 21)):
        Image.fromarray(op.quantize(x.numpy()).transpose(1, 2, 0)).save(f"faces/{i}.png")
    argv = BASE + ["--custom_test_dataset_dir", "faces", "--custom_train_dataset_dir", "faces",
                   "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr",
                   "smiling", "--save_x_origin", "--content_preservation"]
    r, res = _run(argv, cuda_device)
    origin, edited = res[("test", 1)]
    table = _table(os.path.join(r.args.test_image_folder, TSV))
    assert table[0] == ["image", "tuple", "hs_coeff", "PSNR", "SSIM", "MS_SSIM", "LPIPS"] and len(table) == 5
    assert [t[:3] for t in table[1:3]] == [["0", "origin", "-"], ["1", "origin", "-"]]
    rec = torch.tensor([[float(v) for v in t[3:7]] for t in table[1:3]], dtype=torch.float64)
    cp = torch.tensor([[float(v) for v in t[3:7]] for t in table[3:]], dtype=torch.float64)
    assert torch.equal(rec, r.reconstruction["test_1_0"]) and torch.equal(cp, r.content_preservation["test_1_0"][0])
    m = pv.ContentPreservation(synthetic.lpips_state_dict(seed=1234), device=cuda_device)
    x0 = torch.cat(_load_image_folder("faces", 256, 2))
    assert torch.equal(m.scores(x0, origin), rec)
    assert torch.equal(m.scores(origin, edited), cp)
    assert torch.isfinite(rec).all() and (rec[:, 1] < 1).all()
