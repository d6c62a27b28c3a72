"""Face-parsing BiSeNet and the segmentation consistency on the GPU: each kernel against fp64 at the shapes the network
launches and at odd sizes, the full synthetic BiSeNet within the DESIGN.md §2 bound at O(1) and x1e3 inputs, exact
agreement counts, determinism and batch independence, and `main --run_test --seg_consistency` end to end."""
import csv
import os

import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, face_parsing as fp, main as cli, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import face_parsing as of

pytestmark = pytest.mark.gpu
# DESIGN.md §2, TF32 emulation of the full synthetic BiSeNet (scripts/face_parsing_emulate.py), about 3x its max-abs
# logit error (3.3e-2 at O(1) inputs, 8.1e-2 at x1e3, where the clamp saturates the image and the logits are larger).
# A label can differ from fp64's only where the fp64 top-2 margin is at most 2 * LOGIT_TOL.
LOGIT_TOL = {1.0: 0.1, 1e3: 0.25}


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rel(out, ref):
    ref = ref.double()
    return ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2).double().cpu()


def _tf32(x):
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


@pytest.mark.parametrize("H,W", [(256, 256), (512, 512), (97, 300), (1, 1)])
def test_pack(cuda_device, H, W):
    x = torch.rand(2, 3, H, W, generator=_g(H + W)) * 3 - 1.5  # partly outside [-1, 1]: clamped
    out = torch.full((2, 512, 512, 4), float("nan"), device=cuda_device)
    ops.faceparse_pack(x.to(cuda_device), out)
    ref = of.preprocess(x)
    assert (_nchw(out[..., :3]) - ref).abs().max().item() <= 2e-6 * ref.abs().max().item()
    assert torch.equal(out[..., 3].cpu(), torch.zeros(2, 512, 512))


@pytest.mark.parametrize("H,W,C", [(256, 256, 64), (7, 9, 8), (2, 3, 4), (1, 1, 4)])
def test_maxpool_padding(cuda_device, H, W, C):
    """every value negative, the border pixels most negative: a padding tap counted as 0 (or a skipped border tap)
    changes the result"""
    x = -1 - torch.rand(2, C, H, W, generator=_g(H * W))
    x[:, :, 0] -= 10
    x[:, :, :, -1] -= 10
    out = torch.full((2, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), float("nan"), device=cuda_device)
    ops.faceparse_maxpool(_nhwc(x).to(cuda_device), out)
    assert torch.equal(_nchw(out), F.max_pool2d(x.double(), 3, 2, 1))


# (Cin, Cout, k, stride, H): the stem on the packed input, a BasicBlock's 3x3 / 2 and 1x1 / 2 downsample, the head's
# 3x3, the class layer, at sizes with partial tiles
@pytest.mark.parametrize("cin,cout,k,stride,H", [(4, 64, 7, 2, 37), (64, 128, 3, 2, 31), (128, 256, 1, 2, 17),
                                                 (256, 256, 3, 1, 13), (256, 64, 1, 1, 9)])
def test_conv_epilogues(cuda_device, cin, cout, k, stride, H):
    g = _g(cin + H)
    x = torch.randn(2, cin, H, H + 2, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    bias = torch.randn(cout, generator=g)
    pad = k // 2
    ref = F.conv2d(_tf32(x), _tf32(w), stride=stride, padding=pad) + bias.double().view(1, -1, 1, 1)
    res = torch.randn(ref.shape, generator=g)
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    out = torch.empty(2, ref.shape[2], ref.shape[3], cout, device=cuda_device)
    wp, xp = dev(ops.pack_lpips_conv_weight(w)), dev(_nhwc(x))
    ops.faceparse_conv(xp, wp, dev(bias), out, k, stride, pad)
    assert _rel(_nchw(out), ref) <= 1e-5
    ops.faceparse_conv(xp, wp, dev(bias), out, k, stride, pad, relu=True)
    assert _rel(_nchw(out), torch.relu(ref)) <= 1e-5
    ops.faceparse_conv(xp, wp, dev(bias), out, k, stride, pad, residual=dev(_nhwc(res)))
    assert _rel(_nchw(out), torch.relu(ref + res.double())) <= 1e-5
    ops.faceparse_conv(xp, wp, None, out, k, stride, pad, residual=dev(_nhwc(res)))
    assert _rel(_nchw(out), torch.relu(ref - bias.double().view(1, -1, 1, 1) + res.double())) <= 1e-5


def test_conv_refusals(cuda_device):
    x = torch.zeros(1, 4, 4, 4, device=cuda_device)
    w = torch.zeros(64, 64, device=cuda_device)
    out = torch.full((1, 4, 4, 64), 7.0, device=cuda_device)
    lib = _lib.load()
    rc = lib.asyrp_faceparse_conv(ops._ptr(x), ops._ptr(w), None, None, ops._ptr(out), 1, 4, 4, 4, 64, 3, 1, 1, 1,
                                  ops._stream())
    assert rc != 0 and "needs a bias" in lib.asyrp_last_error().decode()
    rc = lib.asyrp_faceparse_conv(ops._ptr(x), ops._ptr(w), None, ops._ptr(out), ops._ptr(out), 1, 4, 4, 4, 64, 3, 1,
                                  1, 0, ops._stream())
    assert rc != 0 and "before the ReLU" in lib.asyrp_last_error().decode()
    torch.cuda.synchronize()
    assert (out == 7).all()


def _mean_ref(x):
    return x.double().mean((2, 3))


# the three gates the network runs: conv_avg (512 -> 128, ReLU), an ARM (128 -> 128, sigmoid), the FFM (256 -> 64
# ReLU -> 256 sigmoid), at the network's map sizes and at an odd one
@pytest.mark.parametrize("C,HW", [(128, (16, 16)), (128, (32, 32)), (256, (64, 64)), (512, (16, 16)), (128, (5, 7)),
                                  (256, (3, 1)), (512, (1, 1))])
def test_gates(cuda_device, C, HW):
    g = _g(C + HW[0])
    x = torch.randn(3, C, *HW, generator=g) + 0.5
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    m = _mean_ref(x)
    if C == 512:
        w, b = torch.randn(128, 512, generator=g) / 512 ** 0.5, torch.randn(128, generator=g)
        out = torch.empty(3, 128, device=cuda_device)
        ops.faceparse_gate(dev(_nhwc(x)), dev(w), dev(b), ops.FP_ACT_RELU, out)
        ref = torch.relu(m @ w.double().t() + b.double())
    elif C == 128:
        w, b = torch.randn(128, 128, generator=g) / 128 ** 0.5, torch.randn(128, generator=g)
        out = torch.empty(3, 128, device=cuda_device)
        ops.faceparse_gate(dev(_nhwc(x)), dev(w), dev(b), ops.FP_ACT_SIGMOID, out)
        ref = torch.sigmoid(m @ w.double().t() + b.double())
    else:
        w1, w2 = torch.randn(64, 256, generator=g) / 16, torch.randn(256, 64, generator=g) / 8
        out = torch.empty(3, 256, device=cuda_device)
        ops.faceparse_gate(dev(_nhwc(x)), dev(w1), None, ops.FP_ACT_RELU, out, w2=dev(w2), act2=ops.FP_ACT_SIGMOID)
        ref = torch.sigmoid(torch.relu(m @ w1.double().t()) @ w2.double().t())
    assert (out.cpu().double() - ref).abs().max().item() <= 2e-6 * max(1.0, ref.abs().max().item())
    # a sample's gate does not depend on its neighbours
    one = torch.empty_like(out[:1])
    if C == 256:
        ops.faceparse_gate(dev(_nhwc(x[1:2])), dev(w1), None, ops.FP_ACT_RELU, one, w2=dev(w2),
                           act2=ops.FP_ACT_SIGMOID)
    else:
        ops.faceparse_gate(dev(_nhwc(x[1:2])), dev(w), dev(b), ops.FP_ACT_RELU if C == 512 else ops.FP_ACT_SIGMOID,
                           one)
    assert torch.equal(one, out[1:2])


@pytest.mark.parametrize("C,H,up,kind", [(128, 16, 2, "vector"), (128, 32, 2, "map"), (256, 64, 1, "self"),
                                         (4, 3, 2, "map"), (8, 5, 1, "vector")])
def test_apply_exact(cuda_device, C, H, up, kind):
    """f * gate + add, one rounding per operation: equal to torch's fp32 product then sum"""
    g = _g(C + H)
    f = torch.randn(2, H, H + 1, C, generator=g)
    gate = torch.rand(2, C, generator=g)
    add = {"vector": torch.randn(2, C, generator=g), "map": torch.randn(2, H, H + 1, C, generator=g), "self": f}[kind]
    out = torch.full((2, H * up, (H + 1) * up, C), float("nan"), device=cuda_device)
    fd = f.to(cuda_device)
    ops.faceparse_apply(fd, gate.to(cuda_device), fd if kind == "self" else add.to(cuda_device), out, up=up)
    ref = f * gate[:, None, None, :] + (add[:, None, None, :] if kind == "vector" else add)
    ref = ref.repeat_interleave(up, 1).repeat_interleave(up, 2)
    assert torch.equal(out.cpu(), ref)


def _labels_ref(lg, ncls, size):
    up = F.interpolate(lg[..., :ncls].permute(0, 3, 1, 2).double().cpu(), size, mode="bilinear", align_corners=True)
    top = up.topk(min(2, ncls), dim=1).values
    margin = top[:, 0] - top[:, 1] if ncls > 1 else torch.full_like(top[:, 0], float("inf"))
    return up.argmax(1), margin


@pytest.mark.parametrize("N,Hi,Wi,ld,ncls,Ho,Wo", [(2, 64, 64, 64, 19, 512, 512), (3, 5, 7, 8, 5, 33, 17),
                                                   (1, 64, 64, 64, 64, 512, 512), (2, 9, 4, 4, 1, 1, 3),
                                                   (1, 2, 2, 20, 19, 511, 2)])
def test_upsample_argmax(cuda_device, N, Hi, Wi, ld, ncls, Ho, Wo):
    lg = torch.randn(N, Hi, Wi, ld, generator=_g(Hi * Wi + ncls)) * 3
    lg[..., ncls:] = 1e9  # padding classes are never read
    labels = torch.full((N, Ho, Wo), 255, dtype=torch.uint8, device=cuda_device)
    ops.faceparse_labels(lg.to(cuda_device), ncls, labels)
    ref, margin = _labels_ref(lg, ncls, (Ho, Wo))
    sure = margin > 1e-4  # fp32 interpolation of O(3) values: error ~1e-6
    assert sure.double().mean().item() > 0.99
    assert torch.equal(labels.cpu().long()[sure], ref[sure])


def test_upsample_argmax_ties_go_to_the_first_class(cuda_device):
    g = _g(4)
    lg = torch.randn(2, 64, 64, 64, generator=g)
    lg[..., 19:] = 0
    lg[0, ..., 11] = lg[0, ..., 3] = 10 + torch.rand(64, 64, generator=g)  # 3 and 11 tie everywhere: 3 wins
    lg[1, :, :, :19] = 0.5                                                # every class ties: 0 wins
    labels = torch.empty(2, 512, 512, dtype=torch.uint8, device=cuda_device)
    ops.faceparse_labels(lg.to(cuda_device), 19, labels)
    assert (labels[0] == 3).all() and (labels[1] == 0).all()


@pytest.mark.parametrize("n,B,row0,Hi,ncls,Ho", [(6, 2, 0, 64, 19, 512), (5, 3, 4, 64, 19, 512), (3, 1, 0, 9, 7, 41)])
def test_agreement_count_is_exact(cuda_device, n, B, row0, Hi, ncls, Ho):
    g = _g(n + B + Hi)
    src = torch.randn(B, Hi, Hi, 64, generator=g)
    # edited rows: their source plus a perturbation of growing size, so that the counts differ from row to row
    edited = torch.stack([src[(row0 + j) % B] + 0.3 * j * torch.randn(Hi, Hi, 64, generator=g) for j in range(n)])
    d_src, d_ed = src.to(cuda_device), edited.to(cuda_device)
    agree = torch.full((n,), -1, dtype=torch.int32, device=cuda_device)
    ops.faceparse_agreement(d_src, d_ed, ncls, (Ho, Ho), agree, row0=row0)
    ls = torch.empty(B, Ho, Ho, dtype=torch.uint8, device=cuda_device)
    le = torch.empty(n, Ho, Ho, dtype=torch.uint8, device=cuda_device)
    ops.faceparse_labels(d_src, ncls, ls)
    ops.faceparse_labels(d_ed, ncls, le)
    ref = torch.stack([(le[j] == ls[(row0 + j) % B]).sum() for j in range(n)]).cpu().int()
    assert torch.equal(agree.cpu(), ref)
    if row0 == 0:
        assert agree[0].item() == Ho * Ho  # row 0 is its source
    assert len(set(ref.tolist())) > 1


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model(cuda_device):
    sd = synthetic.face_parsing_state_dict(seed=7)
    return sd, fp.FaceParser(sd, device=cuda_device)


def _images(n, seed, scale=1.0):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    from clip_image_emulate import smooth_images
    return smooth_images(n, 256, seed) * scale


@pytest.mark.parametrize("scale", [1.0, 1e3])
def test_full_network_within_the_design_bound(model, scale):
    sd, m = model
    tol = LOGIT_TOL[scale]
    x = _images(2, 11, scale)
    edit = x + 0.3 * scale * _images(2, 12)
    lg = m.logits(torch.cat([x, edit]))
    ref = of.logits(sd, torch.cat([x, edit]))
    assert tuple(lg.shape) == (4, 19, 64, 64)
    assert (lg.double().cpu() - ref).abs().max().item() <= tol
    labels = m.labels(torch.cat([x, edit])).cpu().long()
    ref_labels = of.upsample(ref).argmax(1)
    margin = of.top2_margin(ref)
    sure = margin > 2 * tol
    assert sure.double().mean().item() > 0.8
    assert torch.equal(labels[sure], ref_labels[sure])
    sc = m.seg_consistency(x, edit)
    ref_sc = (ref_labels[2:] == ref_labels[:2]).double().mean((1, 2))
    low = (~sure[:2] | ~sure[2:]).double().mean((1, 2))  # pixels where either label may differ from fp64's
    assert ((sc - ref_sc).abs() <= low).all(), (sc, ref_sc, low)
    assert (ref_sc < 0.99).all()  # the edit moved some labels: the comparison is not trivial
    assert torch.equal(m.seg_consistency(x, x), torch.ones(2, dtype=torch.float64))


def test_deterministic_and_batch_independent(model, cuda_device):
    sd, m = model
    x = _images(6, 3)
    x[3:] *= 1e3
    lg = m.logits(x)
    assert torch.equal(m.logits(x), lg)
    for i in (0, 4):
        assert torch.equal(m.logits(x[i:i + 1]), lg[i:i + 1])
    assert torch.equal(m.logits(x[2:5]), lg[2:5])
    assert torch.equal(m.logits(torch.cat([x[5:], x[:2]])), torch.cat([lg[5:], lg[:2]]))
    labels = m.labels(x)
    assert torch.equal(m.labels(x[3:4]), labels[3:4])
    sc = m.seg_consistency(x[:2], x[2:6])
    assert torch.equal(m.seg_consistency(x[:2], x[2:6]), sc)
    ref = torch.stack([(labels[2 + j] == labels[j % 2]).double().mean() for j in range(4)]).cpu()
    assert torch.equal(sc, ref)
    # one image per chunk: the same bits, the pairing kept across chunks
    one = fp.FaceParser(sd, device=cuda_device, max_rows=1)
    assert torch.equal(one.logits(x), lg)
    assert torch.equal(one.seg_consistency(x[:2], x[2:6]), sc)
    assert torch.equal(m.seg_consistency(x[:2], torch.cat([x[4:6], x[2:4]])), torch.cat([sc[2:], sc[:2]]))


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


BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/sc", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500",
        "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
        "--get_h_num", "1"]


@pytest.mark.parametrize("mode", ["single", "interp", "sweep"])
def test_run_test_scores_every_edit(cuda_device, tmp_path, monkeypatch, mode):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    sd = synthetic.face_parsing_state_dict(seed=5)
    torch.save(sd, "79999_iter.pth")
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
    r, res = _run(argv + ["--seg_consistency", "--seg_weights", "79999_iter.pth"], cuda_device)
    _, plain = _run(argv, cuda_device)                              # without the flag
    _, with_origin = _run(argv + ["--save_x_origin"], cuda_device)  # the origin row the score compares against
    rows = res[("test", 1)]
    assert len(rows) == tuples and len(with_origin[("test", 1)]) == tuples + 1
    for a, b, c in zip(rows, plain[("test", 1)], with_origin[("test", 1)][1:]):
        assert torch.equal(a, b) and torch.equal(a, c)  # the score changes no edited image
    origin = with_origin[("test", 1)][0]
    table = _table(os.path.join(r.args.test_image_folder, "test_1_0_ngen4_seg_consistency.tsv"))
    header = ["image", "tuple", "hs_coeff", "SC"] + (["attr"] if mode == "sweep" else [])
    assert table[0] == header and len(table) == 1 + tuples * 2
    assert [(int(t[1]), int(t[0])) for t in table[1:]] == [(k, i) for k in range(tuples) for i in range(2)]
    if mode == "sweep":
        assert [t[4] for t in table[1:]] == ["smiling", "smiling", "angry", "angry"]
    sc = torch.tensor([float(t[3]) for t in table[1:]], dtype=torch.float64)
    assert torch.equal(sc.view(tuples, 2), r.seg_consistency["test_1_0"])
    # the scorer on the run's own saved origin and edited images gives the table's bits
    m = fp.FaceParser(sd, device=cuda_device)
    assert torch.equal(m.seg_consistency(origin, torch.cat(rows)), sc)
    assert ((sc > 0) & (sc <= 1)).all()


def test_run_test_with_all_three_scores_shares_the_origin_pass(cuda_device, tmp_path, monkeypatch):
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
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = BASE + ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling", "--DirectionalClipSmilarity",
                   "--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz", "--id_similarity", "--id_weights",
                   "ir_se50.pth"]
    calls = []
    orig = diffusion_latent.Asyrp.edit_batch

    def counting(self, *a, **kw):
        calls.append(1)
        return orig(self, *a, **kw)
    r1, res1 = _run(argv, cuda_device)
    monkeypatch.setattr(diffusion_latent.Asyrp, "edit_batch", counting)
    r2, res2 = _run(argv + ["--seg_consistency", "--seg_weights", "79999_iter.pth"], cuda_device)
    assert len(calls) == 2  # one origin pass, one edit pass, for all three scores
    assert all(torch.equal(a, b) for a, b in zip(res1[("test", 1)], res2[("test", 1)]))
    assert torch.equal(r1.directional_clip["test_1_0"], r2.directional_clip["test_1_0"])
    assert torch.equal(r1.id_similarity["test_1_0"], r2.id_similarity["test_1_0"])
    assert r2.seg_consistency["test_1_0"].shape == (1, 2)
