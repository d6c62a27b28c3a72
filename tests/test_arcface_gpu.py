"""ArcFace IR-SE50 and the identity similarity on the GPU: each new kernel against fp64, the full synthetic IR-SE50
within the DESIGN.md §2 bound at O(1) and x1e3 inputs, determinism and batch independence, and
`main --run_test --id_similarity` end to end."""
import csv
import os

import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, arcface, main as cli, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import arcface as oa

pytestmark = pytest.mark.gpu
# DESIGN.md §2, TF32 emulation of the full synthetic IR-SE50 (scripts/arcface_emulate.py), about 3x:
FEAT_TOL = {1.0: 2e-3, 1e3: 0.45}  # relative max-abs of the features (emulation 6.4e-4 / 1.5e-1)
ID_TOL = {1.0: 1e-4, 1e3: 4e-2}    # absolute error of ID = 1 - IDLoss (emulation 2.5e-5 / 1.2e-2)


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


@pytest.mark.parametrize("H,W", [(256, 256), (223, 220)])
def test_preprocess(cuda_device, H, W):
    x = torch.rand(3, 3, H, W, generator=_g(H)) * 2e3 - 1e3
    out = torch.full((3, 112, 112, 4), float("nan"), device=cuda_device)
    ops.arcface_preprocess(x.to(cuda_device), out)
    ref = oa.preprocess(x.double())
    assert (_nchw(out[..., :3]) - ref).abs().max().item() <= 4e-7 * ref.abs().max().item()
    assert torch.equal(out[..., 3].cpu(), torch.zeros(3, 112, 112))


def test_preprocess_rejects_small_images(cuda_device):
    with pytest.raises(_lib.AsyrpError, match="H >= 223"):
        ops.arcface_preprocess(torch.zeros(1, 3, 222, 256, device=cuda_device),
                               torch.empty(1, 112, 112, 4, device=cuda_device))


@pytest.mark.parametrize("cin,cout,k,stride,H", [(4, 64, 3, 1, 20), (64, 128, 3, 2, 15), (128, 256, 1, 2, 14),
                                                 (256, 64, 3, 1, 7)])
def test_conv_bias_prelu(cuda_device, cin, cout, k, stride, H):
    """conv + folded-BN bias + PReLU, and the bias-only epilogue, against fp64 on the TF32-rounded operands"""
    g = _g(cin + H)
    x = torch.randn(2, cin, H, H + 3, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    bias, slope = torch.randn(cout, generator=g), 0.25 + 0.05 * torch.randn(cout, generator=g)
    pad = k // 2
    ref = F.conv2d(_tf32(x), _tf32(w), stride=stride, padding=pad) + bias.double().view(1, -1, 1, 1)
    out = torch.empty(ref.shape[0], ref.shape[2], ref.shape[3], cout, device=cuda_device)
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    ops.arcface_conv(dev(_nhwc(x)), dev(ops.pack_lpips_conv_weight(w)), dev(bias), out, k, stride, pad)
    assert _rel(_nchw(out), ref) <= 1e-5
    ops.arcface_conv(dev(_nhwc(x)), dev(ops.pack_lpips_conv_weight(w)), dev(bias), out, k, stride, pad,
                     prelu=dev(slope))
    assert _rel(_nchw(out), oa.prelu(ref, slope.double())) <= 1e-5
    ops.arcface_conv(dev(_nhwc(x)), dev(ops.pack_lpips_conv_weight(w)), None, out, k, stride, pad, prelu=dev(slope))
    assert _rel(_nchw(out), oa.prelu(ref - bias.double().view(1, -1, 1, 1), slope.double())) <= 1e-5


def test_pre_conv_bn_with_a_large_shift_pads_with_zeros(cuda_device):
    """BN0(x) materialised, then the 3x3 conv zero-pads BN0(x): a large shift makes padding x instead visible"""
    g = _g(5)
    C, H = 64, 12
    x = torch.randn(2, C, H, H, generator=g)
    scale, shift = 1 + 0.1 * torch.randn(C, generator=g), 50 + torch.randn(C, generator=g)
    xb = torch.empty(2, H, H, C, device=cuda_device)
    ops.arcface_affine(_nhwc(x).to(cuda_device), scale.to(cuda_device), shift.to(cuda_device), xb)
    ref_b = x.double() * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    assert _rel(_nchw(xb), ref_b) <= 1e-6
    w = torch.randn(64, C, 3, 3, generator=g) / (9 * C) ** 0.5
    out = torch.empty(2, H, H, 64, device=cuda_device)
    ops.arcface_conv(xb, ops.pack_lpips_conv_weight(w).to(cuda_device), None, out, 3, 1, 1)
    ref = F.conv2d(_tf32(xb.permute(0, 3, 1, 2).cpu()), _tf32(w), padding=1)
    assert _rel(_nchw(out), ref) <= 1e-5
    border = (_nchw(out) - ref)[:, :, 0].abs().max().item()
    wrong = F.conv2d(F.pad(_tf32(xb.permute(0, 3, 1, 2).cpu()), (1, 1, 1, 1), value=shift.mean().item()),
                     _tf32(w))[:, :, 0]
    assert border < 1e-3 * (wrong - ref[:, :, 0]).abs().max().item()


@pytest.mark.parametrize("cin,depth,stride", [(128, 128, 1), (64, 64, 2), (256, 512, 2)])
def test_se_block_end(cuda_device, cin, depth, stride):
    """SE gate and block end with the identity, the strided-subsample (block 0) and the conv shortcut, and the next
    block's BN0 as the second output"""
    g = _g(depth + stride)
    H = 14
    Ho = (H - 1) // stride + 1
    r = torch.randn(3, depth, Ho, Ho, generator=g) * 2
    x = torch.randn(3, cin, H, H, generator=g)
    fc1 = torch.randn(depth // 16, depth, generator=g) / depth ** 0.5
    fc2 = torch.randn(depth, depth // 16, generator=g) / (depth // 16) ** 0.5
    bs, bt = 1 + 0.1 * torch.randn(depth, generator=g), torch.randn(depth, generator=g)
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    gate = torch.empty(3, depth, device=cuda_device)
    ops.arcface_se_scale(dev(_nhwc(r)), dev(fc1), dev(fc2), gate)
    ref_gate = torch.sigmoid(torch.relu(r.double().mean((2, 3)) @ fc1.double().t()) @ fc2.double().t())
    assert (gate.cpu().double() - ref_gate).abs().max().item() <= 1e-6
    if cin != depth:  # the conv shortcut's output, at the block's output size
        w = torch.randn(depth, cin, 1, 1, generator=g) / cin ** 0.5
        sc = torch.empty(3, Ho, Ho, depth, device=cuda_device)
        ops.arcface_conv(dev(_nhwc(x)), dev(ops.pack_lpips_conv_weight(w)), None, sc, 1, stride, 0)
        sc_ref, sc_stride = _nchw(sc), 1
    else:
        sc, sc_ref, sc_stride = dev(_nhwc(x)), x.double()[:, :, ::stride, ::stride], stride
    out, out2 = torch.empty(3, Ho, Ho, depth, device=cuda_device), torch.empty(3, Ho, Ho, depth, device=cuda_device)
    ops.arcface_se_apply(dev(_nhwc(r)), gate, sc, out, sc_stride, bn=(dev(bs), dev(bt)), out2=out2)
    ref = r.double() * gate.cpu().double()[:, :, None, None] + sc_ref
    assert _rel(_nchw(out), ref) <= 1e-6
    assert _rel(_nchw(out2), ref * bs.double().view(1, -1, 1, 1) + bt.double().view(1, -1, 1, 1)) <= 1e-6


def test_head_flatten_order(cuda_device):
    """the folded head on an NHWC map equals BN2d, flatten NCHW, linear, BN1d, l2_norm on the NCHW map; asymmetric
    weights, so a wrong column permutation shows"""
    sd = synthetic.arcface_state_dict(seed=2)
    folded = arcface.fold(arcface.load_state_dict(sd))
    h = torch.randn(3, 512, 7, 7, generator=_g(9)) * torch.linspace(0.5, 2, 49).view(1, 1, 7, 7)
    raw = torch.empty(3, 512, device=cuda_device)
    ops.clip_linear(_nhwc(h).reshape(3, -1).to(cuda_device), folded["head"]["weight"].to(cuda_device),
                    folded["head"]["bias"].to(cuda_device), raw)
    feats = torch.empty_like(raw)
    ops.arcface_l2norm(raw, feats)
    g = {k: v.double() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    z = oa.batch_norm(h.double(), g, "output_layer.0").reshape(3, -1) @ g["output_layer.3.weight"].t()
    z = oa.batch_norm(z + g["output_layer.3.bias"], g, "output_layer.4")
    ref = z / z.norm(dim=1, keepdim=True)
    assert (feats.cpu().double() - ref).abs().max().item() <= 2e-4
    assert (feats.cpu().double().norm(dim=1) - 1).abs().max().item() <= 1e-6
    ids = torch.empty(6, device=cuda_device)
    ops.arcface_dot(feats, torch.cat([feats, feats.flip(0)]), ids)
    assert (ids[:3].cpu().double() - 1).abs().max().item() <= 1e-6
    assert (ids[3:].cpu().double() - (ref.flip(0) * ref).sum(-1)).abs().max().item() <= 2e-4


@pytest.fixture(scope="module")
def model(cuda_device):
    sd = synthetic.arcface_state_dict(seed=7)
    return sd, arcface.ArcFace(sd, device=cuda_device)


@pytest.mark.parametrize("scale", [1.0, 1e3])
def test_full_network_within_the_design_bound(model, scale):
    sd, m = model
    g = _g(int(scale) + 1)
    x = (torch.rand(4, 3, 256, 256, generator=g) * 2 - 1) * scale
    edit = x + 0.3 * scale * (torch.rand(4, 3, 256, 256, generator=g) * 2 - 1)
    feats = m.extract_feats(x)
    ref = oa.extract_feats(sd, x)
    assert _rel(feats, ref) <= FEAT_TOL[scale]
    ids = m.id_similarity(x, edit)
    ref_ids = oa.id_similarity(sd, x.double(), edit.double())
    assert (ids.double() - ref_ids).abs().max().item() <= ID_TOL[scale], (ids, ref_ids)
    # a row against itself
    assert (m.id_similarity(x, x).double() - 1).abs().max().item() <= 1e-6


def test_deterministic_and_batch_independent(model):
    _, m = model
    x = torch.rand(6, 3, 256, 256, generator=_g(3)) * 2 - 1
    x[3:] *= 1e3
    feats = m.extract_feats(x)
    assert torch.equal(m.extract_feats(x), feats)
    for i in (0, 4):
        assert torch.equal(m.extract_feats(x[i:i + 1]), feats[i:i + 1])
    assert torch.equal(m.extract_feats(x[2:5]), feats[2:5])
    assert torch.equal(m.extract_feats(torch.cat([x[5:], x[:2]])), torch.cat([feats[5:], feats[:2]]))
    # id_similarity pairs edited row j with source row j % B, sources encoded in the same call
    ids = m.id_similarity(x[:2], x[2:6])
    ref = torch.stack([(feats[2 + j] * feats[j % 2]).sum() for j in range(4)]).cpu()
    assert (ids - ref).abs().max().item() <= 1e-6


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


@pytest.mark.parametrize("interp", [False, True])
def test_run_test_scores_every_edit(cuda_device, tmp_path, monkeypatch, interp):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    sd = synthetic.arcface_state_dict(seed=5)
    torch.save(sd, "ir_se50.pth")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/id", "--do_train", "0", "--do_test", "1",
            "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
            "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500",
            "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
            "--get_h_num", "1", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]
    if interp:
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
    tuples = 3 if interp else 1
    r, res = _run(argv + ["--id_similarity", "--id_weights", "ir_se50.pth"], cuda_device)
    _, plain = _run(argv, cuda_device)                              # without the flag
    _, with_origin = _run(argv + ["--save_x_origin"], cuda_device)  # the origin row the score compares against
    rows = res[("test", 1)]
    assert len(rows) == tuples and len(with_origin[("test", 1)]) == tuples + 1
    for a, b, c in zip(rows, plain[("test", 1)], with_origin[("test", 1)][1:]):
        assert torch.equal(a, b) and torch.equal(a, c)  # the score changes no edited image
    origin = with_origin[("test", 1)][0]
    table = _table(os.path.join(r.args.test_image_folder, "test_1_0_ngen4_id_similarity.tsv"))
    assert table[0] == ["image", "tuple", "hs_coeff", "ID"] and len(table) == 1 + tuples * 2
    assert [(int(t[1]), int(t[0])) for t in table[1:]] == [(k, i) for k in range(tuples) for i in range(2)]
    ids = torch.tensor([float(t[3]) for t in table[1:]], dtype=torch.float64)
    assert torch.equal(ids.float().view(tuples, 2), r.id_similarity["test_1_0"])
    # the oracle, from the run's own origin and edited images (|x_0| ~ 1e3 with synthetic UNet weights)
    ref = oa.id_similarity(sd, origin.double(), torch.cat(rows).double())
    assert (ids - ref).abs().max().item() <= ID_TOL[1e3], (ids, ref)


def test_run_test_with_both_scores_shares_the_origin_pass(cuda_device, tmp_path, monkeypatch):
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
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/both", "--do_train", "0", "--do_test", "1",
            "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--n_inv_step", "4", "--n_train_step", "4",
            "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500", "--user_defined_t_addnoise",
            "0", "--synthetic_weights", "--train_delta_block", "--get_h_num", "1", "--manual_checkpoint_name",
            "smiling_0.pth", "--edit_attr", "smiling", "--DirectionalClipSmilarity", "--clip_weights", "clip.pt",
            "--clip_vocab", "bpe.txt.gz"]
    calls = []
    orig = diffusion_latent.Asyrp.edit_batch

    def counting(self, *a, **kw):
        calls.append(1)
        return orig(self, *a, **kw)
    r1, res1 = _run(argv, cuda_device)
    monkeypatch.setattr(diffusion_latent.Asyrp, "edit_batch", counting)
    r2, res2 = _run(argv + ["--id_similarity", "--id_weights", "ir_se50.pth"], cuda_device)
    assert len(calls) == 2  # one origin pass, one edit pass, for both scores
    assert all(torch.equal(a, b) for a, b in zip(res1[("test", 1)], res2[("test", 1)]))
    assert torch.equal(r1.directional_clip["test_1_0"], r2.directional_clip["test_1_0"])
    assert r2.id_similarity["test_1_0"].shape == (1, 2)
