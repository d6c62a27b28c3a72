"""CLIP image tower and directional similarity on the GPU: each new kernel against fp64, encode_image on synthetic
ViT-B/16 and ViT-B/32 towers within the DESIGN.md §2 bound, determinism and batch independence, and
`main --run_test --DirectionalClipSmilarity` end to end."""
import csv
import os

import pytest
import torch
import yaml

from asyrp_official_b200 import clip_image, main as cli, modules, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import clip_image as oci
from oracle import clip_text as oct
from oracle import ddpm as od

pytestmark = pytest.mark.gpu
FEAT_TOL = 1.5e-3  # relative max-abs of the features (DESIGN.md §2: TF32 emulation up to 5.1e-4)
SDIR_TOL = 1.5e-4  # absolute error of S_dir times |df|/|f| (emulation up to 4.6e-5)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rel(out, ref):
    ref = ref.double()
    return ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()


def _patchify(pre, G, P):
    B = pre.shape[0]
    return pre.reshape(B, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(B * G * G, 3 * P * P)


@pytest.mark.parametrize("S,P,G", [(256, 16, 14), (32, 14, 16), (224, 32, 7), (7, 16, 14)])
def test_preprocess_and_patches(cuda_device, S, P, G):
    """bicubic weights, the edge clamp (upsampling reads past the border), CLIP's normalisation, the patch layout and
    the zero K padding (P = 14: 588 columns padded to 608)"""
    x = torch.rand(3, 3, S, S, generator=_g(S)) * 2 - 1
    x[0, :, 0, :] = 1.0  # a hard edge on the border
    kpad = ops.clip_image_kpad(P)
    out = torch.full((3 * G * G, kpad), float("nan"), device=cuda_device)
    ops.clip_image_patches(x.to(cuda_device), out, G, P)
    ref = _patchify(oci.preprocess(x.double(), G * P), G, P)
    out = out.cpu()
    # the fp32 source coordinate (o + 0.5) * S/R - 0.5 is exact to an ulp of S (1.5e-5 at 256), as in torch's fp32
    # kernel, which moves a sample of this noise image by up to ~1e-4; a wrong weight, tap or clamp is off by 1e-2 or
    # more
    assert (out[:, :3 * P * P].double() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    assert torch.equal(out[:, 3 * P * P:], torch.zeros(3 * G * G, kpad - 3 * P * P))


@pytest.mark.parametrize("T", [50, 197, 257, 1, 33])
def test_full_attention(cuda_device, T):
    heads, P = 12, 3
    w = 64 * heads
    qkv = torch.randn(P, T, 3 * w, generator=_g(T)) * 2
    out = torch.empty(P, T, w, device=cuda_device)
    ops.clip_attention(qkv.to(cuda_device), out, heads, causal=False)
    q, k, v = (t.double().reshape(P, T, heads, 64).transpose(1, 2) for t in qkv.split(w, dim=-1))
    ref = (torch.softmax(q @ k.transpose(-1, -2) / 8, -1) @ v).transpose(1, 2).reshape(P, T, w)
    assert _rel(out, ref) <= 1e-5


def test_full_attention_rejects_more_than_257_tokens(cuda_device):
    from asyrp_official_b200 import _lib
    qkv = torch.zeros(1, 258, 3 * 64, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="T <= 257"):
        ops.clip_attention(qkv, torch.empty(1, 258, 64, device=cuda_device), 1, causal=False)


def test_tokens_and_pooling(cuda_device):
    g = _g(3)
    B, G, w = 3, 7, 768
    T = G * G + 1
    emb, cls, pos = torch.randn(B * G * G, w, generator=g), torch.randn(w, generator=g), torch.randn(T, w, generator=g)
    x = torch.empty(B, T, w, device=cuda_device)
    ops.clip_image_tokens(emb.to(cuda_device), cls.to(cuda_device), pos.to(cuda_device), x)
    ref = torch.cat([cls.expand(B, 1, w), emb.reshape(B, G * G, w)], 1) + pos
    assert torch.equal(x.cpu(), ref)
    x = x * 3 + 1.5
    gam, bet = 1 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    pooled = torch.empty(B, w, device=cuda_device)
    ops.clip_layernorm_rows(x, gam.to(cuda_device), bet.to(cuda_device), pooled)
    assert _rel(pooled, oct.layer_norm(x[:, 0].cpu().double(), gam.double(), bet.double())) <= 2e-6
    dense = torch.empty(B, w, device=cuda_device)  # the same row code as the dense LayerNorm: the same bits
    ops.clip_layernorm(x[:, 0].contiguous(), gam.to(cuda_device), bet.to(cuda_device), dense)
    assert torch.equal(pooled, dense)


def test_direction_kernel(cuda_device):
    g = _g(4)
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    src, trg = torch.randn(6, 512, generator=g), torch.randn(6, 512, generator=g)
    trg[2] = src[2]  # an unedited image: 0 / (0 + 1e-7) = exactly 0
    out = torch.empty(6, 512, device=cuda_device)
    ops.clip_direction(dev(src), dev(trg), out, 1, 1e-7)
    ref = oci.edit_direction(src.double() / src.double().norm(dim=-1, keepdim=True),
                             trg.double() / trg.double().norm(dim=-1, keepdim=True))
    assert (out.cpu().double() - ref).abs().max().item() <= 1e-6
    assert torch.equal(out[2].cpu(), torch.zeros(512))
    # text: one group of all template rows, no eps
    s, t = torch.randn(79, 512, generator=g), torch.randn(79, 512, generator=g)
    d = torch.empty(1, 512, device=cuda_device)
    ops.clip_direction(dev(s), dev(t), d, 79, 0.0)
    sd, td = s.double(), t.double()
    r = (td / td.norm(dim=-1, keepdim=True) - sd / sd.norm(dim=-1, keepdim=True)).mean(0, keepdim=True)
    assert (d.cpu().double() - r / r.norm()).abs().max().item() <= 1e-6
    # the cosine against the text direction, eps 1e-8
    cos = torch.empty(6, device=cuda_device)
    ops.clip_cosine(out, d.expand(6, -1).contiguous(), cos, eps=1e-8)
    rc = torch.nn.CosineSimilarity()(ref, r / r.norm())
    assert (cos.cpu().double() - rc).abs().max().item() <= 1e-6 and cos[2].item() == 0.0


@pytest.mark.parametrize("patch,grid", [(16, 14), (32, 7)])
def test_encode_image_within_the_design_bound(cuda_device, patch, grid):
    sd = synthetic.clip_image_state_dict(seed=1, width=768, layers=12, patch=patch, grid=grid, embed_dim=512)
    m = clip_image.CLIPImage(sd, device=cuda_device)
    assert m.dims == dict(width=768, heads=12, layers=12, patch=patch, grid=grid, resolution=224, embed_dim=512)
    x = torch.rand(6, 3, 256, 256, generator=_g(patch)) * 2 - 1
    x[3:] *= 1e3  # the range synthetic UNet weights produce
    feats = m.encode_image(x)
    ref = oci.encode_image(sd, x)
    for rows in (slice(0, 3), slice(3, 6)):
        e = _rel(feats[rows], ref[rows])
        assert e <= FEAT_TOL, e
    # determinism and batch independence
    assert torch.equal(m.encode_image(x), feats)
    for i in (0, 4):
        assert torch.equal(m.encode_image(x[i:i + 1]), feats[i:i + 1])
    assert torch.equal(m.encode_image(x[2:5]), feats[2:5])
    assert torch.equal(m.encode_image(torch.cat([x[5:], x[:2]])), torch.cat([feats[5:], feats[:2]]))


# ---------------------------------------------------------------------------------------------------------------------
CFG = od.MINI_CFG
TEMPLATES = ["a photo of a {}.", "a drawing of the {}.", "{}"]
SRC, TRG = "face", "smiling face"


def _write_cfg(path):
    cfg = {"data": dict(dataset="CelebA_HQ", category="CelebA_HQ", image_size=CFG["image_size"], channels=3,
                        rescaled=True, num_workers=0),
           "model": dict(type="simple", in_channels=3, out_ch=3, ch=CFG["ch"], ch_mult=list(CFG["ch_mult"]),
                         num_res_blocks=CFG["num_res_blocks"], attn_resolutions=list(CFG["attn_resolutions"]), dropout=0.0,
                         var_type="fixedsmall", ema_rate=0.999, ema=True, resamp_with_conv=True),
           "diffusion": dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
           "sampling": dict(batch_size=4, last_only=True)}
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return path


def _delta_block_ckpt(path, seed):
    from types import SimpleNamespace as NS
    ns = NS(model=NS(**{**CFG, "dropout": 0.0, "resamp_with_conv": True}), data=NS(image_size=CFG["image_size"]))
    m = modules.DDPM(ns)
    m.setattr_layers(1)
    synthetic.randomize_(m, seed=seed, style="jittered")
    torch.save({"0": {k: v.clone() for k, v in m.layer_0.state_dict().items()}}, path)


def _run(argv, dev):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config, device=dev)
    return r, r.run_test()


@pytest.mark.parametrize("interp", [False, True])
def test_run_test_scores_every_edit(cuda_device, tmp_path, monkeypatch, interp):
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    os.makedirs("utils")
    with open("utils/text_dic.py", "w") as f:
        f.write(f"SRC_TRG_TXT_DIC = {{'smiling': (['{SRC}'], ['{TRG}'])}}\n")
    with open("templates.py", "w") as f:
        f.write(f"imagenet_templates = {TEMPLATES!r}\n")
    n = synthetic.write_clip_vocab("bpe.txt.gz", synthetic.clip_bpe_merges([t.format(c) for t in TEMPLATES
                                                                            for c in (SRC, TRG)]))
    sd = synthetic.clip_text_state_dict(seed=5, width=128, layers=2, vocab=n, embed_dim=128)
    sd.update(synthetic.clip_image_state_dict(seed=5, width=128, layers=2, patch=16, grid=14, embed_dim=128))
    torch.save(sd, "clip.pt")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = ["--run_test", "--config", _write_cfg(str(tmp_path / "mini.yml")), "--exp", "./runs/sdir", "--do_train",
            "0", "--do_test", "1", "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999",
            "--n_inv_step", "4", "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise",
            "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0", "--synthetic_weights", "--seed", "1234",
            "--train_delta_block", "--get_h_num", "1", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr",
            "smiling"]
    if interp:
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
    tuples = 3 if interp else 1
    r, res = _run(argv + ["--DirectionalClipSmilarity", "--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz",
                          "--text_templates", "templates.py"], cuda_device)
    _, plain = _run(argv, cuda_device)                      # without the flag
    _, with_origin = _run(argv + ["--save_x_origin"], cuda_device)  # the origin row the score compares against
    rows, rows_plain = res[("test", 1)], plain[("test", 1)]
    assert len(rows) == tuples and len(rows_plain) == tuples and len(with_origin[("test", 1)]) == tuples + 1
    for a, b, c in zip(rows, rows_plain, with_origin[("test", 1)][1:]):
        assert torch.equal(a, b) and torch.equal(a, c)      # the score changes no edited image
    origin = with_origin[("test", 1)][0]
    path = os.path.join(r.args.test_image_folder, "test_1_0_ngen4_directional_clip.tsv")
    with open(path) as f:
        table = list(csv.reader(f, delimiter="\t"))
    assert table[0] == ["image", "tuple", "hs_coeff", "S_dir"] and len(table) == 1 + tuples * 2
    assert [(int(t[1]), int(t[0])) for t in table[1:]] == [(k, i) for k in range(tuples) for i in range(2)]
    s_dir = torch.tensor([float(t[3]) for t in table[1:]], dtype=torch.float64)
    assert torch.equal(s_dir.float().view(tuples, 2), r.directional_clip["test_1_0"])
    # the oracle, from the run's own origin and edited images
    tok = oct.SimpleTokenizer("bpe.txt.gz")
    target = torch.cat(rows).double()
    src = origin.double().repeat(tuples, 1, 1, 1)
    ref = oci.directional_similarity(sd, tok, TEMPLATES, src, SRC, target, TRG)
    f_src, f_trg = oci.get_image_features(sd, src), oci.get_image_features(sd, target)
    ratio = ((f_trg - f_src).norm(dim=-1) / f_src.norm(dim=-1))
    err = (s_dir - ref).abs()
    assert (err <= SDIR_TOL / ratio).all(), (err, ratio)
