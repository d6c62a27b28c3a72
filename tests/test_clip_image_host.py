"""CLIP image tower and directional similarity, host side (no GPU): the CPU oracle pinned against torch's and
torchvision's own modules, the visual weight loader, the templates reader and the --DirectionalClipSmilarity CLI
rejections, which come before any model is loaded."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import clip_image, clip_text, ops, synthetic
from oracle import clip_image as oci
from oracle import clip_text as oct


def _images(B, S, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 3, S, S, generator=g, dtype=torch.float64) * 2 - 1) * scale


@pytest.mark.parametrize("S", [256, 32])
def test_oracle_preprocess_matches_interpolate_and_torchvision(S):
    import torchvision.transforms as T
    from torchvision.transforms import InterpolationMode
    x = _images(2, S, S)
    ref = F.interpolate(x, (224, 224), mode="bicubic", align_corners=False, antialias=False)
    assert (oci.resize_bicubic(x, 224) - ref).abs().max().item() <= 1e-13
    tv = T.Compose([T.Normalize([-1.0] * 3, [2.0] * 3),
                    T.Resize(224, interpolation=InterpolationMode.BICUBIC, antialias=False), T.CenterCrop(224),
                    T.Normalize(oci.MEAN, oci.STD)])
    assert (oci.preprocess(x, 224) - tv(x)).abs().max().item() <= 1e-12


def _torch_modules_encode(sd, x):
    """VisionTransformer.forward with nn.Conv2d / nn.LayerNorm / nn.MultiheadAttention, fp64, on preprocessed x"""
    d = oci.dims_of(sd)
    g = {k[7:]: v.double() for k, v in sd.items() if k.startswith("visual.")}
    w = d["width"]

    def ln(prefix):
        m = torch.nn.LayerNorm(w, eps=1e-5).double()
        m.weight.data, m.bias.data = g[prefix + ".weight"], g[prefix + ".bias"]
        return m
    conv = torch.nn.Conv2d(3, w, d["patch"], d["patch"], bias=False).double()
    conv.weight.data = g["conv1.weight"]
    h = conv(x).flatten(2).transpose(1, 2)
    h = torch.cat([g["class_embedding"].expand(x.shape[0], 1, -1), h], 1) + g["positional_embedding"]
    h = ln("ln_pre")(h)
    for i in range(d["layers"]):
        p = f"transformer.resblocks.{i}."
        mha = torch.nn.MultiheadAttention(w, d["heads"]).double()
        mha.in_proj_weight.data, mha.in_proj_bias.data = g[p + "attn.in_proj_weight"], g[p + "attn.in_proj_bias"]
        mha.out_proj.weight.data, mha.out_proj.bias.data = g[p + "attn.out_proj.weight"], g[p + "attn.out_proj.bias"]
        y = ln(p + "ln_1")(h).transpose(0, 1)  # CLIP runs the transformer sequence-first
        h = h + mha(y, y, y, need_weights=False)[0].transpose(0, 1)
        z = ln(p + "ln_2")(h) @ g[p + "mlp.c_fc.weight"].t() + g[p + "mlp.c_fc.bias"]
        h = h + (z * torch.sigmoid(1.702 * z)) @ g[p + "mlp.c_proj.weight"].t() + g[p + "mlp.c_proj.bias"]
    return ln("ln_post")(h[:, 0]) @ g["proj"]


@pytest.mark.parametrize("S,patch,grid", [(256, 32, 7), (32, 16, 14)])
def test_oracle_encode_image_matches_torch_modules(S, patch, grid):
    sd = synthetic.clip_image_state_dict(seed=3, width=128, layers=2, patch=patch, grid=grid, embed_dim=64)
    x = _images(2, S, 5)
    ref = _torch_modules_encode(sd, oci.preprocess(x, grid * patch))
    out = oci.encode_image(sd, x)
    assert (out - ref).abs().max().item() <= 1e-10 * ref.abs().max().item()


def test_oracle_directional_loss_matches_cosine_similarity():
    g = torch.Generator().manual_seed(1)
    src, trg, text = (torch.randn(4, 64, generator=g, dtype=torch.float64) for _ in range(3))
    e = oci.edit_direction(src / src.norm(dim=-1, keepdim=True), trg / trg.norm(dim=-1, keepdim=True))
    t = text[:1] / text[:1].norm()
    ref = 1 - torch.nn.CosineSimilarity()(e, t)
    assert torch.allclose(ref, 1 - (e @ t.t()).squeeze(1) / e.norm(dim=-1), atol=1e-12)
    same = oci.edit_direction(src, src)
    assert torch.equal(same, torch.zeros_like(same))  # 0 / (0 + 1e-7)


def _vit(width=128, layers=2, patch=16, grid=14, embed=64, text=True):
    sd = synthetic.clip_image_state_dict(seed=2, width=width, layers=layers, patch=patch, grid=grid, embed_dim=embed)
    if text:
        sd.update(synthetic.clip_text_state_dict(seed=2, width=64, layers=1, vocab=600, embed_dim=embed))
    return {k: v.half() for k, v in sd.items()}  # CLIP stores its weights in fp16


@pytest.mark.parametrize("patch,grid,kpad", [(16, 14, 768), (32, 7, 3072), (14, 16, 608)])
def test_loader_derives_the_dimensions(tmp_path, patch, grid, kpad):
    sd = _vit(patch=patch, grid=grid)
    torch.save(sd, tmp_path / "clip.pt")
    for src in (sd, str(tmp_path / "clip.pt")):
        dims, t = clip_image.load_state_dict(src)
        assert dims == dict(width=128, heads=2, layers=2, patch=patch, grid=grid, resolution=grid * patch,
                            embed_dim=64)
        assert set(t) == set(clip_image.image_key_shapes(128, 2, patch, grid, 64))
        assert all(v.dtype == torch.float32 for v in t.values())
    assert ops.clip_image_kpad(patch) == kpad
    # the text loader keeps ignoring visual.*
    assert clip_text.load_state_dict(sd)[0]["width"] == 64


def test_loader_rejects_bad_state_dicts():
    sd = _vit()
    cases = {"missing": {k: v for k, v in sd.items() if k != "visual.transformer.resblocks.1.mlp.c_fc.bias"},
             "missing_top": {k: v for k, v in sd.items() if k != "visual.ln_post.bias"},
             "missing_proj": {k: v for k, v in sd.items() if k != "visual.proj"},
             "shape": {**sd, "visual.transformer.resblocks.0.attn.in_proj_weight": torch.zeros(3 * 128, 64)},
             "shape_cls": {**sd, "visual.class_embedding": torch.zeros(64)},
             "shape_pos": {**sd, "visual.positional_embedding": torch.zeros(196, 128)},
             "too_many_tokens": {**sd, "visual.positional_embedding": torch.zeros(290, 128)},
             "unknown": {**sd, "visual.transformer.resblocks.0.attn.extra": torch.zeros(2)},
             "unknown_top": {**sd, "visual.bias": torch.zeros(2)},
             "resnet": {**sd, "visual.layer1.0.conv1.weight": torch.zeros(64, 64, 1, 1)},
             "embed_dim": {**sd, "text_projection": torch.zeros(64, 128)}}
    for what, bad in cases.items():
        with pytest.raises(ValueError) as e:
            clip_image.load_state_dict(bad)
            pytest.fail(what)
        if what == "resnet":
            assert "ModifiedResNet" in str(e.value)
        if what == "embed_dim":
            assert "text tower" in str(e.value)
    with pytest.raises(ValueError):
        clip_image.load_state_dict(_vit(text=False) | {"visual.layer1.0.bn1.weight": torch.zeros(2)})
    assert clip_image.load_state_dict(_vit(text=False))[0]["embed_dim"] == 64  # no text tower: nothing to compare


def test_templates_are_parsed_not_executed(tmp_path):
    p = tmp_path / "text_templates.py"
    p.write_text("import module_that_does_not_exist\nimagenet_templates = [\n    'a bad photo of a {}.',\n"
                 "    # comment\n    'a {} in a video game.',\n]\npart_templates = ['x']\nraise SystemExit(1)\n")
    assert clip_image.read_templates(str(p)) == ["a bad photo of a {}.", "a {} in a video game."]
    (tmp_path / "empty.py").write_text("part_templates = ['x']\n")
    with pytest.raises(ValueError):
        clip_image.read_templates(str(tmp_path / "empty.py"))
    (tmp_path / "bad.py").write_text("imagenet_templates = []\n")
    with pytest.raises(ValueError):
        clip_image.read_templates(str(tmp_path / "bad.py"))
    with pytest.raises(FileNotFoundError):
        clip_image.read_templates(str(tmp_path / "nope.py"))


def test_cli_rejections_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200 import scoring
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    os.makedirs("utils")
    with open("utils/text_dic.py", "w") as f:
        f.write("SRC_TRG_TXT_DIC = {'smiling': (['face'], ['smiling face'])}\n")
    with open("utils/text_templates.py", "w") as f:
        f.write("imagenet_templates = ['a photo of a {}.']\n")
    for name in ("w.pt", "v.txt.gz"):
        open(name, "w").close()

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    base = ["--run_test", "--config", "celeba.yml", "--edit_attr", "smiling", "--DirectionalClipSmilarity"]
    clip = ["--clip_weights", "w.pt", "--clip_vocab", "v.txt.gz"]
    cases = [(clip + ["--multiple_attr", "smiling old"], "--multiple_attr"),
             (clip + ["--pass_editing"], "--pass_editing"),
             ([], "--clip_weights and --clip_vocab"),
             (["--clip_weights", "w.pt"], "--clip_weights and --clip_vocab"),
             (["--clip_weights", "missing.pt", "--clip_vocab", "v.txt.gz"], "is not a file"),
             (clip + ["--text_templates", "nope.py"], "nope.py"),
             (["--run_test", "--config", "celeba.yml", "--DirectionalClipSmilarity"] + clip, "--src_txts")]
    for extra, match in cases:
        argv = extra if extra and extra[0] == "--run_test" else base + extra
        args, cfg = cli.parse_args_and_config(argv)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, cfg = cli.parse_args_and_config(base + clip)
    assert args.DirectionalClipSmilarity and args.text_templates is None
    assert scoring.directional_clip_setup(Asyrp(args, cfg, device="cpu")) == ("face", "smiling face",
                                                                           ["a photo of a {}."])


def test_oracle_text_direction_uses_every_template(tmp_path):
    templates = ["a photo of a {}.", "a drawing of the {}.", "{}"]
    gz = str(tmp_path / "bpe.txt.gz")
    n = synthetic.write_clip_vocab(gz, synthetic.clip_bpe_merges(["a photo of a face. drawing the smiling"]))
    sd = synthetic.clip_text_state_dict(seed=4, width=64, layers=1, vocab=n, embed_dim=64)
    tok = oct.SimpleTokenizer(gz)
    d = oci.compute_text_direction(sd, tok, templates, "face", "smiling face")
    assert d.shape == (1, 64) and math.isclose(d.norm().item(), 1.0, rel_tol=1e-12)
    d1 = oci.compute_text_direction(sd, tok, templates[:1], "face", "smiling face")
    assert (d - d1).abs().max().item() > 1e-3
