"""Face-parsing BiSeNet and the segmentation consistency, host side (no GPU): the fp64 oracle's backbone against
torchvision's ResNet-18, the load-time folding, the weight loader, the --seg_consistency CLI refusals (which come
before any model loads) and the score tables."""
import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import face_parsing as fp, synthetic
from oracle import face_parsing as of


def _g(seed):
    return torch.Generator().manual_seed(seed)


def test_oracle_backbone_equals_torchvision_resnet18():
    """an independent pin of the ResNet-18 half of the network: the same conv1 / bn1 / layer* tensors in torchvision's
    resnet18, fp64, eval mode"""
    import torchvision
    sd = synthetic.face_parsing_state_dict(seed=2)
    net = torchvision.models.resnet18(weights=None).double().eval()
    pre = "cp.resnet."
    tv = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    missing, unexpected = net.load_state_dict(tv, strict=False)
    assert sorted(missing) == ["fc.bias", "fc.weight"] and not unexpected
    x = of.preprocess(torch.rand(2, 3, 256, 256, generator=_g(1)) * 2 - 1)
    with torch.no_grad():
        h = net.maxpool(net.relu(net.bn1(net.conv1(x))))
        h = net.layer1(h)
        ref = []
        for layer in (net.layer2, net.layer3, net.layer4):
            h = layer(h)
            ref.append(h)
    feats = of.resnet(of._g(sd, torch.float64), x)
    for f, r, shape in zip(feats, ref, ((128, 64), (256, 32), (512, 16))):
        assert tuple(f.shape) == (2, shape[0], shape[1], shape[1])
        assert (f - r).abs().max().item() <= 1e-12 * r.abs().max().item()


def test_oracle_preprocess_and_head_conventions():
    x = torch.rand(1, 3, 256, 256, generator=_g(3), dtype=torch.float64) * 4 - 2  # outside [-1, 1]: clamped
    ref = F.interpolate(x.clamp(-1, 1) * 0.5 + 0.5, (512, 512), mode="bilinear", align_corners=False)
    ref = (ref - torch.tensor(of.MEAN, dtype=torch.float64).view(1, 3, 1, 1)) / \
        torch.tensor(of.STD, dtype=torch.float64).view(1, 3, 1, 1)
    assert torch.equal(of.preprocess(x), ref)
    lg = torch.zeros(1, 19, 64, 64, dtype=torch.float64)
    lg[:, 4] = 1.0
    lg[:, 9] = 1.0  # an exact tie: the first class wins
    assert (of.upsample(lg).argmax(1) == 4).all()


def test_synthetic_weights_have_the_bisenet_layout():
    sd = synthetic.face_parsing_state_dict(seed=3)
    main = fp.state_dict_shapes()
    aux = fp.aux_head_shapes()
    assert set(main) | set(aux) == {k for k in sd if not k.endswith("num_batches_tracked")}
    assert len(main) == 148 and len(aux) == 12
    assert sum(v.numel() for k, v in sd.items() if k in main) == 13_162_688
    assert [k for k in main if ".downsample.0." in k] == [f"cp.resnet.layer{i}.0.downsample.0.weight"
                                                          for i in (2, 3, 4)]
    assert all(sd[k].min() > 0 for k in sd if k.endswith("running_var"))


def test_loader_accepts_a_torch_save_and_rejects_bad_keys(tmp_path):
    sd = synthetic.face_parsing_state_dict(seed=3)
    torch.save(sd, tmp_path / "79999_iter.pth")
    t = fp.load_state_dict(str(tmp_path / "79999_iter.pth"))
    assert set(t) == set(fp.state_dict_shapes())
    bare = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked") and not k.startswith("conv_out1")
            and not k.startswith("conv_out3")}
    torch.save(bare, tmp_path / "bare.pth")
    t2 = fp.load_state_dict(str(tmp_path / "bare.pth"))
    assert set(t2) == set(t) and all(torch.equal(t[k], t2[k]) for k in t)
    # n_classes comes from the class layer
    sd5 = synthetic.face_parsing_state_dict(seed=3, n_classes=5, aux=False)
    assert fp.load_state_dict(sd5)["conv_out.conv_out.weight"].shape == (5, 256, 1, 1)
    cases = {"missing": ({k: v for k, v in sd.items() if k != "cp.resnet.layer3.0.downsample.1.running_var"},
                         "missing key 'cp.resnet.layer3.0.downsample.1.running_var'"),
             "missing_ffm": ({k: v for k, v in sd.items() if k != "ffm.conv2.weight"}, "missing key 'ffm.conv2.weight'"),
             "missing_head": ({k: v for k, v in sd.items() if k != "conv_out.conv_out.weight"},
                              "missing key 'conv_out.conv_out.weight'"),
             "shape": ({**sd, "cp.arm16.conv.conv.weight": torch.zeros(128, 512, 3, 3)},
                       "'cp.arm16.conv.conv.weight' has shape"),
             "shape_aux": ({**sd, "conv_out16.conv.conv.weight": torch.zeros(64, 256, 3, 3)},
                           "'conv_out16.conv.conv.weight' has shape"),
             "shape_classes": ({**sd, "conv_out.conv_out.weight": torch.zeros(19, 128, 1, 1)},
                               "'conv_out.conv_out.weight' has shape"),
             "too_many_classes": ({**sd, "conv_out.conv_out.weight": torch.zeros(65, 256, 1, 1)},
                                  "'conv_out.conv_out.weight' has shape"),
             "unknown": ({**sd, "cp.resnet.fc.weight": torch.zeros(1000, 512)}, "cp.resnet.fc.weight"),
             "unknown_downsample": ({**sd, "cp.resnet.layer1.0.downsample.0.weight": torch.zeros(64, 64, 1, 1)},
                                    "cp.resnet.layer1.0.downsample.0.weight"),
             "unknown_tracked": ({**sd, "ffm.conv1.num_batches_tracked": torch.tensor(0)},
                                 "ffm.conv1.num_batches_tracked"),
             "prefixed": ({f"module.{k}": v for k, v in sd.items()}, "missing key|unexpected keys")}
    for what, (bad, match) in cases.items():
        with pytest.raises(ValueError, match=match):
            fp.load_state_dict(bad)
            pytest.fail(what)
    (tmp_path / "junk.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot be read"):
        fp.load_state_dict(str(tmp_path / "junk.pth"))
    torch.save([1, 2], tmp_path / "list.pth")
    with pytest.raises(ValueError, match="not a state dict"):
        fp.load_state_dict(str(tmp_path / "list.pth"))


def _folded_logits(folded, x):
    """the network on the folded parameters, as the GPU runs it: convblk as two convs, the second adding the first"""
    d = lambda t: None if t is None else t.double()  # noqa: E731
    conv = lambda h, wb, **k: F.conv2d(h, d(wb[0]), d(wb[1]), **k)  # noqa: E731
    h = torch.relu(conv(x, folded["stem"], stride=2, padding=3))
    h = F.max_pool2d(h, 3, 2, 1)
    feats = []
    for li, (_, stride) in enumerate(fp.LAYERS):
        for b in range(2):
            blk = folded[f"layer{li + 1}.{b}"]
            s = stride if b == 0 else 1
            t = torch.relu(conv(h, blk["conv1"], stride=s, padding=1))
            sc = h if blk["downsample"] is None else conv(h, blk["downsample"], stride=s)
            h = torch.relu(sc + conv(t, blk["conv2"], padding=1))
        feats.append(h)
    feat8, feat16, feat32 = feats[1:]
    w, b = folded["conv_avg"]
    avg = torch.relu(feat32.mean((2, 3)) @ d(w).t() + d(b))[:, :, None, None]
    up = None
    for name, feat, head in (("arm32", feat32, "conv_head32"), ("arm16", feat16, "conv_head16")):
        f = torch.relu(conv(feat, folded[name]["conv"], padding=1))
        w, b = folded[name]["atten"]
        g = torch.sigmoid(f.mean((2, 3)) @ d(w).t() + d(b))[:, :, None, None]
        s = f * g + (avg if up is None else up)
        up = torch.relu(conv(F.interpolate(s, scale_factor=2, mode="nearest"), folded[head], padding=1))
    ffm = folded["ffm"]
    fa = conv(feat8, ffm["convblk_a"])
    f = torch.relu(fa + conv(up, ffm["convblk_b"]))
    a = torch.sigmoid(torch.relu(f.mean((2, 3)) @ d(ffm["conv1"]).t()) @ d(ffm["conv2"]).t())[:, :, None, None]
    f = f * a + f
    return F.conv2d(torch.relu(conv(f, folded["conv_out"], padding=1)), d(folded["classes"]))


def test_folding_is_exact_algebra():
    sd = synthetic.face_parsing_state_dict(seed=4)
    folded = fp.fold(fp.load_state_dict(sd))
    x = torch.rand(1, 3, 256, 256, generator=_g(1)) * 2 - 1
    ref = of.logits(sd, x)
    got = _folded_logits(folded, of.preprocess(x))
    assert (got - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()  # the folded tensors are fp32


def test_oracle_seg_consistency_pairs_rows_modulo_the_sources():
    sd = synthetic.face_parsing_state_dict(seed=5)
    src = torch.rand(2, 3, 64, 64, generator=_g(2)) * 2 - 1
    edited = torch.cat([src, src.flip(0)])
    sc = of.seg_consistency(sd, src, edited)
    assert torch.equal(sc[:2], torch.ones(2, dtype=torch.float64))
    lab = of.labels(sd, src)
    ref = (lab.flip(0) == lab).double().mean((1, 2))
    assert torch.equal(sc[2:], ref) and (ref < 1).all()


def test_cli_rejections_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200 import scoring
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    sd = synthetic.face_parsing_state_dict(seed=1)
    torch.save(sd, "79999_iter.pth")
    torch.save({k: v for k, v in sd.items() if k != "cp.arm32.bn_atten.running_mean"}, "partial.pth")
    torch.save({**sd, "cp.resnet.layer4.1.conv2.weight": torch.zeros(512, 256, 3, 3)}, "shape.pth")
    (tmp_path / "junk.pth").write_bytes(b"\x00" * 64)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    base = ["--run_test", "--config", "celeba.yml", "--seg_consistency"]
    cases = [(["--seg_weights", "79999_iter.pth", "--pass_editing"], "--pass_editing"),
             ([], "is not a file"),  # the default pretrained/79999_iter.pth does not exist here
             (["--seg_weights", "missing.pth"], "is not a file"),
             (["--seg_weights", "partial.pth"], "missing key 'cp.arm32.bn_atten.running_mean'"),
             (["--seg_weights", "shape.pth"], "'cp.resnet.layer4.1.conv2.weight' has shape"),
             (["--seg_weights", "junk.pth"], "cannot be read")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml"])
    assert args.seg_weights == "pretrained/79999_iter.pth" and not args.seg_consistency
    args, cfg = cli.parse_args_and_config(base + ["--seg_weights", "79999_iter.pth", "--multiple_attr", "smiling old"])
    assert set(scoring.seg_consistency_setup(Asyrp(args, cfg, device="cpu"))) == set(fp.state_dict_shapes())


def test_score_table_layout(tmp_path):
    from asyrp_official_b200.scoring import write_scores
    sc = torch.tensor([[0.5, 0.25], [0.75, 1.0], [0.125, 0.0]], dtype=torch.float64)
    coeffs = [(1.0, 0.5), (1.0, 1.0), (1.0, 1.5)]
    write_scores(str(tmp_path / "t.tsv"), coeffs, sc, "SC", "segmentation consistency")
    lines = (tmp_path / "t.tsv").read_text().splitlines()
    assert lines[0] == "image\ttuple\ths_coeff\tSC"
    assert lines[1:] == [f"{i}\t{k}\t1,{c}\t{sc[k][i].item()!r}" for k, c in enumerate(("0.5", "1", "1.5"))
                         for i in range(2)]
    attrs = ["smiling", "angry", "young"]  # --attr_sweep: tuple k is attribute k
    sweep = [(1.0, 1.0, 0.0, 0.0), (1.0, 0.0, 1.0, 0.0), (1.0, 0.0, 0.0, 1.0)]
    write_scores(str(tmp_path / "s.tsv"), sweep, sc, "SC", "segmentation consistency", attrs=attrs)
    lines = (tmp_path / "s.tsv").read_text().splitlines()
    assert lines[0] == "image\ttuple\ths_coeff\tSC\tattr"
    assert lines[1:] == [f"{i}\t{k}\t{','.join('1' if j in (0, k + 1) else '0' for j in range(4))}\t"
                         f"{sc[k][i].item()!r}\t{attrs[k]}" for k in range(3) for i in range(2)]
