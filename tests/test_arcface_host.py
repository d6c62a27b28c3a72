"""ArcFace IR-SE50 and the identity similarity, host side (no GPU): the fp64 oracle against the golden fixture the
reference's own Backbone / IDLoss produced (tests/golden/make_arcface_golden.py), the oracle's adaptive pool against
torch's, the weight loader and its folding, and the --id_similarity CLI refusals, which come before any model loads."""
import hashlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import arcface, synthetic
from oracle import arcface as oa

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "arcface_irse50.npz")


def _sha256(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        if sd[k].is_floating_point():
            h.update(k.encode())
            h.update(sd[k].float().contiguous().numpy().tobytes())
    return h.hexdigest()


@pytest.fixture(scope="module")
def golden():
    d = np.load(GOLDEN)
    return {k: d[k] for k in d.files}


def test_oracle_matches_the_reference_golden(golden):
    sd = synthetic.arcface_state_dict(seed=int(golden["seed"]))
    assert _sha256(sd) == str(golden["weights_sha256"])
    # the generator's to_float: uint8 images as the fp32 values the reference saw
    x, x_hat = (torch.from_numpy(golden[k]).float() / 127.5 - 1 for k in ("x_u8", "x_hat_u8"))
    pooled = oa.preprocess(x)
    assert (pooled - torch.from_numpy(golden["pooled"]).double()).abs().max().item() <= 1e-6
    feats, feats_hat = oa.extract_feats(sd, x), oa.extract_feats(sd, x_hat)
    # the reference ran in fp32: |f| = 1, fp32 rounding through 50 layers stays below 1e-5
    assert (feats - torch.from_numpy(golden["feats"]).double()).abs().max().item() <= 1e-5
    assert (feats_hat - torch.from_numpy(golden["feats_hat"]).double()).abs().max().item() <= 1e-5
    loss = oa.id_loss(sd, x, x_hat)
    assert (loss - torch.from_numpy(golden["id_loss"]).double()).abs().max().item() <= 1e-5
    assert (loss > 1e-3).all()  # the edit moved the features: the fixture tests a non-trivial score


@pytest.mark.parametrize("H,W", [(256, 256), (223, 220), (300, 240)])
def test_oracle_pool_equals_adaptive_avg_pool2d(H, W):
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(H), dtype=torch.float64)
    ref = F.adaptive_avg_pool2d(x[:, :, 35:223, 32:220], (112, 112))
    assert (oa.preprocess(x) - ref).abs().max().item() <= 1e-14


def test_synthetic_weights_have_the_reference_layout():
    sd = synthetic.arcface_state_dict(seed=3)
    assert len(sd) == 397
    assert sum(v.numel() for k, v in sd.items() if not k.endswith("num_batches_tracked")) == 43_824_064
    assert all(sd[k].min() > 0 for k in sd if k.endswith("running_var"))
    assert [i for i, (c, d, s) in enumerate(arcface.BLOCKS) if s == 2] == [0, 3, 7, 21]
    assert [i for i, (c, d, s) in enumerate(arcface.BLOCKS) if c != d] == [3, 7, 21]


def test_loader_accepts_a_torch_save_and_rejects_bad_keys(tmp_path):
    sd = synthetic.arcface_state_dict(seed=3)
    torch.save(sd, tmp_path / "ir_se50.pth")
    t = arcface.load_state_dict(str(tmp_path / "ir_se50.pth"))
    assert set(t) == set(arcface.state_dict_shapes()) and len(t) == 343
    no_tracked = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    assert set(arcface.load_state_dict(no_tracked)) == set(t)
    cases = {"missing": {k: v for k, v in sd.items() if k != "body.21.shortcut_layer.1.running_var"},
             "missing_fc": {k: v for k, v in sd.items() if k != "body.5.res_layer.5.fc2.weight"},
             "shape": {**sd, "body.3.res_layer.1.weight": torch.zeros(128, 64, 1, 1)},
             "shape_head": {**sd, "output_layer.3.weight": torch.zeros(512, 512 * 14 * 14)},
             "unknown": {**sd, "body.24.res_layer.0.weight": torch.zeros(512)},
             "unknown_tracked": {**sd, "body.0.res_layer.1.num_batches_tracked": torch.tensor(0)},
             "shortcut_on_identity_block": {**sd, "body.1.shortcut_layer.0.weight": torch.zeros(64, 64, 1, 1)}}
    for what, bad in cases.items():
        with pytest.raises(ValueError):
            arcface.load_state_dict(bad)
            pytest.fail(what)
    (tmp_path / "junk.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot be read"):
        arcface.load_state_dict(str(tmp_path / "junk.pth"))
    torch.save([1, 2], tmp_path / "list.pth")
    with pytest.raises(ValueError, match="not a state dict"):
        arcface.load_state_dict(str(tmp_path / "list.pth"))


def _folded_forward(folded, x):
    """the backbone on the folded parameters, NHWC head: checks the folding algebra and the column permutation"""
    fi = folded["input"]
    h = F.conv2d(x, fi["weight"].double(), padding=1) + fi["bias"].double().view(1, -1, 1, 1)
    h = oa.prelu(h, fi["prelu"].double())
    for i, (cin, depth, stride) in enumerate(arcface.BLOCKS):
        b = {k: (tuple(t.double() for t in v) if isinstance(v, tuple) else (None if v is None else v.double()))
             for k, v in folded[f"body.{i}"].items()}
        xb = h * b["bn0"][0].view(1, -1, 1, 1) + b["bn0"][1].view(1, -1, 1, 1)
        t = oa.prelu(F.conv2d(xb, b["w1"], padding=1), b["prelu"])
        r = F.conv2d(t, b["w2"], stride=stride, padding=1) + b["b2"].view(1, -1, 1, 1)
        gate = torch.sigmoid(torch.relu(r.mean((2, 3)) @ b["fc1"].t()) @ b["fc2"].t())
        sc = h[:, :, ::stride, ::stride] if b["sc_w"] is None else \
            F.conv2d(h, b["sc_w"], stride=stride) + b["sc_b"].view(1, -1, 1, 1)
        h = r * gate[:, :, None, None] + sc
    flat = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)  # NHWC
    z = flat @ folded["head"]["weight"].double().t() + folded["head"]["bias"].double()
    return z / z.norm(dim=1, keepdim=True)


def test_folding_is_exact_algebra():
    sd = synthetic.arcface_state_dict(seed=4)
    folded = arcface.fold(arcface.load_state_dict(sd))
    x = oa.preprocess(torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(1)) * 2 - 1)
    ref = oa.backbone(sd, x)
    assert (_folded_forward(folded, x) - ref).abs().max().item() <= 2e-5  # the folded tensors are fp32


def test_cli_rejections_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200 import scoring
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    sd = synthetic.arcface_state_dict(seed=1)
    torch.save(sd, "ir_se50.pth")
    torch.save({k: v for k, v in sd.items() if k != "output_layer.3.bias"}, "partial.pth")
    (tmp_path / "small.yml").write_text("data: {image_size: 128, dataset: CelebA_HQ, category: CelebA_HQ}\n"
                                        "model: {var_type: fixedsmall}\n"
                                        "diffusion: {beta_start: 0.0001, beta_end: 0.02, "
                                        "num_diffusion_timesteps: 1000}\n")

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    base = ["--run_test", "--config", "celeba.yml", "--id_similarity"]
    cases = [(["--id_weights", "ir_se50.pth", "--pass_editing"], "--pass_editing"),
             ([], "is not a file"),  # the default pretrained/model_ir_se50.pth does not exist here
             (["--id_weights", "missing.pth"], "is not a file"),
             (["--id_weights", "partial.pth"], "missing key 'output_layer.3.bias'"),
             (["--id_weights", "ir_se50.pth", "--config", "small.yml"], "223 x 220")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml"])
    assert args.id_weights == "pretrained/model_ir_se50.pth" and not args.id_similarity
    # --multiple_attr needs no text pair: accepted
    args, cfg = cli.parse_args_and_config(base + ["--id_weights", "ir_se50.pth", "--multiple_attr", "smiling old"])
    assert set(scoring.id_similarity_setup(Asyrp(args, cfg, device="cpu"))) == set(arcface.state_dict_shapes())


def test_score_table_layout(tmp_path):
    from asyrp_official_b200.scoring import write_scores
    ids = torch.tensor([[0.5, 0.25], [0.75, 1.0], [0.125, 0.0]])
    coeffs = [(1.0, 0.5), (1.0, 1.0), (1.0, 1.5)]
    write_scores(str(tmp_path / "t.tsv"), coeffs, ids, "ID", "identity similarity")
    lines = (tmp_path / "t.tsv").read_text().splitlines()
    assert lines[0] == "image\ttuple\ths_coeff\tID"
    assert lines[1:] == [f"{i}\t{k}\t1,{c}\t{ids[k][i].item()!r}" for k, c in enumerate(("0.5", "1", "1.5"))
                         for i in range(2)]
