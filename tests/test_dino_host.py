"""--dino_structure without a GPU: the fp64 oracle against transformers' ViTModel and torchvision's Resize + Normalize,
the structure distance against an explicit T x T computation, the weight loader's refusals, the CLI refusals, the C
symbols, both score tables, and the --diff_style table's gather and sort on a gloo world of 2."""
import csv
import os
import socket
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, dino, scoring, synthetic
from oracle import dino as od


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _images(n, S, seed):
    return (torch.rand(n, 3, S, S, generator=_g(seed)) * 2 - 1)


# ---------------------------------------------------------------------------------------------------------------------
def _hf_model(sd, dim, depth, patch, grid):
    from transformers import ViTConfig, ViTModel
    cfg = ViTConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=dim // 64, intermediate_size=4 * dim,
                    image_size=grid * patch, patch_size=patch, layer_norm_eps=1e-6, hidden_act="gelu", qkv_bias=True,
                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    m = ViTModel(cfg, add_pooling_layer=False).double().eval()
    hf = {"embeddings.cls_token": sd["cls_token"], "embeddings.position_embeddings": sd["pos_embed"],
          "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
          "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
          "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"]}
    for i in range(depth):
        p, q = f"blocks.{i}.", f"encoder.layer.{i}."
        for j, n in enumerate(("query", "key", "value")):
            hf[q + f"attention.attention.{n}.weight"] = sd[p + "attn.qkv.weight"][j * dim:(j + 1) * dim]
            hf[q + f"attention.attention.{n}.bias"] = sd[p + "attn.qkv.bias"][j * dim:(j + 1) * dim]
        for a, b in (("attention.output.dense", "attn.proj"), ("intermediate.dense", "mlp.fc1"),
                     ("output.dense", "mlp.fc2"), ("layernorm_before", "norm1"), ("layernorm_after", "norm2")):
            hf[q + a + ".weight"], hf[q + a + ".bias"] = sd[p + b + ".weight"], sd[p + b + ".bias"]
    m.load_state_dict({k: v.double() for k, v in hf.items()})
    return m


@pytest.mark.parametrize("patch,grid", [(8, 4), (16, 3)])
def test_oracle_against_transformers_vit(patch, grid):
    dim, depth = 128, 2
    sd = synthetic.dino_state_dict(seed=3, dim=dim, depth=depth, patch=patch, grid=grid)
    m = _hf_model(sd, dim, depth, patch, grid)
    R = grid * patch
    x = _images(2, R, 5).double()
    keys = {}
    m.encoder.layer[-1].attention.attention.key.register_forward_hook(lambda mod, i, o: keys.setdefault("k", o))
    with torch.no_grad():
        y = (x + 1) / 2
        y = (y - torch.tensor(od.MEAN).view(1, 3, 1, 1)) / torch.tensor(od.STD).view(1, 3, 1, 1)
        hidden = m(pixel_values=y).last_hidden_state.numpy()
    k, tokens = od.forward({n: v.numpy() for n, v in sd.items()}, x.numpy())
    np.testing.assert_allclose(tokens, hidden, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(k, keys["k"].numpy(), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("S", [32, 224, 256])
@pytest.mark.parametrize("R", [224, 64])
def test_oracle_pack_against_torchvision(S, R):
    from torchvision import transforms
    x = _images(2, S, S + R)
    tf = transforms.Compose([transforms.Resize(R, antialias=True),
                             transforms.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))])
    ref = tf(((x.double() + 1) / 2)).numpy()
    np.testing.assert_allclose(od.preprocess(x.numpy(), R), ref, rtol=0, atol=1e-12)
    patches = od.pack(x.numpy(), R // 8, 8)
    y = ref.reshape(2, 3, R // 8, 8, R // 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(-1, 192)
    np.testing.assert_allclose(patches, y, rtol=0, atol=1e-12)


def test_structure_distance_against_explicit_sum():
    rng = np.random.default_rng(0)
    ka, kb = rng.normal(size=(17, 64)), rng.normal(size=(17, 64))
    kb[3] = 0.0  # a zero row: normalised by eps, so its similarities are 0
    T = ka.shape[0]
    total = 0.0
    for i in range(T):
        for j in range(T):
            sa = ka[i] @ ka[j] / (max(np.linalg.norm(ka[i]), 1e-8) * max(np.linalg.norm(ka[j]), 1e-8))
            sb = kb[i] @ kb[j] / (max(np.linalg.norm(kb[i]), 1e-8) * max(np.linalg.norm(kb[j]), 1e-8))
            total += (sa - sb) ** 2
    assert od.structure_distance(ka, kb) == pytest.approx(total / T ** 2, rel=1e-12)
    assert od.structure_distance(ka, ka) == 0.0
    assert od.cls_cos(ka[0], 2 * ka[0]) == pytest.approx(1.0, rel=1e-15)


# ---------------------------------------------------------------------------------------------------------------------
def _small_sd():
    return synthetic.dino_state_dict(seed=1, dim=128, depth=2, patch=8, grid=4)


@pytest.mark.parametrize("dim,patch,grid", [(384, 8, 28), (384, 16, 14), (768, 8, 28), (768, 16, 14)])
def test_loader_accepts_the_released_layouts(dim, patch, grid):
    sd = {k: torch.zeros(s) for k, s in dino.key_shapes(dim, 12, patch, grid).items()}
    dims, out = dino.load_state_dict(sd)
    assert dims == dict(dim=dim, heads=dim // 64, depth=12, patch=patch, grid=grid, tokens=grid * grid + 1,
                        resolution=grid * patch)
    assert set(out) == set(sd)


def _refused(sd, match):
    with pytest.raises(ValueError, match=match):
        dino.load_state_dict(sd)


def test_loader_refusals():
    sd = _small_sd()
    dino.load_state_dict(sd)
    _refused({k: v for k, v in sd.items() if k != "blocks.1.mlp.fc2.bias"}, "missing key 'blocks.1.mlp.fc2.bias'")
    _refused({**sd, "blocks.0.attn.proj.weight": torch.zeros(128, 64)}, "'blocks.0.attn.proj.weight' has shape")
    _refused({**sd, "head.weight": torch.zeros(10, 128)}, "unexpected key 'head.weight'")
    _refused({**sd, "blocks.x.norm1.weight": torch.zeros(128)}, "unexpected key 'blocks.x.norm1.weight'")
    _refused({"module." + k: v for k, v in sd.items()}, "key 'module.")
    _refused({"backbone." + k: v for k, v in sd.items()}, "key 'backbone.")
    odd = synthetic.dino_state_dict(seed=1, dim=128, depth=1, patch=8, grid=4)
    odd["patch_embed.proj.weight"] = torch.zeros(96, 3, 8, 8)
    _refused(odd, "'patch_embed.proj.weight' gives D = 96")
    _refused({k: v for k, v in sd.items() if k != "pos_embed"}, "missing key 'pos_embed'")
    big = {k: torch.zeros(s) for k, s in dino.key_shapes(64, 1, 8, 33).items()}
    _refused(big, "'pos_embed' has 1090 tokens, above 1025")
    ok = {k: torch.zeros(s) for k, s in dino.key_shapes(64, 1, 8, 32).items()}
    assert dino.load_state_dict(ok)[0]["tokens"] == 1025
    _refused({**sd, "pos_embed": torch.zeros(1, 18, 128)}, "'pos_embed' has 18 tokens")


def _runner(tmp_path, **kw):
    a = dict(run_test=True, diff_style=False, lpips=False, h_directions=False, pass_editing=False,
             dino_weights=str(tmp_path / "dino.pth"))
    a.update(kw)
    return NS(args=NS(**a))


def test_cli_refusals(tmp_path):
    torch.save(_small_sd(), tmp_path / "dino.pth")
    sd = scoring.dino_structure_setup(_runner(tmp_path))
    assert dino.load_state_dict(sd)[0]["dim"] == 128 and sd["pos_embed"].dtype == torch.float32
    scoring.dino_structure_setup(_runner(tmp_path, run_test=False, diff_style=True))
    for kw, match in ((dict(pass_editing=True), "--pass_editing"), (dict(run_test=False), "--run_test"),
                      (dict(lpips=True), "--lpips"), (dict(h_directions=True), "--h_directions"),
                      (dict(dino_weights=str(tmp_path / "none.pth")), "is not a file")):
        with pytest.raises(ValueError, match=match):
            scoring.dino_structure_setup(_runner(tmp_path, **kw))
    torch.save({"module." + k: v for k, v in _small_sd().items()}, tmp_path / "bad.pth")
    with pytest.raises(ValueError, match="--dino_structure: DINO state dict: key 'module."):
        scoring.dino_structure_setup(_runner(tmp_path, dino_weights=str(tmp_path / "bad.pth")))
    (tmp_path / "junk.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot read"):
        scoring.dino_structure_setup(_runner(tmp_path, dino_weights=str(tmp_path / "junk.pth")))


def test_cli_parses_the_flags():
    from asyrp_official_b200 import main as cli
    a = cli.build_parser().parse_args(["--run_test", "--config", "celeba.yml"])
    assert a.dino_structure is False and a.dino_weights == "pretrained/dino_vitbase8_pretrain.pth"
    a = cli.build_parser().parse_args(["--diff_style", "--config", "celeba.yml", "--dino_structure", "--dino_weights",
                                       "w.pth"])
    assert a.dino_structure is True and a.dino_weights == "w.pth"


def test_c_symbols():
    lib = _lib.load()
    for name in ("asyrp_dino_pack", "asyrp_dino_layernorm", "asyrp_dino_attention", "asyrp_dino_selfsim_partials",
                 "asyrp_dino_selfsim_distance"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    header = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "asyrp_b200.h")).read()
    for name in ("asyrp_dino_pack", "asyrp_dino_selfsim_distance"):
        assert f"int {name}(" in header
    assert [lib.asyrp_dino_selfsim_partials(T) for T in (0, 1, 64, 65, 785, 1025, 1026)] == [-1, 1, 1, 3, 91, 153, -1]


# ---------------------------------------------------------------------------------------------------------------------
def _table(path):
    with open(path) as f:
        return list(csv.reader(f, delimiter="\t"))


@pytest.mark.parametrize("attrs", [None, ["smiling", "angry"]])
def test_score_table_layout(tmp_path, attrs):
    sc = torch.arange(2 * 3 * 2, dtype=torch.float64).view(2, 3, 2) / 7
    origin = torch.tensor([[0.0, 1.0], [0.0, 0.5], [0.0, 0.25]], dtype=torch.float64)
    path = tmp_path / "t.tsv"
    scoring.write_scores(str(path), [(1.0, 0.5), (1.0, 1.0)], sc, scoring.DINO_COLUMNS, "DINO", attrs=attrs,
                         origin=origin)
    t = _table(path)
    assert t[0] == ["image", "tuple", "hs_coeff", "structure", "cls_cos"] + (["attr"] if attrs else [])
    assert t[1][:5] == ["0", "origin", "-", "0.0", "1.0"] and len(t) == 1 + 3 + 6
    assert t[4][:3] == ["0", "0", "1,0.5"] and float(t[5][3]) == sc[0, 1, 0].item()
    if attrs:
        assert [r[5] for r in t[1:]] == ["-"] * 3 + ["smiling"] * 3 + ["angry"] * 3


def test_diff_style_table_sorted(tmp_path):
    rows = [("c/b.png", "s/a.png", 0.5, 0.1, 0.2, 0.9, 0.8), ("c/a.png", "s/b.png", 0.9, 0.3, 0.4, 0.7, 0.6),
            ("c/a.png", "s/b.png", 0.5, 0.5, 0.6, 0.5, 0.4), ("c/a.png", "s/a.png", 0.9, 0.0, 0.1, 1.0, 0.2)]
    out = scoring.write_diff_style_dino(str(tmp_path / "d.tsv"), rows)
    t = _table(tmp_path / "d.tsv")
    assert t[0] == list(scoring.DIFF_STYLE_DINO_COLUMNS)
    assert [r[:3] for r in t[1:]] == [["c/a.png", "s/a.png", "0.9"], ["c/a.png", "s/b.png", "0.5"],
                                      ["c/a.png", "s/b.png", "0.9"], ["c/b.png", "s/a.png", "0.5"]]
    assert out[1] == rows[2] and t[2][3:] == [repr(v) for v in rows[2][3:]]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gather_worker(rank, world, port, path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runner = NS(rank=rank, world=world)
        # rank r holds the rows of the chunks r, r + world, ... as run_diff_style shards them
        mine = [(f"c{c}.png", f"s{s}.png", g, c + s + g, 0.0, 1.0, 1.0)
                for k, (c, s) in enumerate([(c, s) for c in range(3) for s in range(2)]) if k % world == rank
                for g in (0.9, 0.5)]
        rows = scoring.gather_rows(runner, mine)
        if rank == 0:
            scoring.write_diff_style_dino(path, rows)
        else:
            assert rows is None
    finally:
        dist.destroy_process_group()


def test_diff_style_gather_world2(tmp_path):
    import torch.multiprocessing as mp
    path2 = str(tmp_path / "w2.tsv")
    mp.spawn(_gather_worker, args=(2, _free_port(), path2), nprocs=2, join=True)
    runner = NS(rank=0, world=1)
    rows = scoring.gather_rows(runner, [(f"c{c}.png", f"s{s}.png", g, c + s + g, 0.0, 1.0, 1.0)
                                        for c in range(3) for s in range(2) for g in (0.9, 0.5)])
    scoring.write_diff_style_dino(str(tmp_path / "w1.tsv"), rows)
    assert open(path2).read() == open(tmp_path / "w1.tsv").read()
    assert len(_table(path2)) == 1 + 12


def test_scorers_without_the_flag_build_no_dino(tmp_path):
    a = NS(DirectionalClipSmilarity=False, id_similarity=False, seg_consistency=False, fid=False,
           content_preservation=False, dino_structure=False, load_random_noise=False)
    s = scoring.Scorers(NS(args=a))
    assert s.specs == {} and not s.needs_origin and not s.keeps_source
    a.dino_structure = True
    torch.save(_small_sd(), tmp_path / "dino.pth")
    runner = NS(args=a, dino_structure_setup=lambda: "sd")
    s = scoring.Scorers(runner)
    assert s.specs == {"dino": "sd"} and s.needs_origin and s.keeps_source
    a.load_random_noise = True
    assert not scoring.Scorers(runner).keeps_source
