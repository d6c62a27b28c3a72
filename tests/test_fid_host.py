"""FID / KID on the host: the oracle against torchvision's Inception3, the input mapping against a written PNG, BN
folding, the loader, the host statistics against their restatements, the CLI refusals, the TSV layout and the
end-of-run gather of the pool features over a gloo world of 2."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from asyrp_official_b200 import fid, synthetic
from oracle import fid as ofid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def sd():
    return synthetic.inception_state_dict(seed=3)


def test_oracle_stem_and_shared_blocks_equal_torchvision(sd):
    tv = ofid.torchvision_inception(sd, dtype=torch.float32)
    m = ofid.fid_inception(sd, dtype=torch.float32)
    x = torch.randn(2, 3, 83, 83, generator=_g(1))
    with torch.no_grad():
        ref = tv.maxpool2(tv.Conv2d_4a_3x3(tv.Conv2d_3b_1x1(tv.maxpool1(
            tv.Conv2d_2b_3x3(tv.Conv2d_2a_3x3(tv.Conv2d_1a_3x3(x)))))))
        assert torch.equal(ofid.stem(m, x), ref)
        h = torch.randn(2, 288, 11, 11, generator=_g(2))
        assert torch.equal(m.Mixed_6a(h), tv.Mixed_6a(h))  # InceptionB
        h = torch.randn(2, 768, 9, 9, generator=_g(3))
        assert torch.equal(m.Mixed_7a(h), tv.Mixed_7a(h))  # InceptionD


@pytest.mark.parametrize("name,cin", [("Mixed_5b", 192), ("Mixed_6b", 768), ("Mixed_7b", 1280)])
def test_fid_blocks_equal_torchvision_away_from_the_border(sd, name, cin):
    tv = ofid.torchvision_inception(sd, dtype=torch.float32)
    m = ofid.fid_inception(sd, dtype=torch.float32)
    x = torch.rand(1, cin, 8, 9, generator=_g(4))
    with torch.no_grad():
        a, b = getattr(m, name)(x), getattr(tv, name)(x)
    assert torch.equal(a[..., 1:-1, 1:-1], b[..., 1:-1, 1:-1])
    border = torch.ones(8, 9, dtype=torch.bool)
    border[1:-1, 1:-1] = False
    assert (a[..., border] != b[..., border]).any()  # count_include_pad=False only changes border pixels


def test_fid_e2_pools_with_max(sd):
    tv = ofid.torchvision_inception(sd, dtype=torch.float32)
    m = ofid.fid_inception(sd, dtype=torch.float32)
    x = torch.randn(1, 2048, 8, 8, generator=_g(5))
    with torch.no_grad():
        a, b = m.Mixed_7c(x), tv.Mixed_7c(x)
        assert torch.equal(a[:, :1856], b[:, :1856])  # the branches without a pool
        assert torch.equal(a[:, 1856:], tv.Mixed_7c.branch_pool(F.max_pool2d(x, 3, 1, 1)))
        assert not torch.equal(a[:, 1856:], b[:, 1856:])


def test_input_mapping_equals_the_written_png(tmp_path):
    import torchvision.utils as tvu
    from PIL import Image
    x = torch.rand(2, 3, 37, 45, generator=_g(6)) * 2.4 - 1.2  # past [-1, 1]: the clamp
    x[0, 0, 0, :6] = torch.tensor([-1.0, 1.0, -1 + 1 / 255, 0.0, 2 / 255 - 1, 1 - 0.5 / 255])
    for i in range(2):
        path = str(tmp_path / f"{i}.png")
        tvu.save_image((x[i:i + 1] + 1) * 0.5, path)
        u8 = torch.from_numpy(np.asarray(Image.open(path).convert("RGB")).copy()).permute(2, 0, 1)
        assert torch.equal(ofid.quantise(x[i:i + 1])[0], u8)
        ref = F.interpolate(u8[None].float() / 255, size=(299, 299), mode="bilinear", align_corners=False) * 2 - 1
        assert torch.equal(ofid.preprocess(x[i:i + 1], dtype=torch.float32), ref)


def test_folding_is_exact_algebra(sd):
    raw = fid.load_state_dict(sd)
    folded = fid.fold(raw)
    for name in ("Conv2d_1a_3x3", "Mixed_6b.branch7x7_2", "Mixed_7c.branch3x3dbl_3b"):
        cin, cout, kh, kw, stride, ph, pw = fid.conv_specs()[name]
        x = torch.randn(2, cin, 9, 9, generator=_g(7), dtype=torch.float64)
        conv = F.conv2d(x, raw[f"{name}.conv.weight"].double(), stride=stride, padding=(ph, pw))
        g = {s: raw[f"{name}.bn.{s}"].double() for s in fid.BN_STATS}
        ref = F.batch_norm(conv, g["running_mean"], g["running_var"], g["weight"], g["bias"], False, 0.0, fid.BN_EPS)
        w, b = folded[name]
        out = F.conv2d(x, w.double(), b.double(), stride=stride, padding=(ph, pw))
        assert (out - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()  # fp32 storage of the folded pair
        s = g["weight"] / torch.sqrt(g["running_var"] + fid.BN_EPS)
        assert torch.equal(w, (raw[f"{name}.conv.weight"].double() * s[:, None, None, None]).float())
        assert torch.equal(b, (g["bias"] - g["running_mean"] * s).float())


def test_loader_accepts_the_layout_and_refuses_bad_keys(sd, tmp_path):
    assert sum(k.endswith(".conv.weight") for k in sd) == 94
    assert "fc.weight" in sd and "Conv2d_1a_3x3.bn.num_batches_tracked" in sd
    path = str(tmp_path / "pt_inception.pth")
    torch.save(sd, path)
    out = fid.load_state_dict(path)
    assert set(out) == set(fid.state_dict_shapes())  # fc.* and num_batches_tracked ignored
    assert set(fid.load_state_dict({k: v for k, v in sd.items()
                                    if not k.startswith("fc.") and "num_batches" not in k})) == set(out)
    with pytest.raises(ValueError, match="missing key 'Mixed_6c.branch7x7dbl_4.bn.running_var'"):
        fid.load_state_dict({k: v for k, v in sd.items() if k != "Mixed_6c.branch7x7dbl_4.bn.running_var"})
    with pytest.raises(ValueError, match="'Mixed_5b.branch_pool.conv.weight' has shape"):
        fid.load_state_dict({**sd, "Mixed_5b.branch_pool.conv.weight": torch.zeros(64, 192, 1, 1)})
    with pytest.raises(ValueError, match="unexpected keys.*AuxLogits.fc.weight"):
        fid.load_state_dict({**sd, "AuxLogits.fc.weight": torch.zeros(1008, 768)})
    with pytest.raises(ValueError, match="'fc.weight' has shape"):
        fid.load_state_dict({**sd, "fc.weight": torch.zeros(1000, 2048)})
    (tmp_path / "junk.pth").write_bytes(b"\x00" * 64)
    with pytest.raises(ValueError, match="cannot be read"):
        fid.load_state_dict(str(tmp_path / "junk.pth"))


def _feats(n, d, seed, shift=0.0):
    g = np.random.default_rng(seed)
    return g.standard_normal((n, d)) @ g.standard_normal((d, d)) * 0.3 + shift


def test_frechet_distance():
    f = _feats(3000, 8, 1)
    mu, s = ofid.moments(f)
    assert abs(fid.frechet_distance(mu, s, mu, s)) < 1e-10
    shift = np.linspace(-1, 1, 8)
    mu2, s2 = ofid.moments(f + shift)
    assert np.isclose(fid.frechet_distance(mu, s, mu2, s2), shift @ shift, rtol=1e-10, atol=1e-10)
    g = _feats(2500, 8, 2, shift=0.5)
    mu3, s3 = ofid.moments(g)
    ref = ofid.frechet_distance_sqrtm(mu, s, mu3, s3)
    assert abs(fid.frechet_distance(mu, s, mu3, s3) - ref) <= 1e-8 * abs(ref)
    # rank-deficient covariances (n < d): defined, non-negative, 0 against itself
    few = _feats(5, 64, 3)
    m4, s4 = ofid.moments(few)
    # the null space's eigenvalues are rounding noise ~1e-16 tr S, each adding its square root: ~1e-7 tr S in all
    assert abs(fid.frechet_distance(m4, s4, m4, s4)) < 1e-6 * np.trace(s4)
    assert fid.frechet_distance(m4, s4, *ofid.moments(_feats(5, 64, 4))) > 0


def test_kid_matches_a_direct_double_loop():
    f1, f2 = _feats(9, 16, 5), _feats(7, 16, 6, shift=0.2)
    d = 16
    k = {key: (a @ b.T / d + 1) ** 3 for key, (a, b) in {"xx": (f1, f1), "yy": (f2, f2), "xy": (f1, f2)}.items()}
    got = fid.kid_from_sums(k["xx"].sum() - np.trace(k["xx"]), k["yy"].sum() - np.trace(k["yy"]), k["xy"].sum(), 9, 7)
    assert np.isclose(got, ofid.kid_loop(f1, f2), rtol=1e-12, atol=1e-14)


def test_cli_rejections_come_before_any_model_load(tmp_path, monkeypatch):
    from asyrp_official_b200 import main as cli
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    sd = synthetic.inception_state_dict(seed=1, fc=False)
    torch.save(sd, "pt_inception.pth")
    torch.save({k: v for k, v in sd.items() if k != "Mixed_7a.branch3x3_2.conv.weight"}, "partial.pth")
    (tmp_path / "junk.pth").write_bytes(b"\x00" * 64)

    def fail_load(*a, **k):
        raise AssertionError("a model was loaded before the requirements were checked")
    monkeypatch.setattr(Asyrp, "load_pretrained_model", fail_load)
    monkeypatch.setattr(Asyrp, "set_t_edit_t_addnoise", fail_load)
    base = ["--run_test", "--config", "celeba.yml", "--fid"]
    cases = [(["--fid_weights", "pt_inception.pth", "--pass_editing"], "--pass_editing"),
             ([], "is not a file"),  # the default pretrained/pt_inception-2015-12-05-6726825d.pth does not exist here
             (["--fid_weights", "partial.pth"], "missing key 'Mixed_7a.branch3x3_2.conv.weight'"),
             (["--fid_weights", "junk.pth"], "cannot be read")]
    for extra, match in cases:
        args, cfg = cli.parse_args_and_config(base + extra)
        with pytest.raises(ValueError, match=match):
            Asyrp(args, cfg, device="cpu").run_test()
    args, cfg = cli.parse_args_and_config(["--diff_style", "--config", "celeba.yml", "--fid", "--fid_weights",
                                           "pt_inception.pth"])
    with pytest.raises(ValueError, match="--diff_style is not scored"):
        Asyrp(args, cfg, device="cpu").run_diff_style()
    args, _ = cli.parse_args_and_config(["--run_test", "--config", "celeba.yml"])
    assert args.fid_weights == "pretrained/pt_inception-2015-12-05-6726825d.pth" and not args.fid


def test_fid_table_layout(tmp_path, capsys):
    from asyrp_official_b200.scoring import write_fid
    rows = [(12.5, 0.25), (float("nan"), float("nan")), (0.1 + 0.2, 1e-17)]
    coeffs = [(1.0, 0.5), (1.0, 1.0), (1.0, 1.5)]
    write_fid(str(tmp_path / "t.tsv"), coeffs, rows, 40, "test")
    lines = (tmp_path / "t.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tFID\tKID"
    assert lines[1:] == [f"{k}\t1,{c}\t40\t{rows[k][0]!r}\t{rows[k][1]!r}" for k, c in enumerate(("0.5", "1", "1.5"))]
    assert "hs_coeff (1.0, 0.5): FID 12.500000, KID 0.250000" in capsys.readouterr().out
    attrs = ["smiling", "angry", "young"]
    write_fid(str(tmp_path / "s.tsv"), [(1.0, 1.0, 0.0, 0.0), (1.0, 0.0, 1.0, 0.0), (1.0, 0.0, 0.0, 1.0)], rows, 3,
              "train", attrs=attrs)
    lines = (tmp_path / "s.tsv").read_text().splitlines()
    assert lines[0] == "tuple\ths_coeff\tn\tFID\tKID\tattr"
    assert [ln.split("\t")[5] for ln in lines[1:]] == attrs and lines[2].split("\t")[1] == "1,0,1,0"


# ---------------------------------------------------------------------------------------------------------------------
N_IMAGES, BS = 7, 2  # batches of image indices (0, 1), (2, 3), (4, 5), (6,): rank b % 2 holds batch b


def _batches():
    g = torch.Generator().manual_seed(9)
    feats = {key: torch.randn(N_IMAGES, 64, generator=g) for key in ("origin", 0, 1)}
    return [list(range(i, min(i + BS, N_IMAGES))) for i in range(0, N_IMAGES, BS)], feats


def _collect(rank, world):
    batches, feats = _batches()
    sets = fid.FeatureSets()
    for b, ids in enumerate(batches):
        if b % world == rank:
            for key in ("origin", 0, 1):
                sets.add("test", key, ids, feats[key][ids])
    return sets


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    got = _collect(rank, world).gather(rank, world)
    q.put((rank, got))
    dist.destroy_process_group()


def test_gather_world2_reassembles_image_order():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + os.getpid() % 90
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res[1] is None
    one = _collect(0, 1).gather(0, 1)
    _, feats = _batches()
    assert set(res[0]) == set(one) == {("test", "origin"), ("test", 0), ("test", 1)}
    for key, (ids, f) in one.items():
        assert torch.equal(ids, torch.arange(N_IMAGES)) and torch.equal(f, feats[key[1]])
        assert torch.equal(res[0][key][0], ids) and torch.equal(res[0][key][1], f)
    ref = ofid.moments(one[("test", "origin")][1].double().numpy())
    for k in (0, 1):
        a = fid.frechet_distance(*ref, *ofid.moments(one[("test", k)][1].double().numpy()))
        b = fid.frechet_distance(*ref, *ofid.moments(res[0][("test", k)][1].double().numpy()))
        assert a == b and a > 0


def test_feature_sets_refuse_an_image_twice():
    sets = fid.FeatureSets()
    sets.add("test", "origin", [0, 1], torch.zeros(2, 4))
    sets.add("test", "origin", [1], torch.zeros(1, 4))
    with pytest.raises(ValueError, match="occurs twice"):
        sets.gather()
