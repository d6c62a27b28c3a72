"""FID / KID against real images on the GPU: the u8 pack and features_u8 bit for bit against the fp32 path, the subset
kernel sum bit for bit against the plain kernel sum of the gathered rows and against fp64, kid_subsets against the
restatement of torch-fidelity, the --save-stats command end to end, and `main --run_test --fid --fid_ref`."""
import csv
import os

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, fid, ops, synthetic
from test_fid_gpu import BASE, _bytes, _delta_block_ckpt, _run
from test_fid_real_host import kid_subsets_oracle

pytestmark = pytest.mark.gpu


def _u8(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    u = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    u.view(-1)[:min(256, u.numel())] = torch.arange(256, dtype=torch.uint8)[:min(256, u.numel())]  # every value
    return u


def _as_float(u):
    """u / 127.5 - 1 as fp32 NCHW: the image whose save_image u8 is u"""
    return (u.permute(0, 3, 1, 2).float() / 127.5 - 1).contiguous()


@pytest.mark.parametrize("B,H,W", [(2, 256, 256), (1, 1024, 1024), (3, 37, 45), (1, 1, 1), (1, 512, 300)])
def test_pack_u8_equals_pack_of_the_float_image(cuda_device, B, H, W):
    u = _u8(B, H, W, H * W)
    got = torch.empty(B, 299, 299, 4, device=cuda_device)
    ref = torch.full((B, 299, 299, 4), 7.0, device=cuda_device)
    ops.fid_pack_u8(u.to(cuda_device), got)
    ops.fid_pack(_as_float(u).to(cuda_device), ref)
    assert torch.equal(got, ref)
    if H == W and H <= 299:  # at S = H the resize is the identity: u / 255 * 2 - 1 exactly
        same = torch.empty(B, H, H, 4, device=cuda_device)
        ops.fid_pack_u8(u.to(cuda_device), same)
        assert torch.equal(same[..., :3].cpu(), u.float() / 255 * 2 - 1)


@pytest.fixture(scope="module")
def net(cuda_device):
    return fid.FIDInception(synthetic.inception_state_dict(seed=7), device=cuda_device)


def test_features_u8_equal_features(net, cuda_device):
    u = _u8(5, 80, 64, 3)
    f = net.features(_as_float(u))
    assert torch.equal(net.features_u8(u), f)
    assert torch.equal(net.features_u8(u.pin_memory()), f)
    assert torch.equal(net.features_u8(u.to(cuda_device)), f)
    chunked = fid.FIDInception(synthetic.inception_state_dict(seed=7), device=cuda_device, max_rows=2)
    assert torch.equal(chunked.features_u8(u), f)
    with pytest.raises(ValueError, match="uint8"):
        net.features_u8(u.float())


def _gathered_cases():
    """(n, m, s, subsets): s of 2, 63, 64, 65 and 1000, n != m"""
    return [(5, 3, 2, 4), (100, 70, 63, 3), (64, 200, 64, 2), (130, 66, 65, 3), (1200, 1500, 1000, 2)]


def _indices(n, s, subsets, seed):
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(n, s, replace=s > n) for _ in range(subsets)]).astype(np.int32)
    idx[0, 0], idx[-1, -1] = 0, n - 1  # the first and the last row
    if subsets > 1:
        idx[1, :s // 2] = idx[0, :s // 2]  # rows that repeat across subsets
    return idx


@pytest.mark.parametrize("n,m,s,subsets", _gathered_cases())
def test_subset_sums_equal_the_kernel_sum_of_the_gathered_rows(cuda_device, n, m, s, subsets):
    d = 2048 if s == 1000 else 48
    g = np.random.default_rng(n + m)
    x, y = (torch.from_numpy(g.random((k, d)).astype(np.float32)).to(cuda_device) for k in (n, m))
    ix, iy = _indices(n, s, subsets, 1), _indices(m, s, subsets, 2)
    tx, ty = torch.from_numpy(ix).to(cuda_device), torch.from_numpy(iy).to(cuda_device)
    x64, y64 = x.cpu().double().numpy(), y.cpu().double().numpy()
    for excl in (False, True):
        got = ops.fid_kernel_sum_subsets(x, y, tx, ty, exclude_diag=excl)
        assert got.shape == (subsets,) and got.dtype == torch.float64
        for z in range(subsets):
            xz, yz = x[tx[z].long()].contiguous(), y[ty[z].long()].contiguous()
            assert torch.equal(got[z], ops.fid_kernel_sum(xz, yz, excl)), (excl, z)
            k = (x64[ix[z]] @ y64[iy[z]].T / d + 1) ** 3
            ref = k.sum() - (np.trace(k) if excl else 0.0)
            assert abs(got[z].item() - ref) <= 1e-12 * abs(ref)
    # within one set (x = y, the same indices): what kid_subsets launches
    same = ops.fid_kernel_sum_subsets(x, x, tx, tx, exclude_diag=True)
    for z in range(subsets):
        xz = x[tx[z].long()].contiguous()
        assert torch.equal(same[z], ops.fid_kernel_sum(xz, xz, True))


def test_subset_sum_refusals(cuda_device):
    x = torch.zeros(10, 32, device=cuda_device)
    idx = torch.zeros(3, 4, dtype=torch.int32, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match=r"idx_y holds rows in \[0, 10\], outside \[0, 10\)"):
        bad = idx.clone()
        bad[2, 3] = 10
        ops.fid_kernel_sum_subsets(x, x, idx, bad)
    with pytest.raises(_lib.AsyrpError, match="outside"):
        ops.fid_kernel_sum_subsets(x, x, idx - 1, idx)
    with pytest.raises(_lib.AsyrpError, match="int32"):
        ops.fid_kernel_sum_subsets(x, x, idx.long(), idx.long())
    with pytest.raises(_lib.AsyrpError, match="exclude_diag needs s >= 2"):
        one = idx[:, :1].contiguous()
        ops.fid_kernel_sum_subsets(x, x, one, one, exclude_diag=True)
    odd = torch.zeros(10, 24, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="multiple of 16"):
        ops.fid_kernel_sum_subsets(odd, odd, idx, idx)
    many = torch.zeros(65536, 2, dtype=torch.int32, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="subsets=65536 above 65535"):
        ops.fid_kernel_sum_subsets(x, x, many, many)
    ops.fid_kernel_sum_subsets(x, x, many[:65535], many[:65535])  # the limit itself runs


def test_kid_subsets_equal_torch_fidelity(cuda_device, capsys):
    g = np.random.default_rng(5)
    f1 = (g.random((300, 2048)) * 0.5).astype(np.float32)
    f2 = (g.random((450, 2048)) * 0.5 + 0.1).astype(np.float32)
    t1, t2 = torch.from_numpy(f1).to(cuda_device), torch.from_numpy(f2).to(cuda_device)
    for subsets, size in ((10, 100), (3, 300), (1, 2)):
        mean, std = fid.kid_subsets(t1, t2, subsets, size)
        rm, rs = kid_subsets_oracle(f1, f2, subsets, size)
        assert abs(mean - rm) <= 1e-10 * abs(rm), (subsets, size, mean, rm)
        assert abs(std - rs) <= 1e-10 * abs(rm) + 1e-10 * rs, (subsets, size, std, rs)
    assert all(np.isnan(v) for v in fid.kid_subsets(t1[:50], t2, 2, 51))
    assert "smaller than the subset size 51" in capsys.readouterr().out


# ---------------------------------------------------------------------------------------------------------------------
def _write_folder(folder, seed):
    """seeded PNG / JPG images of mixed sizes, one grayscale PNG and one RGBA PNG"""
    from PIL import Image
    os.makedirs(folder)
    g = np.random.default_rng(seed)
    sizes = [(64, 64), (64, 64), (48, 80), (64, 64), (33, 47), (48, 80), (64, 64), (21, 21), (64, 64), (48, 80)]
    for i, (h, w) in enumerate(sizes):
        a = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if i == 3:
            Image.fromarray(a[..., 0]).save(os.path.join(folder, f"{i:02d}.png"))
        elif i == 5:
            rgba = np.concatenate([a, g.integers(0, 256, (h, w, 1), dtype=np.uint8)], axis=2)
            Image.fromarray(rgba).save(os.path.join(folder, f"{i:02d}.png"))
        elif i % 3 == 1:
            Image.fromarray(a).save(os.path.join(folder, f"{i:02d}.jpg"), quality=90)
        else:
            Image.fromarray(a).save(os.path.join(folder, f"{i:02d}.png"))
    with open(os.path.join(folder, "notes.txt"), "w") as f:
        f.write("not an image\n")


def test_save_stats_command(cuda_device, tmp_path, capsys):
    from PIL import Image
    folder = str(tmp_path / "real")
    _write_folder(folder, 3)
    sd = synthetic.inception_state_dict(seed=5)
    torch.save(sd, str(tmp_path / "w.pth"))
    outs = {}
    for bs, nw in ((1, 0), (7, 0), (7, 2), (50, 2)):
        out = str(tmp_path / f"s_{bs}_{nw}.npz")
        assert fid.main(["--save-stats", folder, out, "--fid_weights", str(tmp_path / "w.pth"), "--batch_size",
                         str(bs), "--num_workers", str(nw)]) == 0
        outs[(bs, nw)] = _bytes(out)
    assert "--save-stats: 10 images" in capsys.readouterr().out
    assert len(set(outs.values())) == 1  # the same file for any batch size and worker count
    # the pytorch-fid way: each file opened, converted to RGB, one image at a time through features(u / 127.5 - 1)
    net = fid.FIDInception(sd, device=cuda_device)
    files = sorted(os.path.join(folder, f) for f in os.listdir(folder) if not f.endswith(".txt"))
    feats = torch.cat([net.features(_as_float(torch.from_numpy(np.asarray(Image.open(p).convert("RGB")).copy())[None]))
                       for p in files])
    mu, sigma = fid.set_moments(feats)
    z = np.load(str(tmp_path / "s_1_0.npz"))
    assert np.array_equal(z["mu"], mu) and np.array_equal(z["sigma"], sigma)
    assert np.array_equal(z["features"], feats.cpu().numpy())
    assert z["kid_kxx"] == ops.fid_kernel_sum(feats, feats, exclude_diag=True).item()
    assert fid.validate_stats(str(tmp_path / "s_1_0.npz")) == (10, True)


# ---------------------------------------------------------------------------------------------------------------------
def _table(path):
    with open(path) as f:
        return list(csv.reader(f, delimiter="\t"))


def _stats(path, sd, device, features=True):
    net = fid.FIDInception(sd, device=device)
    feats = net.features_u8(_u8(6, 64, 64, 17))
    if features:
        fid.save_stats(path, feats)
    else:
        mu, sigma = fid.set_moments(feats)
        np.savez_compressed(path, mu=mu, sigma=sigma)  # pytorch-fid's --save-stats layout


@pytest.mark.parametrize("mode", ["single", "interp", "sweep"])
def test_run_test_fid_ref(cuda_device, tmp_path, monkeypatch, mode):
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    sd = synthetic.inception_state_dict(seed=5)
    torch.save(sd, "pt_inception.pth")
    _stats("ref.npz", sd, cuda_device)
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)
    argv = BASE + ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling", "--bs_train", "2"]
    tuples, attrs = 1, None
    if mode == "interp":
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
        tuples = 3
    elif mode == "sweep":
        argv = BASE + ["--attr_sweep", "smiling angry", "--manual_checkpoint_name", "attribute_0.pth",
                       "--bs_train", "2"]
        tuples, attrs = 2, ["smiling", "angry"]
    fid_argv = ["--fid", "--fid_weights", "pt_inception.pth"]
    ref_argv = ["--fid_ref", "ref.npz", "--kid_subsets", "3", "--kid_subset_size", "2"]
    captured = []
    finish = Asyrp.finish_fid

    def capturing(self, sets, *a, **kw):
        captured.append(sets)
        return finish(self, sets, *a, **kw)
    monkeypatch.setattr(Asyrp, "finish_fid", capturing)
    r, _ = _run(argv + fid_argv + ref_argv, cuda_device)
    folder = r.args.test_image_folder
    names = ["test_ngen4_fid.tsv", "test_1_0_ngen4.png"]
    with_ref = [_bytes(os.path.join(folder, nm)) for nm in names]
    real_tsv = os.path.join(folder, "test_ngen4_fid_real.tsv")
    table = _table(real_tsv)
    os.remove(real_tsv)
    _run(argv + fid_argv, cuda_device)  # without --fid_ref: the same _fid.tsv and PNG, no _fid_real.tsv
    assert [_bytes(os.path.join(folder, nm)) for nm in names] == with_ref
    assert not os.path.exists(real_tsv)
    header = ["tuple", "hs_coeff", "n", "n_ref", "FID", "KID", "KID_mean", "KID_std"] + (["attr"] if attrs else [])
    assert table[0] == header and len(table) == 2 + tuples
    assert [t[0] for t in table[1:]] == ["origin"] + [str(k) for k in range(tuples)] and table[1][1] == "-"
    assert all(t[2] == "2" and t[3] == "6" for t in table[1:])
    if attrs:
        assert [t[8] for t in table[1:]] == ["-"] + attrs
    vals = torch.tensor([[float(v) for v in t[4:8]] for t in table[1:]], dtype=torch.float64)
    assert torch.equal(vals, r.fid_real["test"]) and torch.isfinite(vals).all()
    # the table recomputed from the gathered features and the file
    got = captured[0].gather()
    real = fid.load_stats("ref.npz")
    real["features"] = torch.from_numpy(real["features"]).to(cuda_device)
    keys = ["origin"] + list(range(tuples))
    ref_rows = [fid.score_against_stats(got[("test", k)][1].to(cuda_device).contiguous(), real, 3, 2) for k in keys]
    assert torch.equal(torch.tensor(ref_rows, dtype=torch.float64), vals)
    if mode == "single":  # a mu / sigma-only file: FID, and nan KID
        _stats("ref_fid_only.npz", sd, cuda_device, features=False)
        r2, _ = _run(argv + fid_argv + ["--fid_ref", "ref_fid_only.npz"], cuda_device)
        t2 = _table(real_tsv)
        assert all(t[3] == "-" for t in t2[1:])
        v2 = r2.fid_real["test"]
        assert torch.equal(v2[:, 0], vals[:, 0]) and torch.isnan(v2[:, 1:]).all()
