"""Precision / recall / density / coverage on the GPU: asyrp_fid_knn_radii and asyrp_fid_knn_counts against the fp64
restatement (bit for bit on integer-valued features, where every distance is an exact integer), their argument limits,
and `main --run_test --fid --prdc` end to end."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from asyrp_official_b200 import _lib, fid, ops, synthetic
from test_fid_gpu import BASE, _bytes, _delta_block_ckpt, _run
from test_fid_real_gpu import _stats, _table
from test_prdc_host import counts_oracle, prdc_oracle, radii_oracle

pytestmark = pytest.mark.gpu

KS = (1, 3, 5, 32)


def _dist(a, b):
    """D fp64 [n][m] of a [n][d], b [m][d] on the device, the definition written out in torch (differences in fp64,
    squared, summed), in row chunks"""
    a, b = a.double(), b.double()
    rows = max(1, (1 << 27) // max(1, b.shape[0] * b.shape[1]))
    return torch.cat([((a[i:i + rows, None, :] - b[None]) ** 2).sum(-1) for i in range(0, a.shape[0], rows)])


def _kth(D, k):
    return torch.sort(D, dim=1).values[:, k]


def _random(n, d, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g).to(dev)


def _integers(n, d, seed, dev, lo=-4, hi=5):
    """integer-valued fp32 features with planted duplicate rows (radius exactly 0 once k of them coincide)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(lo, hi, (n, d), generator=g).float()
    if n >= 6:
        x[1] = x[0]
        x[n - 1] = x[0]
        x[n // 2] = x[3]
    return x.to(dev)


# ---- knn_radii ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", ["k+1", 63, 64, 65, 129, 4097])
@pytest.mark.parametrize("d", [1, 2048])
def test_radii_against_the_definition(cuda_device, n, d):
    sets = {}
    for k in KS:
        rows = k + 1 if n == "k+1" else n
        if rows not in sets:
            x, xi = _random(rows, d, rows * d, cuda_device), _integers(rows, d, rows + d, cuda_device)
            sets[rows] = (x, _dist(x, x), xi, _dist(xi, xi))
        x, Dx, xi, D = sets[rows]
        got = ops.fid_knn_radii(x, k)
        assert got.dtype == torch.float64 and got.shape == (rows,)
        ref = _kth(Dx, k)
        assert torch.all((got - ref).abs() <= 1e-12 * ref.abs()), (k, (got - ref).abs().max().item())
        exact = ops.fid_knn_radii(xi, k)
        assert torch.equal(exact, _kth(D, k)), k
        assert torch.equal(ops.fid_knn_radii(xi, k), exact)  # launch to launch
        if d == 1 and rows <= 129:  # the numpy restatement
            assert np.array_equal(exact.cpu().numpy(), radii_oracle(xi.cpu().numpy(), k))


def test_planted_duplicates_have_radius_zero(cuda_device):
    x = _integers(200, 16, 3, cuda_device)
    x[10:14] = x[9]  # five equal rows: each has four others at distance 0
    r = ops.fid_knn_radii(x, 4)
    assert torch.all(r[9:14] == 0) and torch.all(r[[0, 1, 199]] > 0)  # rows 0, 1, 199 are three equal rows
    assert torch.equal(ops.fid_knn_radii(x, 2)[[0, 1, 199]].cpu(), torch.zeros(3, dtype=torch.float64))
    assert torch.equal(r, _kth(_dist(x, x), 4))


def test_radii_do_not_depend_on_the_row_order(cuda_device):
    x = _random(700, 96, 9, cuda_device)
    perm = torch.randperm(700, generator=torch.Generator().manual_seed(1)).to(cuda_device)
    for k in (1, 7, 32):
        assert torch.equal(ops.fid_knn_radii(x, k)[perm], ops.fid_knn_radii(x[perm].contiguous(), k))


def test_radii_30000_rows_sampled_against_the_cpu(cuda_device):
    x = _random(30000, 2048, 30, cuda_device)
    k = 5
    got = ops.fid_knn_radii(x, k).cpu()
    rows = torch.randperm(30000, generator=torch.Generator().manual_seed(2))[:256]
    rows[0], rows[1] = 0, 29999
    xc = x.cpu().double()

    def radius(i):
        t = xc - xc[i]
        return t.mul_(t).sum(1).kthvalue(k + 1).values
    ref = torch.stack([radius(i) for i in rows.tolist()])
    assert torch.all((got[rows] - ref).abs() <= 1e-12 * ref), (got[rows] - ref).abs().max().item()


# ---- knn_counts -----------------------------------------------------------------------------------------------------
def _check_counts(a, ra, b, rb):
    D = _dist(a, b)
    ref = ((D < ra[:, None]).sum(0), (D < rb[None, :]).sum(1), (D < ra[:, None]).sum(1))
    got = ops.fid_knn_counts(a, ra, b, rb)
    for g, r in zip(got, ref):
        assert g.dtype == torch.int32 and torch.equal(g.long(), r)
    return got, D


@pytest.mark.parametrize("n,m", [(1, 1), (1, 70), (70, 1), (63, 64), (64, 65), (65, 63), (129, 200), (300, 4097)])
def test_counts_integer_features_bit_exact(cuda_device, n, m):
    d = 40
    a, b = _integers(n, d, n, cuda_device, -2, 3), _integers(m, d, m + 1, cuda_device, -2, 3)
    D = _dist(a, b)
    # radii that are distances of the pairs themselves: D == r ties everywhere, which < must not count
    ra = D[:, torch.arange(n, device=cuda_device) % m].diagonal().contiguous()
    rb = D[torch.arange(m, device=cuda_device) % n, torch.arange(m, device=cuda_device)].contiguous()
    assert torch.any(D == ra[:, None]) and torch.any(D == rb[None, :])
    _check_counts(a, ra, b, rb)
    if n <= 129 and m <= 200:  # the numpy restatement
        got = ops.fid_knn_counts(a, ra, b, rb)
        ref = counts_oracle(a.cpu().numpy(), ra.cpu().numpy(), b.cpu().numpy(), rb.cpu().numpy())
        assert all(np.array_equal(g.cpu().numpy(), r) for g, r in zip(got, ref))


@pytest.mark.parametrize("n,m,d", [(1, 5, 2048), (65, 129, 2048), (500, 300, 2048), (257, 191, 3)])
def test_counts_random_features(cuda_device, n, m, d):
    a, b = _random(n, d, 1, cuda_device), _random(m, d, 2, cuda_device) * 1.05
    ka, kb = min(3, n - 1), min(3, m - 1)
    ra = ops.fid_knn_radii(a, ka) if n > 1 else torch.full((1,), 1e9, dtype=torch.float64, device=cuda_device)
    rb = ops.fid_knn_radii(b, kb) if m > 1 else torch.full((1,), 1e9, dtype=torch.float64, device=cuda_device)
    got, D = _check_counts(a, ra, b, rb)
    # exact, not by luck: no pair is within 1e-9 relative of a radius it is compared with
    assert torch.all((D - ra[:, None]).abs() > 1e-9 * ra[:, None]) and torch.all((D - rb[None]).abs() > 1e-9 * rb[None])
    assert sum(int(g.sum()) for g in got) > 0


def test_counts_split_and_overwrite(cuda_device):
    n, m, m1, d = 150, 230, 97, 64
    a, b = _integers(n, d, 5, cuda_device, -3, 4), _integers(m, d, 6, cuda_device, -3, 4)
    ra, rb = ops.fid_knn_radii(a, 3), ops.fid_knn_radii(b, 2)
    whole = ops.fid_knn_counts(a, ra, b, rb)
    p1 = ops.fid_knn_counts(a, ra, b[:m1].contiguous(), rb[:m1].contiguous())
    p2 = ops.fid_knn_counts(a, ra, b[m1:].contiguous(), rb[m1:].contiguous())
    assert torch.equal(whole[0], torch.cat([p1[0], p2[0]]))
    assert torch.equal(whole[1], p1[1] + p2[1]) and torch.equal(whole[2], p1[2] + p2[2])
    out = tuple(torch.full((s,), 12345, dtype=torch.int32, device=cuda_device) for s in (m, n, n))
    for _ in range(2):  # overwritten, not added to
        ops.fid_knn_counts(a, ra, b, rb, out=out)
        assert all(torch.equal(o, w) for o, w in zip(out, whole))


def test_worked_examples_on_the_gpu(cuda_device):
    def col(v):
        return torch.tensor(v, dtype=torch.float32, device=cuda_device)[:, None]
    assert fid.prdc(col([0, 1, 2, 3]), col([0.5, 10]), 1) == (0.5, 1.0, 1.0, 0.5)
    assert torch.equal(fid.knn_radii(col([0, 0, 0, 5]), 1).cpu(), torch.tensor([0.0, 0.0, 0.0, 25.0], dtype=torch.float64))
    assert fid.prdc(col([0, 0, 0, 5]), col([0, 7]), 1) == (0.5, 1.0, 0.5, 0.25)


@pytest.mark.parametrize("n,m,d,k", [(40, 30, 2048, 3), (129, 65, 8, 5), (70, 90, 2, 32), (33, 33, 1, 32)])
def test_prdc_against_the_restatement(cuda_device, n, m, d, k):
    g = np.random.default_rng(n * m)
    real = g.integers(-3, 4, (n, d)).astype(np.float32)
    fake = (g.integers(-3, 4, (m, d)) + (g.random((m, 1)) < 0.3)).astype(np.float32)
    got = fid.prdc(torch.from_numpy(real).to(cuda_device), torch.from_numpy(fake).to(cuda_device), k)
    ref = prdc_oracle(real, fake, k)
    assert got == ref
    rr = fid.knn_radii(torch.from_numpy(real).to(cuda_device), k)
    assert fid.prdc(torch.from_numpy(real).to(cuda_device), torch.from_numpy(fake).to(cuda_device), k, rr) == ref


# ---- limits ---------------------------------------------------------------------------------------------------------
def _radii_rc(x_ptr, n, d, k, radii=None, work=None):
    lib = _lib.load()
    return lib.asyrp_fid_knn_radii(x_ptr, radii, work, n, d, k, ops._stream())


def test_radii_limits(cuda_device):
    lib = _lib.load()
    x = _random(40, 4, 1, cuda_device)
    radii = torch.empty(40, dtype=torch.float64, device=cuda_device)
    work = torch.empty(max(1, lib.asyrp_fid_knn_radii_workspace(40, 32)), dtype=torch.float64, device=cuda_device)
    xp, rp, wp = (C.c_void_p(t.data_ptr()) for t in (x, radii, work))
    ok = 0
    for n, d, k, good in [(40, 4, 1, True), (40, 4, 0, False), (40, 4, 32, True), (40, 4, 33, False),
                          (33, 4, 32, True), (32, 4, 32, False), (2, 4, 1, True), (1, 4, 1, False),
                          (40, 1, 5, True), (40, 0, 5, False), (40, -1, 5, False)]:
        rc = _radii_rc(xp, n, d, k, rp, wp)
        assert (rc == ok) == good, (n, d, k, rc, lib.asyrp_last_error())
        if not good:
            assert rc == -1 and lib.asyrp_last_error()
    torch.cuda.synchronize()
    assert _radii_rc(C.c_void_p(x.data_ptr() + 2), 40, 4, 1, rp, wp) == -1  # misaligned x
    assert b"aligned" in lib.asyrp_last_error()
    assert _radii_rc(xp, 40, 4, 1, C.c_void_p(radii.data_ptr() + 4), wp) == -1
    assert _radii_rc(xp, 40, 4, 1, rp, rp) == -1 and b"alias" in lib.asyrp_last_error()
    assert _radii_rc(xp, 40, 4, 1, None, wp) == -1
    assert lib.asyrp_fid_knn_radii_workspace(40, 33) == -1 and lib.asyrp_fid_knn_radii_workspace(0, 3) == -1
    assert lib.asyrp_fid_knn_radii_workspace(40, 32) >= 40 * 33
    with pytest.raises(_lib.AsyrpError, match="k=33 not in 1..32"):
        fid.knn_radii(x, 33)
    with pytest.raises(_lib.AsyrpError, match="needs at least k \\+ 1 = 11"):
        fid.knn_radii(x[:10].contiguous(), 10)


def test_counts_limits(cuda_device):
    lib = _lib.load()
    cap = 65535 * 64
    a = torch.zeros(cap, 1, device=cuda_device)
    a[-1] = 3.0
    ra = torch.full((cap,), 0.5, dtype=torch.float64, device=cuda_device)
    b = torch.full((1, 1), 3.0, device=cuda_device)
    rb = torch.full((1,), 0.5, dtype=torch.float64, device=cuda_device)
    outs = [torch.empty(s, dtype=torch.int32, device=cuda_device) for s in (1, cap, cap)]
    p = [C.c_void_p(t.data_ptr()) for t in (a, ra, b, rb, *outs)]

    def rc(n, m, d, o=None, ptrs=None):
        q = list(ptrs or p)
        o = o or (q[4], q[5], q[6])
        return lib.asyrp_fid_knn_counts(q[0], q[1], n, q[2], q[3], m, d, o[0], o[1], o[2], ops._stream())
    assert rc(cap, 1, 1) == 0  # the largest n: only the last row lies next to b
    assert outs[0].item() == 1 and outs[1].sum().item() == 1 and outs[2].sum().item() == 1 and outs[1][-1].item() == 1
    assert rc(cap + 1, 1, 1) == -1 and b"above" in lib.asyrp_last_error()
    for n, m, d in ((0, 1, 1), (1, 0, 1), (1, 1, 0)):
        assert rc(n, m, d) == -1
    assert rc(1, 1, 1) == 0
    assert rc(1, 1, 1, o=(p[4], p[4], p[6])) == -1 and b"distinct" in lib.asyrp_last_error()
    assert rc(1, 1, 1, o=(p[4], p[5], p[5])) == -1 and rc(1, 1, 1, o=(p[6], p[5], p[6])) == -1
    assert rc(1, 1, 1, o=(p[4], None, p[6])) == -1
    bad = list(p)
    bad[1] = C.c_void_p(ra.data_ptr() + 4)
    assert rc(1, 1, 1, ptrs=bad) == -1 and b"aligned" in lib.asyrp_last_error()
    torch.cuda.synchronize()


def test_rows_past_2_to_the_31_elements(cuda_device):
    """the row offsets are 64-bit: sets of more than 2^31 fp32 values"""
    n, d = (1 << 20) + 1, 2048  # n * d > 2^31
    a = torch.zeros(n, d, device=cuda_device)
    a[-1, -1] = 2.0
    a[-2, 0] = 1.0
    b = torch.zeros(2, d, device=cuda_device)
    b[1, -1] = 2.0
    ra = torch.full((n,), 0.5, dtype=torch.float64, device=cuda_device)
    rb = torch.full((2,), 0.5, dtype=torch.float64, device=cuda_device)
    b_in_a, a_in_b, a_cov = ops.fid_knn_counts(a, ra, b, rb)
    assert b_in_a.tolist() == [n - 2, 1]  # b_0 = 0 lies in every ball but those of the two nonzero rows
    assert a_in_b[-1].item() == 1 and a_in_b[-2].item() == 0 and a_in_b[0].item() == 1
    assert a_cov[-1].item() == 1 and a_cov[-2].item() == 0 and int(a_cov.sum()) == n - 1
    del a, a_in_b, a_cov, ra
    torch.cuda.empty_cache()
    n, d = 1100, (1 << 21)  # n * d > 2^31 in one set
    g = torch.Generator(device=cuda_device).manual_seed(3)
    x = torch.randint(-1, 2, (n, d), generator=g, device=cuda_device, dtype=torch.float32)
    x[7] = x[1000]
    got = ops.fid_knn_radii(x, 2)
    x64 = x.double()
    sq = (x64 * x64).sum(1)
    D = sq[:, None] + sq[None, :] - 2 * (x64 @ x64.T)  # exact: integers far below 2^53
    del x64
    assert torch.equal(got, _kth(D, 2))


# ---- main --run_test --fid --prdc -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["single", "interp", "sweep", "ref"])
def test_run_test_prdc(cuda_device, tmp_path, monkeypatch, mode):
    from asyrp_official_b200.diffusion_latent import Asyrp
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    sd = synthetic.inception_state_dict(seed=5)
    torch.save(sd, "pt_inception.pth")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)
    argv = BASE + ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]
    tuples, attrs = 1, None
    if mode == "interp":
        argv += ["--delta_interpolation", "--num_delta", "3", "--min_delta", "0.5", "--max_delta", "1.5"]
        tuples = 3
    elif mode == "sweep":
        argv = BASE + ["--attr_sweep", "smiling angry", "--manual_checkpoint_name", "attribute_0.pth"]
        tuples, attrs = 2, ["smiling", "angry"]
    argv += ["--fid", "--fid_weights", "pt_inception.pth"]
    if mode == "ref":
        _stats("ref.npz", sd, cuda_device)
        argv += ["--fid_ref", "ref.npz", "--kid_subsets", "3", "--kid_subset_size", "2"]
    prdc_argv = ["--prdc", "--prdc_k", "1"]
    captured = []
    finish = Asyrp.finish_fid

    def capturing(self, sets, *a, **kw):
        captured.append(sets)
        return finish(self, sets, *a, **kw)
    monkeypatch.setattr(Asyrp, "finish_fid", capturing)
    r, _ = _run(argv + ["--bs_train", "2"] + prdc_argv, cuda_device)
    folder = r.args.test_image_folder
    tsv, real_tsv = (os.path.join(folder, f"test_ngen4_{s}.tsv") for s in ("prdc", "prdc_real"))
    keep = ["test_ngen4_fid.tsv", "test_1_0_ngen4.png"] + (["test_ngen4_fid_real.tsv"] if mode == "ref" else [])
    with_prdc = [_bytes(os.path.join(folder, nm)) for nm in keep]
    tables = [_bytes(tsv)] + ([_bytes(real_tsv)] if mode == "ref" else [])
    table = _table(tsv)
    header = ["tuple", "hs_coeff", "n", "precision", "recall", "density", "coverage"] + (["attr"] if attrs else [])
    assert table[0] == header and len(table) == 1 + tuples
    assert [t[0] for t in table[1:]] == [str(k) for k in range(tuples)] and all(t[2] == "2" for t in table[1:])
    if attrs:
        assert [t[7] for t in table[1:]] == attrs
    vals = torch.tensor([[float(v) for v in t[3:7]] for t in table[1:]], dtype=torch.float64)
    assert torch.equal(vals, r.prdc["test"]) and torch.isfinite(vals).all()
    # recomputed from the gathered features
    got = captured[0].gather()
    origin = got[("test", "origin")][1].to(cuda_device).contiguous()
    ref_rows = [fid.prdc(origin, got[("test", k)][1].to(cuda_device).contiguous(), 1) for k in range(tuples)]
    assert torch.equal(torch.tensor(ref_rows, dtype=torch.float64), vals)
    if mode == "ref":
        rt = _table(real_tsv)
        assert rt[0] == ["tuple", "hs_coeff", "n", "n_ref", "precision", "recall", "density", "coverage"]
        assert [t[0] for t in rt[1:]] == ["origin"] + [str(k) for k in range(tuples)]
        assert all(t[2] == "2" and t[3] == "6" for t in rt[1:])
        rv = torch.tensor([[float(v) for v in t[4:8]] for t in rt[1:]], dtype=torch.float64)
        assert torch.equal(rv, r.prdc_real["test"]) and torch.isfinite(rv).all()
        real = torch.from_numpy(fid.load_stats("ref.npz")["features"]).to(cuda_device)
        sets = [origin] + [got[("test", k)][1].to(cuda_device).contiguous() for k in range(tuples)]
        assert torch.equal(torch.tensor([fid.prdc(real, f, 1) for f in sets], dtype=torch.float64), rv)
    # the same tables for another batch size
    os.remove(tsv)
    _run(argv + ["--bs_train", "1"] + prdc_argv, cuda_device)
    assert [_bytes(tsv)] + ([_bytes(real_tsv)] if mode == "ref" else []) == tables
    # without --prdc: the same other outputs, no prdc tables
    os.remove(tsv)
    if mode == "ref":
        os.remove(real_tsv)
    _run(argv + ["--bs_train", "2"], cuda_device)
    assert [_bytes(os.path.join(folder, nm)) for nm in keep] == with_prdc
    assert not os.path.exists(tsv) and not os.path.exists(real_tsv)
    if mode == "ref":  # a mu / sigma-only file: n_ref '-', nan
        _stats("ref_fid_only.npz", sd, cuda_device, features=False)
        r2, _ = _run(argv[:argv.index("--fid_ref")] + ["--fid_ref", "ref_fid_only.npz", "--bs_train", "2"] + prdc_argv,
                     cuda_device)
        t2 = _table(real_tsv)
        assert all(t[3] == "-" for t in t2[1:]) and len(t2) == 2 + tuples
        assert torch.isnan(r2.prdc_real["test"]).all() and torch.equal(r2.prdc["test"], vals)
