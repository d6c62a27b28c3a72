"""--dino_structure on the GPU: the pack against fp64 (and exact at S = R), the GELU epilogue and the eps LayerNorm
against fp64 with the CLIP entries unchanged, the flash attention against fp64 within its TF32 bound and batch
independent bit for bit, the self-similarity distance (exact 0 on equal rows, fp64 bound, strided views, shared
indices, batching, refusals, a launch past 2^31 key elements), ViT-S/8 and B/8 against the fp64 oracle, and
`--run_test` / `--diff_style` end to end.  DESIGN.md (--dino_structure) states the bounds."""
import csv
import ctypes
import math
import os

import numpy as np
import pytest
import torch
import yaml

from asyrp_official_b200 import _lib, dino, main as cli, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from oracle import dino as od

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _images(n, S, seed):
    g = _g(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, S), torch.linspace(0, 1, S), indexing="ij")
    base = torch.stack([torch.sin(5 * xx + 3 * c * yy) * torch.cos(4 * yy + c) for c in range(3)])
    return (0.7 * base + 0.3 * torch.randn(n, 3, S, S, generator=g)).clamp(-1, 1)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [32, 224, 256])
@pytest.mark.parametrize("P", [8, 16])
def test_pack_against_fp64(cuda_device, S, P):
    G = 224 // P
    x = _images(2, S, S + P)
    out = torch.full((2 * G * G, ops.clip_image_kpad(P)), float("nan"), device=cuda_device)
    ops.dino_pack(x.to(cuda_device), out, G, P)
    ref = od.pack(x.double().numpy(), G, P)
    got = out.double().cpu().numpy()
    assert np.all(got[:, 3 * P * P:] == 0)
    err = np.abs(got[:, :3 * P * P] - ref).max()
    # fp32 arithmetic, plus the tap positions scale (i + 0.5), computed in fp32 as PyTorch does, off by up to (S + 1) u:
    # each of the 2 max(1, S/R) + 2 taps per axis moves by that over its support, on values up to 1 / std
    taps = 2 * max(1.0, S / 224) + 2
    assert err <= 64 * U * (1 + np.abs(ref).max()) + 4 * taps * (S + 1) * U / 0.224, err
    if S == 224:  # the identity resize: exactly the fp32 normalisation of the input
        mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
        std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
        y = (((x + 1) / 2) - mean) / std
        y = y.reshape(2, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(2 * G * G, 3 * P * P)
        assert torch.equal(out[:, :3 * P * P].cpu(), y)


def test_gelu_epilogue_against_fp64(cuda_device):
    M, K, N = 300, 384, 1536
    x = torch.randn(M, K, generator=_g(1))
    W = torch.randn(N, K, generator=_g(2)) * K ** -0.5
    b = torch.randn(N, generator=_g(3))
    out = torch.empty(M, N, device=cuda_device)
    ops.clip_linear(x.to(cuda_device), W.to(cuda_device), b.to(cuda_device), out, ops.CLIP_EPI_GELU)
    z = x.double() @ W.double().t() + b.double()
    ref = 0.5 * z * (1 + torch.special.erf(z / math.sqrt(2)))
    # TF32 operands: |dz| <= 2^-10 |x| @ |W|^T; GELU's slope is at most 1.13; plus the epilogue's fp32 roundings
    bound = 1.13 * 2.0 ** -10 * (x.double().abs() @ W.double().abs().t()) + 16 * U * (ref.abs() + z.abs())
    assert ((out.double().cpu() - ref).abs() <= bound).all()


def test_layernorm_eps_against_fp64_and_clip_unchanged(cuda_device):
    B, T, D = 3, 785, 384
    x = (torch.randn(B, T, D, generator=_g(4)) * 3 + 1).to(cuda_device)
    gam, bet = torch.randn(D, generator=_g(5)).to(cuda_device), torch.randn(D, generator=_g(6)).to(cuda_device)
    out = torch.empty(B, T, D, device=cuda_device)
    ops.dino_layernorm(x, gam, bet, out, eps=1e-6)
    xd = x.double()
    ref = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-6) * \
        gam.double() + bet.double()
    assert ((out.double() - ref).abs() <= 64 * U * (ref.abs() + bet.double().abs() + gam.double().abs() * 8)).all()
    cls = torch.empty(B, D, device=cuda_device)  # strided rows: the CLS token of each image
    ops.dino_layernorm(x.view(B, T * D)[:, :D], gam, bet, cls, eps=1e-6)
    assert torch.equal(cls, out[:, 0])
    # the CLIP entries keep eps 1e-5 and their bits: equal to this kernel at eps 1e-5
    a, c = torch.empty_like(out), torch.empty_like(out)
    ops.clip_layernorm(x, gam, bet, a)
    ops.dino_layernorm(x, gam, bet, c, eps=1e-5)
    assert torch.equal(a, c)
    r = torch.empty(B, D, device=cuda_device)
    ops.clip_layernorm_rows(x, gam, bet, r)
    assert torch.equal(r, c[:, 0])


# ---------------------------------------------------------------------------------------------------------------------
def _attention64(qkv, heads):
    B, T, D3 = qkv.shape
    D = D3 // 3
    q, k, v = (qkv[..., i * D:(i + 1) * D].double().reshape(B, T, heads, 64).transpose(1, 2) for i in range(3))
    s = q @ k.transpose(-1, -2) / 8
    o = torch.softmax(s, -1) @ v
    # TF32 bound (DESIGN.md): scores off by <= 2^-10 |q| . |k| / 8 (both operands rounded), probabilities rounded to
    # TF32 (2^-11) and V rounded (2^-11): |do| <= (2 max_j dS_ij + 2^-10 + 2^-9) max|v| per query row and head
    ds = (q.abs() @ k.abs().transpose(-1, -2) / 8).amax(-1) * 2.0 ** -10
    vmax = v.abs().amax((-1, -2))
    bound = (2 * torch.expm1(2 * ds) + 2.0 ** -9 + 2.0 ** -10) * vmax[..., None]
    return o.transpose(1, 2).reshape(B, T, D), bound.transpose(1, 2).repeat_interleave(64, -1).reshape(B, T, D)


@pytest.mark.parametrize("T", [2, 17, 64, 65, 197, 785, 1025])
@pytest.mark.parametrize("heads", [6, 12])
def test_attention_against_fp64(cuda_device, T, heads):
    B, D = 2, 64 * heads
    qkv = (torch.randn(B, T, 3 * D, generator=_g(T + heads)) * 1.5).to(cuda_device)
    out = torch.full((B, T, D), float("nan"), device=cuda_device)
    ops.dino_attention(qkv, out, heads)
    ref, bound = _attention64(qkv, heads)
    assert ((out.double() - ref).abs() <= bound).all(), ((out.double() - ref).abs() / bound).max().item()
    one = torch.empty(1, T, D, device=cuda_device)  # every image the same bits alone
    for b in range(B):
        ops.dino_attention(qkv[b:b + 1].contiguous(), one, heads)
        assert torch.equal(one[0], out[b])


def test_attention_refusals(cuda_device):
    heads, D = 6, 384
    ok = torch.randn(1, 1025, 3 * D, device=cuda_device)
    ops.dino_attention(ok, torch.empty(1, 1025, D, device=cuda_device), heads)
    with pytest.raises(_lib.AsyrpError, match="T <= 1025"):
        ops.dino_attention(torch.randn(1, 1026, 3 * D, device=cuda_device),
                           torch.empty(1, 1026, D, device=cuda_device), heads)
    flat = torch.randn(65 * 3 * D + 4, device=cuda_device)
    out = torch.empty(1, 65, D, device=cuda_device)
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        ops.dino_attention(flat[1:1 + 65 * 3 * D].view(1, 65, 3 * D), out, heads)
    ops.dino_attention(flat[4:4 + 65 * 3 * D].view(1, 65, 3 * D), out, heads)
    with pytest.raises(_lib.AsyrpError, match="heads"):
        ops.dino_attention(flat[:65 * 3 * D].view(1, 65, 3 * D), out, 5)
    lib = _lib.load()
    assert lib.asyrp_dino_attention(None, ctypes.c_void_p(out.data_ptr()), 1, 65, heads, None) != 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
def _distance_bound(d64, D):
    e = (2 * D + 8) * U  # per-entry error of a normalised fp32 dot product of D terms
    return 4 * e * math.sqrt(d64) + 4 * e * e


def _d64(keys, ia, ib, T):
    k = keys.double().cpu().numpy()
    return [od.structure_distance(k[a:a + T], k[b:b + T]) for a, b in zip(ia, ib)]


def _dist(keys, ia, ib, T):
    dev = keys.device
    out = torch.empty(len(ia), dtype=torch.float64, device=dev)
    ops.dino_selfsim_distance(keys, torch.tensor(ia, device=dev), torch.tensor(ib, device=dev), T, out)
    return out.cpu()


@pytest.mark.parametrize("T", [2, 65, 197, 785, 1025])
def test_distance_against_fp64(cuda_device, T):
    D = 384
    base = torch.randn(T, D, generator=_g(T))
    keys = torch.cat([base, base + 0.3 * torch.randn(T, D, generator=_g(T + 1)),
                      torch.randn(T, D, generator=_g(T + 2)), base]).to(cuda_device)
    ia, ib = [0, 0, T, 0], [T, 2 * T, 2 * T, 3 * T]
    got = _dist(keys, ia, ib, T)
    want = _d64(keys, ia, ib, T)
    for g, w in zip(got.tolist(), want):
        assert abs(g - w) <= _distance_bound(w, D), (g, w)
    assert got[3] == 0.0  # equal rows in other buffer rows: exactly 0
    assert _dist(keys, [T], [T], T).item() == 0.0
    for p in range(4):  # each pair the same bits alone
        assert _dist(keys, ia[p:p + 1], ib[p:p + 1], T).item() == got[p].item()


def test_distance_strided_views_and_shared_origin(cuda_device):
    B, T, D = 3, 197, 384
    qkv = torch.randn(B * T, 3 * D, generator=_g(7)).to(cuda_device)
    view = qkv[:, D:2 * D]  # the keys in place, row stride 3D
    dense = view.contiguous()
    ia, ib = [0, 0, 0, T], [T, 2 * T, 0, 2 * T]  # origin 0 shared by three pairs
    got = _dist(view, ia, ib, T)
    assert torch.equal(got, _dist(dense, ia, ib, T)) and got[2] == 0.0
    for g, w in zip(got.tolist(), _d64(dense, ia, ib, T)):
        assert abs(g - w) <= _distance_bound(w, D)


def test_distance_refusals(cuda_device):
    lib = _lib.load()
    T, D = 65, 64
    keys = torch.randn(2 * 1026, D, device=cuda_device)
    ia = torch.zeros(3, dtype=torch.int64, device=cuda_device)
    ib = torch.full((3,), 65, dtype=torch.int64, device=cuda_device)
    part = torch.empty(3 * 153 + 1, dtype=torch.float64, device=cuda_device)
    out = torch.empty(4, dtype=torch.float64, device=cuda_device)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    off = lambda t, b: ctypes.c_void_p(t.data_ptr() + b)  # noqa: E731

    def call(k=None, ld=D, a=None, b=None, n=1, t=T, d=D, eps=1e-8, pt=None, o=None):
        return lib.asyrp_dino_selfsim_distance(k or P(keys), ld, a or P(ia), b or P(ib), n, t, d, eps, pt or P(part),
                                               o or P(out), None)
    assert call() == 0
    assert call(t=1025) == 0 and call(t=1026) != 0
    assert call(n=0) != 0 and call(d=0) != 0 and call(ld=D - 1) != 0 and call(eps=0.0) != 0
    assert call(k=off(keys, 4)) == 0 and call(k=off(keys, 2)) != 0
    assert call(a=off(ia, 8)) == 0 and call(a=off(ia, 4)) != 0 and call(b=off(ib, 4)) != 0
    assert call(pt=off(part, 8)) == 0 and call(pt=off(part, 4)) != 0 and call(o=off(out, 4)) != 0
    for name in ("k", "a", "b", "pt", "o"):
        args = {name: ctypes.c_void_p(0)}
        assert lib.asyrp_dino_selfsim_distance(
            args.get("k", P(keys)), D, args.get("a", P(ia)), args.get("b", P(ib)), 1, T, D, 1e-8,
            args.get("pt", P(part)), args.get("o", P(out)), None) != 0
    with pytest.raises(_lib.AsyrpError, match="must lie"):
        ops.dino_selfsim_distance(keys[:100], ia[:1], ib[:1], T, out[:1])
    torch.cuda.synchronize()


def test_distance_past_2_31_key_elements(cuda_device):
    T, D = 65, 64
    far = (1 << 31) // D  # row far * D is element 2^31
    keys = torch.empty((far + T) * D, device=cuda_device).view(far + T, D)
    a = torch.randn(T, D, generator=_g(9))
    b = a + 0.5 * torch.randn(T, D, generator=_g(10))
    keys[:T] = a.to(cuda_device)
    keys[T:2 * T] = b.to(cuda_device)
    keys[far:] = a.to(cuda_device)
    got = _dist(keys, [0, T], [far, far], T)
    assert got[0] == 0.0
    w = od.structure_distance(b.double().numpy(), a.double().numpy())
    assert abs(got[1].item() - w) <= _distance_bound(w, D)
    del keys
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [384, 768])
def test_network_against_oracle(cuda_device, dim):
    """ViT-S/8 and B/8 (random weights, 224^2 from 256^2 input): keys, CLS rows, D and cls_cos against fp64"""
    sd = synthetic.dino_state_dict(seed=2, dim=dim, depth=12, patch=8, grid=28)
    net = dino.DINO(sd, device=cuda_device)
    x = _images(2, 256, 3)
    k, c = net.features(x)
    k64, tok64 = od.forward({n: v.numpy() for n, v in sd.items()}, x.double().numpy())
    kr = np.abs(k.double().cpu().numpy() - k64).max() / np.abs(k64).max()
    cr = np.abs(c.double().cpu().numpy() - tok64[:, 0]).max() / np.abs(tok64[:, 0]).max()
    # 12 blocks of TF32 GEMMs and attention: the relative error stays within 2^-7 (DESIGN.md)
    assert kr <= 2.0 ** -7 and cr <= 2.0 ** -7, (kr, cr)
    s = net.scores(x[:1], x[1:])
    d64 = od.structure_distance(k64[0], k64[1])
    assert abs(s[0, 0, 0].item() - d64) <= 2.0 ** -5 * d64 + 1e-6, (s[0, 0, 0].item(), d64)
    assert abs(s[0, 0, 1].item() - od.cls_cos(tok64[0, 0], tok64[1, 0])) <= 2.0 ** -7
    # batch and chunk independence
    k3, c3 = net.features(torch.cat([x, x[:1]]))
    for b in range(2):
        kb, cb = net.features(x[b:b + 1])
        assert torch.equal(kb[0], k3[b]) and torch.equal(cb[0], c3[b]) and torch.equal(kb[0], k[b])
    e = torch.cat([x, x.flip(0), x])
    whole = net.scores(x, e)
    net.max_rows = 1
    assert torch.equal(net.scores(x, e), whole)
    assert whole[0, 0, 0].item() == 0.0 and whole[2, 1, 0].item() == 0.0


# ---------------------------------------------------------------------------------------------------------------------
def _table(path):
    with open(path) as f:
        return list(csv.reader(f, delimiter="\t"))


def _small_dino(path):
    torch.save(synthetic.dino_state_dict(seed=4, dim=128, depth=2, patch=8, grid=8), path)


BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/dino", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--user_defined_t_edit", "500", "--user_defined_t_addnoise", "0",
        "--synthetic_weights", "--seed", "1234", "--train_delta_block", "--get_h_num", "1"]
DINO = ["--dino_structure", "--dino_weights", "dino.pth"]


def _setup(tmp_path, monkeypatch):
    from test_preservation_gpu import _delta_block_ckpt
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/angry_0.pth", 12)
    _small_dino("dino.pth")


def _run(argv, dev):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config, device=dev)
    return r, r.run_test()


def _files(folder):
    out = {}
    for root, _, names in os.walk(folder):
        for n in names:
            with open(os.path.join(root, n), "rb") as f:
                out[os.path.relpath(os.path.join(root, n), folder)] = f.read()
    return out


@pytest.mark.parametrize("mode", ["single", "sweep"])
def test_run_test_scores_every_edit(cuda_device, tmp_path, monkeypatch, mode):
    _setup(tmp_path, monkeypatch)
    argv = BASE + ["--load_random_noise", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling",
                   "--save_x_origin"]
    tuples = 1
    if mode == "sweep":
        argv = BASE + ["--load_random_noise", "--attr_sweep", "smiling angry", "--manual_checkpoint_name",
                       "attribute_0.pth", "--save_x_origin"]
        tuples = 2
    r, res = _run(argv + DINO, cuda_device)
    folder = r.args.test_image_folder
    with_flag = _files(folder)
    table = _table(os.path.join(folder, "test_1_0_ngen4_dino.tsv"))
    header = ["image", "tuple", "hs_coeff", "structure", "cls_cos"] + (["attr"] if mode == "sweep" else [])
    assert table[0] == header and len(table) == 1 + 2 * tuples
    vals = torch.tensor([[float(v) for v in t[3:5]] for t in table[1:]], dtype=torch.float64)
    assert torch.equal(vals.view(tuples, 2, 2), r.dino["test_1_0"])
    origin, edited = res[("test", 1)][0], res[("test", 1)][1:]
    net = dino.DINO(synthetic.dino_state_dict(seed=4, dim=128, depth=2, patch=8, grid=8), device=cuda_device)
    assert torch.equal(net.scores(origin, torch.cat(edited)).view(-1, 2), vals)
    # every other output byte-identical without the flag
    import shutil
    shutil.rmtree("runs")
    r2, res2 = _run(argv, cuda_device)
    plain = _files(r2.args.test_image_folder)
    assert plain == {k: v for k, v in with_flag.items() if not k.endswith("_dino.tsv")}
    assert all(torch.equal(a, b) for a, b in zip(res[("test", 1)], res2[("test", 1)]))


def test_run_test_exact_inversion_origin_rows(cuda_device, tmp_path, monkeypatch):
    from test_exact_inversion_gpu import _faces
    _setup(tmp_path, monkeypatch)
    _faces(2, 256)
    argv = BASE + ["--custom_test_dataset_dir", "faces", "--custom_train_dataset_dir", "faces", "--exact_inversion",
                   "--save_x_origin", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"] + DINO
    r, res = _run(argv, cuda_device)
    table = _table(os.path.join(r.args.test_image_folder, "test_1_0_ngen4_dino.tsv"))
    assert [t[:3] for t in table[1:3]] == [["0", "origin", "-"], ["1", "origin", "-"]] and len(table) == 5
    assert [float(t[3]) for t in table[1:3]] == [0.0, 0.0]  # the origin pass is the input image bit for bit
    assert torch.equal(r.dino_origin["test_1_0"][:, 0], torch.zeros(2, dtype=torch.float64))


def test_diff_style_table(cuda_device, tmp_path, monkeypatch):
    from oracle import ddpm as oddpm
    from test_diff_style_host import _write_pngs
    monkeypatch.chdir(tmp_path)
    _small_dino("dino.pth")
    cfg = oddpm.MINI_CFG
    _write_pngs("content", ["c0.png", "c1.jpg"], [(40, 32), (32, 48)])  # test_main_diff_style_end_to_end's images
    _write_pngs("style", ["s0.png", "s1.png"], [(32, 32), (64, 40)])
    conf = {"data": dict(dataset="CelebA_HQ", category="CelebA_HQ", image_size=cfg["image_size"], channels=3,
                         rescaled=True, num_workers=0),
            "model": dict(type="simple", in_channels=3, out_ch=3, ch=cfg["ch"], ch_mult=list(cfg["ch_mult"]),
                          num_res_blocks=cfg["num_res_blocks"], attn_resolutions=list(cfg["attn_resolutions"]),
                          dropout=0.0, var_type="fixedsmall", ema_rate=0.999, ema=True, resamp_with_conv=True),
            "diffusion": dict(beta_schedule="linear", beta_start=0.0001, beta_end=0.02, num_diffusion_timesteps=1000),
            "sampling": dict(batch_size=4, last_only=True)}
    with open("mini.yml", "w") as f:
        yaml.safe_dump(conf, f)
    argv = ["--diff_style", "--config", os.path.join(str(tmp_path), "mini.yml"), "--content_dir", "content",
            "--style_dir", "style", "--user_defined_t_edit", "500", "--hs_coeff_list", "0.9 0.6",
            "--t_noise", "300", "--dt_lambda", "0.9985", "--n_inv_step", "8", "--bs_train", "3",
            "--synthetic_weights", "--seed", "1234"]

    def run(save_dir, *extra):
        args, config = cli.parse_args_and_config(argv + ["--save_dir", save_dir] + list(extra))
        r = Asyrp(args, config, device=cuda_device)
        return r, r.run_diff_style()

    r16, res = run("o16", "--max_rows_per_replay", "16", *DINO)
    r2, _ = run("o2", "--max_rows_per_replay", "2", *DINO)
    _, res_plain = run("plain", "--max_rows_per_replay", "16")
    t16 = open(os.path.join("o16", "diff_style_dino.tsv")).read()
    assert t16 == open(os.path.join("o2", "diff_style_dino.tsv")).read()
    table = _table(os.path.join("o16", "diff_style_dino.tsv"))
    assert table[0] == ["content", "style", "hs_coeff", "structure_content", "structure_style", "cls_cos_content",
                        "cls_cos_style"] and len(table) == 1 + 8
    assert [(os.path.basename(t[0]), os.path.basename(t[1]), t[2]) for t in table[1:3]] == \
        [("c0.png", "s0.png", "0.6"), ("c0.png", "s0.png", "0.9")]
    plain = _files("plain")
    assert plain == {k: v for k, v in _files("o16").items() if k != "diff_style_dino.tsv"}
    for k in res:
        assert torch.isfinite(res[k]).all() and torch.equal(res[k], res_plain[k])
    # a row against the scorer on the run's own images
    net = dino.DINO(synthetic.dino_state_dict(seed=4, dim=128, depth=2, patch=8, grid=8), device=cuda_device)
    (c, s_), out = next(iter(res.items()))
    from asyrp_official_b200.diffusion_latent import diff_style_image
    sc = net.scores(diff_style_image(c, cfg["image_size"]), out)[:, 0]
    row = [t for t in table[1:] if t[0] == c and t[1] == s_ and t[2] == "0.9"][0]
    assert float(row[3]) == sc[0, 0].item() and float(row[5]) == sc[0, 1].item()
