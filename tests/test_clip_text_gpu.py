"""CLIP text tower on the GPU: each kernel against the fp64 oracle, the whole encoder within the DESIGN.md §2 bound,
determinism and batch independence, and t_edit chosen from CLIP's cosine through `main --run_test`."""
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

from asyrp_official_b200 import clip_text, main as cli, modules, ops, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp, _read_tsv
from oracle import clip_text as oct
from oracle import ddpm as od

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEAT_TOL = 3e-3  # relative max-abs of the features (DESIGN.md §2: TF32 emulation up to 1.1e-3)
COS_TOL = 6e-4   # absolute error of the cosine (emulation up to 2.1e-4)
PROMPTS = ["face", "smiling face", "person", "person with blond hair", "photo", "painting by gogh",
           "a photo of a red sports car on the street", "Person with curly hair and a very long beard, in a garden"]
DIC = {"smiling": (["face"], ["smiling face"]), "car": (["face"], ["a photo of a red sports car on the street"])}


def _rel(out, ref):
    ref = ref.double()
    return ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()


@pytest.fixture(scope="module")
def vocab(tmp_path_factory):
    gz = str(tmp_path_factory.mktemp("clip") / "bpe.txt.gz")
    n = synthetic.write_clip_vocab(gz, synthetic.clip_bpe_merges(PROMPTS))
    return gz, n


def _g(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def test_embed_layernorm_pool_and_cosine(cuda_device):
    g = _g(1)
    P, T, w, V = 3, 77, 512, 700
    tok, pos = torch.randn(V, w, generator=g), torch.randn(T, w, generator=g)
    ids = torch.randint(0, V - 1, (P, T), generator=g, dtype=torch.int32)
    ids[0, 5] = ids[0, 9] = V - 1  # the first of two maxima is the pooled row
    ids[1, 76] = V - 1
    ids[2, 0] = V - 1
    dev = lambda t: t.to(cuda_device)  # noqa: E731
    x = torch.empty(P, T, w, device=cuda_device)
    ops.clip_embed(dev(ids), dev(tok), dev(pos), x)
    assert torch.equal(x.cpu(), (tok.double()[ids.long()] + pos.double()).float())
    x = x * 3 + 1.5
    gam, bet = 1 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)
    y = torch.empty_like(x)
    ops.clip_layernorm(x, dev(gam), dev(bet), y)
    ref = oct.layer_norm(x.cpu().double(), gam.double(), bet.double())
    assert _rel(y, ref) <= 2e-6
    ops.clip_layernorm(x, dev(gam), dev(bet), x)  # in place
    assert torch.equal(x, y)
    pooled = torch.empty(P, w, device=cuda_device)
    ops.clip_pool(y, dev(ids), dev(gam), dev(bet), pooled)
    rows = y.cpu().double()[torch.arange(P), torch.tensor([5, 76, 0])]
    assert _rel(pooled, oct.layer_norm(rows, gam.double(), bet.double())) <= 2e-6
    proj = torch.randn(w, 512, generator=g) / w ** 0.5
    feats = torch.empty(P, 512, device=cuda_device)
    ops.clip_linear(pooled, dev(proj.t().contiguous()), None, feats)
    assert _rel(feats, pooled.cpu().double() @ proj.double()) <= 2e-3
    a, b = torch.randn(6, 512, generator=g), torch.randn(6, 512, generator=g)
    a[5] *= 1e-9  # below eps: the norm is clamped as CosineSimilarity clamps it
    b[2] = a[2] * 0.5 + 1e-3 * b[2]
    cos = torch.empty(6, device=cuda_device)
    ops.clip_cosine(dev(a), dev(b), cos)
    ref = torch.nn.CosineSimilarity(dim=1, eps=1e-6)(a.double(), b.double())
    assert (cos.cpu().double() - ref).abs().max().item() <= 1e-6


@pytest.mark.parametrize("epi", [ops.CLIP_EPI_BIAS, ops.CLIP_EPI_QUICK_GELU, ops.CLIP_EPI_RESIDUAL])
def test_linear_epilogues(cuda_device, epi):
    """the LPIPS conv's TF32 GEMM as a linear layer: |err| <= 2^-10 (|x| @ |W|^T) + fp32 rounding of the epilogue"""
    g = _g(10 + epi)
    M, K, N = 3 * 77, (512, 512, 2048)[epi - 1], (1536, 2048, 512)[epi - 1]
    x, W, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    out = res.clone().to(cuda_device) if epi == ops.CLIP_EPI_RESIDUAL else torch.empty(M, N, device=cuda_device)
    ops.clip_linear(x.to(cuda_device), W.to(cuda_device), bias.to(cuda_device), out, epi,
                    residual=out if epi == ops.CLIP_EPI_RESIDUAL else None)
    z = x.double() @ W.double().t() + bias.double()
    ref = {ops.CLIP_EPI_BIAS: z, ops.CLIP_EPI_QUICK_GELU: oct.quick_gelu(z), ops.CLIP_EPI_RESIDUAL: res.double() + z}[epi]
    bound = 2.0 ** -10 * (x.double().abs() @ W.double().abs().t()) * (1.1 if epi == ops.CLIP_EPI_QUICK_GELU else 1)
    err = (out.cpu().double() - ref).abs()
    assert (err <= bound + 1e-6 * (1 + ref.abs())).all(), (err / bound).max().item()
    if epi == ops.CLIP_EPI_BIAS:  # no bias: the identity epilogue alone
        o2 = torch.empty(M, N, device=cuda_device)
        ops.clip_linear(x.to(cuda_device), W.to(cuda_device), None, o2)
        ref2 = z - bias.double()
        assert ((o2.cpu().double() - ref2).abs() <= bound + 1e-6 * (1 + ref2.abs())).all()


@pytest.mark.parametrize("heads,T", [pytest.param(8, 77, id="8"), pytest.param(12, 77, id="12"),
                                     pytest.param(8, 1, id="8-T1"), pytest.param(8, 33, id="8-T33"),
                                     pytest.param(12, 128, id="12-T128")])  # T <= 128: the most the kernel admits
def test_causal_attention(cuda_device, heads, T):
    g = _g(heads + T)
    P, w = 3, 64 * heads
    qkv = torch.randn(P, T, 3 * w, generator=g) * 2
    out = torch.empty(P, T, w, device=cuda_device)
    ops.clip_attention(qkv.to(cuda_device), out, heads)
    q, k, v = (t.double().reshape(P, T, heads, 64).transpose(1, 2) for t in qkv.split(w, dim=-1))
    s = q @ k.transpose(-1, -2) / 8 + torch.full((T, T), float("-inf"), dtype=torch.float64).triu(1)
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(P, T, w)
    assert _rel(out, ref) <= 1e-5


@pytest.mark.parametrize("width,heads", [(512, 8), (768, 12)])
def test_encoder_within_the_design_bound(cuda_device, vocab, width, heads):
    gz, n = vocab
    sd = synthetic.clip_text_state_dict(seed=1, width=width, layers=12, vocab=n, embed_dim=512)
    m = clip_text.CLIPText(sd, gz, device=cuda_device)
    assert m.dims == dict(width=width, heads=heads, layers=12, context=77, vocab=n, embed_dim=512)
    ids = m.tokenize(PROMPTS)
    feats = m.encode_text(ids)
    ref = oct.encode_text(sd, ids)
    e = _rel(feats, ref)
    assert e <= FEAT_TOL, e
    half = len(PROMPTS) // 2
    cos = m.text_cosine(PROMPTS[:half], PROMPTS[half:])
    ce = (cos.double() - oct.cosine(ref[:half], ref[half:])).abs().max().item()
    assert ce <= COS_TOL, ce
    # determinism and batch independence
    assert torch.equal(m.encode_text(ids), feats)
    for i in (0, 3, 7):
        assert torch.equal(m.encode_text(ids[i:i + 1]), feats[i:i + 1])
    assert torch.equal(m.encode_text(ids[2:5]), feats[2:5])
    assert torch.equal(m.text_cosine(PROMPTS[1], PROMPTS[5]), m.text_cosine([PROMPTS[1]], [PROMPTS[5]]))


# ---------------------------------------------------------------------------------------------------------------------
CFG = od.MINI_CFG
SEED, WIDTH, LAYERS = 7, 128, 2


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


def _scratch(tmp_path, monkeypatch):
    """scratch directory: mini config, SRC_TRG_TXT_DIC at utils/text_dic.py, the golden CelebA x0_t table under the
    config's stem, synthetic CLIP weights and vocabulary; returns (argv prefix, oracle cosine of each attribute)"""
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    os.makedirs("utils")
    with open("utils/text_dic.py", "w") as f:
        f.write(f"SRC_TRG_TXT_DIC = {DIC!r}\n")
    shutil.copy(os.path.join(ROOT, "tests", "golden", "lpips", "celeba_LPIPS_distance_x0_t.tsv"),
                "utils/mini_LPIPS_distance_x0_t.tsv")
    texts = [t for src, trg in DIC.values() for t in src + trg]
    n = synthetic.write_clip_vocab("bpe.txt.gz", synthetic.clip_bpe_merges(texts))
    sd = synthetic.clip_text_state_dict(seed=SEED, width=WIDTH, layers=LAYERS, vocab=n, embed_dim=128)
    torch.save(sd, "clip.pt")
    tok = oct.SimpleTokenizer("bpe.txt.gz")
    cos = {k: oct.cosine(oct.encode_text(sd, tok.tokenize(s)), oct.encode_text(sd, tok.tokenize(t))).item()
           for k, (s, t) in DIC.items()}
    cfg = _write_cfg(os.path.join(str(tmp_path), "mini.yml"))
    argv = ["--run_test", "--config", cfg, "--exp", "./runs/attr", "--do_train", "0", "--do_test", "1",
            "--n_test_img", "1", "--n_train_img", "0", "--bs_train", "1", "--t_0", "999", "--n_inv_step", "4",
            "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_addnoise", "0",
            "--synthetic_weights", "--seed", "1234", "--train_delta_block"]
    return argv, cos


def _oracle_t_edit(cos, th=0.33):
    """t_edit of the table for cosine cos, asserting the table's margin around th*cos is wider than th*COS_TOL"""
    table = _read_tsv("utils/mini_LPIPS_distance_x0_t.tsv")
    thr = th * cos
    i = next(i for i, (_, v) in enumerate(table) if v >= thr)
    below = max((v for _, v in table[:i]), default=-np.inf)
    assert table[i][1] - thr > th * COS_TOL and thr - below > th * COS_TOL, (table[i], below, thr)
    return table[i][0]


def _run(argv, dev):
    args, config = cli.parse_args_and_config(argv)
    r = Asyrp(args, config, device=dev)
    return r, r.run_test()


def test_run_test_takes_t_edit_from_clip(cuda_device, tmp_path, monkeypatch):
    argv, cos = _scratch(tmp_path, monkeypatch)
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    argv = argv + ["--get_h_num", "1", "--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling"]
    r, res = _run(argv + ["--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz"], cuda_device)
    t_edit = _oracle_t_edit(cos["smiling"])
    assert r.t_edit == t_edit and r.t_addnoise == 0
    r2, res2 = _run(argv + ["--user_defined_t_edit", str(t_edit)], cuda_device)
    (row,), (row2,) = res[("test", 0)], res2[("test", 0)]
    assert torch.equal(row, row2)


def test_multiple_attr_takes_the_largest_cosine(cuda_device, tmp_path, monkeypatch):
    argv, cos = _scratch(tmp_path, monkeypatch)
    assert abs(cos["smiling"] - cos["car"]) > 10 * COS_TOL, cos
    for i, a in enumerate(DIC):
        _delta_block_ckpt(f"checkpoint/{a}_0.pth", 11 + i)
    argv = argv + ["--get_h_num", "2", "--manual_checkpoint_name", "attribute_0.pth", "--edit_attr", "attribute",
                   "--multiple_attr", " ".join(DIC), "--clip_weights", "clip.pt", "--clip_vocab", "bpe.txt.gz"]
    r, res = _run(argv, cuda_device)
    best = max(DIC, key=lambda k: cos[k])
    assert (r.src_txts, r.trg_txts) == (DIC[best][0], DIC[best][1])
    assert r.t_edit == _oracle_t_edit(cos[best])
    assert len(res[("test", 0)]) == 1
