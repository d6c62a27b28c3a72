"""--region_compose on the GPU: the compose kernel bit for bit against its fp32 restatement (K attributes, B images,
the float4 and the scalar path, soft / hard / overlapping masks, K = 1 against the blend kernel), its refusals and a
launch past 2^31 elements, composed per-row trajectories on mini DDPM / ADM and DDPM CelebA 256² (K = 1 against
Schedule + blend, all-zero masks, identical rows, graph = eager, one graph for new masks, the launch count, the fp64
restatement), and `--run_test --region_compose` end to end."""
import csv
import ctypes
import os

import numpy as np
import pytest
import torch

import compose_oracle as oc
from asyrp_official_b200 import _lib, main as cli, ops, region, synthetic
from asyrp_official_b200.diffusion_latent import Asyrp
from asyrp_official_b200.schedule import RowSchedule, Schedule, make_sequences
from oracle import adm as oa, ddpm as od, region as orr, sampler as osmp
from test_attr_sweep_gpu import _module, _single
from test_diff_style_gpu import TOL_TRAJ
from test_edit_region_gpu import _labels

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# compose kernel
# ------------------------------------------------------------------------------------------------------------------
def _masks(kind, K, B, H, W, g):
    if kind == "soft":
        m = torch.rand(K, B, H, W, generator=g) / K
        m.view(-1)[::5] = 0.0
    elif kind == "hard":   # one attribute or none per pixel
        own = torch.randint(0, K + 1, (B, H, W), generator=g)
        m = torch.stack([(own == k + 1) for k in range(K)]).float()
    else:                  # overlapping: sums above 1
        m = torch.rand(K, B, H, W, generator=g)
        m[:, :, :H // 2] = 1.0
    return m


@pytest.mark.parametrize("H,W", [(32, 32), (256, 256), (31, 33)])
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
def test_compose_rows_exact(cuda_device, K, B, H, W):
    dev = cuda_device
    C = 3
    g = torch.Generator().manual_seed(K * 100 + B * 10 + H)
    x = torch.randn(K * B, C, H, W, generator=g)
    ref = torch.randn(B, C, H, W, generator=g)
    for kind in ("soft", "hard", "overlap"):
        m = _masks(kind, K, B, H, W, g)
        out = x.to(dev)
        ops.compose_rows(out, ref.to(dev), m.to(dev))
        out = out.cpu()
        want = torch.from_numpy(oc.compose_fp32(x.view(K, B, C, H, W).numpy(), ref.numpy(), m.numpy()))
        for k in range(K):
            assert torch.equal(out[k * B:(k + 1) * B], want), f"{kind}: attribute row {k}"
        if kind == "overlap" and K > 1:
            assert bool((m.sum(0) > 1).any())
        if K == 1:
            bl = x.to(dev)
            ops.blend_rows(bl, ref.to(dev), m[0].to(dev))
            assert torch.equal(out, bl.cpu()), f"{kind}: K = 1 differs from blend_rows"
    zero = x.to(dev)
    ops.compose_rows(zero, ref.to(dev), torch.zeros(K, B, H, W, device=dev))
    assert torch.equal(zero.cpu(), ref.repeat(K, 1, 1, 1)), "all-zero masks must give the origin"


def test_compose_rows_refusals(cuda_device):
    dev = cuda_device
    K, B, C, H, W = 2, 2, 3, 8, 8
    x = torch.randn(K * B, C, H, W, device=dev)
    ref = torch.randn(B, C, H, W, device=dev)
    masks = torch.rand(K, B, H, W, device=dev)
    before = x.clone()
    for bad in ((x, ref, masks[:1]), (x, ref[:1].contiguous(), masks), (x.half(), ref, masks), (x, ref.cpu(), masks),
                (x, ref, masks.cpu()), (x[:, :, :, :4], ref, masks), (x, ref, masks[:, :, :4].contiguous()),
                (x, ref, masks[0]), (x, ref.double(), masks)):
        with pytest.raises(_lib.AsyrpError):
            ops.compose_rows(*bad)
    nine = torch.randn(9 * B, C, H, W, device=dev)
    nine_before = nine.clone()
    with pytest.raises(_lib.AsyrpError, match="K=9 outside 1..8"):
        ops.compose_rows(nine, ref, torch.rand(9, B, H, W, device=dev))
    # float4 loads need 16-byte alignment: a tensor one element into its storage is refused
    buf = torch.randn(K * B * C * H * W + 1, device=dev)
    buf_before = buf.clone()
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        ops.compose_rows(buf[1:].view(K * B, C, H, W), ref, masks)
    mbuf = torch.rand(K * B * H * W + 1, device=dev)
    with pytest.raises(_lib.AsyrpError, match="aligned"):
        ops.compose_rows(x, ref, mbuf[1:].view(K, B, H, W))
    lib = _lib.load()
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    HW = H * W
    for args in ((0, B, C, HW), (9, B, C, HW), (-1, B, C, HW), (K, 0, C, HW), (K, B, 0, HW), (K, B, C, 0),
                 (K, B, C, -4), (K, -2, C, HW)):
        assert lib.asyrp_compose_rows(P(x), P(ref), P(masks), *args, s) == -1, args
    assert lib.asyrp_compose_rows(None, P(ref), P(masks), K, B, C, HW, s) == -1
    assert lib.asyrp_compose_rows(P(x), None, P(masks), K, B, C, HW, s) == -1
    assert lib.asyrp_compose_rows(P(x), P(ref), None, K, B, C, HW, s) == -1
    assert lib.asyrp_compose_rows(P(x), ctypes.c_void_p(ref.data_ptr() + 4), P(masks), K, B, C, HW, s) == -1
    torch.cuda.synchronize()
    assert torch.equal(x, before) and torch.equal(buf, buf_before) and torch.equal(nine, nine_before), \
        "a refused call launched"
    # odd HW takes one element per thread and only 4-byte alignment
    xo = torch.randn(K * B * C * 9 + 1, device=dev)
    ro, mo = torch.randn(B, C, 3, 3, device=dev), torch.rand(K, B, 3, 3, device=dev)
    tgt = xo[1:].view(K * B, C, 3, 3)
    want = oc.compose_fp32(tgt.view(K, B, C, 3, 3).cpu().numpy(), ro.cpu().numpy(), mo.cpu().numpy())
    ops.compose_rows(tgt, ro, mo)
    assert np.array_equal(tgt[:B].cpu().numpy(), want)


def test_compose_rows_past_2_31_elements(cuda_device):
    """K B C HW = 2.4e9 > 2^31 elements of x (16 GB in all): the rows past the 32-bit range against the restatement"""
    dev = cuda_device
    K, B, C, H, W = 3, 2, 3, 8192, 16384
    HW = H * W
    need = 4 * (K * B * C * HW + B * C * HW + K * B * HW)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need + (2 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory and 2 GiB to spare; {free / 2**30:.1f} GiB free")
    assert K * B * C * HW > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(K * B, C, H, W, device=dev, generator=g)
    ref = torch.randn(B, C, H, W, device=dev, generator=g)
    masks = torch.rand(K, B, H, W, device=dev, generator=g) * 0.6
    tail = slice(HW - 4096, HW)   # the last pixels of every plane: offsets up to K B C HW
    xt = x.view(K, B, C, HW)[..., tail].cpu().numpy()
    rt, mt = ref.view(B, C, HW)[..., tail].cpu().numpy(), masks.view(K, B, HW)[..., tail].cpu().numpy()
    head = slice(0, 4096)
    xh = x.view(K, B, C, HW)[..., head].cpu().numpy()
    rh, mh = ref.view(B, C, HW)[..., head].cpu().numpy(), masks.view(K, B, HW)[..., head].cpu().numpy()
    ops.compose_rows(x, ref, masks)
    out = x.view(K, B, C, HW)
    for sl, xs, rs, ms in ((tail, xt, rt, mt), (head, xh, rh, mh)):
        want = oc.compose_fp32(xs[..., None], rs[..., None], ms[..., None])[..., 0]
        for k in range(K):
            assert np.array_equal(out[k][..., sl].cpu().numpy(), want), k
    del x, ref, masks, out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# composed trajectories
# ------------------------------------------------------------------------------------------------------------------
def _fwd(family, sd, cfg=None):
    if family == "ddpm":
        return lambda *a, **k: od.ddpm_forward(sd, cfg or od.MINI_CFG, *a, **k)
    return lambda *a, **k: oa.adm_forward(sd, cfg or oa.MINI_HP, *a, **k)


def _row_schedule(betas, seq, seq_next, times, coeffs, b):
    K = len(times)
    return RowSchedule(betas, seq, seq_next, [times[k][0] for k in range(K) for _ in range(b)],
                       [times[k][1] for k in range(K) for _ in range(b)], [coeffs[k] for k in range(K) for _ in range(b)])


@pytest.mark.parametrize("family", ["ddpm", "adm"])
def test_composed_trajectories(cuda_device, family):
    dev = cuda_device
    m = _module(family, 2)
    synthetic.randomize_(m, 1234, "jittered")
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    singles = [_single(family, sd, k, dev) for k in range(2)]
    b, S, K = 2, 32, 2
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 6)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(b, 3, S, S, generator=g).to(dev)
    origin = Schedule(betas, seq, seq_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False)
    o = singles[0].engine.sample(x, origin, record_process=True)
    ref = singles[0].engine.last_records["x"].clone()
    coarse = torch.randint(0, 19, (b, 1, 8, 8), generator=g).float()   # blobs of classes, no scattered pixels
    lab = torch.nn.functional.interpolate(coarse, size=(512, 512), mode="nearest")[:, 0].to(torch.uint8)
    masks = torch.stack([torch.from_numpy(orr.feather(orr.select(lab.numpy(), cls, S), 1.0)).float()
                         for cls in ([3, 4, 7], [4, 5, 8])]).to(dev)
    assert bool((masks.sum(0) > 1).any()) and bool((masks.sum(0) == 0).any()), "overlaps and uncovered pixels"
    # K = 1: a per-row schedule with compose= equals the Schedule with blend=, bit for bit
    rs1 = _row_schedule(betas, seq, seq_next, [(500, 450)], [(1.0, 1.2)], b)
    sch1 = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=450, hs_coeff=(1.0, 1.2))
    assert rs1.n_stochastic == sch1.n_stochastic > 0
    z1 = torch.randn(rs1.n_stochastic, b, 3, S, S, generator=g).to(dev)
    a1 = singles[0].engine.sample(x, rs1, noise=z1, compose=(masks[:1].contiguous(), ref))
    assert torch.equal(a1, singles[0].engine.sample(x, sch1, noise=z1, blend=(masks[0], ref))), "K = 1 != blend"
    # K = 2 attributes, each its own block, t_edit and t_addnoise; the images' noise shared by their rows
    times, coeffs = [(700, 0), (400, 450)], [(1.0, 1.0, 0.0), (1.0, 0.0, 1.3)]
    rs = _row_schedule(betas, seq, seq_next, times, coeffs, b)
    z = torch.randn(rs.n_stochastic, b, 3, S, S, generator=g).to(dev)
    nz, xs = z.repeat(1, K, 1, 1, 1), x.repeat(K, 1, 1, 1)
    plain = eng.sample(xs, rs, noise=nz)
    launches = eng.last_launches
    out = eng.sample(xs, rs, noise=nz, compose=(masks, ref))
    assert eng.last_launches == launches + len(rs.steps)
    n_graphs = len(eng.graphs)
    for k in range(K):
        assert torch.equal(out[k * b:(k + 1) * b], out[:b]), f"attribute row {k}"
    assert not torch.equal(out[:b], o) and not torch.equal(out[:b], plain[:b]) and not torch.equal(out[b:], plain[b:])
    w0 = (masks.sum(0) == 0)[:, None].expand_as(o)
    assert torch.equal(out[:b][w0], o[w0]), "pixels outside every mask must equal the origin pass"
    zeros = torch.zeros_like(masks)
    assert torch.equal(eng.sample(xs, rs, noise=nz, compose=(zeros, ref)), o.repeat(K, 1, 1, 1)), "all-zero masks"
    flipped = masks.flip(0).contiguous()
    other = eng.sample(xs, rs, noise=nz, compose=(flipped, ref))
    assert len(eng.graphs) == n_graphs, "new masks must replay the same graph"
    assert not torch.equal(other, out)
    assert torch.equal(eng.sample(xs, rs, noise=nz, compose=(masks, ref), use_graph=False), out), "graph vs eager"
    rec_out = eng.sample(xs, rs, noise=nz, compose=(masks, ref), record_process=True)
    assert torch.equal(rec_out, out)
    rec = eng.last_records["x"]
    for k_step in range(len(rs.steps)):
        for k in range(1, K):
            assert torch.equal(rec[k_step][k * b:(k + 1) * b], rec[k_step][:b]), f"step {k_step}, attribute {k}"
    assert torch.equal(eng.sample(xs, rs, noise=nz), plain), "without compose the trajectory is unchanged"
    # refusals
    bad = [(masks[:1].contiguous(), ref), (masks, ref[1:]), (masks.cpu(), ref), (masks, ref.cpu()),
           (masks.double(), ref), (masks[:, :, :4].contiguous(), ref), (masks[:, :1].contiguous(), ref[:, :1]), masks]
    for c in bad:
        with pytest.raises(_lib.AsyrpError):
            eng.sample(xs, rs, noise=nz, compose=c)
    with pytest.raises(_lib.AsyrpError, match="per-row schedule"):
        singles[0].engine.sample(x, sch1, noise=z1, compose=(masks[:1].contiguous(), ref))
    # the fp64 restatement
    fwds = [_fwd(family, {k_: v.cpu() for k_, v in s_.state_dict().items()}) for s_ in singles]
    noises = {s_.t: z[zi].cpu() for zi, s_ in enumerate([s_ for s_ in rs.steps if s_.stochastic])}
    want = oc.run_composed_trajectory(fwds, x.cpu(), masks.cpu().numpy(), ref.cpu(), betas=betas, seq=seq,
                                      seq_next=seq_next, t_edit=[t[0] for t in times],
                                      t_addnoise=[t[1] for t in times], hs_coeff=[(1.0, 1.0), (1.0, 1.3)],
                                      learn_sigma=family == "adm", noises=noises)
    got = out[:b].cpu()
    for j in range(b):
        e, mx = (got[j].double() - want[j].double()).abs().max().item(), want[j].abs().max().item()
        print(f"\n{family} image {j}: max-abs {e:.3e} of {mx:.3e}")
        assert e <= TOL_TRAJ * max(1.0, mx), f"{family} image {j}: {e:.3e} of {mx:.3e}"


def test_celeba256_composed_trajectory(cuda_device):
    """DDPM CelebA 256², two seeded attributes: pixels outside both masks equal the origin pass, and the composite is
    within the trajectory tolerance of the fp64 restatement"""
    dev = cuda_device
    m = _module("ddpm", 2, od.CELEBA_CFG)
    synthetic.randomize_(m, 1234, "torch_default")
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    m = m.to(dev)
    eng = m.engine
    S, b, K = 256, 1, 2
    betas = osmp.make_betas()
    seq, seq_next = make_sequences(999, 5)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(b, 3, S, S, generator=g)
    origin = Schedule(betas, seq, seq_next, t_edit=10 ** 9, t_addnoise=0, hs_coeff=(1.0,), edit=False)
    times, coeffs = [(600, 0), (400, 0)], [(1.0, 1.0, 0.0), (1.0, 0.0, 0.8)]
    rs = _row_schedule(betas, seq, seq_next, times, coeffs, b)
    singles = [_single("ddpm", sd, k, dev, od.CELEBA_CFG) for k in range(K)]
    o = singles[0].engine.sample(x.to(dev), origin, record_process=True)
    ref = singles[0].engine.last_records["x"].clone()
    lab = _labels(b, 8).to(dev)
    masks = torch.stack([region.masks_from_labels(lab, cls, S, 2, 1.5) for cls in ([17], [1, 10])])
    out = eng.sample(x.to(dev).repeat(K, 1, 1, 1), rs, compose=(masks, ref))
    assert torch.equal(out[:b], out[b:])
    w0 = (masks.sum(0) == 0)[:, None].expand_as(o)
    assert 0 < w0.float().mean().item() < 1
    assert torch.equal(out[:b][w0], o[w0]), "pixels with w_0 = 1 must equal the origin pass"
    out, masks_h, ref_h = out[:b].cpu(), masks.cpu().numpy(), ref.cpu()
    fwds = [_fwd("ddpm", {k_: v.cpu() for k_, v in s_.state_dict().items()}, od.CELEBA_CFG) for s_ in singles]
    del m, eng, singles
    torch.cuda.empty_cache()
    want = oc.run_composed_trajectory(fwds, x, masks_h, ref_h, betas=betas, seq=seq, seq_next=seq_next,
                                      t_edit=[t[0] for t in times], t_addnoise=[t[1] for t in times],
                                      hs_coeff=[(1.0, 1.0), (1.0, 0.8)])
    e, mx = (out[0].double() - want[0].double()).abs().max().item(), want[0].abs().max().item()
    print(f"\nceleba256 composite: max-abs {e:.3e} of {mx:.3e}")
    assert e <= TOL_TRAJ * max(1.0, mx), f"{e:.3e} of {mx:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# end to end (DDPM CelebA-HQ 256², synthetic weights)
# ------------------------------------------------------------------------------------------------------------------
BASE = ["--run_test", "--config", "celeba.yml", "--exp", "./runs/rc", "--do_train", "0", "--do_test", "1",
        "--n_test_img", "2", "--n_train_img", "0", "--bs_train", "2", "--t_0", "999", "--n_inv_step", "4",
        "--n_train_step", "4", "--n_test_step", "4", "--load_random_noise", "--user_defined_t_edit", "500",
        "--user_defined_t_addnoise", "400", "--synthetic_weights", "--seed", "1234", "--train_delta_block",
        "--get_h_num", "1", "--save_x_origin", "--seg_weights", "79999_iter.pth", "--edit_region_dilate", "1"]


def _png(path):
    from PIL import Image
    return np.asarray(Image.open(path).convert("RGB"))


def _run(argv, dev):
    args, cfg = cli.parse_args_and_config(argv)
    r = Asyrp(args, cfg, device=dev)
    return r, r.run_test()[("test", 1)]


def test_run_test_region_compose_end_to_end(cuda_device, tmp_path, monkeypatch):
    """two synthetic DeltaBlocks and the seeded face parser.  Which classes that parser finds is arbitrary, so the
    regions are taken from the labels of the origin pass: the second and third most frequent classes, which leaves the
    most frequent one outside every mask"""
    from test_seg_consistency_gpu import _delta_block_ckpt
    from asyrp_official_b200 import face_parsing
    monkeypatch.chdir(tmp_path)
    os.makedirs("checkpoint")
    _delta_block_ckpt("checkpoint/smiling_0.pth", 11)
    _delta_block_ckpt("checkpoint/grey_hair_0.pth", 12)
    torch.save(synthetic.face_parsing_state_dict(seed=5), "79999_iter.pth")
    compose = BASE + ["--manual_checkpoint_name", "attribute_0.pth", "--seg_consistency", "--content_preservation"]
    _, rows = _run(compose + ["--region_compose", "smiling=mouth grey_hair=hair"], cuda_device)
    origin = rows[0]
    parser = face_parsing.FaceParser(torch.load("79999_iter.pth", weights_only=True), device=cuda_device)
    counts = torch.bincount(parser.labels(origin).flatten().long(), minlength=19)
    order = [int(c) for c in counts.argsort(descending=True) if counts[c] > 0]
    print(f"\nlabels of the origin pass: {[(region.CLASSES[c], int(counts[c])) for c in order]}")
    assert len(order) >= 3, "the seeded parser finds fewer than three classes"
    a, b = region.CLASSES[order[1]], region.CLASSES[order[2]]
    compose += ["--region_compose", f"smiling={a} grey_hair={b}"]
    r, rows = _run(compose + ["--max_rows_per_replay", "16"], cuda_device)
    assert r.compose_times == {"smiling": (500, 400), "grey_hair": (500, 400)}
    folder = r.args.test_image_folder
    files = os.listdir(folder)
    for name in ("test_1_0_ngen4.png", "test_1_0_ngen4_region_compose.png", "test_1_0_ngen4_seg_consistency.tsv",
                 "test_1_0_ngen4_content_preservation.tsv"):
        assert name in files, name
    for name in ("seg_consistency", "content_preservation"):
        with open(os.path.join(folder, f"test_1_0_ngen4_{name}.tsv")) as f:
            table = list(csv.reader(f, delimiter="\t"))
        assert table[0][-1] == "attr" and table[0][:3] == ["image", "tuple", "hs_coeff"], name
        body = [t for t in table[1:] if t[1] != "origin"]
        assert [(t[0], t[1], t[-1]) for t in body] == [("0", "0", "smiling+grey_hair"), ("1", "0", "smiling+grey_hair")]
        assert body[0][2] == "1,1,1", body[0][2]   # (hs_coeff_origin_h, s, s)
    assert len(rows) == 2  # the origin row and the composite
    assert torch.equal(rows[0], origin)
    comp = rows[1]
    masks = region.compose_masks(parser, origin, [[order[1]], [order[2]]], 1, 0.0).cpu()
    print(f"masks of {a} and {b} cover {masks[0].mean().item():.3f} and {masks[1].mean().item():.3f} of the image")
    assert masks[0].mean() > 0 and masks[1].mean() > 0
    S = 256
    grid_mask = _png(os.path.join(folder, "test_1_0_ngen4_region_compose.png"))
    for k in range(2):
        for i in range(2):
            cell = grid_mask[1 + k * (S + 1):1 + k * (S + 1) + S, 1 + i * (S + 1):1 + i * (S + 1) + S, 0]
            assert np.array_equal(cell, (masks[k, i].numpy() * 255).astype(np.uint8)), (k, i)
    grid = _png(os.path.join(folder, "test_1_0_ngen4.png"))
    cell = lambda row, col: grid[1 + row * (S + 1):1 + row * (S + 1) + S, 1 + col * (S + 1):1 + col * (S + 1) + S]  # noqa: E731
    outside = masks.sum(0) == 0
    assert 0 < outside.float().mean().item() < 1
    for i in range(2):
        assert np.array_equal(cell(1, i)[outside[i].numpy()], cell(0, i)[outside[i].numpy()]), f"image {i} PNG"
        keep = outside[i][None].expand(3, S, S)
        assert torch.equal(comp[i][keep], origin[i][keep]), f"image {i}"
    assert not torch.equal(comp, origin)
    # the output does not depend on the chunking
    for max_rows in ("2", "4"):
        _, again = _run(compose + ["--max_rows_per_replay", max_rows], cuda_device)
        assert all(torch.equal(x, y) for x, y in zip(again, rows)), f"--max_rows_per_replay {max_rows}"
    # K = 1 is --edit_region, bit for bit, in the tensors and in the PNGs
    _, one = _run(BASE + ["--manual_checkpoint_name", "attribute_0.pth", "--region_compose", f"smiling={a}"],
                  cuda_device)
    png_one = _png(os.path.join(folder, "test_1_0_ngen4.png"))
    _, er = _run(BASE + ["--manual_checkpoint_name", "smiling_0.pth", "--edit_attr", "smiling", "--edit_region", a],
                 cuda_device)
    png_er = _png(os.path.join(folder, "test_1_0_ngen4.png"))
    assert len(one) == len(er) == 2
    assert not torch.equal(one[1], one[0]), "the region must change the image"
    assert torch.equal(one[0], er[0]) and torch.equal(one[1], er[1]), f"--region_compose smiling={a} != --edit_region"
    assert np.array_equal(png_one, png_er)
