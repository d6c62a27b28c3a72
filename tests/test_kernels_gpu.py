"""Kernel-level parity: every C-ABI op against a plain fp64/fp32 torch CPU evaluation of the same formula on
the same fp16-rounded operands.  Tolerances are fp16-output rounding (2^-11 relative) plus fp32 accumulation
order effects; stated per test."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from asyrp_official_b200 import ops
    return ops


def _rand(shape, gen, scale=1.0):
    return (torch.randn(shape, generator=gen) * scale)


def _nhwc_half(x_nchw, dev):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(torch.float16).to(dev)


def _from_nhwc(t):
    return t.float().cpu().permute(0, 3, 1, 2)


def _h(x):
    """fp16 rounding applied on the CPU reference side (the operands the kernel actually sees)"""
    return x.to(torch.float16).double()


def _check(out, ref, tol_rel, what):
    err = (out.double() - ref).abs().max().item()
    mag = ref.abs().max().item()
    assert err <= tol_rel * mag + 1e-6, f"{what}: max-abs err {err:.3e} vs max|ref| {mag:.3e}"


def _stats_ref(ref_nchw):
    n, c, h, w = ref_nchw.shape
    r = ref_nchw.reshape(n, c // 2, 2, h * w)
    return torch.stack([r.sum(dim=(2, 3)), (r * r).sum(dim=(2, 3))], dim=-1)  # [N][C/2][2]


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 32, 32, 64, 64), (2, 32, 32, 128, 128), (1, 16, 48, 128, 256),
                                            (3, 8, 8, 128, 128), (5, 4, 4, 64, 128), (2, 64, 64, 192, 192)])
def test_conv3x3_bias_residual_stats(cuda_device, N, H, W, Cin, Cout):
    ops = _ops()
    g = torch.Generator().manual_seed(1)
    x = _rand((N, Cin, H, W), g)
    w = _rand((Cout, Cin, 3, 3), g, 1.0 / math.sqrt(9 * Cin))
    eb = _rand((N, Cout), g)
    res = _rand((N, Cout, H, W), g)
    ref = F.conv2d(_h(x), _h(w), padding=1) + eb.double()[:, :, None, None]
    ref = 0.75 * ref + 1.5 * _h(res)
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=cuda_device)
    stats = ops.new_stats(N, H, W, Cout, cuda_device, True)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3)], ops.pack_conv_weight(w).to(cuda_device), out=out,
                    ebias=eb.to(cuda_device), ebias_stride=Cout, residual=_nhwc_half(res, cuda_device),
                    res_scale=1.5, acc_scale=0.75, stats=stats)
    op.launch()
    op.launch()  # idempotent relaunch (persistent barriers re-initialised per launch)
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 1.5e-3, "conv3x3")
    st = stats.sum(dim=1).cpu().double()
    sref = _stats_ref(ref)
    assert (st - sref).abs().max().item() <= 2e-3 * sref.abs().max().item() + 1e-3


def test_conv1x1_concat_two_sources(cuda_device):
    ops = _ops()
    g = torch.Generator().manual_seed(2)
    N, H, W, C1, C2, Cout = 2, 16, 16, 128, 64, 128
    x1, x2 = _rand((N, C1, H, W), g), _rand((N, C2, H, W), g)
    w = _rand((Cout, C1 + C2, 1, 1), g, 1.0 / math.sqrt(C1 + C2))
    b = _rand((Cout,), g)
    ref = F.conv2d(torch.cat([_h(x1), _h(x2)], 1), _h(w)) + b.double()[None, :, None, None]
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x1, cuda_device), ops.MODE_1x1), (_nhwc_half(x2, cuda_device), ops.MODE_1x1)],
                    ops.pack_conv_weight(w).to(cuda_device), out=out, ebias=b.to(cuda_device))
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 1.5e-3, "conv1x1 concat")


def test_conv3x3_with_fused_1x1_shortcut(cuda_device):
    """conv2(a2) + nin_shortcut(cat(x1, x2)) accumulated in one accumulator tile (ddpm/diffusion.py:159-170)."""
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    N, H, W, C1, C2, Cout = 2, 32, 32, 128, 64, 128
    a2, x1, x2 = _rand((N, Cout, H, W), g), _rand((N, C1, H, W), g), _rand((N, C2, H, W), g)
    w3 = _rand((Cout, Cout, 3, 3), g, 1.0 / math.sqrt(9 * Cout))
    w1 = _rand((Cout, C1 + C2, 1, 1), g, 1.0 / math.sqrt(C1 + C2))
    ref = F.conv2d(_h(a2), _h(w3), padding=1) + F.conv2d(torch.cat([_h(x1), _h(x2)], 1), _h(w1))
    wp = torch.cat([ops.pack_conv_weight(w3), ops.pack_conv_weight(w1[:, :C1]), ops.pack_conv_weight(w1[:, C1:])], 1)
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(a2, cuda_device), ops.MODE_3x3), (_nhwc_half(x1, cuda_device), ops.MODE_1x1),
                     (_nhwc_half(x2, cuda_device), ops.MODE_1x1)], wp.contiguous().to(cuda_device), out=out)
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 1.5e-3, "conv3x3+shortcut")


def test_conv3x3_stride2_asymmetric_pad(cuda_device):
    """Downsample: pad (0,1,0,1) then 3x3 stride 2 (ddpm/diffusion.py:103-108)."""
    ops = _ops()
    g = torch.Generator().manual_seed(4)
    N, Hi, Wi, C = 2, 32, 32, 128
    x = _rand((N, C, Hi, Wi), g)
    w = _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    b = _rand((C,), g)
    ref = F.conv2d(F.pad(_h(x), (0, 1, 0, 1)), _h(w), stride=2) + b.double()[None, :, None, None]
    out = torch.empty(N, Hi // 2, Wi // 2, C, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3_S2)], ops.pack_conv_weight(w).to(cuda_device),
                    out=out, ebias=b.to(cuda_device))
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 1.5e-3, "conv3x3 s2")


def test_conv_planar_fp32_output(cuda_device):
    """conv_out: 3 (or 6) real output channels written as fp32 NCHW (ddpm/diffusion.py:424-428)."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    N, H, W, C, Co = 2, 32, 32, 128, 6
    x = _rand((N, C, H, W), g)
    w = torch.zeros(64, C, 3, 3)
    w[:Co] = _rand((Co, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    b = torch.zeros(64)
    b[:Co] = _rand((Co,), g)
    ref = F.conv2d(_h(x), _h(w[:Co]), padding=1) + b[:Co].double()[None, :, None, None]
    outp = torch.zeros(N, Co, H, W, dtype=torch.float32, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3)], ops.pack_conv_weight(w).to(cuda_device),
                    out_shape=(N, H, W, 64), ebias=b.to(cuda_device), out_planar=outp)
    op.launch()
    torch.cuda.synchronize()
    _check(outp.cpu(), ref, 2e-5, "planar fp32")


def test_batched_gemm_mode(cuda_device):
    """H=1 'image' rows x per-sample weight matrix: logits = q k^T as used by a tensor-core attention."""
    ops = _ops()
    g = torch.Generator().manual_seed(6)
    N, T, D = 3, 256, 128
    q, k = _rand((N, T, D), g), _rand((N, T, D), g)
    ref = torch.einsum("ntd,nsd->nts", _h(q), _h(k))
    out = torch.empty(N, 1, T, T, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp([(q.to(torch.float16).to(cuda_device).reshape(N, 1, T, D), ops.MODE_1x1)],
                    k.to(torch.float16).to(cuda_device).contiguous(), out=out, weight_batched=True)
    op.launch()
    torch.cuda.synchronize()
    _check(out.float().cpu().reshape(N, T, T), ref, 1.5e-3, "batched gemm")


@pytest.mark.parametrize("Ca,Cb,resample,act", [(128, 0, 0, 1), (128, 64, 0, 1), (64, 128, 0, 0), (128, 0, 1, 1),
                                                (128, 0, 2, 1), (64, 0, 2, 0)])
def test_groupnorm_finalize_and_apply(cuda_device, Ca, Cb, resample, act):
    """GroupNorm(32) over a (possibly concatenated) tensor from conv-epilogue partial sums, then
    SiLU / avg-pool / nearest-up.  The statistics come from a real conv epilogue (1x1 identity-free conv)."""
    ops = _ops()
    g = torch.Generator().manual_seed(7)
    N, H, W = 2, 16, 16
    C = Ca + Cb
    srcs, stats, refs = [], [], []
    for Cs in [c for c in (Ca, Cb) if c]:
        xin = _rand((N, 64, H, W), g)
        w = _rand((Cs, 64, 1, 1), g, 0.2)
        b = _rand((Cs,), g)
        out = torch.empty(N, H, W, Cs, dtype=torch.float16, device=cuda_device)
        st = ops.new_stats(N, H, W, Cs, cuda_device, False)
        ops.ConvOp([(_nhwc_half(xin, cuda_device), ops.MODE_1x1)], ops.pack_conv_weight(w).to(cuda_device), out=out,
                   ebias=b.to(cuda_device), stats=st).launch()
        srcs.append(out)
        stats.append(st)
        refs.append(F.conv2d(_h(xin), _h(w)) + b.double()[None, :, None, None])
    torch.cuda.synchronize()
    xcat = torch.cat([_from_nhwc(s).double() for s in srcs], 1)  # what apply actually reads (fp16-rounded)
    gamma, beta = _rand((C,), g) + 1.0, _rand((C,), g)
    ss = _rand((N, 2 * C), g, 0.3)
    eps = 1e-6
    # statistics are taken on the fp32 pre-rounding values
    xstat = torch.cat(refs, 1)
    xg = xstat.reshape(N, 32, -1)
    mean, var = xg.mean(-1), xg.var(-1, unbiased=False)
    cpg = C // 32
    mean_c = mean.repeat_interleave(cpg, 1)[:, :, None, None]
    rstd_c = (1.0 / torch.sqrt(var + eps)).repeat_interleave(cpg, 1)[:, :, None, None]
    y = (xcat - mean_c) * rstd_c * gamma.double()[None, :, None, None] + beta.double()[None, :, None, None]
    y = y * (1 + ss[:, :C].double()[:, :, None, None]) + ss[:, C:].double()[:, :, None, None]
    if act:
        y = y * torch.sigmoid(y)
    if resample == 1:
        y = F.avg_pool2d(y, 2)
    elif resample == 2:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    affine = torch.empty(N, C, 2, dtype=torch.float32, device=cuda_device)
    ops.gn_finalize(stats[0], Ca, stats[1] if Cb else None, Cb, gamma.to(cuda_device), beta.to(cuda_device), eps, N,
                    H * W, affine, scale_shift=ss.to(cuda_device), ss_stride=2 * C)
    Ho, Wo = y.shape[2:]
    out = torch.empty(N, Ho, Wo, C, dtype=torch.float16, device=cuda_device)
    ops.apply(srcs[0], srcs[1] if Cb else None, affine, out, act, resample)
    torch.cuda.synchronize()
    _check(_from_nhwc(out), y, 2e-3, "gn+apply")


@pytest.mark.parametrize("N,T,heads,D", [(2, 256, 1, 512), (2, 64, 1, 256), (1, 1024, 8, 64), (3, 200, 2, 128)])
def test_attention(cuda_device, N, T, heads, D):
    ops = _ops()
    g = torch.Generator().manual_seed(8)
    C = heads * D
    qkv = _rand((N, T, 3 * C), g)
    qh = _h(qkv)
    q, k, v = [qh[:, :, i * C:(i + 1) * C].reshape(N, T, heads, D).permute(0, 2, 1, 3) for i in range(3)]
    scale = D ** -0.5
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
    ref = (p @ v).permute(0, 2, 1, 3).reshape(N, T, C)
    out = torch.empty(N, T, C, dtype=torch.float16, device=cuda_device)
    ops.attention(qkv.to(torch.float16).to(cuda_device), out, heads, D, scale)
    torch.cuda.synchronize()
    _check(out.float().cpu(), ref, 1.5e-3, "attention")


def test_pack_embedding_linear_ddim(cuda_device):
    ops = _ops()
    g = torch.Generator().manual_seed(9)
    dev = cuda_device
    # pack_input
    x = _rand((2, 3, 16, 16), g)
    packed = torch.empty(2, 16, 16, 64, dtype=torch.float16, device=dev)
    ops.pack_input(x.to(dev), packed)
    ref = torch.zeros(2, 16, 16, 64)
    ref[..., :3] = x.permute(0, 2, 3, 1).to(torch.float16).float()
    assert torch.equal(packed.float().cpu(), ref)
    # timestep embeddings, both conventions
    t = torch.tensor([999.0, 512.0, 25.0, 0.0])
    for variant, dim in ((0, 128), (1, 256)):
        half = dim // 2
        if variant == 0:
            fr = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
            e = t[:, None] * fr[None]
            ref = torch.cat([torch.sin(e), torch.cos(e)], 1)
        else:
            fr = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half)
            e = t[:, None] * fr[None]
            ref = torch.cat([torch.cos(e), torch.sin(e)], 1)
        out = torch.empty(4, dim, dtype=torch.float32, device=dev)
        ops.timestep_embedding(t.to(dev), out, variant)
        assert (out.cpu() - ref).abs().max().item() < 2e-4  # sin/cos of arguments up to ~1e3 in fp32
    # linear with SiLU on the input / output
    inp, w, b = _rand((4, 96), g), _rand((40, 96), g, 0.1), _rand((40,), g)
    out = torch.empty(4, 40, dtype=torch.float32, device=dev)
    ops.linear(inp.to(dev), w.to(dev), b.to(dev), out, act_in=True)
    ref = F.silu(inp.double()) @ w.double().t() + b.double()
    assert (out.cpu().double() - ref).abs().max().item() < 1e-5
    ops.linear(inp.to(dev), w.to(dev), b.to(dev), out, act_out=True)
    ref = F.silu(inp.double() @ w.double().t() + b.double())
    assert (out.cpu().double() - ref).abs().max().item() < 1e-5
    # DDIM update, eta = 0 and eta > 0 (utils/diffusion_utils.py:84-97), fp32 op order as the reference
    xt, et, em, z = (_rand((2, 3, 8, 8), g) for _ in range(4))
    et6 = torch.cat([et, _rand((2, 3, 8, 8), g)], 1)
    em6 = torch.cat([em, _rand((2, 3, 8, 8), g)], 1)
    at, an = torch.tensor(0.3, dtype=torch.float32), torch.tensor(0.6, dtype=torch.float32)
    x0 = (xt - em * (1 - at).sqrt()) / at.sqrt()
    nxt0 = an.sqrt() * x0 + (1 - an).sqrt() * et
    c1 = 1.0 * ((1 - at / an) * (1 - an) / (1 - at)).sqrt()
    c2 = ((1 - an) - c1 ** 2).sqrt()
    nxt1 = an.sqrt() * x0 + c2 * et + c1 * z
    o_next, o_x0 = torch.empty(2, 3, 8, 8, device=dev), torch.empty(2, 3, 8, 8, device=dev)
    ops.ddim_update(xt.to(dev), et6.to(dev), em6.to(dev), None, o_next, o_x0, at.item(), an.item(), 0.0,
                    (1 - an).sqrt().item())
    assert torch.equal(o_x0.cpu(), x0) and torch.equal(o_next.cpu(), nxt0)
    ops.ddim_update(xt.to(dev), et6.to(dev), em6.to(dev), z.to(dev), o_next, o_x0, at.item(), an.item(), c1.item(),
                    c2.item())
    assert (o_next.cpu() - nxt1).abs().max().item() <= 1e-6


@pytest.mark.parametrize("N,H,W,C1,C2,Cout,mode,act", [(2, 32, 32, 128, 0, 128, "3x3", 1), (2, 32, 32, 128, 64, 128, "3x3", 1),
                                                       (3, 8, 8, 128, 64, 128, "3x3", 1), (2, 16, 16, 128, 0, 384, "1x1", 0),
                                                       (1, 64, 64, 64, 0, 256, "3x3", 1), (2, 16, 24, 64, 64, 64, "3x3", 1),
                                                       (2, 8, 8, 256, 256, 256, "3x3", 1), (2, 8, 8, 256, 0, 256, "3x3", 1),
                                                       (2, 16, 16, 256, 128, 128, "3x3", 1), (2, 8, 8, 256, 128, 256, "3x3", 1)])
def test_conv_with_fused_groupnorm_silu_operand(cuda_device, N, H, W, C1, C2, Cout, mode, act):
    """conv(act(GroupNorm(cat(x1, x2)))) with the affine + SiLU applied to the operand tile in shared memory
    (ResnetBlock norm1-swish-conv1 over the decoder's concatenated input, ddpm/diffusion.py:153-155,549).
    The zero padding must be applied after the activation."""
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    C = C1 + C2
    xs = [_rand((N, c, H, W), g) * 1.5 + 0.3 for c in (C1, C2) if c]
    aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()  # (a, b) pairs
    k = 3 if mode == "3x3" else 1
    w = _rand((Cout, C, k, k), g, 1.0 / math.sqrt(k * k * C))
    b = _rand((Cout,), g)
    xcat = torch.cat([_h(x) for x in xs], 1)
    y = xcat * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
    if act:
        y = y * torch.sigmoid(y)
    y = _h(y.float())  # the transformed operand is rounded to fp16 before the MMA
    ref = F.conv2d(y, _h(w), padding=k // 2) + b.double()[None, :, None, None]
    m = ops.MODE_3x3 if mode == "3x3" else ops.MODE_1x1
    affd = aff.to(cuda_device)
    segs, off, wparts = [], 0, []
    for x in xs:
        segs.append((_nhwc_half(x, cuda_device), m, affd, off, act))
        wparts.append(ops.pack_conv_weight(w[:, off:off + x.shape[1]]))
        off += x.shape[1]
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp(segs, torch.cat(wparts, 1).contiguous().to(cuda_device), out=out, ebias=b.to(cuda_device))
    op.launch()
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 2.5e-3, f"fused gn+silu conv {mode}")


@pytest.mark.parametrize("H,W,C,C1,C2", [(32, 32, 128, 128, 64), (8, 8, 128, 128, 64), (8, 8, 256, 256, 256),
                                         (16, 16, 256, 256, 128)])
def test_fused_operand_plus_raw_shortcut_segments(cuda_device, H, W, C, C1, C2):
    """conv2(silu(gn(h))) + nin_shortcut(cat(x1, x2)): one transformed 3x3 segment and two raw 1x1 segments in the
    same accumulator (ResnetBlock of the decoder, ddpm/diffusion.py:159-170)"""
    ops = _ops()
    g = torch.Generator().manual_seed(12)
    N = 2
    h, x1, x2 = _rand((N, C, H, W), g), _rand((N, C1, H, W), g), _rand((N, C2, H, W), g)
    aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()
    w3 = _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    w1 = _rand((C, C1 + C2, 1, 1), g, 1.0 / math.sqrt(C1 + C2))
    y = _h(h) * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
    y = _h((y * torch.sigmoid(y)).float())
    ref = F.conv2d(y, _h(w3), padding=1) + F.conv2d(torch.cat([_h(x1), _h(x2)], 1), _h(w1))
    wp = torch.cat([ops.pack_conv_weight(w3), ops.pack_conv_weight(w1[:, :C1]), ops.pack_conv_weight(w1[:, C1:])], 1)
    out = torch.empty(N, H, W, C, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(h, cuda_device), ops.MODE_3x3, aff.to(cuda_device), 0, 1),
                     (_nhwc_half(x1, cuda_device), ops.MODE_1x1), (_nhwc_half(x2, cuda_device), ops.MODE_1x1)],
                    wp.contiguous().to(cuda_device), out=out)
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 2.5e-3, "fused + raw shortcut")


def test_fused_operand_planar_output(cuda_device):
    """norm_out - swish - conv_out (ddpm/diffusion.py:575-578): fused operand, 64-wide padded N tile, fp32 planar store"""
    ops = _ops()
    g = torch.Generator().manual_seed(13)
    N, H, W, C, Co = 2, 32, 32, 64, 3
    x = _rand((N, C, H, W), g)
    aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()
    w = torch.zeros(64, C, 3, 3)
    w[:Co] = _rand((Co, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    y = _h(x) * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
    y = _h((y * torch.sigmoid(y)).float())
    ref = F.conv2d(y, _h(w[:Co]), padding=1)
    outp = torch.zeros(N, Co, H, W, dtype=torch.float32, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3, aff.to(cuda_device), 0, 1)],
                    ops.pack_conv_weight(w).to(cuda_device), out_shape=(N, H, W, 64), out_planar=outp)
    op.launch()
    torch.cuda.synchronize()
    _check(outp.cpu(), ref, 2.5e-3, "fused planar")


def test_tensor_core_attention_pieces(cuda_device):
    """q k^T and P v as batched GEMMs on channel slices of one qkv tensor (pixel pitch 3C), v -> v^T, row softmax:
    the single-head attention path of AttnBlock (ddpm/diffusion.py:200-221) on tensor cores"""
    ops = _ops()
    g = torch.Generator().manual_seed(21)
    N, T, Cc = 3, 256, 128
    qkv = _rand((N, T, 3 * Cc), g).to(torch.float16)
    qd = qkv.to(cuda_device)
    q, k, v = (qkv[..., i * Cc:(i + 1) * Cc].double() for i in range(3))
    S = torch.empty(N, 1, T, T, dtype=torch.float32, device=cuda_device)  # fp32 logits
    ops.ConvOp([(qd.view(N, 1, T, 3 * Cc)[..., :Cc], ops.MODE_1x1)], qd[:, :, Cc:2 * Cc], out=S, weight_batched=True).launch()
    s_ref = torch.einsum("ntc,nsc->nts", q, k)
    torch.cuda.synchronize()
    _check(S.cpu().reshape(N, T, T), s_ref, 2e-5, "q k^T on slices")
    P = torch.empty(N, 1, T, T, dtype=torch.float16, device=cuda_device)
    scale = Cc ** -0.5
    ops.softmax_rows(S, P, scale)
    p_ref = torch.softmax(S.double().cpu().reshape(N, T, T) * scale, dim=-1)
    torch.cuda.synchronize()
    assert (P.double().cpu().reshape(N, T, T) - p_ref).abs().max().item() < 6e-4
    vT = torch.empty(N, Cc, T, dtype=torch.float16, device=cuda_device)
    ops.transpose_tc(qd[:, :, 2 * Cc:], vT)
    torch.cuda.synchronize()
    assert torch.equal(vT.cpu(), qkv[..., 2 * Cc:].transpose(1, 2).contiguous())
    O = torch.empty(N, 1, T, Cc, dtype=torch.float16, device=cuda_device)
    ops.ConvOp([(P, ops.MODE_1x1)], vT, out=O, weight_batched=True).launch()
    torch.cuda.synchronize()
    o_ref = torch.einsum("nts,nsc->ntc", P.double().cpu().reshape(N, T, T), v)
    _check(O.float().cpu().reshape(N, T, Cc), o_ref, 1.5e-3, "P v")


def test_multi_head_attention_gemms(cuda_device):
    """QKVAttentionLegacy (improved_ddpm/unet.py:379-396) on tensor cores: S_h = q_h k_h^T and O_h = P_h v_h batched
    over (sample, head), heads being 64-channel slices of one qkv tensor; O_h lands in its channel slice"""
    ops = _ops()
    g = torch.Generator().manual_seed(22)
    N, T, heads, d = 2, 256, 4, 64
    Cc = heads * d
    qkv = _rand((N, T, 3 * Cc), g).to(torch.float16)
    qd = qkv.to(cuda_device)
    q, k, v = (qkv[..., i * Cc:(i + 1) * Cc].double().reshape(N, T, heads, d).permute(0, 2, 1, 3) for i in range(3))
    S = torch.empty(N * heads, 1, T, T, dtype=torch.float32, device=cuda_device)
    ops.ConvOp([(qd.view(N, 1, T, 3 * Cc)[..., :d], ops.MODE_1x1)], qd[:, :, Cc:Cc + d], out=S, weight_batched=True,
               a_heads=heads, b_heads=heads).launch()
    torch.cuda.synchronize()
    _check(S.cpu().reshape(N, heads, T, T), q @ k.transpose(-1, -2), 2e-5, "multi-head q k^T")
    P = torch.empty(N * heads, 1, T, T, dtype=torch.float16, device=cuda_device)
    ops.softmax_rows(S, P, d ** -0.5)
    vT = torch.empty(N, Cc, T, dtype=torch.float16, device=cuda_device)
    ops.transpose_tc(qd[:, :, 2 * Cc:], vT)
    O = torch.empty(N, 1, T, Cc, dtype=torch.float16, device=cuda_device)
    ops.ConvOp([(P, ops.MODE_1x1)], vT.view(N * heads, d, T), out=O, weight_batched=True, out_heads=heads).launch()
    torch.cuda.synchronize()
    o_ref = (P.double().cpu().reshape(N, heads, T, T) @ v).permute(0, 2, 1, 3).reshape(N, T, Cc)
    _check(O.float().cpu().reshape(N, T, Cc), o_ref, 1.5e-3, "multi-head P v")


@pytest.mark.parametrize("N,H,W,C", [(2, 16, 16, 128), (1, 32, 24, 128), (2, 16, 16, 256), (17, 16, 8, 64),
                                      (3, 64, 64, 128)])
def test_upsample_conv_subpixel(cuda_device, N, H, W, C):
    """Upsample.conv (ddpm/diffusion.py:77-87): conv3x3(F.interpolate(x, 2, 'nearest')) evaluated as four sub-pixel
    phase convs on the source (AsyrpConvDesc.up2).  Reference: the plain formula on the fp16-rounded input with the
    fp16-rounded PACKED (pre-summed) weights' fp32 originals — the pre-summing changes the rounding points, hence the
    tolerance of a few fp16 ulps of the largest output."""
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    x = _rand((N, C, H, W), g)
    w = _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    eb = _rand((C,), g)
    ref = F.conv2d(F.interpolate(_h(x), scale_factor=2.0, mode="nearest"), w.double(), padding=1) \
        + eb.double()[None, :, None, None]
    tiles = ops.conv_stats_tiles_up2(H, W, C)
    assert tiles > 0
    out = torch.zeros(N, 2 * H, 2 * W, C, dtype=torch.float16, device=cuda_device)
    stats = torch.zeros(N, tiles, C // 2, 2, dtype=torch.float32, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3)], ops.pack_upconv_weight(w).to(cuda_device), out=out,
                    ebias=eb.to(cuda_device), stats=stats, up2=True)
    op.launch()
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 2.5e-3, "up2 conv")
    st = stats.sum(dim=1).cpu().double()
    sref = _stats_ref(ref)
    assert (st - sref).abs().max().item() <= 3e-3 * sref.abs().max().item() + 1e-3


def test_fused_silu_one_mufu_vs_two_mufu(cuda_device):
    """SiLU inside the operand transform: h + h*tanh.approx(h) (default, one special-function op) against
    x*rcp(1 + ex2(-x log2 e)) and against the fp64 formula.  Stated bound: the element-wise error of the tanh form is
    <= 2^-12 |x| + fp16 rounding, so the conv output (K = 1152 products) stays within 1.5e-3 of max|ref| either way."""
    ops = _ops()
    lib = ops._lib.load()
    g = torch.Generator().manual_seed(43)
    N, C, H = 2, 128, 64
    x, w = _rand((N, C, H, H), g, 2.0), _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()
    y = _h(x) * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
    ref = F.conv2d(y * torch.sigmoid(y), _h(w), padding=1)   # operand NOT rounded: the bound covers its fp16 rounding
    errs = []
    try:
        for mode in (1, 0):
            lib.asyrp_set_silu_tanh(mode)
            out = torch.zeros(N, H, H, C, dtype=torch.float16, device=cuda_device)
            op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3, aff.to(cuda_device), 0, 1)],
                            ops.pack_conv_weight(w).to(cuda_device), out=out, stats=ops.new_stats(N, H, H, C, cuda_device, True))
            op.launch()
            torch.cuda.synchronize()
            errs.append((_from_nhwc(out).double() - ref).abs().max().item() / ref.abs().max().item())
    finally:
        lib.asyrp_set_silu_tanh(-1)
    print(f"fused SiLU conv, max-abs error / max|ref|: tanh form {errs[0]:.2e}, ex2+rcp form {errs[1]:.2e}")
    assert errs[0] <= 1.5e-3 and errs[1] <= 1.5e-3, errs
    assert errs[0] <= 2.0 * errs[1] + 2e-4, errs


@pytest.mark.parametrize("Co,fused", [(3, False), (6, True)])
def test_conv_out_narrow_tile(cuda_device, Co, fused):
    """conv_out as a 16-wide N tile (BN=16): 3 / 6 real channels, fp32 planar store, bias, optional fused GN+SiLU"""
    ops = _ops()
    g = torch.Generator().manual_seed(41)
    N, H, W, C = 2, 32, 32, 128
    x = _rand((N, C, H, W), g)
    w = torch.zeros(16, C, 3, 3)
    w[:Co] = _rand((Co, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    b = torch.zeros(16)
    b[:Co] = _rand((Co,), g)
    y = _h(x)
    seg = (_nhwc_half(x, cuda_device), ops.MODE_3x3)
    if fused:
        aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()
        y = y * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
        y = _h((y * torch.sigmoid(y)).float())
        seg = seg + (aff.to(cuda_device), 0, 1)
    ref = F.conv2d(y, _h(w[:Co]), padding=1) + b[:Co].double()[None, :, None, None]
    outp = torch.zeros(N, Co, H, W, dtype=torch.float32, device=cuda_device)
    op = ops.ConvOp([seg], ops.pack_conv_weight(w).to(cuda_device), out_shape=(N, H, W, 16), ebias=b.to(cuda_device),
                    out_planar=outp)
    op.launch()
    op.launch()
    torch.cuda.synchronize()
    _check(outp.cpu(), ref, 2.5e-3 if fused else 2e-5, "narrow conv_out tile")


@pytest.mark.parametrize("C,H,mode", [(128, 32, "up"), (256, 32, "up"), (128, 64, "down"), (256, 32, "down"), (512, 16, "down"),
                                      (128, 16, "up"), (128, 64, "up")])
def test_resampled_residual_in_the_epilogue(cuda_device, C, H, mode):
    """skip branch of the ADM ResBlock(up / down) (improved_ddpm/unet.py:279-284,297): out = conv3x3(a) + resample(x),
    x read by the epilogue through the nearest-x2 / 2x2-average index map (AsyrpConvDesc.res_mode), on 64- and
    128-channel tiles"""
    ops = _ops()
    g = torch.Generator().manual_seed(51)
    N = 2
    a = _rand((N, C, H, H), g)
    w = _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    b = _rand((C,), g)
    if mode == "up":
        x = _rand((N, C, H // 2, H // 2), g)
        skip = F.interpolate(_h(x), scale_factor=2, mode="nearest")
    else:
        x = _rand((N, C, 2 * H, 2 * H), g)
        skip = F.avg_pool2d(_h(x), 2)
    ref = F.conv2d(_h(a), _h(w), padding=1) + b.double()[None, :, None, None] + skip
    out = torch.empty(N, H, H, C, dtype=torch.float16, device=cuda_device)
    stats = ops.new_stats(N, H, H, C, cuda_device, True)
    op = ops.ConvOp([(_nhwc_half(a, cuda_device), ops.MODE_3x3)], ops.pack_conv_weight(w).to(cuda_device), out=out,
                    ebias=b.to(cuda_device), residual=_nhwc_half(x, cuda_device), stats=stats,
                    res_mode=1 if mode == "up" else 2)
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 1.5e-3, f"resampled residual {mode}")
    st = stats.sum(dim=1).cpu().double()
    sref = _stats_ref(ref)
    assert (st - sref).abs().max().item() <= 2e-3 * sref.abs().max().item() + 1e-3


@pytest.mark.parametrize("C,H", [(128, 32), (256, 16)])
def test_subpixel_upconv_with_fused_groupnorm_silu(cuda_device, C, H):
    """in_layers of the ADM ResBlock(up=True): conv3x3(nearest-x2(silu(GN(x)))) on the source image — sub-pixel phases
    with the affine + SiLU applied to the operand tile in shared memory (improved_ddpm/unet.py:224-228,279-283)"""
    ops = _ops()
    g = torch.Generator().manual_seed(52)
    N = 2
    x = _rand((N, C, H, H), g) * 1.5 + 0.2
    aff = torch.stack([_rand((N, C), g) * 0.5 + 1.0, _rand((N, C), g) * 0.5], dim=-1).contiguous()
    w = _rand((C, C, 3, 3), g, 1.0 / math.sqrt(9 * C))
    y = _h(x) * aff[..., 0].double()[:, :, None, None] + aff[..., 1].double()[:, :, None, None]
    y = _h((y * torch.sigmoid(y)).float())
    ref = F.conv2d(F.interpolate(y, scale_factor=2.0, mode="nearest"), w.double(), padding=1)
    out = torch.zeros(N, 2 * H, 2 * H, C, dtype=torch.float16, device=cuda_device)
    stats = torch.zeros(N, ops.conv_stats_tiles_up2(H, H, C), C // 2, 2, dtype=torch.float32, device=cuda_device)
    op = ops.ConvOp([(_nhwc_half(x, cuda_device), ops.MODE_3x3, aff.to(cuda_device), 0, 1)],
                    ops.pack_upconv_weight(w).to(cuda_device), out=out, stats=stats, up2=True)
    op.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), ref, 3e-3, "fused up2 conv")


@pytest.mark.parametrize("C1,C2,H,mode,ss", [(128, 0, 32, "3x3", False), (128, 64, 32, "3x3", False), (64, 0, 16, "1x1", False),
                                             (256, 128, 16, "3x3", True), (256, 0, 64, "3x3", True), (512, 256, 16, "1x1", False)])
def test_groupnorm_finalised_inside_the_consumer_conv(cuda_device, C1, C2, H, mode, ss):
    """AsyrpConvSeg.gn_*: the producers' epilogues add (sum, sum of squares) per (sample, channel pair) into int64
    accumulators (integer atomics: deterministic); the consuming conv computes GroupNorm(32) [*(1+scale)+shift] + SiLU of its
    operand from them — no asyrp_gn_finalize launch, no affine table.  Reference: torch GroupNorm over the concatenated
    producers' outputs (statistics on the fp32 pre-rounding values, normalisation of the fp16-stored tensor)."""
    ops = _ops()
    g = torch.Generator().manual_seed(61)
    N, W, Cout = 3, H, 128
    C = C1 + C2
    srcs, sums, refs = [], [], []
    for Cs in [c for c in (C1, C2) if c]:
        xin = _rand((N, 64, H, W), g)
        w = _rand((Cs, 64, 1, 1), g, 0.3)
        b = _rand((Cs,), g)
        out = torch.empty(N, H, W, Cs, dtype=torch.float16, device=cuda_device)
        st = ops.new_stats(N, H, W, Cs, cuda_device, False)
        sm = ops.new_sums(N, Cs, cuda_device)
        op = ops.ConvOp([(_nhwc_half(xin, cuda_device), ops.MODE_1x1)], ops.pack_conv_weight(w).to(cuda_device), out=out,
                        ebias=b.to(cuda_device), stats=st, sums_out=sm)
        op.launch()
        srcs.append(out)
        sums.append(sm)
        refs.append(F.conv2d(_h(xin), _h(w)) + b.double()[None, :, None, None])
    torch.cuda.synchronize()
    # the accumulators equal the per-tile slots' totals (fixed point, 2^18)
    xstat = torch.cat(refs, 1)
    for sm, r in zip(sums, refs):
        got = sm.double().cpu() / ops.STAT_SCALE
        want = _stats_ref(r)
        assert (got - want).abs().max().item() <= 2e-3 * want.abs().max().item() + 1e-3
    gamma, beta = _rand((C,), g) * 0.3 + 1.0, _rand((C,), g) * 0.3
    ssv = _rand((N, 2 * C + 5), g, 0.3)[:, 3:3 + 2 * C] if ss else None  # a slice of a wider row, as the engine passes it
    eps = 1e-5
    xg = xstat.reshape(N, 32, -1)
    mean, var = xg.mean(-1), xg.var(-1, unbiased=False)
    cpg = C // 32
    mean_c = mean.repeat_interleave(cpg, 1)[:, :, None, None]
    rstd_c = (1.0 / torch.sqrt(var + eps)).repeat_interleave(cpg, 1)[:, :, None, None]
    xcat = torch.cat([_from_nhwc(s).double() for s in srcs], 1)
    y = (xcat - mean_c) * rstd_c * gamma.double()[None, :, None, None] + beta.double()[None, :, None, None]
    if ss:
        y = y * (1 + ssv[:, :C].double()[:, :, None, None]) + ssv[:, C:].double()[:, :, None, None]
    y = _h((y * torch.sigmoid(y)).float())
    k = 3 if mode == "3x3" else 1
    w2 = _rand((Cout, C, k, k), g, 1.0 / math.sqrt(k * k * C))
    ref = F.conv2d(y, _h(w2), padding=k // 2)
    ssd = None
    if ss:
        wide = torch.zeros(N, 2 * C + 5)
        wide[:, 3:3 + 2 * C] = ssv
        ssd = wide.to(cuda_device)[:, 3:3 + 2 * C]
    spec = ops.GNSpec(sums, [c for c in (C1, C2) if c], gamma.to(cuda_device), beta.to(cuda_device), eps, H * W,
                      ssd, 2 * C + 5 if ss else 0)
    m = ops.MODE_3x3 if mode == "3x3" else ops.MODE_1x1
    segs, off, wparts = [], 0, []
    for x in srcs:
        segs.append((x, m, spec, off, 1))
        wparts.append(ops.pack_conv_weight(w2[:, off:off + x.shape[-1]]))
        off += x.shape[-1]
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=cuda_device)
    op = ops.ConvOp(segs, torch.cat(wparts, 1).contiguous().to(cuda_device), out=out)
    op.launch()
    a = out.clone()
    op.launch()
    torch.cuda.synchronize()
    assert torch.equal(a, out)
    _check(_from_nhwc(out), ref, 3e-3, f"in-kernel GroupNorm {mode} C={C1}+{C2}")
