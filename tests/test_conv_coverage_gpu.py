"""Coverage of the conv kernel's tile configurations and of the kernels that test_kernels_gpu.py does not reach.

Every conv case below is driven from a small spec and checked against one CPU fp64 evaluation of the whole ConvOp
descriptor.  Each case
  * asserts the tile instantiation (BN, MT) it is meant to exercise, and that it launches at least two waves of tiles
    (the kernel is persistent: only a CTA that owns two or more tiles runs the producers ahead across a tile boundary,
    wraps its mbarrier parities and reuses its epilogue staging tile and statistics scratch);
  * fills the output, the statistics slots and the planar output with NaN, each with one extra sample behind it as a
    guard: a pixel or slot the kernel fails to write stays NaN, and a store past the end shows up in the guard (the
    engine's buffers come from a pool of torch.empty allocations, so a skipped store reads stale data there);
  * compares the output and the per-sample statistics with the reference, and a second launch bit for bit.

Conventions of the reference (those of test_kernels_gpu.py): operands are rounded to fp16, a transformed operand is
rounded to fp16 before the MMA, GroupNorm statistics come from the producer's fp32 values, up2 uses the unrounded 3x3
weights.  Tolerances, relative to max|ref|: 1.5e-3 raw fp16 operands (fp16 output rounding plus fp32 accumulation
order), 2.5e-3 with a fused affine+SiLU operand (its fp16 rounding and the one-MUFU SiLU) or the up2 conv's pre-summed
weights, 3e-3 with the GroupNorm finalised in the kernel (fp32 (a, b) from fixed-point sums) or a fused up2 operand,
2e-5 for fp32 outputs of raw operands; statistics 2e-3 (3e-3 for up2).
"""
import math
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL_RAW, TOL_FUSED, TOL_GN, TOL_F32, TOL_STATS = 1.5e-3, 2.5e-3, 3e-3, 2e-5, 2e-3


def _ops():
    from asyrp_official_b200 import ops
    return ops


def _h(x):
    """fp16 rounding of an operand, evaluated in fp64"""
    return x.to(torch.float16).double()


def _nhwc(x_nchw, dev, dtype=torch.float16):
    return x_nchw.permute(0, 2, 3, 1).contiguous().to(dtype).to(dev)


def _from_nhwc(t):
    return t.double().cpu().permute(0, 3, 1, 2)


def _check(out, ref, tol_rel, what):
    err = (out.double() - ref).abs().max().item()
    mag = ref.abs().max().item()
    assert err <= tol_rel * mag + 1e-6, f"{what}: max-abs err {err:.3e} vs max|ref| {mag:.3e}"


def _stats_ref(ref_nchw):
    n, c, h, w = ref_nchw.shape
    r = ref_nchw.reshape(n, c // 2, 2, h * w)
    return torch.stack([r.sum(dim=(2, 3)), (r * r).sum(dim=(2, 3))], dim=-1)  # [N][C/2][2]


def _check_stats(got, want, tol, what):
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= tol * want.abs().max().item() + 1e-3, f"{what}: max-abs err {err:.3e}"


def _guarded(shape, dtype, dev, fill=float("nan")):
    """(full, view): a buffer of shape[0] + 1 samples filled with `fill`; the view holds the first shape[0], the last
    sample is the guard region"""
    full = torch.full((shape[0] + 1,) + tuple(shape[1:]), fill, dtype=dtype, device=dev)
    return full, full[:shape[0]]


def _check_guarded(full, what):
    used, guard = full[:-1], full[-1]
    bad = (~torch.isfinite(used)).sum().item()
    assert bad == 0, f"{what}: {bad} of {used.numel()} elements were not written"
    assert torch.isnan(guard).all(), f"{what}: the guard region after the buffer was overwritten"


def _silu(y):
    return y * torch.sigmoid(y)


# ------------------------------------------------------------------------------------------------------------------
# spec-driven conv harness
# ------------------------------------------------------------------------------------------------------------------
# segs: (mode, C, transform) with mode "3x3" | "1x1" | "s2" and transform None | "affine" (fused act(a*x+b) from a
# table) | "gn" (GroupNorm finalised in the kernel from the sums of 1x1 producer convs; all "gn" segments form one
# concatenated GroupNorm).  H, W: the output geometry, except for up2 where they are the source's.
CASES = {
    # <128,1>, 3x3 from one halo tile, raw operand + residual + per-sample bias, 384 tiles
    "halo128_raw_residual": dict(inst=(128, 1), N=6, H=64, W=64, Cout=256, segs=[("3x3", 64, None)], ebias="sample",
                                 residual=0, res_scale=1.5, acc_scale=0.75, stats=True),
    # three dx-shifted copies with fused affine+SiLU: partial x tiles (W=40 in 16-wide tiles), 270 tiles
    "copies128_fused_partial_x": dict(inst=(128, 1), N=30, H=24, W=40, Cout=128, segs=[("3x3", 64, "affine")],
                                      ebias="shared", stats=True),
    # ... partial x and y tiles (W=24 in 16-wide, H=20 in 8-row tiles), 288 tiles
    "copies64_fused_partial_xy": dict(inst=(64, 1), N=24, H=20, W=24, Cout=128, segs=[("3x3", 64, "affine")],
                                      ebias="sample", stats=True),
    # <64,2>: in-kernel GroupNorm over the concat of two producers, with scale/shift, stats + sums_out, 288 tiles
    "halo64x2_gn_concat_ss": dict(inst=(64, 2), N=6, H=64, W=64, Cout=192, segs=[("3x3", 64, "gn"), ("3x3", 64, "gn")],
                                  gn_ss=True, stats=True, sums=True),
    # ... without scale/shift, 272 tiles
    "halo64x2_gn_concat": dict(inst=(64, 2), N=17, H=64, W=64, Cout=64, segs=[("3x3", 64, "gn"), ("3x3", 64, "gn")],
                               stats=True, sums=True),
    # <64,1>: fused 3x3 halo segment + two raw 1x1 segments (separate light ring), 10 K chunks, 320 tiles
    "halo64_fused_two_raw_1x1": dict(inst=(64, 1), N=40, H=16, W=16, Cout=256,
                                     segs=[("3x3", 256, "affine"), ("1x1", 256, None), ("1x1", 128, None)],
                                     ebias="sample", stats=True),
    # tiles of two samples (8x8), N odd: the last tile is half empty, 272 tiles
    "nb2_fused": dict(inst=(64, 1), NB=2, N=67, H=8, W=8, Cout=512, segs=[("3x3", 64, "affine")], ebias="sample",
                      stats=True),
    # tiles of eight samples (4x4), N = 8*33+1, with a 2x2-average-pooled residual, 272 tiles
    "nb8_raw_avgpool_residual": dict(inst=(64, 1), NB=8, N=265, H=4, W=4, Cout=512, segs=[("3x3", 64, None)],
                                     ebias="shared", residual=2, res_scale=0.5, stats=True),
    # stride 2 (parity view of the 2x source) with a nearest-x2 residual, 320 tiles
    "s2_nearest_residual": dict(inst=(128, 1), N=40, H=32, W=32, Cout=128, segs=[("s2", 64, None)], ebias="shared",
                                residual=1, stats=True),
    # sub-pixel up2 conv over a 16x16 source, 8 slots per sample: >= 272 tiles
    "up2_raw": dict(up2=True, slots=8, N=34, H=16, W=16, Cout=128, segs=[("3x3", 64, None)], ebias="shared",
                    stats=True),
    "up2_fused": dict(up2=True, slots=8, N=34, H=16, W=16, Cout=128, segs=[("3x3", 64, "affine")], stats=True),
    # conv_out: 16-wide channel tile, fp32 planar store, 320 / 288 tiles
    "conv_out16x2_fused": dict(inst=(16, 2), N=20, H=64, W=64, Cout=16, planar=6, segs=[("3x3", 64, "affine")],
                               ebias="shared"),
    "conv_out16x1_raw": dict(inst=(16, 1), N=48, H=24, W=24, Cout=16, planar=3, segs=[("3x3", 64, None)],
                             ebias="shared"),
    # batched GEMM (H = 1 rows x per-sample weights): T = 200 is a partial 128-row tile, 288 tiles; T = 384 with
    # Cout = 384 is three 128-channel tiles, fp32 out, 270 tiles
    "gemm_T200": dict(inst=(64, 1), batched=True, N=36, H=1, W=200, Cout=256, segs=[("1x1", 128, None)]),
    "gemm_T384_f32": dict(inst=(128, 1), batched=True, N=30, H=1, W=384, Cout=384, segs=[("1x1", 128, None)],
                          out="f32"),
}


def _gn_producers(spec, g, dev):
    """1x1 producer convs writing the sources of the "gn" segments and their int64 sums; returns the fp16 outputs,
    the sums and the fp64 references of the producers' fp32 values"""
    ops = _ops()
    N, H, W = spec["N"], spec["H"], spec["W"]
    srcs, sums, refs = [], [], []
    for mode, C, tf in spec["segs"]:
        if tf != "gn":
            continue
        xin = torch.randn(N, 64, H, W, generator=g)
        w = torch.randn(C, 64, 1, 1, generator=g) * 0.3
        b = torch.randn(C, generator=g)
        out = torch.empty(N, H, W, C, dtype=torch.float16, device=dev)
        sm = ops.new_sums(N, C, dev)
        ops.ConvOp([(_nhwc(xin, dev), ops.MODE_1x1)], ops.pack_conv_weight(w).to(dev), out=out, ebias=b.to(dev),
                   stats=ops.new_stats(N, H, W, C, dev, False), sums_out=sm).launch()
        srcs.append(out)
        sums.append(sm)
        refs.append(F.conv2d(_h(xin), _h(w)) + b.double()[None, :, None, None])
    return srcs, sums, refs


def _run_case(spec, dev, seed):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    N, H, W, Cout = spec["N"], spec["H"], spec["W"], spec["Cout"]
    up2, batched = spec.get("up2", False), spec.get("batched", False)
    segs = spec["segs"]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count

    # ---- configuration and wave count, before anything is launched
    has3 = any(m == "3x3" for m, _, _ in segs) and not up2
    if up2:
        slots = ops.conv_stats_tiles_up2(H, W, Cout)
        assert slots == spec["slots"], slots
        tiles = N * slots  # lower bound: the up2 tiles also split Cout
    else:
        assert ops.conv_tile_config(H, W, Cout, has3) == spec["inst"], ops.conv_tile_config(H, W, Cout, has3)
        slots = ops.conv_stats_tiles(H, W, Cout, has3)
        BN = spec["inst"][0]
        NB = spec.get("NB", 1)
        if NB == 1:
            tiles = N * slots * (Cout // BN)
        else:  # whole images per tile, one slot per lane quarter of the epilogue
            assert H * W * NB == 128 and slots == 4, (H, W, NB, slots)
            tiles = -(-N // NB) * (Cout // BN)
    assert tiles >= 2 * sms, f"{tiles} tiles on {sms} SMs: fewer than two waves"

    # ---- operands and the fp64 reference of the whole descriptor
    Ho, Wo = (2 * H, 2 * W) if up2 else (H, W)
    ktot = sum(C * (1 if m == "1x1" else 9) for m, C, _ in segs)
    c_aff = sum(C for _, C, tf in segs if tf == "affine")
    aff = None
    if c_aff:  # O(1) shift: an out-of-image pixel that is not re-zeroed after the SiLU is far from zero
        aff = torch.stack([torch.randn(N, c_aff, generator=g) * 0.5 + 1.0,
                           torch.randn(N, c_aff, generator=g) * 0.5 + 1.0], dim=-1).contiguous()
        affd = aff.to(dev)
    gn_srcs, gn_sums, gn_refs = _gn_producers(spec, g, dev) if any(tf == "gn" for _, _, tf in segs) else ([], [], [])
    gn_spec, gn_y = None, None
    if gn_srcs:
        Cg = sum(s.shape[-1] for s in gn_srcs)
        gamma = torch.randn(Cg, generator=g) * 0.3 + 1.0
        beta = torch.randn(Cg, generator=g) * 0.3
        eps = 1e-5
        xs = torch.cat(gn_refs, 1).reshape(N, 32, -1)
        cpg = Cg // 32
        mean = xs.mean(-1).repeat_interleave(cpg, 1)[:, :, None, None]
        rstd = (1.0 / torch.sqrt(xs.var(-1, unbiased=False) + eps)).repeat_interleave(cpg, 1)[:, :, None, None]
        xcat = torch.cat([_from_nhwc(s) for s in gn_srcs], 1)
        y = (xcat - mean) * rstd * gamma.double()[None, :, None, None] + beta.double()[None, :, None, None]
        ssd, ss_stride = None, 0
        if spec.get("gn_ss"):  # scale | shift: a slice of a wider row, as the engine passes it
            wide = torch.randn(N, 2 * Cg + 5, generator=g) * 0.3
            ss = wide[:, 3:3 + 2 * Cg]
            y = y * (1 + ss[:, :Cg].double()[:, :, None, None]) + ss[:, Cg:].double()[:, :, None, None]
            ssd, ss_stride = wide.to(dev)[:, 3:3 + 2 * Cg], 2 * Cg + 5
        gn_y = _h(_silu(y).float())
        gn_spec = ops.GNSpec(gn_sums, [s.shape[-1] for s in gn_srcs], gamma.to(dev), beta.to(dev), eps, H * W, ssd,
                             ss_stride)

    conv_segs, wparts, acc = [], [], 0.0
    a_off = g_off = gi = 0
    mode_id = {"3x3": ops.MODE_3x3, "1x1": ops.MODE_1x1, "s2": ops.MODE_3x3_S2}
    for mode, C, tf in segs:
        k = 1 if mode == "1x1" else 3
        if tf == "gn":
            y = gn_y[:, g_off:g_off + C]
            conv_segs.append((gn_srcs[gi], mode_id[mode], gn_spec, g_off, 1))
            g_off += C
            gi += 1
        elif batched:
            x = torch.randn(N, W, C, generator=g)
            conv_segs.append((x.to(torch.float16).to(dev).reshape(N, 1, W, C), mode_id[mode]))
            y = _h(x)
        else:
            Hs, Ws = (2 * H, 2 * W) if mode == "s2" else (H, W)
            if tf == "affine":
                x = torch.randn(N, C, Hs, Ws, generator=g) * 1.5 + 0.3
                a = aff[:, a_off:a_off + C]
                y = _h(x) * a[..., 0].double()[:, :, None, None] + a[..., 1].double()[:, :, None, None]
                y = _h(_silu(y).float())
                conv_segs.append((_nhwc(x, dev), mode_id[mode], affd, a_off, 1))
                a_off += C
            else:
                x = torch.randn(N, C, Hs, Ws, generator=g)
                y = _h(x)
                conv_segs.append((_nhwc(x, dev), mode_id[mode]))
        if batched:
            w = torch.randn(N, Cout, C, generator=g) / math.sqrt(C)
            wparts.append(w.to(torch.float16))
            acc = acc + torch.einsum("ntk,nok->not", y, _h(w))[:, :, None, :]  # [N][Cout][1][T]
            continue
        w = torch.randn(Cout, C, k, k, generator=g) / math.sqrt(ktot)
        if spec.get("planar"):
            w[spec["planar"]:] = 0
        if up2:
            wparts.append(ops.pack_upconv_weight(w))
            acc = acc + F.conv2d(F.interpolate(y, scale_factor=2.0, mode="nearest"), w.double(), padding=1)
        else:
            wparts.append(ops.pack_conv_weight(w))
            if mode == "s2":
                acc = acc + F.conv2d(F.pad(y, (0, 1, 0, 1)), _h(w), stride=2)
            else:
                acc = acc + F.conv2d(y, _h(w), padding=k // 2)
    weight = torch.cat(wparts, -1).contiguous().to(dev)  # batched: one segment, [N][Cout][K]

    ref = acc
    kw = {}
    if spec.get("ebias"):  # O(1) bias: statistics that count out-of-image pixels are visibly off
        eb = torch.randn(N if spec["ebias"] == "sample" else 1, Cout, generator=g) * 0.5 + 1.0
        if spec.get("planar"):
            eb[:, spec["planar"]:] = 0
        ref = ref + eb.double()[:, :, None, None]
        kw.update(ebias=(eb if spec["ebias"] == "sample" else eb[0]).contiguous().to(dev),
                  ebias_stride=Cout if spec["ebias"] == "sample" else 0)
    acc_scale, res_scale = spec.get("acc_scale", 1.0), spec.get("res_scale", 1.0)
    kw.update(res_scale=res_scale, acc_scale=acc_scale)
    ref = ref * acc_scale
    if spec.get("residual") is not None:
        rm = spec["residual"]
        rs = {0: (H, W), 1: (H // 2, W // 2), 2: (2 * H, 2 * W)}[rm]
        res = torch.randn(N, Cout, *rs, generator=g)
        r = _h(res)
        r = F.interpolate(r, scale_factor=2, mode="nearest") if rm == 1 else (F.avg_pool2d(r, 2) if rm == 2 else r)
        ref = ref + res_scale * r
        kw.update(residual=_nhwc(res, dev), res_mode=rm)
    if spec.get("planar"):
        ref = ref[:, :spec["planar"]]

    # ---- sentinel-filled outputs with a guard sample behind each
    bufs = {}
    if spec.get("planar"):
        bufs["out_planar"] = _guarded((N, spec["planar"], H, W), torch.float32, dev)
        kw.update(out_planar=bufs["out_planar"][1], out_shape=(N, H, W, Cout))
    else:
        odt = torch.float32 if spec.get("out") == "f32" else torch.float16
        bufs["out"] = _guarded((N, Ho, Wo, Cout), odt, dev)
        kw.update(out=bufs["out"][1])
    if spec.get("stats"):
        bufs["stats"] = _guarded((N, slots, Cout // 2, 2), torch.float32, dev)
        kw.update(stats=bufs["stats"][1])
    sums_full = None
    if spec.get("sums"):
        sums_full, sums = _guarded((N, Cout // 2, 2), torch.int64, dev, fill=0)
        kw.update(sums_out=sums)
    op = ops.ConvOp(conv_segs, weight, up2=up2, weight_batched=batched, **kw)
    op.launch()
    torch.cuda.synchronize()

    # ---- results
    if gn_srcs or (up2 and c_aff):
        tol = TOL_GN  # the fused up2 conv adds the pre-summed weights' rounding to the transform's
    elif c_aff or up2:
        tol = TOL_FUSED
    elif spec.get("out") == "f32" or spec.get("planar"):
        tol = TOL_F32
    else:
        tol = TOL_RAW
    for name, (full, _) in bufs.items():
        _check_guarded(full, name)
    if spec.get("planar"):
        out = bufs["out_planar"][1].double().cpu()
    else:
        out = _from_nhwc(bufs["out"][1])
    _check(out, ref, tol, "output")
    if spec.get("stats"):
        _check_stats(bufs["stats"][1].sum(dim=1), _stats_ref(ref), TOL_STATS * (1.5 if up2 else 1.0), "stats slots")
    if sums_full is not None:
        assert not sums_full[-1].any(), "sums_out: the guard sample was written"
        _check_stats(sums_full[:-1].double() / ops.STAT_SCALE, _stats_ref(ref), TOL_STATS, "sums_out")

    # ---- determinism: a second launch of the same op gives the same bits
    first = {name: full.clone() for name, (full, _) in bufs.items()}
    for full, _ in bufs.values():
        full.fill_(float("nan"))
    if sums_full is not None:
        sums_first = sums_full.clone()
        sums_full.zero_()
    op.launch()
    torch.cuda.synchronize()
    for name, (full, _) in bufs.items():
        assert torch.equal(full[:-1], first[name][:-1]), f"{name}: second launch differs"
    if sums_full is not None:
        assert torch.equal(sums_full, sums_first), "sums_out: second launch differs"


@pytest.mark.parametrize("case", list(CASES))
def test_conv_tile_configurations_past_one_wave(cuda_device, case):
    t0 = time.perf_counter()
    _run_case(CASES[case], cuda_device, seed=100 + list(CASES).index(case))
    print(f"{case}: {time.perf_counter() - t0:.2f} s")


# ------------------------------------------------------------------------------------------------------------------
# batch invariance and device-side coefficients
# ------------------------------------------------------------------------------------------------------------------
# (H, W, Cout, fused operand, residual, sums_out): NB = 1 (16x16 halo tiles), NB = 2 (8x8), NB = 8 (4x4)
INVARIANCE_GEOMETRIES = {"nb1": (16, 16, 128, True, False, True), "nb2": (8, 8, 128, True, False, False),
                         "nb8": (4, 4, 128, False, True, False)}


@pytest.mark.parametrize("geom", list(INVARIANCE_GEOMETRIES))
def test_sample_result_is_independent_of_its_batch(cuda_device, geom):
    """DESIGN.md §2/§5: a sample's conv output, statistics slots, sums_out and GroupNorm affine are bit-identical
    whether it runs alone or at any position of a batch of 5 (the tile partition does not depend on the batch, and
    tiles that hold several samples reduce each sample's statistics separately)"""
    ops = _ops()
    dev = cuda_device
    H, W, Cout, fused, with_res, with_sums = INVARIANCE_GEOMETRIES[geom]
    C = 64
    g = torch.Generator().manual_seed(7)
    pool = 5
    x = torch.randn(pool, C, H, W, generator=g) * 1.5 + 0.3
    aff = torch.stack([torch.randn(pool, C, generator=g) * 0.5 + 1.0, torch.randn(pool, C, generator=g) * 0.5 + 1.0], -1)
    eb = torch.randn(pool, Cout, generator=g) + 1.0
    res = torch.randn(pool, Cout, H, W, generator=g)
    w = ops.pack_conv_weight(torch.randn(Cout, C, 3, 3, generator=g) / math.sqrt(9 * C)).to(dev)
    gamma, beta = (torch.randn(Cout, generator=g) * 0.3 + 1.0).to(dev), (torch.randn(Cout, generator=g) * 0.3).to(dev)
    slots = ops.conv_stats_tiles(H, W, Cout, True)
    k = 2  # the sample under test; pool entries != k are its batch neighbours

    def run(order):
        n = len(order)
        seg = (_nhwc(x[order], dev), ops.MODE_3x3)
        if fused:
            seg = seg + (aff[order].contiguous().to(dev), 0, 1)
        out = torch.full((n, H, W, Cout), float("nan"), dtype=torch.float16, device=dev)
        stats = torch.full((n, slots, Cout // 2, 2), float("nan"), dtype=torch.float32, device=dev)
        sums = ops.new_sums(n, Cout, dev) if with_sums else None
        ops.ConvOp([seg], w, out=out, ebias=eb[order].contiguous().to(dev), ebias_stride=Cout, stats=stats,
                   residual=_nhwc(res[order], dev) if with_res else None, res_scale=0.5, sums_out=sums).launch()
        affine = torch.full((n, Cout, 2), float("nan"), dtype=torch.float32, device=dev)
        ops.gn_finalize(stats, Cout, None, 0, gamma, beta, 1e-6, n, H * W, affine)
        torch.cuda.synchronize()
        return out, stats, sums, affine

    alone = run([k])
    assert torch.isfinite(alone[0]).all() and torch.isfinite(alone[1]).all() and torch.isfinite(alone[3]).all()
    others = [i for i in range(pool) if i != k]
    for pos in range(pool):
        order = others[:pos] + [k] + others[pos:]
        batch = run(order)
        for name, a, b in zip(("output", "stats slots", "sums_out", "gn_finalize affine"), alone, batch):
            if a is None:
                continue
            assert torch.equal(a[0], b[pos]), f"{geom}: {name} of the sample differs at batch position {pos}"


def test_device_side_conv_coefficients(cuda_device):
    """scales= (a device pair (acc_scale, res_scale)) overrides the by-value pair, and rewriting it between launches of
    the same op changes the result as out = acc_scale * (conv + bias) + res_scale * residual says; set_scales changes
    the by-value pair of an op without a device pair"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(8)
    N, H, W, C, Cout = 2, 16, 16, 64, 64
    x = torch.randn(N, C, H, W, generator=g)
    w = torch.randn(Cout, C, 3, 3, generator=g) / math.sqrt(9 * C)
    eb = torch.randn(N, Cout, generator=g)
    res = torch.randn(N, Cout, H, W, generator=g)
    conv = F.conv2d(_h(x), _h(w), padding=1) + eb.double()[:, :, None, None]
    r = _h(res)
    args = ([(_nhwc(x, dev), ops.MODE_3x3)], ops.pack_conv_weight(w).to(dev))
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=dev)
    kw = dict(out=out, ebias=eb.to(dev), ebias_stride=Cout, residual=_nhwc(res, dev))
    scales = torch.tensor([0.75, 1.5], dtype=torch.float32, device=dev)
    op = ops.ConvOp(*args, acc_scale=0.5, res_scale=0.25, scales=scales, **kw)
    for a, b in ((0.75, 1.5), (-1.25, 0.5), (1.0, 0.0)):
        scales.copy_(torch.tensor([a, b]))
        out.fill_(float("nan"))
        op.launch()
        torch.cuda.synchronize()
        _check(_from_nhwc(out), a * conv + b * r, TOL_RAW, f"device scales ({a}, {b})")
    op2 = ops.ConvOp(*args, acc_scale=0.5, res_scale=0.25, **kw)
    op2.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), 0.5 * conv + 0.25 * r, TOL_RAW, "by-value scales")
    op2.set_scales(0.3, -2.0)
    op2.launch()
    torch.cuda.synchronize()
    _check(_from_nhwc(out), 0.3 * conv - 2.0 * r, TOL_RAW, "set_scales")


# ------------------------------------------------------------------------------------------------------------------
# kernels without another kernel-level test
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("use_mask", [0, 1])
@pytest.mark.parametrize("shared_dh", [True, False])
def test_slerp_h(cuda_device, t, use_mask, shared_dh):
    """asyrp_slerp_h against oracle.ddpm.slerp and the masked / norm-matched branches of oracle.ddpm.ddpm_forward;
    the statistics of h2 land in slot 0 and every other slot is zeroed"""
    from oracle import ddpm as od
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(9)
    N, C, H, W, T = 3, 64, 8, 8, 4
    h = torch.randn(N, C, H, W, generator=g).to(torch.float16)
    dh = torch.randn(1 if shared_dh else N, C, H, W, generator=g) * 3.0
    hd = h.double()
    dhd = dh.double().expand(N, C, H, W)
    if use_mask:
        mask = torch.zeros_like(hd)
        mask[:, :, 4:-1, 3:5] = 1.0
        ref = od.slerp(t, hd * mask, dhd * mask) + (1 - mask) * hd
    else:
        hn = torch.norm(hd.reshape(N, -1), dim=1)[:, None, None, None]
        dn = torch.norm(dhd.reshape(N, -1), dim=1)[:, None, None, None]
        ref = od.slerp(t, hd, hn * dhd / dn)
    h2 = torch.full((N, H, W, C), float("nan"), dtype=torch.float16, device=dev)
    stats = torch.full((N, T, C // 2, 2), float("nan"), dtype=torch.float32, device=dev)
    dh_dev = dh[0].contiguous().to(dev) if shared_dh else dh.contiguous().to(dev)
    ops.slerp_h(_nhwc(h.float(), dev), dh_dev, h2, stats, t, use_mask=bool(use_mask))
    torch.cuda.synchronize()
    _check(_from_nhwc(h2), ref, 1e-3, "slerp_h")
    st = stats.cpu()
    assert torch.isfinite(st).all()
    _check_stats(st[:, 0], _stats_ref(ref), TOL_STATS, "slerp_h stats slot 0")
    assert not st[:, 1:].any(), "slerp_h: slots other than 0 are not zero"


@pytest.mark.parametrize("learned", [0, 1])
@pytest.mark.parametrize("mask", [0.0, 1.0])
def test_ddpm_update(cuda_device, learned, mask):
    """x_next = 1/sqrt(1-bt) * (x - bt/sqrt(1-at) * et) + mask * exp(0.5 logvar) * z with a fixed logvar or the learned
    channels [Cx, 2Cx) of the model output; x_next aliases x, as in the engine's sampler step"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(10)
    N, Cx, H, W = 3, 3, 17, 19
    Ce = 2 * Cx if learned else Cx
    x, z = torch.randn(N, Cx, H, W, generator=g), torch.randn(N, Cx, H, W, generator=g)
    et = torch.randn(N, Ce, H, W, generator=g)
    at, bt, logvar = 0.35, 0.02, -4.5
    xd, ed = x.double(), et.double()
    lv = ed[:, Cx:] if learned else torch.full_like(xd, logvar)
    ref = 1 / math.sqrt(1 - bt) * (xd - bt / math.sqrt(1 - at) * ed[:, :Cx]) + mask * torch.exp(0.5 * lv) * z.double()
    xg = x.to(dev)
    ops.ddpm_update(xg, et.to(dev), z.to(dev), xg, at, bt, logvar, learned, mask)
    torch.cuda.synchronize()
    err = (xg.cpu().double() - ref).abs().max().item()
    assert err <= 2e-6 * ref.abs().max().item(), err


def test_axpby_and_unpack_nchw(cuda_device):
    """axpby: alpha*a + beta*b evaluated in fp32 and rounded to fp16.  Bound: one fp16 ulp of the exact value, plus the
    fp32 rounding of the two products and their sum, which is what remains where they cancel (the compiler may contract
    one product into an FMA, so the fp32 evaluation order is not fixed).  unpack_nchw: NHWC fp16 -> NCHW fp32, exact"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(11)
    a = torch.randn(5, 64, 64, 128, generator=g).to(torch.float16)
    b = torch.randn(5, 64, 64, 128, generator=g).to(torch.float16)
    out = torch.full_like(a, float("nan"), device=dev)
    ops.axpby(a.to(dev), b.to(dev), out, 0.8, -1.7)
    torch.cuda.synchronize()
    al, be = (torch.tensor(v, dtype=torch.float32).double() for v in (0.8, -1.7))  # the kernel's fp32 coefficients
    ta, tb = al * a.double(), be * b.double()
    ref = ta + tb
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 10)
    bound = ulp + 2.0 ** -23 * (ta.abs() + tb.abs())
    err = (out.cpu().double() - ref).abs()
    assert (err <= bound).all(), f"{(err > bound).sum().item()} elements off by more than the bound"
    x = torch.randn(3, 5, 7, 192, generator=g).to(torch.float16)
    o = torch.full((4, 192, 5, 7), float("nan"), dtype=torch.float32, device=dev)
    ops.unpack_nchw(x.to(dev), o[:3])
    torch.cuda.synchronize()
    assert torch.equal(o[:3].cpu(), x.float().permute(0, 3, 1, 2)) and torch.isnan(o[3]).all()


@pytest.mark.parametrize("I", [128, 256, 512, 1024])
def test_linear_fast_path(cuda_device, I):
    """asyrp_linear at the widths of the engine's timestep MLP and projections (the linear_rows_kernel path): more
    samples than one staging pass holds, O not a multiple of 32, input / output rows inside wider rows (the engine's
    emb_all row), SiLU on the input and on the output"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(12)
    N = 2 * (32 * 1024 // (4 * I)) + 1  # samples staged per pass: 32 KB of shared memory
    O = 200
    inp = torch.randn(N, I + 40, generator=g)
    w, b = torch.randn(O, I, generator=g) / math.sqrt(I), torch.randn(O, generator=g)
    x = inp[:, 8:8 + I].double()
    for act_in, act_out in ((False, False), (True, False), (False, True)):
        ref = (F.silu(x) if act_in else x) @ w.double().t() + b.double()
        if act_out:
            ref = F.silu(ref)
        wide = torch.full((N + 1, O + 24), float("nan"), dtype=torch.float32, device=dev)
        ops.linear(inp.to(dev)[:, 8:8 + I], w.to(dev), b.to(dev), wide[:N, 16:16 + O], act_in=act_in, act_out=act_out)
        torch.cuda.synchronize()
        got = wide.cpu()
        assert torch.isnan(got[:, :16]).all() and torch.isnan(got[:, 16 + O:]).all() and torch.isnan(got[N]).all()
        err = (got[:N, 16:16 + O].double() - ref).abs().max().item()
        assert err <= 1e-5 * ref.abs().max().item() + 1e-6, (act_in, act_out, err)


@pytest.mark.parametrize("T", [64, 200, 1024])
def test_softmax_rows(cuda_device, T):
    """fp32 row softmax over logits of magnitude ~50, a row count that is not a multiple of the 8 rows per block"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(13)
    rows = 8 * 5 + 3
    S = torch.randn(rows, T, generator=g) * 50.0
    P = torch.full((rows + 1, T), float("nan"), dtype=torch.float16, device=dev)
    ops.softmax_rows(S.to(dev), P[:rows], 0.7)
    torch.cuda.synchronize()
    ref = torch.softmax(S.double() * 0.7, dim=-1)
    got = P.cpu()
    assert torch.isnan(got[rows]).all()
    assert (got[:rows].double() - ref).abs().max().item() < 6e-4


def test_transpose_tc_ragged(cuda_device):
    """[N][T][C] channel slice of a wider row (ld > C), T not a multiple of 32 -> [N][C][T], exact"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(14)
    N, T, C, ld = 3, 200, 96, 3 * 96 + 32
    full = torch.randn(N, T, ld, generator=g).to(torch.float16)
    out = torch.full((N + 1, C, T), float("nan"), dtype=torch.float16, device=dev)
    ops.transpose_tc(full.to(dev)[:, :, 64:64 + C], out[:N])
    torch.cuda.synchronize()
    assert torch.equal(out[:N].cpu(), full[:, :, 64:64 + C].transpose(1, 2)) and torch.isnan(out[N].cpu()).all()


def test_gn_finalize_from_two_sample_tiles(cuda_device):
    """asyrp_gn_finalize over the 4-slots-per-tile statistics of a producer whose 8x8 tiles hold two samples (N odd: the
    last tile's second sample does not exist), stats buffer NaN-filled before the producer runs"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(15)
    N, H, W, C, Cout = 5, 8, 8, 64, 256
    assert ops.conv_stats_tiles(H, W, Cout, True) == 4
    x = torch.randn(N, C, H, W, generator=g)
    w = torch.randn(Cout, C, 3, 3, generator=g) / math.sqrt(9 * C)
    b = torch.randn(Cout, generator=g) * 0.5
    ref = F.conv2d(_h(x), _h(w), padding=1) + b.double()[None, :, None, None]
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device=dev)
    stats = torch.full((N, 4, Cout // 2, 2), float("nan"), dtype=torch.float32, device=dev)
    ops.ConvOp([(_nhwc(x, dev), ops.MODE_3x3)], ops.pack_conv_weight(w).to(dev), out=out, ebias=b.to(dev),
               stats=stats).launch()
    gamma, beta = torch.randn(Cout, generator=g) * 0.3 + 1.0, torch.randn(Cout, generator=g) * 0.3
    ss = torch.randn(N, 2 * Cout, generator=g) * 0.3
    affine = torch.full((N, Cout, 2), float("nan"), dtype=torch.float32, device=dev)
    ops.gn_finalize(stats, Cout, None, 0, gamma.to(dev), beta.to(dev), 1e-6, N, H * W, affine, scale_shift=ss.to(dev),
                    ss_stride=2 * Cout)
    torch.cuda.synchronize()
    xg = ref.reshape(N, 32, -1)
    cpg = Cout // 32
    mean = xg.mean(-1).repeat_interleave(cpg, 1)
    rstd = (1.0 / torch.sqrt(xg.var(-1, unbiased=False) + 1e-6)).repeat_interleave(cpg, 1)
    a = gamma.double() * rstd
    bb = beta.double() - mean * a
    sc, sh = 1 + ss[:, :Cout].double(), ss[:, Cout:].double()
    got = affine.cpu().double()
    _check(got[..., 0], a * sc, 1e-4, "gn_finalize a")
    _check(got[..., 1], bb * sc + sh, 1e-4, "gn_finalize b")


def test_apply_with_affine_offset(cuda_device):
    """asyrp_apply reading its (a, b) pairs at a channel offset inside a wider affine table"""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(16)
    N, H, W, C, Ctot, off = 2, 12, 10, 64, 192, 128
    x = torch.randn(N, C, H, W, generator=g)
    aff = torch.stack([torch.randn(N, Ctot, generator=g) * 0.5 + 1.0, torch.randn(N, Ctot, generator=g)], -1)
    a, b = aff[:, off:off + C, 0].double(), aff[:, off:off + C, 1].double()
    y = _silu(_h(x) * a[:, :, None, None] + b[:, :, None, None])
    out = torch.full((N, H, W, C), float("nan"), dtype=torch.float16, device=dev)
    ops.apply(_nhwc(x, dev), None, aff.contiguous().to(dev), out, 1, affine_offset=off)
    torch.cuda.synchronize()
    _check(_from_nhwc(out), y, 1e-3, "apply with affine offset")
