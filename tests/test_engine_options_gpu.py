"""The engine's shipped non-default paths, held to the default path's standard.

1. Programmatic dependent launch (asyrp_set_pdl(1) / ASYRP_PDL=1) changes no bit: one edit evaluation of every
   bench.WORKLOADS plan run eagerly (every buffer of the plan compared), and whole trajectories through the captured
   graph with its two decoder streams, DeltaBlock and explicit-delta_h schedules.
2. Every launch of the plans that engine.GN_FOLD, GN_FOLD_PRODUCERS_ONLY (ASYRP_GN_FOLD=1 / 2), FUSE_MIN_H=8 and
   SKIP_AS_K=False build, against fp64 with the harness of test_plans_gpu.py, plus: in-kernel GroupNorm operands
   (GNSpec) against an fp64 GroupNorm of the producers' int64 sums, each producer's sums_out slice exactly the sum of
   its statistics slots in fixed point, no two producers sharing a slice, and the memset that zeroes the sums arena.
   Each option is checked to have taken effect (launch counts against the default plan).
3. Whole trajectories under each option: the production engine (pool, two streams, graph) equals a never-reusing,
   single-stream, eager engine bit for bit; with GN_FOLD also row B-1 at the benchmark batch equals its B=1 trajectory
   and the golden rows stay within TOL_TRAJ of the reference's own output.
4. In-kernel GroupNorm past one wave in the instantiations the GN_FOLD plans use: <128,1>, <64,1> over a concat,
   up2, and a GroupNorm 3x3 segment followed by a raw 1x1 shortcut.  Every CTA owns several tiles, consecutive tiles
   of a CTA lie in different samples, and every sample's group statistics are far from every other sample's, so
   statistics taken from the wrong sample or from the stale half of the one-tile-ahead buffer fail.
"""
import contextlib
import functools
import os
import time
from collections import Counter

import numpy as np
import pytest
import torch

import bench
from asyrp_official_b200 import _lib, engine, ops
from asyrp_official_b200.arch import Res
from asyrp_official_b200.schedule import Schedule, make_sequences
from oracle import sampler as osmp
from test_conv_coverage_gpu import _run_case
from test_plans_gpu import G, TOL_TRAJ, Recorder, _bits, _drive, _extent, _install, _model

pytestmark = pytest.mark.gpu

WORKLOADS = list(bench.WORKLOADS)
ARCH_OF = {"ddpm_celeba_b16": "ddpm_celeba", "ddpm_church_b32": "ddpm_church", "iddpm_afhq_b8": "adm_afhq",
           "adm_imagenet_b4": "adm_imagenet"}
WORKLOAD_OF = {a: w for w, a in ARCH_OF.items()}
OPTIONS = {
    "gn_fold": dict(GN_FOLD=True),
    "gn_fold_producers_only": dict(GN_FOLD=True, GN_FOLD_PRODUCERS_ONLY=True),
    "fuse_min_h_8": dict(FUSE_MIN_H=8),
    "skip_in_epilogue": dict(SKIP_AS_K=False),
}
OPTION_WORKLOADS = {
    "gn_fold": WORKLOADS,
    "gn_fold_producers_only": ["ddpm_celeba_b16", "iddpm_afhq_b8"],
    "fuse_min_h_8": ["ddpm_celeba_b16", "adm_imagenet_b4"],
    "skip_in_epilogue": ["ddpm_celeba_b16", "iddpm_afhq_b8"],
}
OPTION_CASES = [(o, w) for o in OPTIONS for w in OPTION_WORKLOADS[o]]
SENTINEL = 0x5A5A5A5A5A5A5A5A  # int64 pattern the sums arena holds before its memset


def _set_options(monkeypatch, option):
    for k, v in OPTIONS[option].items():
        monkeypatch.setattr(engine, k, v)


@contextlib.contextmanager
def _pdl(on):
    """PDL on / off for the library's launches, the previous setting restored afterwards"""
    lib = _lib.load()
    prev = lib.asyrp_get_pdl()
    lib.asyrp_set_pdl(int(on))
    try:
        assert lib.asyrp_get_pdl() == int(on)
        yield
    finally:
        lib.asyrp_set_pdl(prev)


def _trajectory_inputs(m, dev, B=2):
    """the schedules and inputs of test_plans_gpu's buffer-reuse test: edit, non-edit and stochastic steps"""
    g = torch.Generator().manual_seed(41)
    x = torch.randn(B, 3, 256, 256, generator=g).to(dev)
    seq, seq_next = make_sequences(999, 6)
    betas = osmp.make_betas()
    sch = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(1.0, 0.8))
    sch_dh = Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=300, hs_coeff=(0.6, 1.0))
    assert sch.n_edit and sch.n_edit < len(sch.steps) and sch.n_stochastic
    noise = torch.randn(sch.n_stochastic, *x.shape, generator=g).to(dev)
    h = m.arch.image_size // 32
    dh = (torch.randn(sch_dh.n_edit, B, m.arch.mid_ch, h, h, generator=g) * 2.0).to(dev)
    return x, sch, sch_dh, noise, dh


def _launch_kinds(m, dev):
    """launch kinds of one edit evaluation of the plan the current switches build (batch 1: counts do not depend on
    the batch)"""
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    kinds = Counter(L.kind for L in eng.plan(1).launches(edit=True))
    del eng
    return kinds


# ------------------------------------------------------------------------------------------------------------------
# 1. programmatic dependent launch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("workload", WORKLOADS)
def test_pdl_changes_no_bit_eager(cuda_device, monkeypatch, workload):
    """one edit evaluation at the benchmark batch, launched back to back with PDL off and on: every buffer of the plan
    (both pools, et, et_mod, the embedding rows) bit-identical.  Each arm starts from buffers filled with NaN, so a
    kernel that reads its input before its predecessor has finished writing it cannot read the other arm's values"""
    dev = cuda_device
    B = bench.WORKLOADS[workload][2]
    m = _model(workload, dev)
    raws = {}
    alloc = engine.Pool.alloc

    def recording_alloc(self, shape, dtype):
        t = alloc(self, shape, dtype)
        raws[t._asyrp_raw.data_ptr()] = t._asyrp_raw
        return t

    monkeypatch.setattr(engine.Pool, "alloc", recording_alloc)
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    P = eng.plan(B)
    monkeypatch.undo()
    g = torch.Generator().manual_seed(31)
    P.x.copy_(torch.randn(P.x.shape, generator=g))
    P.t.copy_(torch.linspace(999.0, 500.0, B))
    P.set_coeffs((0.9, 1.3))
    seq = P.launches(edit=True)
    named = {"et": P.et, "et_mod": P.et_mod, "middle_h": P.middle_h.t, "h2": P.h2.t, "delta_h": P.delta_h.t,
             "emb_all": P.emb_all}
    for i, a in enumerate(P.hs):
        named[f"hs[{i}]"] = a.t
        if a.stats is not None:
            named[f"hs[{i}].stats"] = a.stats
    bufs = list(raws.values()) + [P.et, P.et_mod, P.emb_all, P.temb]

    def arm(on):
        for b in bufs:
            b.view(torch.uint8).fill_(0xFF)  # NaN in fp16 and fp32
        torch.cuda.synchronize()
        with _pdl(on):
            assert _lib.load().asyrp_get_pdl() == on
            for L in seq:
                L()
            torch.cuda.synchronize()

    arm(0)
    off_named = {k: v.clone() for k, v in named.items()}
    off_raws = [r.clone() for r in raws.values()]
    assert all(torch.isfinite(v).all() for k, v in off_named.items() if not k.endswith("stats"))
    arm(1)
    bad = [k for k, v in named.items() if not torch.equal(_bits(v), _bits(off_named[k]))]
    assert not bad, f"{workload}: PDL changes {bad}"
    bad_raw = sum(not torch.equal(r, o) for r, o in zip(raws.values(), off_raws))
    assert bad_raw == 0, f"{workload}: PDL changes {bad_raw} of {len(raws)} pool buffers"
    print(f"\n{workload} B={B}: {len(seq)} launches, {len(named)} named tensors and {len(raws)} pool buffers "
          f"({sum(r.numel() for r in raws.values()) / 2**30:.2f} GiB) bit-identical with PDL on")
    del P, eng, m, raws, off_raws, off_named, named, bufs
    torch.cuda.empty_cache()


@pytest.mark.parametrize("arch", list(WORKLOAD_OF))
def test_pdl_changes_no_bit_graph(cuda_device, arch):
    """sample(use_graph=True) at B=2, a fresh engine per arm (the launch attribute is recorded at capture): x_0 of a
    DeltaBlock and of an explicit-delta_h schedule bit-identical with PDL on"""
    dev = cuda_device
    m = _model(WORKLOAD_OF[arch], dev)
    x, sch, sch_dh, noise, dh = _trajectory_inputs(m, dev)
    assert engine.DUAL_STREAM
    res = {}
    for on in (0, 1):
        with _pdl(on):
            eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
            a = eng.sample(x, sch, noise=noise, use_graph=True)
            a_dh = eng.sample(x, sch_dh, noise=noise, use_graph=True, delta_hs=dh)
            assert _lib.load().asyrp_get_pdl() == on
            torch.cuda.synchronize()
            res[on] = (a, a_dh)
            del eng
    (a, a_dh), (b, b_dh) = res[0], res[1]
    assert torch.isfinite(a).all() and torch.isfinite(a_dh).all() and not torch.equal(a, a_dh)
    assert torch.equal(a, b), f"{arch}: DeltaBlock schedule differs with PDL by {(a - b).abs().max().item():.3e}"
    assert torch.equal(a_dh, b_dh), f"{arch}: explicit-delta_h schedule differs with PDL by " \
                                    f"{(a_dh - b_dh).abs().max().item():.3e}"
    del m
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# 2. every launch of the option plans against fp64
# ------------------------------------------------------------------------------------------------------------------
class OptionRecorder(Recorder):
    """Recorder plus the in-kernel GroupNorm operand, the int64 sums a producer accumulates and the sums-arena memset"""

    def __init__(self, B):
        super().__init__(B)
        self.P = None
        self.slices = []            # (first byte, last byte + 1, launch index, desc) of every sums_out
        self.gn_consumed = set()    # GroupNorms (keyed by their sources' sums) finalised inside a consuming conv
        self.gn_launches = set()    # indices of the launches of such consumers
        self.up2_gn = 0             # up2 convs with an in-kernel GroupNorm operand
        self.nb2_fused = 0          # fused-operand convs over 8x8 images (tiles of two samples)
        self.epilogue_skip = 0      # convs adding a same-geometry residual to one 3x3 segment (no identity K block)

    def seg_inputs(self, i, aff):
        if not isinstance(aff, ops.GNSpec):
            return super().seg_inputs(i, aff)
        d = {f"gn{i}.gamma": aff.gamma, f"gn{i}.beta": aff.beta}
        for j, s in enumerate(aff.sums):
            d[f"gn{i}.sums{j}"] = s
        if aff.ss is not None:
            d[f"gn{i}.ss"] = torch.as_strided(aff.ss, (self.B, 2 * sum(aff.C)), (aff.ss_stride, 1),
                                              aff.ss.storage_offset())
        return d

    def seg_affine(self, snap, i, aff, off, C, idx):
        """GroupNorm(32) over the concat of the producers, in fp64 from the snapshot of their int64 sums (groups may
        straddle the seam), then the ADM (1 + scale, shift) rows"""
        if not isinstance(aff, ops.GNSpec):
            return super().seg_affine(snap, i, aff, off, C, idx)
        Ct = sum(aff.C)
        s = torch.cat([snap[f"gn{i}.sums{j}"][idx].double() for j in range(len(aff.sums))], 1) / ops.STAT_SCALE
        s = s.reshape(len(idx), 32, -1, 2).sum(2)
        cnt = aff.hw * (Ct // 32)
        mean = s[..., 0] / cnt
        var = (s[..., 1] / cnt - mean * mean).clamp_min(0.0)
        rstd = 1.0 / torch.sqrt(var + aff.eps)
        a = snap[f"gn{i}.gamma"].double() * rstd.repeat_interleave(Ct // 32, 1)
        b = snap[f"gn{i}.beta"].double() - mean.repeat_interleave(Ct // 32, 1) * a
        if aff.ss is not None:
            ss = snap[f"gn{i}.ss"][idx].double()
            a, b = a * (1 + ss[:, :Ct]), b * (1 + ss[:, :Ct]) + ss[:, Ct:]
        return a[:, off:off + C], b[:, off:off + C]

    def conv(self, op):
        segs, weight, kw = op._rec
        idx, desc = self.label
        for sg in segs:
            if isinstance(sg[2], ops.GNSpec):
                self.gn_consumed.add(tuple(s.data_ptr() for s in sg[2].sums))
                self.gn_launches.add(idx)
                self.up2_gn += bool(kw.get("up2"))
        out = kw.get("out")
        if out is not None and out.shape[1] * out.shape[2] == 64 and any(sg[2] is not None for sg in segs):
            self.nb2_fused += 1
        if kw.get("residual") is not None and kw.get("res_mode", 0) == 0 and len(segs) == 1 and \
                segs[0][1] == ops.MODE_3x3:
            self.epilogue_skip += 1
        sums = kw.get("sums_out")
        if sums is not None:
            lo, hi = _extent(sums)
            a_lo, a_hi = _extent(self.P.sums_arena)
            assert a_lo <= lo and hi <= a_lo + self.P.sums_used * 8, f"launch {idx} ({desc}): sums_out outside the " \
                                                                       f"used part of the arena"
            others = [sg[0] for sg in segs] + [s for sg in segs if isinstance(sg[2], ops.GNSpec) for s in sg[2].sums]
            others += [t for t in (weight, kw.get("residual"), out, kw.get("stats")) if t is not None]
            for t in others:
                b_lo, b_hi = _extent(t)
                assert hi <= b_lo or b_hi <= lo, f"launch {idx} ({desc}): sums_out overlaps an operand"
            assert not sums.any(), f"launch {idx} ({desc}): the sums_out slice is not zero before its producer runs"
            self.slices.append((lo, hi, idx, desc))
        super().conv(op)
        if sums is not None:
            # the epilogue adds __float2ll_rn(slot * 2^18) of the very value it stores in each statistics slot
            want = torch.round(kw["stats"].double() * ops.STAT_SCALE).long().sum(1)
            assert torch.equal(sums, want), f"launch {idx} ({desc}): sums_out differs from its statistics slots " \
                                            f"in {(sums != want).sum().item()} places"

    def memset(self, fn):
        """the launch that zeroes the sums arena at the start of an evaluation: exactly [0, sums_used)"""
        arena, used = self.P.sums_arena, self.P.sums_used
        idx, desc = self.label
        arena.fill_(SENTINEL)
        fn()
        torch.cuda.synchronize()
        assert not arena[:used].any(), f"launch {idx} ({desc}): the memset leaves part of [0, sums_used) non-zero"
        assert bool((arena[used:] == SENTINEL).all()), f"launch {idx} ({desc}): the memset writes past sums_used"
        self.checks += 1
        self.entries.add("memset")


def _track_gns(monkeypatch):
    """every GroupNorm the plan builds: (GN, the Res layer it belongs to or None, whether a conv segment asked for it)"""
    gns, cur = [], [None]
    build_gn, res_block, operand = engine.Plan._gn, engine.Plan._res_block, engine.GN.operand

    def _gn(self, srcs, *a, **k):
        g = build_gn(self, srcs, *a, **k)
        gns.append([g, cur[0], False])
        return g

    def _res_block(self, layer, srcs):
        cur[0] = layer
        try:
            return res_block(self, layer, srcs)
        finally:
            cur[0] = None

    def _operand(self):
        for e in gns:
            if e[0] is self:
                e[2] = True
        return operand(self)

    monkeypatch.setattr(engine.Plan, "_gn", _gn)
    monkeypatch.setattr(engine.Plan, "_res_block", _res_block)
    monkeypatch.setattr(engine.GN, "operand", _operand)
    return gns


@pytest.mark.parametrize("option,workload", OPTION_CASES)
def test_every_launch_of_the_option_plan_vs_fp64(cuda_device, monkeypatch, option, workload):
    """one edit evaluation of the option's plan at the benchmark batch, then the explicit-delta_h path (mask off and
    on), every launch checked; under GN_FOLD the re-drive starts with the arena memset and the encoder that refills it,
    as an evaluation does"""
    t0 = time.perf_counter()
    dev = cuda_device
    B = bench.WORKLOADS[workload][2]
    m = _model(workload, dev)
    base = _launch_kinds(m, dev)
    _set_options(monkeypatch, option)
    gns = _track_gns(monkeypatch)
    rec = OptionRecorder(B)
    _install(monkeypatch, rec)
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    P = eng.plan(B)
    rec.P = P
    memsets = [L for L in P.launches(edit=True) if L.kind == "memset"]
    if engine.GN_FOLD:
        assert len(memsets) == 1 and P.enc_ops[0] is memsets[0], "the sums arena is zeroed once, before any producer"
        memsets[0].fn = functools.partial(rec.memset, memsets[0].fn)
    else:
        assert not memsets and P.sums_arena is None
    g = torch.Generator().manual_seed(31)
    P.x.copy_(torch.randn(P.x.shape, generator=g))
    P.t.copy_(torch.linspace(999.0, 500.0, B))
    P.set_coeffs((0.9, 1.3))
    eng.state.update(ignore_timestep=False, slerp_t=0.0, use_mask=False)
    seq = P.launches(edit=True)
    _drive(rec, seq)
    n = len(seq)
    # no two producers of one evaluation add into the same int64 sums
    sl = sorted(rec.slices)
    for (lo0, hi0, i0, d0), (lo1, hi1, i1, d1) in zip(sl, sl[1:]):
        assert hi0 <= lo1, f"launches {i0} ({d0}) and {i1} ({d1}) share sums_arena bytes [{lo1}, {min(hi0, hi1)})"
    n_producers = len(sl)
    P.dh_user.copy_(torch.randn(P.dh_user.shape, generator=g) * 2.0)
    eng.state["slerp_t"] = 0.3
    redrive = (P.enc_ops if engine.GN_FOLD else []) + P.slerp_ops + P.dec_mod_ops
    for use_mask in (False, True):
        eng.state["use_mask"] = use_mask
        _drive(rec, redrive, n)
        n += len(redrive)
    assert rec.checks == n, (rec.checks, n)

    kinds = Counter(L.kind for L in seq)
    tables16 = [(g_, layer) for g_, layer, asked in gns if g_.srcs[0].H >= 16]
    if option == "gn_fold":
        assert "memset" in rec.entries and n_producers > 0
        assert kinds["gn_finalize"] < base["gn_finalize"], (kinds, base)
        for g_, layer, asked in gns:
            if g_.srcs[0].H < 16:
                continue
            key = tuple(s.sums.data_ptr() if s.sums is not None else None for s in g_.srcs)
            if asked:  # a fused conv segment: the GroupNorm is finalised inside it
                assert key in rec.gn_consumed, f"{workload}: a {g_.srcs[0].H}x{g_.srcs[0].W} GroupNorm has no " \
                                               f"in-kernel consumer"
            else:      # only the ADM downsampling ResBlock feeds a table to the pointwise apply + avg-pool kernel
                assert isinstance(layer, Res) and layer.resample == "down", (layer, g_.srcs[0].H)
        if m.arch.family == "adm":
            assert rec.up2_gn > 0, f"{workload}: no up2 conv with an in-kernel GroupNorm operand"
    elif option == "gn_fold_producers_only":
        assert "memset" in rec.entries and n_producers > 0 and not rec.gn_consumed
        assert kinds["gn_finalize"] == base["gn_finalize"], (kinds, base)
    elif option == "fuse_min_h_8":
        assert kinds["apply"] < base["apply"] and rec.nb2_fused > 0, (kinds, base, rec.nb2_fused)
    elif option == "skip_in_epilogue":
        assert rec.epilogue_skip > 0, "no ResBlock reads its identity skip in the epilogue"
        assert kinds["conv"] == base["conv"], (kinds, base)
    total, total0 = sum(kinds.values()), sum(base.values())
    worst = sorted(rec.worst, key=lambda w: -w[0])[:3]
    worst_gn = sorted((w for w in rec.worst if w[1] in rec.gn_launches), key=lambda w: -w[0])[:1]
    fmt = lambda ws: "; ".join(f"#{i} {d} {w}: {r:.2e} (tol {tol:g}, {mg:.2f} of it)"  # noqa: E731
                               for mg, i, d, w, r, tol in ws)
    print(f"\n{option} {workload} B={B}: {total} launches per edit evaluation (default {total0}: "
          f"{', '.join(f'{k} {kinds[k]}/{base[k]}' for k in sorted(set(kinds) | set(base)))}); "
          f"{n_producers} sums_out producers, {len(rec.gn_consumed)} in-kernel GroupNorms "
          f"({rec.up2_gn} up2 consumers) of {len(tables16)} >= 16x16, {rec.nb2_fused} fused 8x8 convs, "
          f"{rec.epilogue_skip} epilogue skips; {rec.checks} launches checked, {time.perf_counter() - t0:.1f} s; "
          f"worst: {fmt(worst)}" + (f"; worst in-kernel GroupNorm consumer: {fmt(worst_gn)}" if worst_gn else ""))
    monkeypatch.undo()
    del P, eng, m, rec, gns
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# 3. whole trajectories under each option
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("option,arch", [(o, ARCH_OF[w]) for o, w in OPTION_CASES])
def test_option_trajectories_production_equals_serial(cuda_device, monkeypatch, option, arch):
    """production engine (pooled buffers, two decoder streams, CUDA graph) == an engine whose plan never reuses a
    buffer, run on one stream without a graph, bit for bit, with the option on"""
    dev = cuda_device
    _set_options(monkeypatch, option)
    m = _model(WORKLOAD_OF[arch], dev)
    x, sch, sch_dh, noise, dh = _trajectory_inputs(m, dev)
    prod = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    assert engine.DUAL_STREAM
    a = prod.sample(x, sch, noise=noise, use_graph=True)
    a_dh = prod.sample(x, sch_dh, noise=noise, use_graph=True, delta_hs=dh)

    ref = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    with monkeypatch.context() as mp:
        mp.setattr(engine.Pool, "release", lambda self, t: None)
        P = ref.plan(2)
    assert P.pool.total > prod.plan(2).pool.total, "the reference plan reuses buffers"
    monkeypatch.setattr(engine, "DUAL_STREAM", False)
    b = ref.sample(x, sch, noise=noise, use_graph=False)
    b_dh = ref.sample(x, sch_dh, noise=noise, use_graph=False, delta_hs=dh)
    assert torch.isfinite(a).all() and torch.isfinite(a_dh).all()
    assert not torch.equal(a, a_dh)
    assert torch.equal(a, b), f"{option} {arch}: DeltaBlock schedule differs by {(a - b).abs().max().item():.3e}"
    assert torch.equal(a_dh, b_dh), f"{option} {arch}: explicit-delta_h schedule differs by " \
                                    f"{(a_dh - b_dh).abs().max().item():.3e}"
    del P, ref, prod, m
    torch.cuda.empty_cache()


@pytest.mark.parametrize("workload", WORKLOADS)
def test_gn_fold_benchmark_batch_reproduces_the_reference_row_for_row(cuda_device, monkeypatch, workload):
    """test_plans_gpu.py's batch-sharding test with GN_FOLD: row B-1 bit-identical to its B=1 trajectory, the golden
    rows within TOL_TRAJ of the reference's own output"""
    dev = cuda_device
    _set_options(monkeypatch, "gn_fold")
    B, golden = bench.WORKLOADS[workload][2], bench.WORKLOADS[workload][5]
    gold = np.load(os.path.join(G, golden))
    Bg = int(gold["batch"])
    assert Bg in (1, B), Bg
    m = _model(workload, dev)
    seq = gold["seq"].tolist()
    seq_next = [-1] + seq[:-1]
    g = torch.Generator().manual_seed(int(gold["x_seed"]))
    xg = torch.randn(Bg, 3, 256, 256, generator=g)
    gn = torch.Generator().manual_seed(int(gold["noise_seed"]))
    noises = {i: torch.randn(xg.shape, generator=gn) for i in seq}
    sch = Schedule(osmp.make_betas(), seq, seq_next, t_edit=int(gold["t_edit"]), t_addnoise=int(gold["t_addnoise"]),
                   hs_coeff=(1.0, 1.0))
    nzg = torch.stack([noises[s.t] for s in sch.steps if s.stochastic])
    gr = torch.Generator().manual_seed(51)
    xb = torch.cat([torch.randn(B - Bg, 3, 256, 256, generator=gr), xg])
    nzb = torch.cat([torch.randn(nzg.shape[0], B - Bg, 3, 256, 256, generator=gr), nzg], dim=1)
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    assert eng.plan(1).sums_arena is not None
    one = eng.sample(xb[B - 1:].to(dev), sch, noise=nzb[:, B - 1:].contiguous().to(dev))
    full = eng.sample(xb.to(dev), sch, noise=nzb.to(dev))
    row = full[B - 1:]
    e = (full[B - Bg:, :, ::4, ::4].double().cpu() - torch.from_numpy(gold["x0_sub"]).double()).abs().max().item()
    mx = float(np.abs(gold["x0_sub"]).max())
    print(f"\ngn_fold {workload}: rows {B - Bg}..{B - 1} of {B} vs the reference: max-abs {e:.4f} of max|x_0| "
          f"{mx:.2f} -> {e / mx:.2e} (default path 3.8e-4..5.1e-4)")
    assert torch.equal(row, one), f"{workload}: row {B - 1} of a batch of {B} differs from its B=1 run by " \
                                  f"{(row - one).abs().max().item():.3e}"
    assert e <= TOL_TRAJ * mx, f"{workload}: max-abs err {e:.3e} of max|ref| {mx:.3e}"
    del eng, m
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# 4. in-kernel GroupNorm past one wave, in the instantiations the GN_FOLD plans use
# ------------------------------------------------------------------------------------------------------------------
# specs of test_conv_coverage_gpu._run_case; "bn": output channels per tile of the up2 conv (asyrp_conv_tile_config
# does not cover the four-phase tiling), for the tile-order check below
GN_CASES = {
    # <128,1> halo tiles at 32x32, 128 -> 128 (the 256^2 UNets' 32x32 ResBlocks), ADM scale/shift, sums_out; 400 tiles
    "gn128_halo32_ss": dict(inst=(128, 1), N=50, H=32, W=32, Cout=128, segs=[("3x3", 128, "gn")], gn_ss=True,
                            gn_per_sample=True, ebias="sample", stats=True, sums=True),
    # <64,1> at 16x16 over the concat of two producers (a decoder ResBlock's conv1), scale/shift; 536 tiles
    "gn64_halo16_concat_ss": dict(inst=(64, 1), N=67, H=16, W=16, Cout=256,
                                  segs=[("3x3", 128, "gn"), ("3x3", 128, "gn")], gn_ss=True, gn_per_sample=True,
                                  ebias="sample", stats=True),
    # up2 over a 16x16 source with the GroupNorm finalised in the kernel (ADM up ResBlock conv1); 400 tiles
    "up2_gn": dict(up2=True, slots=8, bn=128, N=50, H=16, W=16, Cout=128, segs=[("3x3", 128, "gn")],
                   gn_per_sample=True, ebias="shared", stats=True, sums=True),
    # GroupNorm 3x3 segment + raw 1x1 shortcut (a ResBlock conv2 with cin != cout) at 64x64, <128,1>; 416 tiles
    "gn128_halo64_with_1x1": dict(inst=(128, 1), N=13, H=64, W=64, Cout=128,
                                  segs=[("3x3", 128, "gn"), ("1x1", 64, None)], gn_per_sample=True, ebias="sample",
                                  stats=True, sums=True),
}


@pytest.mark.parametrize("case", list(GN_CASES))
def test_in_kernel_groupnorm_past_one_wave(cuda_device, case):
    spec = GN_CASES[case]
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    H, W, Cout, N = spec["H"], spec["W"], spec["Cout"], spec["N"]
    if spec.get("up2"):
        per_sample, n_tiles = ops.conv_stats_tiles_up2(H, W, Cout) // 4, Cout // spec["bn"] * 4
    else:
        per_sample, n_tiles = ops.conv_stats_tiles(H, W, Cout, True), Cout // spec["inst"][0]
    m_tiles = N * per_sample
    tiles = m_tiles * n_tiles
    assert tiles >= 3 * sms + 1, f"{tiles} tiles on {sms} SMs"
    assert tiles % sms != 0, "every CTA would own the same number of tiles"
    # the kernel's tile order (channel tile, sample, row, column): tile t + grid follows tile t on the same CTA
    grid = min(tiles, sms)
    same = [t for t in range(tiles - grid) if (t % m_tiles) // per_sample == ((t + grid) % m_tiles) // per_sample]
    assert not same, f"tiles {same[:4]} and their successors on the same CTA lie in one sample"
    _run_case(spec, cuda_device, seed=400 + list(GN_CASES).index(case))
