"""The kernel plans the benchmark times, checked launch by launch and as a whole.

1. Every launch of one edit evaluation of each bench.WORKLOADS plan, at its benchmark batch, is checked against an fp64
   reference computed on the device from a snapshot of its inputs: the conv descriptors (3x3, 1x1, stride 2, up2, fused
   GroupNorm-affine+SiLU operands, per-sample bias, residual modes, device scales, weight-batched attention GEMMs,
   planar fp32 output, per-sample statistics), gn_finalize, apply, both attention paths, softmax_rows, transpose_tc, the
   timestep MLP, pack_input and slerp_h; plus the explicit-delta_h path (mask off and on) and the ignore_timestep
   DeltaBlock conv.  Each launch must not write into its inputs, must leave them unchanged, and must write every
   element of its outputs (they are NaN-filled before it runs).
2. Buffer reuse (Pool) and the concurrent decoder pass change nothing: the production engine (pooled buffers, two
   streams, CUDA graph) equals an engine whose buffers are never reused, run serially without a graph, bit for bit.
3. A sample's trajectory at the benchmark batch equals its B=1 trajectory bit for bit and stays within the golden
   tolerance of the reference's own output.

Tolerances (relative to max|ref| of the compared sample, or of the (sample, head) entry of a batched GEMM) are those of
test_conv_coverage_gpu.py: conv 1.5e-3 raw, 2.5e-3 fused operand or up2, 3e-3 fused up2, 2e-5 fp32 output of raw
operands; statistics 2e-3 (3e-3 up2).  The pointwise kernels use the bounds of their kernel tests: gn_finalize 1e-4,
apply 1e-3, scalar attention 1.5e-3, softmax 6e-4 absolute, linear 1e-5, timestep embedding 2e-4 absolute, slerp 1e-3
(statistics 2e-3); transpose and pack_input are exact.
"""
import math
import os
import time
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bench
from asyrp_official_b200 import engine, modules, ops, synthetic
from asyrp_official_b200.schedule import Schedule, make_sequences
from oracle import adm as oa, ddpm as od, sampler as osmp

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")

TOL_RAW, TOL_FUSED, TOL_FUSED_UP2, TOL_F32, TOL_STATS = 1.5e-3, 2.5e-3, 3e-3, 2e-5, 2e-3
TOL_GN, TOL_APPLY, TOL_ATTN, TOL_SOFTMAX_ABS, TOL_LINEAR, TOL_TEMB_ABS, TOL_SLERP = \
    1e-4, 1e-3, 1.5e-3, 6e-4, 1e-5, 2e-4, 1e-3
TOL_GN_FOLD = 3e-3  # test_conv_coverage_gpu.py: GroupNorm finalised inside the consuming conv
TOL_TRAJ = 1e-3  # test_model_gpu.py: N-step x_0 vs the reference's own output
# fp64 work (multiply-adds) per launch above which only samples 0, B//2 and B-1 are compared
FULL_BATCH_MACS = 1 << 36

WORKLOADS = list(bench.WORKLOADS)
ENTRY_POINTS = {"ConvOp", "gn_finalize", "apply", "attention", "softmax_rows", "transpose_tc", "linear",
                "timestep_embedding", "pack_input", "slerp_h"}
# (kernel, shape) pairs the plans reach that the synthetic suites only sample
REQUIRED_TAGS = {
    "ddpm_celeba_b16": {"attention T=64 heads=1 d=512", "gemm S heads=1 T=256"},
    "ddpm_church_b32": {"attention T=64 heads=1 d=512", "gemm S heads=1 T=256"},
    "iddpm_afhq_b8": {"attention T=64 heads=8 d=64", "gemm S heads=8 T=256"},
    "adm_imagenet_b4": {"attention T=64 heads=16 d=64", "gemm S heads=8 T=1024", "gemm S heads=16 T=256",
                        "softmax_rows rows=32768 T=1024", "gn_finalize C=1024+1024",
                        "apply C=1024 at 1024 of 2048"},
}


# ------------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------------
def _model(workload, dev):
    """the workload's UNet as test_model_gpu.py builds it for the goldens: torch-default random init (seed 1234) and
    the shipped DeltaBlock (seeded random for ImageNet, which ships none)"""
    family, key, _, _, ckpt, _ = bench.WORKLOADS[workload]
    if family == "ddpm":  # LSUN-Church uses the CelebA-HQ UNet
        cfg = od.CELEBA_CFG
        m = modules.DDPM(NS(model=NS(**{**cfg, "dropout": 0.0, "resamp_with_conv": True}),
                            data=NS(image_size=cfg["image_size"])))
    else:
        m = modules._create_adm({"afhq": oa.AFHQ_HP, "imagenet": oa.IMAGENET_HP}[key])
    m.setattr_layers(1)
    synthetic.randomize_(m, 1234, "torch_default")
    if ckpt:
        sd = torch.load(os.path.join(G, "checkpoint", ckpt), map_location="cpu", weights_only=True)["0"]
        m.layer_0.load_state_dict(sd)
    return m.to(dev)


# ------------------------------------------------------------------------------------------------------------------
# launch recorder
# ------------------------------------------------------------------------------------------------------------------
def _extent(t):
    """[first byte, last byte + 1) of the memory a strided view addresses"""
    lo = t.data_ptr()
    span = sum((s - 1) * st for s, st in zip(t.shape, t.stride()) if s > 0) + 1
    return lo, lo + span * t.element_size()


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _silu(y):
    return y * torch.sigmoid(y)


def _h32(y):
    """an fp32-evaluated operand rounded to fp16, as the kernels store it"""
    return y.float().half().double()


def _pair_stats(ref):
    """[n][C][H][W] -> [n][C/2][2] (sum, sum of squares) per channel pair"""
    n, c = ref.shape[:2]
    r = ref.reshape(n, c // 2, 2, -1)
    return torch.stack([r.sum(dim=(2, 3)), (r * r).sum(dim=(2, 3))], dim=-1)


class Recorder:
    """Wraps the kernel entry points.  Each wrapped launch asserts that its outputs do not overlap its inputs, snapshots
    the inputs, NaN-fills the outputs, launches, synchronises, and checks: every output element written, every input
    bit-for-bit unchanged, the outputs equal to an fp64 reference of the snapshot."""

    def __init__(self, B):
        self.B = B
        self.checks = 0
        self.entries = set()
        self.tags = set()
        self.worst = []     # (margin, index, desc, what, rel err, tol)
        self.label = (None, "")
        self.last_conv = None  # the ConvOp of the latest conv launch

    def samples(self, macs_per_sample):
        B = self.B
        if B * macs_per_sample <= FULL_BATCH_MACS:
            return list(range(B))
        return sorted({0, B // 2, B - 1})

    def compare(self, what, got, want, tol, absolute=False, ids=None):
        """got / want [entries, ...]: per-entry max-abs error against tol (relative to that entry's max|want|); ids:
        the sample (or batch entry) each row is"""
        err = (got.double() - want).reshape(want.shape[0], -1).abs().amax(1)
        mag = want.reshape(want.shape[0], -1).abs().amax(1)
        bound = torch.full_like(mag, tol) if absolute else tol * mag + 1e-6
        rel = err / (torch.ones_like(mag) if absolute else mag.clamp_min(1e-30))
        k = int(torch.argmax(err / bound))
        idx, desc = self.label
        self.worst.append(((err[k] / bound[k]).item(), idx, desc, what, rel[k].item(), tol))
        bad = (err > bound).nonzero().flatten().tolist()
        assert not bad, (f"launch {idx} ({desc}) {what}: entries {[ids[b] if ids else b for b in bad[:8]]} exceed the tolerance {tol}"
                         f"{'' if absolute else ' x max|ref|'}: max-abs err {err[bad[0]].item():.3e}, "
                         f"max|ref| {mag[bad[0]].item():.3e}")

    def run(self, entry, inputs, outputs, launch, reference, tag=None):
        idx, desc = self.label
        ins = {k: v for k, v in inputs.items() if v is not None}
        outs = {k: v for k, v in outputs.items() if v is not None}
        for ko, o in outs.items():
            lo, hi = _extent(o)
            for ki, i in ins.items():
                a, b = _extent(i)
                assert hi <= a or b <= lo, f"launch {idx} ({desc}, {entry}): output {ko} overlaps input {ki}"
        snap = {k: v.clone() for k, v in ins.items()}
        for o in outs.values():
            o.fill_(float("nan"))
        launch()
        torch.cuda.synchronize()
        for k, o in outs.items():
            bad = (~torch.isfinite(o)).sum().item()
            assert bad == 0, f"launch {idx} ({desc}, {entry}): {bad} of {o.numel()} elements of {k} not written"
        for k, i in ins.items():
            assert torch.equal(_bits(i), _bits(snap[k])), f"launch {idx} ({desc}, {entry}): input {k} was modified"
        reference(snap, outs)
        self.checks += 1
        self.entries.add(entry)
        if tag:
            self.tags.add(tag)

    # ---------------------------------------------------------------------------------------------- conv
    def seg_inputs(self, i, aff):
        """the tensors segment i's operand transform reads (snapshotted, checked unchanged)"""
        assert not isinstance(aff, ops.GNSpec), "in-kernel GroupNorm operands are not part of the default plans"
        return {f"aff{i}": aff}

    def seg_affine(self, snap, i, aff, off, C, idx):
        """(a, b), each [samples idx][C], of segment i's operand transform y = a*x + b, from the snapshot"""
        ab = snap[f"aff{i}"][idx].double()[:, off:off + C]
        return ab[..., 0], ab[..., 1]

    def conv(self, op):
        segs, weight, kw = op._rec
        if kw.get("weight_batched"):
            return self._gemm(op)
        N = self.B
        up2 = bool(kw.get("up2"))
        out, planar = kw.get("out"), kw.get("out_planar")
        if out is not None:
            _, Ho, Wo, Cout = out.shape
        else:
            _, Ho, Wo, Cout = kw["out_shape"]
        ins = {"weight": weight, "residual": kw.get("residual"), "scales": kw.get("scales")}
        eb = kw.get("ebias")
        if eb is not None:
            st = kw.get("ebias_stride", 0)
            ins["ebias"] = torch.as_strided(eb, (N, Cout), (st, 1), eb.storage_offset())
        for i, (src, mode, aff, off, act) in enumerate(segs):
            ins[f"src{i}"] = src
            if aff is not None:
                ins.update(self.seg_inputs(i, aff))
        outs = {"out": out, "stats": kw.get("stats"), "out_planar": planar}
        ktot = weight.shape[-1]
        ns = self.samples(Ho * Wo * Cout * ktot)
        fused = any(sg[2] is not None for sg in segs)
        tol = (TOL_FUSED_UP2 if fused else TOL_FUSED) if up2 else \
            (TOL_FUSED if fused else (TOL_F32 if planar is not None or out.dtype == torch.float32 else TOL_RAW))
        if any(isinstance(sg[2], ops.GNSpec) for sg in segs):
            tol = TOL_GN_FOLD

        def reference(snap, got):
            idx = torch.tensor(ns, device=weight.device)
            w_all = snap["weight"].double()
            acc, k0 = 0.0, 0
            for i, (src, mode, aff, off, act) in enumerate(segs):
                y = _nchw(snap[f"src{i}"][idx])
                C = y.shape[1]
                if aff is not None:
                    a, b = self.seg_affine(snap, i, aff, off, C, idx)
                    y = y * a[..., None, None] + b[..., None, None]
                    if act:
                        y = _silu(y)
                    y = _h32(y)
                taps = 1 if mode == ops.MODE_1x1 else (4 if up2 else 9)
                w = w_all[:, k0:k0 + taps * C]
                k0 += taps * C
                if up2:
                    H, W = y.shape[2:]
                    yp = F.pad(y, (1, 1, 1, 1))
                    o = y.new_empty(len(ns), Cout, 2 * H, 2 * W)
                    for a in (0, 1):
                        for b in (0, 1):
                            wp = w[(2 * a + b) * Cout:(2 * a + b + 1) * Cout].reshape(Cout, 2, 2, C).permute(0, 3, 1, 2)
                            o[:, :, a::2, b::2] = F.conv2d(yp[:, :, a:a + H + 1, b:b + W + 1], wp)
                elif mode == ops.MODE_1x1:
                    o = F.conv2d(y, w.reshape(Cout, C, 1, 1))
                else:
                    w3 = w.reshape(Cout, 3, 3, C).permute(0, 3, 1, 2)
                    o = F.conv2d(F.pad(y, (0, 1, 0, 1)), w3, stride=2) if mode == ops.MODE_3x3_S2 else \
                        F.conv2d(y, w3, padding=1)
                acc = acc + o
            assert k0 == ktot
            if "ebias" in snap:
                acc = acc + snap["ebias"][idx].double()[:, :, None, None]
            acc_s, res_s = kw.get("acc_scale", 1.0), kw.get("res_scale", 1.0)
            if "scales" in snap:
                acc_s, res_s = snap["scales"][0].item(), snap["scales"][1].item()
            acc = acc * acc_s
            if "residual" in snap:
                r = _nchw(snap["residual"][idx])
                rm = kw.get("res_mode", 0)
                r = F.interpolate(r, scale_factor=2, mode="nearest") if rm == 1 else (F.avg_pool2d(r, 2) if rm == 2 else r)
                acc = acc + res_s * r
            if planar is not None:
                self.compare("planar out", got["out_planar"][idx], acc[:, :planar.shape[1]], tol, ids=ns)
            else:
                self.compare("out", _nchw(got["out"][idx]), acc, tol, ids=ns)
            if "stats" in got:
                self.compare("stats", got["stats"][idx].double().sum(1), _pair_stats(acc),
                             TOL_STATS * (1.5 if up2 else 1.0), ids=ns)

        self.last_conv = op
        self.run("ConvOp", ins, outs, lambda: _BaseConvOp.launch(op), reference)

    def _gemm(self, op):
        """weight-batched GEMM: batch entry e = (sample, head) computes out_e[t][o] = sum_k A_e[t][k] * W_e[o][k]"""
        segs, weight, kw = op._rec
        assert len(segs) == 1 and segs[0][1] == ops.MODE_1x1 and segs[0][2] is None
        src = segs[0][0]
        out = kw["out"]
        ah, bh, oh = kw.get("a_heads", 1), kw.get("b_heads", 1), kw.get("out_heads", 1)
        No, Ho, Wo, Cw = out.shape
        Nb, Cout, T = No * oh, Cw // oh, Ho * Wo
        Na, _, _, K = src.shape
        assert Na * ah == Nb and weight.dim() == 3 and weight.shape[0] * bh == Nb and weight.shape[-1] == K
        a_eff = torch.as_strided(src, (Na, ah, T, K), (src.stride(0), K, src.stride(2), 1), src.storage_offset())
        w_eff = torch.as_strided(weight, (weight.shape[0], bh, Cout, K), (weight.stride(0), K, weight.stride(1), 1),
                                 weight.storage_offset())
        heads = Nb // self.B
        ns = self.samples(heads * T * Cout * K)
        ents = [n * heads + h for n in ns for h in range(heads)]
        tol = TOL_F32 if out.dtype == torch.float32 else TOL_RAW

        def reference(snap, got):
            e = torch.tensor(ents, device=out.device)
            A = snap["A"].reshape(Nb, T, K)[e].double()
            Wm = snap["W"].reshape(Nb, Cout, K)[e].double()
            o = got["out"].view(No, T, oh, Cout).permute(0, 2, 1, 3).reshape(Nb, T, Cout)[e]
            self.compare("gemm out", o, A @ Wm.transpose(1, 2), tol, ids=ents)

        what = "S" if out.dtype == torch.float32 else "O"
        self.last_conv = op
        self.run("ConvOp", {"A": a_eff, "W": w_eff}, {"out": out}, lambda: _BaseConvOp.launch(op), reference,
                 tag=f"gemm {what} heads={heads} T={T}")

    # ---------------------------------------------------------------------------------------------- the rest
    def gn_finalize(self, stats_a, Ca, stats_b, Cb, gamma, beta, eps, N, HW, affine, scale_shift=None, ss_stride=0):
        C = Ca + Cb
        ins = {"stats_a": stats_a, "stats_b": stats_b, "gamma": gamma, "beta": beta}
        if scale_shift is not None:
            ins["ss"] = torch.as_strided(scale_shift, (N, 2 * C), (ss_stride, 1), scale_shift.storage_offset())

        def reference(snap, got):
            pairs = [snap["stats_a"].double().sum(1)]  # [N][C/2][2]
            if stats_b is not None:
                pairs.append(snap["stats_b"].double().sum(1))
            s = torch.cat(pairs, 1).reshape(N, 32, -1, 2).sum(2)  # groups straddle the concat seam
            cnt = HW * (C // 32)
            mean = s[..., 0] / cnt
            var = (s[..., 1] / cnt - mean * mean).clamp_min(0.0)
            rstd = 1.0 / torch.sqrt(var + eps)
            mean_c, rstd_c = mean.repeat_interleave(C // 32, 1), rstd.repeat_interleave(C // 32, 1)
            a = snap["gamma"].double() * rstd_c
            b = snap["beta"].double() - mean_c * a
            if "ss" in snap:
                ss = snap["ss"].double()
                a, b = a * (1 + ss[:, :C]), b * (1 + ss[:, :C]) + ss[:, C:]
            self.compare("gn a", got["affine"][..., 0], a, TOL_GN)
            self.compare("gn b", got["affine"][..., 1], b, TOL_GN)

        self.run("gn_finalize", ins, {"affine": affine},
                 lambda: _ORIG["gn_finalize"](stats_a, Ca, stats_b, Cb, gamma, beta, eps, N, HW, affine, scale_shift,
                                              ss_stride),
                 reference, tag=f"gn_finalize C={Ca}+{Cb}" if Cb else f"gn_finalize C={Ca}")

    def apply(self, src_a, src_b, affine, out, act, resample=ops.RESAMPLE_NONE, affine_offset=0):
        C = src_a.shape[-1] + (src_b.shape[-1] if src_b is not None else 0)
        ns = self.samples(out[0].numel())

        def reference(snap, got):
            idx = torch.tensor(ns, device=out.device)
            x = _nchw(snap["a"][idx])
            if src_b is not None:
                x = torch.cat([x, _nchw(snap["b"][idx])], 1)
            if affine is not None:
                ab = snap["affine"][idx].double()[:, affine_offset:affine_offset + C]
                x = x * ab[..., 0, None, None] + ab[..., 1, None, None]
            if act:
                x = _silu(x)
            if resample == ops.RESAMPLE_AVGPOOL2:
                x = F.avg_pool2d(x, 2)
            elif resample == ops.RESAMPLE_UP2:
                x = F.interpolate(x, scale_factor=2, mode="nearest")
            self.compare("apply", _nchw(got["out"][idx]), x, TOL_APPLY, ids=ns)

        tag = f"apply C={C} at {affine_offset} of {affine.shape[1]}" if affine is not None else f"apply C={C}"
        self.run("apply", {"a": src_a, "b": src_b, "affine": affine}, {"out": out},
                 lambda: _ORIG["apply"](src_a, src_b, affine, out, act, resample, affine_offset), reference, tag=tag)

    def attention(self, qkv, out, heads, head_dim, scale):
        N, T, C3 = qkv.shape
        C = C3 // 3

        def reference(snap, got):
            q, k, v = (snap["qkv"].double()[:, :, i * C:(i + 1) * C].reshape(N, T, heads, head_dim).transpose(1, 2)
                       for i in range(3))
            p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
            self.compare("attention", got["out"], (p @ v).transpose(1, 2).reshape(N, T, C), TOL_ATTN)

        self.run("attention", {"qkv": qkv}, {"out": out},
                 lambda: _ORIG["attention"](qkv, out, heads, head_dim, scale), reference,
                 tag=f"attention T={T} heads={heads} d={head_dim}")

    def softmax_rows(self, S, P, scale):
        T = S.shape[-1]

        def reference(snap, got):
            want = torch.softmax(snap["S"].double() * scale, dim=-1)
            self.compare("softmax", got["P"].reshape(S.shape[0], -1), want.reshape(S.shape[0], -1), TOL_SOFTMAX_ABS,
                         absolute=True)

        self.run("softmax_rows", {"S": S}, {"P": P}, lambda: _ORIG["softmax_rows"](S, P, scale), reference,
                 tag=f"softmax_rows rows={S.numel() // T} T={T}")

    def transpose_tc(self, inp, out):
        def reference(snap, got):
            assert torch.equal(got["out"], snap["in"].transpose(1, 2)), f"launch {self.label}: transpose_tc"

        self.run("transpose_tc", {"in": inp}, {"out": out}, lambda: _ORIG["transpose_tc"](inp, out), reference)

    def linear(self, inp, weight, bias, out, act_in=False, act_out=False):
        O = weight.shape[0]

        def reference(snap, got):
            x = snap["in"].double()
            y = (_silu(x) if act_in else x) @ snap["w"].double().t() + snap["b"].double()
            self.compare("linear", got["out"][:, :O], _silu(y) if act_out else y, TOL_LINEAR)

        self.run("linear", {"in": inp, "w": weight, "b": bias}, {"out": out},
                 lambda: _ORIG["linear"](inp, weight, bias, out, act_in=act_in, act_out=act_out), reference)

    def timestep_embedding(self, t, out, variant):
        def reference(snap, got):
            half = out.shape[1] // 2
            i = torch.arange(half, dtype=torch.float32, device=t.device)
            fr = torch.exp(i * -(math.log(10000) / (half - 1))) if variant == 0 else \
                torch.exp(-math.log(10000) * i / half)  # the reference's fp32 frequencies
            e = snap["t"].double()[:, None] * fr.double()[None]
            want = torch.cat([e.sin(), e.cos()] if variant == 0 else [e.cos(), e.sin()], 1)
            self.compare("timestep embedding", got["out"], want, TOL_TEMB_ABS, absolute=True)

        self.run("timestep_embedding", {"t": t}, {"out": out},
                 lambda: _ORIG["timestep_embedding"](t, out, variant), reference)

    def pack_input(self, x, out):
        def reference(snap, got):
            want = torch.zeros_like(got["out"])
            want[..., :x.shape[1]] = snap["x"].permute(0, 2, 3, 1).half()
            assert torch.equal(got["out"], want), f"launch {self.label}: pack_input"

        self.run("pack_input", {"x": x}, {"out": out}, lambda: _ORIG["pack_input"](x, out), reference)

    def slerp_h(self, h, dh, h2, stats, t, use_mask=False):
        def reference(snap, got):
            hd = _nchw(snap["h"])
            N, C, H, W = hd.shape
            dhd = snap["dh"].double().expand(N, C, H, W)
            if use_mask:
                mask = torch.zeros_like(hd)
                mask[:, :, 4:H - 1, 3:5] = 1.0
                want = od.slerp(t, hd * mask, dhd * mask) + (1 - mask) * hd
            else:
                hn = torch.norm(hd.reshape(N, -1), dim=1)[:, None, None, None]
                dn = torch.norm(dhd.reshape(N, -1), dim=1)[:, None, None, None]
                want = od.slerp(t, hd, hn * dhd / dn)
            self.compare("slerp h2", _nchw(got["h2"]), want, TOL_SLERP)
            self.compare("slerp stats", got["stats"][:, 0], _pair_stats(want), TOL_STATS)
            assert not got["stats"][:, 1:].any(), f"launch {self.label}: slerp_h slots other than 0 not zero"

        self.run("slerp_h", {"h": h, "dh": dh}, {"h2": h2, "stats": stats},
                 lambda: _ORIG["slerp_h"](h, dh, h2, stats, t, use_mask), reference,
                 tag=f"slerp_h mask={int(bool(use_mask))}")


_BaseConvOp = ops.ConvOp
_WRAPPED = ("gn_finalize", "apply", "attention", "softmax_rows", "transpose_tc", "linear", "timestep_embedding",
            "pack_input", "slerp_h")
_ORIG = {name: getattr(ops, name) for name in _WRAPPED}


def _install(monkeypatch, rec):
    class RecordingConvOp(_BaseConvOp):
        def __init__(self, segs, weight, **kw):
            super().__init__(segs, weight, **kw)
            segs = [tuple(sg) + (None, 0, 0) * (len(sg) == 2) for sg in segs]
            self._rec = (segs, weight, kw)

        def launch(self):
            rec.conv(self)

        __call__ = launch

    monkeypatch.setattr(ops, "ConvOp", RecordingConvOp)
    for name in _WRAPPED:
        monkeypatch.setattr(ops, name, getattr(rec, name))


def _drive(rec, launches, first_index=0):
    """run each launch once; each must trigger exactly one check.  Returns the ConvOp each conv launch ran"""
    convs = {}
    for i, L in enumerate(launches):
        rec.label = (first_index + i, L.desc)
        before = rec.checks
        rec.last_conv = None
        L()
        assert rec.checks == before + 1, f"launch {first_index + i} ({L.desc}) triggered {rec.checks - before} checks"
        convs[L] = rec.last_conv
    return convs


@pytest.mark.parametrize("workload", WORKLOADS)
def test_every_launch_of_the_benchmark_plan_vs_fp64(cuda_device, monkeypatch, workload):
    """one edit evaluation of the benchmark plan, driven launch by launch, then the explicit-delta_h path (mask off and
    on) and the ignore_timestep DeltaBlock conv: every launch triggers exactly one recorded check"""
    assert not engine.GN_FOLD, "the default plans finalise GroupNorm in gn_finalize launches"
    t0 = time.perf_counter()
    dev = cuda_device
    B = bench.WORKLOADS[workload][2]
    m = _model(workload, dev)
    rec = Recorder(B)
    _install(monkeypatch, rec)
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    P = eng.plan(B)
    g = torch.Generator().manual_seed(31)
    # distinct timesteps per sample: every per-sample embedding row, bias and scale/shift differs
    P.x.copy_(torch.randn(P.x.shape, generator=g))
    P.t.copy_(torch.linspace(999.0, 500.0, B))
    P.set_coeffs((0.9, 1.3))
    eng.state.update(ignore_timestep=False, slerp_t=0.0, use_mask=False)
    seq = P.launches(edit=True)
    convs = _drive(rec, seq)
    n = len(seq)
    # explicit delta_h: h2 = slerp(t, h, |h| dh/|dh|) into the DeltaBlock's h2 buffer, then the edited decoder
    P.dh_user.copy_(torch.randn(P.dh_user.shape, generator=g) * 2.0)
    eng.state["slerp_t"] = 0.3
    for use_mask in (False, True):
        eng.state["use_mask"] = use_mask
        _drive(rec, P.slerp_ops + P.dec_mod_ops, n)
        n += len(P.slerp_ops) + len(P.dec_mod_ops)
    # the ignore_timestep variant of the DeltaBlock's first conv: the shared conv bias instead of the embedding row
    (sel,) = [L for L in P.delta_ops if L.kind == "conv" and L.desc == "conv"]
    op_t = convs[sel]
    assert op_t._rec[2].get("ebias_stride", 0) == eng.emb_total
    eng.state["ignore_timestep"] = True
    op_nt = _drive(rec, [sel], n)[sel]
    assert op_nt is not op_t and op_nt._rec[2].get("ebias_stride", 0) == 0
    expected = len(seq) + 2 * (len(P.slerp_ops) + len(P.dec_mod_ops)) + 1
    assert rec.checks == expected, (rec.checks, expected)
    assert rec.entries == ENTRY_POINTS, rec.entries ^ ENTRY_POINTS
    missing = REQUIRED_TAGS[workload] - rec.tags
    assert not missing, f"{workload}: the plan no longer reaches {missing}"
    worst = sorted(rec.worst, key=lambda w: -w[0])[:3]
    print(f"\n{workload} B={B}: {rec.checks} launches checked ({len(seq)} edit evaluation + "
          f"{expected - len(seq)} explicit-delta_h / ignore_timestep), {time.perf_counter() - t0:.1f} s; worst: " +
          "; ".join(f"#{i} {d} {w}: {r:.2e} (tol {tol:g}, {mg:.2f} of it)" for mg, i, d, w, r, tol in worst))
    monkeypatch.undo()
    del P, eng, m, rec, convs, op_t, op_nt
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# buffer reuse and the concurrent decoder pass
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["ddpm_celeba", "ddpm_church", "adm_afhq", "adm_imagenet"])
def test_buffer_reuse_and_concurrent_decoder_change_nothing(cuda_device, monkeypatch, arch):
    """production engine (pooled buffers, decoder passes on two streams, CUDA graph) == an engine whose plan never
    reuses a buffer, run on one stream without a graph, bit for bit"""
    dev = cuda_device
    workload = {"ddpm_celeba": "ddpm_celeba_b16", "ddpm_church": "ddpm_church_b32", "adm_afhq": "iddpm_afhq_b8",
                "adm_imagenet": "adm_imagenet_b4"}[arch]
    m = _model(workload, dev)
    B = 2
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

    prod = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    assert engine.DUAL_STREAM
    a = prod.sample(x, sch, noise=noise, use_graph=True)
    a_dh = prod.sample(x, sch_dh, noise=noise, use_graph=True, delta_hs=dh)

    monkeypatch.setattr(engine.Pool, "release", lambda self, t: None)
    ref = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    P = ref.plan(B)
    monkeypatch.undo()
    assert P.pool.total > prod.plan(B).pool.total, "the reference plan reuses buffers"
    monkeypatch.setattr(engine, "DUAL_STREAM", False)
    b = ref.sample(x, sch, noise=noise, use_graph=False)
    b_dh = ref.sample(x, sch_dh, noise=noise, use_graph=False, delta_hs=dh)
    assert torch.isfinite(a).all() and torch.isfinite(a_dh).all()
    assert not torch.equal(a, a_dh)
    assert torch.equal(a, b), f"{arch}: DeltaBlock schedule differs by {(a - b).abs().max().item():.3e}"
    assert torch.equal(a_dh, b_dh), f"{arch}: explicit-delta_h schedule differs by {(a_dh - b_dh).abs().max().item():.3e}"
    del P, ref, prod, m
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# batch sharding at the benchmark batch
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("workload", WORKLOADS)
def test_benchmark_batch_reproduces_the_reference_row_for_row(cuda_device, workload):
    """the golden fixture's samples in the last rows of a benchmark-size batch (the other rows seeded random): row B-1
    is bit-identical to its B=1 trajectory (the batch-sharding contract bench.py states) and the fixture's rows are
    within TOL_TRAJ of the reference's own output"""
    dev = cuda_device
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
    eng = m.engine
    one = eng.sample(xb[B - 1:].to(dev), sch, noise=nzb[:, B - 1:].contiguous().to(dev))
    full = eng.sample(xb.to(dev), sch, noise=nzb.to(dev))
    row = full[B - 1:]
    e = (full[B - Bg:, :, ::4, ::4].double().cpu() - torch.from_numpy(gold["x0_sub"]).double()).abs().max().item()
    mx = float(np.abs(gold["x0_sub"]).max())
    print(f"\n{workload}: rows {B - Bg}..{B - 1} of {B} vs the reference: max-abs {e:.4f} of max|x_0| {mx:.2f} -> "
          f"{e / mx:.2e}")
    assert torch.equal(row, one), f"{workload}: row {B - 1} of a batch of {B} differs from its B=1 run by " \
                                  f"{(row - one).abs().max().item():.3e}"
    assert e <= TOL_TRAJ * mx, f"{workload}: max-abs err {e:.3e} of max|ref| {mx:.3e}"
    del eng, m
    torch.cuda.empty_cache()
