"""The face-parsing kernels (csrc/face_parsing.cu) at the limits their entry points admit.

  * Every ASYRP_REQUIRE of the seven asyrp_faceparse_* entry points has a row in REFUSALS: the refused call (made
    through the C ABI, since the ops wrappers assert shapes first) raises AsyrpError naming the entry point and leaves
    a NaN-filled output (a sentinel-filled one for labels and agree) untouched, and its nearest accepted neighbour
    launches and is checked.  Compound shape conditions get a row per clause:
      pack: B, H, W, S = 0.  conv: Cin = 6 and 0, Cout = 96, H + 2 pad = k - 1 (accepted: = k), stride 0, relu = 2,
      a residual without the ReLU, the ReLU with neither bias nor residual, in == out, and the M guard
      N Ho Wo >= 2^31 / 128 * 128 (tiny buffers: the refusal comes before any read; the accepted side, 2^31 - 1
      output pixels, cannot be allocated, so that row has no accepted neighbour).  maxpool: C = 6.  gate: C = 48,
      1024 and 0, C1 = 0 and 513, C2 = 513 with w2, act1 / act2 = 3 and -1, HW = 0, N = 0.  apply: up = 3,
      add_map = 2, C = 6, out == f, out == add.  labels: N = 65536 (accepted 65535), ncls = 65, ld < ncls,
      Wi ncls = 12289 (accepted 12288).  agreement: n = 65536, row0 = -1, B = 0, Wi ncls = 6145 (accepted 6144).
    Not tabled, with the reason: the remaining positivity clauses of the shape conditions (maxpool N, H, W; apply N,
    H, W; labels / agreement Hi, Wi, Ho, Wo; conv N, k, pad, W + 2 pad >= k) share the message and the branch of a
    tabled clause of the same REQUIRE; the conv's Cout % 64 and Cin % 4 clauses are tabled through Cout = 96 and
    Cin = 6.
  * The largest admitted shapes and the edges of each kernel against references: the TF32 conv against TF32-rounded
    operands (round to nearest, ties away, as cvt.rna) summed in fp64, within (Kpad/8 + 2) u (|a_t| @ |b_t|) plus a
    few u of the bias, residual and result, and exactly where one weight per output channel is non-zero; the gate at
    every C dividing 512 within (ceil(HW/J) + J + ceil(C/32) + C1 + 16) u of the magnitudes (1/4 of that through a
    sigmoid); the upsample-argmax kernels bit for bit on every pixel against an fp32 restatement of their explicitly
    rounded arithmetic; pack within the first-order error of its fp32 source position; max-pool and apply exactly.
  * Outputs past 2^31 elements: pack (8 GiB), labels (2.1 GB of uint8) and apply (8 GiB), from tiny or integer
    inputs, compared exactly on the first and last sample and every k-th between.

u = 2^-24 throughout.  Outputs sit in front of a NaN (or sentinel) tail that must stay so.  Large cases check free
device memory first and skip, naming the amount they need, when it is short.  The whole file takes about 19 s on an
NVIDIA H100 80GB HBM3 at a 700 W power limit (6 s of it in the tests, the rest collection), with a peak of 10.07 GiB
of device memory (torch.cuda.max_memory_allocated), in test_apply_past_2_to_the_31_elements.  asyrp_faceparse_agreement launches with
2 Wi ncls floats of dynamic shared memory next to its kernel's 32 bytes of static warp_same[]: from Wi ncls = 6141 on
that passes the default 48 KB per block, so the entry points opt in to the 48 KB they admit
(test_agreement_at_the_shared_memory_limit).  NaN inputs are out of scope: fminf / fmaxf in pack's clamp, the ReLU
epilogues and max-pool drop a NaN where torch propagates it.
"""
import itertools
import math
import re
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from asyrp_official_b200 import _lib, ops

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
NAN = float("nan")
GiB = float(1 << 30)
TAIL = 64
BIG = 65536  # one past the largest grid y dimension
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
WORST = {}  # kernel -> worst err / bound seen, printed at the end of the file (pytest -s)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _p(t):
    return ops._ptr(t)


def _st():
    return ops._stream()


def _tf32(x):
    """round fp32 to TF32, to nearest with ties away from zero (cvt.rna.tf32.f32), as fp64"""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


def _need_memory(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + GiB // 2:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")


SENTINEL = {torch.float32: NAN, torch.uint8: 255, torch.int32: -1}


def _buf(shape, dev, dtype=torch.float32):
    """(whole buffer, front view of `shape`): the buffer holds TAIL more elements, all of it sentinel-filled"""
    n = math.prod(shape)
    full = torch.full((n + TAIL,), SENTINEL[dtype], dtype=dtype, device=dev)
    return full, full[:n].view(shape)


def _untouched(t):
    return bool(torch.isnan(t).all()) if t.dtype == torch.float32 else bool((t == SENTINEL[t.dtype]).all())


def _tail_ok(full, n):
    assert _untouched(full[n:]), "written past the output"
    front = full[:n]
    if front.dtype == torch.float32:
        assert not torch.isnan(front).any(), "output not written"


def _record(kernel, ratio):
    WORST[kernel] = max(WORST.get(kernel, 0.0), ratio)


def _within(kernel, err, bound, what=""):
    ratio = (err / bound).max().item()
    _record(kernel, ratio)
    assert (err <= bound).all(), f"{kernel} {what}: error {ratio:.3g}x the bound"


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def _conv_ref(x, w, stride, pad):
    """x [N][H][W][Cin], w [Cout][Cin][k][k] fp32 -> (TF32-operand conv in fp64, |a_t| @ |b_t|), NHWC"""
    xt, wt = _tf32(x.cpu()).permute(0, 3, 1, 2), _tf32(w.cpu())
    z = F.conv2d(xt, wt, stride=stride, padding=pad).permute(0, 2, 3, 1)
    s = F.conv2d(xt.abs(), wt.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return z, s


def _ac_taps(n_in, n_out):
    """ac_taps of csrc/face_parsing.cu in fp32: s = o * ((in - 1) / (out - 1)), i0 = min(floor s, in - 1),
    i1 = min(i0 + 1, in - 1), l = s - i0"""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    s = torch.arange(n_out, dtype=torch.float32) * torch.tensor(scale, dtype=torch.float32)
    i0 = s.long().clamp(max=n_in - 1)  # s >= 0: truncation is floor
    i1 = (i0 + 1).clamp(max=n_in - 1)
    return i0, i1, s - i0.float()


def _lerp(a, b, l):
    """lerp_rn: fl(fl(fl(1 - l) a) + fl(l b)), every operation rounded to fp32 (torch's CPU ops do not fuse)"""
    return (1 - l) * a + l * b


def _labels_ref(lg, ncls, Ho, Wo):
    """the upsample-argmax kernel restated in fp32 on the CPU: rows blended first, then columns, argmax with the
    first class winning a tie; lg [N][Hi][Wi][ld] -> uint8 [N][Ho][Wo]"""
    lg = lg.cpu().float()[..., :ncls]
    N, Hi, Wi, _ = lg.shape
    y0, y1, ly = _ac_taps(Hi, Ho)
    x0, x1, lx = _ac_taps(Wi, Wo)
    out = torch.empty(N, Ho, Wo, dtype=torch.uint8)
    step = max(1, (1 << 24) // max(1, N * max(Wo, Wi) * ncls))
    for a in range(0, Ho, step):
        sl = slice(a, min(Ho, a + step))
        rows = _lerp(lg[:, y0[sl]], lg[:, y1[sl]], ly[sl].view(1, -1, 1, 1))
        v = _lerp(rows[:, :, x0], rows[:, :, x1], lx.view(1, 1, -1, 1))
        out[:, sl] = v.argmax(-1).to(torch.uint8)  # torch.argmax returns the first maximal index
    return out


def _agreement_ref(src, edited, ncls, Ho, Wo, row0):
    B, n = src.shape[0], edited.shape[0]
    ls, le = _labels_ref(src, ncls, Ho, Wo), _labels_ref(edited, ncls, Ho, Wo)
    return (le == ls[(row0 + torch.arange(n)) % B]).flatten(1).sum(1)


def _pack_ref(x, S):
    """fp64: clamp, [0, 1], F.interpolate(bilinear, align_corners=False) to S x S, ImageNet normalisation, NHWC"""
    v = F.interpolate(x.double().cpu().clamp(-1, 1) * 0.5 + 0.5, (S, S), mode="bilinear", align_corners=False)
    v = (v - torch.tensor(MEAN, dtype=torch.float64).view(1, 3, 1, 1)) / torch.tensor(STD, dtype=torch.float64).view(
        1, 3, 1, 1)
    return v.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------------------------
# refusals: one row per ASYRP_REQUIRE clause; each maker returns (call, outputs that must stay untouched, check)
# ------------------------------------------------------------------------------------------------------------------
def _pack(dev, B=2, H=3, W=5, S=4):
    x = (torch.rand(max(B, 1), 3, max(H, 1), max(W, 1), generator=_g(1)) * 4 - 2).to(dev)
    full, out = _buf((max(B, 1), max(S, 1), max(S, 1), 4), dev)

    def check():
        _tail_ok(full, out.numel())
        ref = _pack_ref(x, S)
        assert (out[..., :3].double().cpu() - ref).abs().max().item() < 1e-5
        assert (out[..., 3] == 0).all()
    return lambda: _lib.load().asyrp_faceparse_pack(_p(x), _p(out), B, H, W, S, _st()), [full], check


def _conv(dev, N=1, H=4, W=4, Cin=4, Cout=64, k=3, stride=1, pad=1, relu=0, bias=True, res=False, alias=False,
          tiny=False):
    """a conv through the C ABI; tiny: buffers of one element (the call must refuse before any read)"""
    g = _g(2)
    if tiny:
        x, w, b = (torch.zeros(64, device=dev) for _ in range(3))
        out = torch.full((64,), NAN, device=dev)
        return (lambda: _lib.load().asyrp_faceparse_conv(_p(x), _p(w), _p(b), None, _p(out), N, H, W, Cin, Cout, k,
                                                         stride, pad, relu, _st()), [out], None)
    cin = max(Cin, 4)
    x = torch.randn(N, H, W, cin, generator=g)
    w = torch.randn(max(Cout, 64), cin, max(k, 1), max(k, 1), generator=g) / math.sqrt(cin * k * k)
    Ho = (H + 2 * pad - k) // max(stride, 1) + 1
    Wo = (W + 2 * pad - k) // max(stride, 1) + 1
    shape = (N, max(Ho, 1), max(Wo, 1), max(Cout, 64))
    bv = torch.randn(shape[-1], generator=g).to(dev) if bias else None
    rv = torch.randn(shape, generator=g).to(dev) if res else None
    xd = x.to(dev)
    wp = ops.pack_lpips_conv_weight(w).to(dev) if k > 0 else torch.zeros(64, device=dev)
    if alias:
        assert cin == shape[-1] and (H, W) == shape[1:3]
        xd.fill_(NAN)
        full, out = xd.view(-1), xd
    else:
        full, out = _buf(shape, dev)

    def check():
        _tail_ok(full, out.numel())
        z, s = _conv_ref(x, w, stride, pad)
        v = z + (bv.double().cpu() if bv is not None else 0)
        if rv is not None:
            v = v + rv.double().cpu()
        want = v.clamp_min(0) if relu else v
        bound = (wp.shape[1] / 8 + 2) * U * s + 4 * U * (v.abs() + (rv.double().cpu().abs() if rv is not None else 0)
                                                        + (bv.double().cpu().abs() if bv is not None else 0))
        _within("conv", (out.double().cpu() - want).abs(), bound, "accepted neighbour")
    return (lambda: _lib.load().asyrp_faceparse_conv(_p(xd), _p(wp), _p(bv), _p(rv), _p(out), N, H, W, Cin, Cout, k,
                                                     stride, pad, relu, _st()), [full], check)


def _maxpool(dev, C=4, N=2, H=5, W=6):
    x = torch.randn(N, H, W, max(C, 4), generator=_g(3)).to(dev)
    full, out = _buf((N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, max(C, 4)), dev)

    def check():
        _tail_ok(full, out.numel())
        want = F.max_pool2d(x.cpu().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
        assert torch.equal(out.cpu(), want)
    return lambda: _lib.load().asyrp_faceparse_maxpool(_p(x), _p(out), N, H, W, C, _st()), [full], check


def _gate(dev, C=64, C1=8, C2=None, act1=1, act2=2, HW=5, N=2):
    g = _g(4)
    Cp, C1p = max(C, 1), max(C1, 1)
    x = torch.randn(max(N, 1), max(HW, 1), min(Cp, 1024), generator=g).to(dev)
    w1 = (torch.randn(C1p, min(Cp, 1024), generator=g) / math.sqrt(Cp)).to(dev)
    b1 = torch.randn(C1p, generator=g).to(dev)
    w2 = (torch.randn(C2, C1p, generator=g) / math.sqrt(C1p)).to(dev) if C2 else None
    full, out = _buf((max(N, 1), C2 or C1p), dev)

    def check():
        _tail_ok(full, out.numel())
        h = x.double().cpu().mean(1) @ w1.double().cpu().t() + b1.double().cpu()
        h = _act(h, act1)
        if w2 is not None:
            h = _act(h @ w2.double().cpu().t(), act2)
        assert (out.double().cpu() - h).abs().max().item() < 1e-5
    return (lambda: _lib.load().asyrp_faceparse_gate(_p(x), _p(w1), _p(b1), C1, act1, _p(w2), None, C2 or 0, act2,
                                                     _p(out), N, HW, C, _st()), [full], check)


def _act(v, act):
    return v.clamp_min(0) if act == 1 else torch.sigmoid(v) if act == 2 else v


def _apply(dev, C=4, up=2, add_map=1, alias=None, N=2, H=3, W=5):
    g = _g(5)
    Cp = max(C, 4)
    f = torch.randn(N, H, W, Cp, generator=g).to(dev)
    gate = torch.rand(N, Cp, generator=g).to(dev)
    add = torch.randn(N, H, W, Cp, generator=g).to(dev) if add_map else torch.randn(N, Cp, generator=g).to(dev)
    upo = up if up in (1, 2) else 1
    full, out = _buf((N, H * upo, W * upo, Cp), dev)
    if alias == "f":
        f.fill_(NAN)
        full, out = f.view(-1), f
    elif alias == "add":
        add.fill_(NAN)
        full, out = add.view(-1), add

    def check():
        _tail_ok(full, out.numel())
        a = add.cpu() if add_map else add.cpu()[:, None, None, :]
        want = (f.cpu() * gate.cpu()[:, None, None, :] + a).repeat_interleave(up, 1).repeat_interleave(up, 2)
        assert torch.equal(out.cpu(), want)
    return (lambda: _lib.load().asyrp_faceparse_apply(_p(f), _p(gate), _p(add), add_map, _p(out), N, H, W, C, up,
                                                      _st()), [full], check)


def _labels(dev, N=2, Hi=3, Wi=4, ld=8, ncls=5, Ho=7, Wo=9):
    lg = (torch.randn(N, Hi, Wi, max(ld, ncls), generator=_g(6)) * 3).to(dev)
    full, out = _buf((N, Ho, Wo), dev, torch.uint8)

    def check():
        _tail_ok(full, out.numel())
        assert torch.equal(out.cpu(), _labels_ref(lg, ncls, Ho, Wo))
    return (lambda: _lib.load().asyrp_faceparse_labels(_p(lg), _p(out), N, Hi, Wi, ld, ncls, Ho, Wo, _st()), [full],
            check)


def _agreement(dev, n=3, B=2, row0=1, Hi=3, Wi=4, ld=8, ncls=5, Ho=7, Wo=9):
    g = _g(7)
    src = (torch.randn(max(B, 1), Hi, Wi, ld, generator=g) * 3).to(dev)
    edited = src[torch.arange(n) % max(B, 1)] + torch.randn(n, Hi, Wi, ld, generator=g).to(dev)
    full, agree = _buf((n,), dev, torch.int32)

    def check():
        _tail_ok(full, n)
        want = _agreement_ref(src, edited, ncls, Ho, Wo, row0)
        assert torch.equal(agree.cpu().long(), want)
    return (lambda: _lib.load().asyrp_faceparse_agreement(_p(src), _p(edited), _p(agree), n, B, row0, Hi, Wi, ld, ncls,
                                                          Ho, Wo, _st()), [full], check)


M_GUARD = dict(N=1 << 15, H=256, W=256, Cin=4, Cout=64, k=1, stride=1, pad=0, tiny=True)  # N Ho Wo = 2^31
assert M_GUARD["N"] * M_GUARD["H"] * M_GUARD["W"] == (1 << 31) // 128 * 128

# (row, entry point, message fragment, refused call, accepted call or None)
REFUSALS = [
    ("pack_b_0", "asyrp_faceparse_pack", "B=0", lambda d: _pack(d, B=0), lambda d: _pack(d, B=1)),
    ("pack_h_0", "asyrp_faceparse_pack", "H=0", lambda d: _pack(d, H=0), lambda d: _pack(d, H=1)),
    ("pack_w_0", "asyrp_faceparse_pack", "W=0", lambda d: _pack(d, W=0), lambda d: _pack(d, W=1)),
    ("pack_s_0", "asyrp_faceparse_pack", "S=0", lambda d: _pack(d, S=0), lambda d: _pack(d, S=1)),
    ("conv_cin_6", "asyrp_faceparse_conv", "Cin=6", lambda d: _conv(d, Cin=6), lambda d: _conv(d, Cin=8)),
    ("conv_cin_0", "asyrp_faceparse_conv", "Cin=0", lambda d: _conv(d, Cin=0), lambda d: _conv(d, Cin=4)),
    ("conv_cout_96", "asyrp_faceparse_conv", "Cout=96", lambda d: _conv(d, Cout=96), lambda d: _conv(d, Cout=128)),
    ("conv_h_below_k", "asyrp_faceparse_conv", "bad geometry", lambda d: _conv(d, H=4, k=7, pad=1),
     lambda d: _conv(d, H=5, k=7, pad=1, W=5)),
    ("conv_stride_0", "asyrp_faceparse_conv", "stride=0", lambda d: _conv(d, stride=0), lambda d: _conv(d, stride=1)),
    ("conv_relu_2", "asyrp_faceparse_conv", "relu=2", lambda d: _conv(d, relu=2), lambda d: _conv(d, relu=1)),
    ("conv_residual_without_relu", "asyrp_faceparse_conv", "before the ReLU", lambda d: _conv(d, res=True),
     lambda d: _conv(d, res=True, relu=1)),
    ("conv_relu_without_bias", "asyrp_faceparse_conv", "needs a bias", lambda d: _conv(d, relu=1, bias=False),
     lambda d: _conv(d, relu=1)),
    ("conv_in_is_out", "asyrp_faceparse_conv", "must not alias", lambda d: _conv(d, Cin=64, k=1, pad=0, alias=True),
     lambda d: _conv(d, Cin=64, k=1, pad=0)),
    ("conv_m_2_to_the_31", "asyrp_faceparse_conv", "too many output pixels", lambda d: _conv(d, **M_GUARD), None),
    ("maxpool_c_6", "asyrp_faceparse_maxpool", "C=6", lambda d: _maxpool(d, C=6), lambda d: _maxpool(d, C=8)),
    ("gate_c_48", "asyrp_faceparse_gate", "C=48", lambda d: _gate(d, C=48), lambda d: _gate(d, C=64)),
    ("gate_c_1024", "asyrp_faceparse_gate", "C=1024", lambda d: _gate(d, C=1024), lambda d: _gate(d, C=512)),
    ("gate_c_0", "asyrp_faceparse_gate", "C=0", lambda d: _gate(d, C=0), lambda d: _gate(d, C=1)),
    ("gate_c1_0", "asyrp_faceparse_gate", "C1=0", lambda d: _gate(d, C1=0), lambda d: _gate(d, C1=1)),
    ("gate_c1_513", "asyrp_faceparse_gate", "C1=513", lambda d: _gate(d, C1=513), lambda d: _gate(d, C1=512)),
    ("gate_c2_513", "asyrp_faceparse_gate", "C2=513", lambda d: _gate(d, C2=513), lambda d: _gate(d, C2=512)),
    ("gate_act1_3", "asyrp_faceparse_gate", "act1=3", lambda d: _gate(d, act1=3), lambda d: _gate(d, act1=2)),
    ("gate_act1_neg", "asyrp_faceparse_gate", "act1=-1", lambda d: _gate(d, act1=-1), lambda d: _gate(d, act1=0)),
    ("gate_act2_3", "asyrp_faceparse_gate", "act2=3", lambda d: _gate(d, C2=8, act2=3),
     lambda d: _gate(d, C2=8, act2=2)),
    ("gate_act2_neg", "asyrp_faceparse_gate", "act2=-1", lambda d: _gate(d, C2=8, act2=-1),
     lambda d: _gate(d, C2=8, act2=0)),
    ("gate_hw_0", "asyrp_faceparse_gate", "HW=0", lambda d: _gate(d, HW=0), lambda d: _gate(d, HW=1)),
    ("gate_n_0", "asyrp_faceparse_gate", "N=0", lambda d: _gate(d, N=0), lambda d: _gate(d, N=1)),
    ("apply_up_3", "asyrp_faceparse_apply", "up=3", lambda d: _apply(d, up=3), lambda d: _apply(d, up=2)),
    ("apply_add_map_2", "asyrp_faceparse_apply", "add_map=2", lambda d: _apply(d, add_map=2),
     lambda d: _apply(d, add_map=1)),
    ("apply_c_6", "asyrp_faceparse_apply", "C=6", lambda d: _apply(d, C=6), lambda d: _apply(d, C=8)),
    ("apply_out_is_f", "asyrp_faceparse_apply", "must not alias", lambda d: _apply(d, up=1, alias="f"),
     lambda d: _apply(d, up=1)),
    ("apply_out_is_add", "asyrp_faceparse_apply", "must not alias", lambda d: _apply(d, up=1, alias="add"),
     lambda d: _apply(d, up=1)),
    ("labels_n_big", "asyrp_faceparse_labels", f"N={BIG}", lambda d: _labels(d, N=BIG, Hi=1, Wi=1, ld=2, ncls=2, Ho=1,
                                                                           Wo=1),
     lambda d: _labels(d, N=BIG - 1, Hi=1, Wi=1, ld=2, ncls=2, Ho=1, Wo=1)),
    ("labels_ncls_65", "asyrp_faceparse_labels", "ncls=65", lambda d: _labels(d, ld=65, ncls=65),
     lambda d: _labels(d, ld=65, ncls=64)),
    ("labels_ld_below_ncls", "asyrp_faceparse_labels", "ld=4", lambda d: _labels(d, ld=4, ncls=5),
     lambda d: _labels(d, ld=5, ncls=5)),
    ("labels_smem_12289", "asyrp_faceparse_labels", "too large", lambda d: _labels(d, Hi=2, Wi=12289, ld=1, ncls=1),
     lambda d: _labels(d, Hi=2, Wi=192, ld=64, ncls=64, Wo=300)),
    ("agreement_n_big", "asyrp_faceparse_agreement", f"n={BIG}",
     lambda d: _agreement(d, n=BIG, Hi=1, Wi=1, ld=2, ncls=2, Ho=1, Wo=1),
     lambda d: _agreement(d, n=BIG - 1, Hi=1, Wi=1, ld=2, ncls=2, Ho=1, Wo=1)),
    ("agreement_row0_neg", "asyrp_faceparse_agreement", "row0=-1", lambda d: _agreement(d, row0=-1),
     lambda d: _agreement(d, row0=0)),
    ("agreement_b_0", "asyrp_faceparse_agreement", "B=0", lambda d: _agreement(d, B=0), lambda d: _agreement(d, B=1)),
    ("agreement_smem_6145", "asyrp_faceparse_agreement", "too large",
     lambda d: _agreement(d, Hi=2, Wi=1229, ld=5, ncls=5),
     lambda d: _agreement(d, Hi=2, Wi=96, ld=64, ncls=64, Wo=300)),
]


@pytest.mark.parametrize("row", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_entry_point_refusals(cuda_device, row):
    name, entry, fragment, bad, good = row
    call, outs, _ = bad(cuda_device)
    torch.cuda.synchronize()
    with pytest.raises(_lib.AsyrpError, match=f"{re.escape(entry)}: .*{re.escape(fragment)}") as exc:
        _lib.check(call(), entry)
    assert f"{entry}: " in str(exc.value)
    torch.cuda.synchronize()
    for o in outs:
        assert _untouched(o), f"{name}: the refused call wrote its output"
    if good is None:
        return
    call, outs, check = good(cuda_device)
    _lib.check(call(), entry)
    torch.cuda.synchronize()
    check()


# ------------------------------------------------------------------------------------------------------------------
# conv: every epilogue at the admitted edges, against TF32 operands in fp64
# ------------------------------------------------------------------------------------------------------------------
# (N, H, W, Cin, Cout, k, stride, pad): M = 1 with H + 2 pad = k = 7 (the stem, Ho = 1); M = 127 with K padded
# (Cin 516) and nine channel tiles; M = 128; M = 129 (samples of 43 pixels: boundaries inside the first tile, one
# pixel in the second); two samples of 100 pixels (a boundary inside a tile) with Cin 516 / Cout 576 through a 3x3;
# stride > k (1x1 / 3, 3x3 / 4); the stem at a size with partial tiles
CONV_CASES = {
    "m1_stem_ho1": (1, 1, 1, 4, 64, 7, 2, 3),
    "m127_k_padded_9_tiles": (1, 127, 1, 516, 576, 1, 1, 0),
    "m128": (1, 8, 16, 8, 64, 3, 1, 1),
    "m129_3_samples": (3, 43, 1, 4, 64, 3, 1, 1),
    "sample_boundary_in_tile": (2, 10, 10, 516, 576, 3, 1, 1),
    "k1_stride3": (2, 13, 11, 8, 128, 1, 3, 0),
    "k3_stride4": (2, 17, 15, 12, 64, 3, 4, 1),
    "stem_37": (2, 37, 37, 4, 64, 7, 2, 3),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_every_epilogue_within_the_tf32_bound(cuda_device, case):
    """kEpiBias (bias present and null), kEpiRelu, kEpiResidualRelu (bias present and null, and residual == out, which
    must give the bits of a separate residual buffer)"""
    N, H, W, Cin, Cout, k, stride, pad = CONV_CASES[case]
    dev = cuda_device
    g = _g(H * 31 + Cin)
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / math.sqrt(Cin * k * k)
    bias = torch.randn(Cout, generator=g)
    z, s = _conv_ref(x, w, stride, pad)
    res = torch.randn(z.shape, generator=g)
    wp = ops.pack_lpips_conv_weight(w).to(dev)
    kpad = wp.shape[1]
    xd, bd, rd = x.to(dev), bias.to(dev), res.to(dev)
    full, out = _buf(tuple(z.shape), dev)
    bb, rr = bias.double().view(1, 1, 1, -1), res.double()
    for what, b, relu, r in (("bias", True, False, False), ("no bias", False, False, False),
                             ("relu", True, True, False), ("residual relu", True, True, True),
                             ("residual relu, no bias", False, True, True)):
        full.fill_(NAN)
        ops.faceparse_conv(xd, wp, bd if b else None, out, k, stride, pad, relu=relu, residual=rd if r else None)
        torch.cuda.synchronize()
        _tail_ok(full, out.numel())
        v = z + (bb if b else 0) + (rr if r else 0)
        want = v.clamp_min(0) if relu else v
        bound = (kpad / 8 + 2) * U * s + 4 * U * (v.abs() + (bb.abs() if b else 0) + (rr.abs() if r else 0))
        _within("conv", (out.double().cpu() - want).abs(), bound, f"{case} {what}")
        if r:
            sep = out.clone()
            out.copy_(rd)
            ops.faceparse_conv(xd, wp, bd if b else None, out, k, stride, pad, residual=out)
            torch.cuda.synchronize()
            assert torch.equal(out, sep), f"{case} {what}: residual == out differs from a separate residual"


def _ties(n, g):
    """fp32 values whose 13 low mantissa bits are exactly 0x1000: a TF32 tie, rounded away from zero by cvt.rna"""
    b = torch.randint(0, 1 << 10, (n,), generator=g, dtype=torch.int32) << 13 | 0x1000
    e = torch.randint(120, 131, (n,), generator=g, dtype=torch.int32) << 23
    sgn = torch.randint(0, 2, (n,), generator=g, dtype=torch.int32) << 31
    return (b | e | sgn).view(torch.float32)


@pytest.mark.parametrize("case", ["m1_stem_ho1", "m129_3_samples", "sample_boundary_in_tile", "k3_stride4"])
def test_conv_single_tap_weights_are_exact(cuda_device, case):
    """one non-zero weight per output channel: the accumulator holds one exact TF32 product, so every epilogue must
    equal an fp32 CPU restatement fl(fl(acc + b) + r) and the max bit for bit; half the operands are TF32 ties"""
    N, H, W, Cin, Cout, k, stride, pad = CONV_CASES[case]
    dev = cuda_device
    g = _g(77 + H)
    x = torch.randn(N, H, W, Cin, generator=g)
    tie = torch.rand(x.shape, generator=g) < 0.5
    x[tie] = _ties(int(tie.sum()), g)
    o = torch.arange(Cout)
    ci, ky, kx = (o * 7 + 1) % Cin, (o * 5) % k, (o * 3 + 1) % k
    wv = torch.randn(Cout, generator=g)
    wv[::2] = _ties(len(wv[::2]), g)
    w = torch.zeros(Cout, Cin, k, k)
    w[o, ci, ky, kx] = wv
    # acc[n, y, x, o] = tf32(x[n, y*s - pad + ky, x*s - pad + kx, ci]) * tf32(wv[o]) (zero outside the image)
    xt = _tf32(x).permute(0, 3, 1, 2)
    xp = F.pad(xt, (pad, pad, pad, pad))
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    yy = torch.arange(Ho).view(Ho, 1, 1) * stride + ky.view(1, 1, Cout)
    xx = torch.arange(Wo).view(1, Wo, 1) * stride + kx.view(1, 1, Cout)
    acc = (xp[:, ci.view(1, 1, Cout), yy, xx] * _tf32(wv)).float()  # exact: two 11-bit significands
    bias = torch.randn(Cout, generator=g)
    res = torch.randn(acc.shape, generator=g)
    wp = ops.pack_lpips_conv_weight(w).to(dev)
    xd, bd, rd = x.to(dev), bias.to(dev), res.to(dev)
    full, out = _buf(tuple(acc.shape), dev)
    for what, b, relu, r in (("bias", True, False, False), ("no bias", False, False, False),
                             ("relu", True, True, False), ("residual relu", True, True, True),
                             ("residual relu, no bias", False, True, True)):
        full.fill_(NAN)
        ops.faceparse_conv(xd, wp, bd if b else None, out, k, stride, pad, relu=relu, residual=rd if r else None)
        v = acc + bias if b else acc.clone()
        if r:
            v = res + v
        if relu:
            v = torch.maximum(v, torch.zeros_like(v))
        torch.cuda.synchronize()
        _tail_ok(full, out.numel())
        assert torch.equal(out.cpu(), v), f"{case} {what}: {int((out.cpu() != v).sum())} elements differ"
        if r:
            assert (v == 0).any() and (v > 0).any(), "the max must act"


# ------------------------------------------------------------------------------------------------------------------
# gate
# ------------------------------------------------------------------------------------------------------------------
GATE_C = [1 << i for i in range(10)]  # every C dividing 512: J = 512 / C partials per channel
GATE_CONFIGS = list(itertools.product([1, 33, 512], [None, 1, 512], [False, True]))  # C1, C2 (None: no w2), biases
ACTS = list(itertools.product(range(3), range(3)))


@pytest.mark.parametrize("HW", [1, 128 * 128])
@pytest.mark.parametrize("C", GATE_C)
def test_gate_every_channel_count(cuda_device, C, HW):
    """each (C1, C2, biases) configuration, cycling through all nine (act1, act2) pairs; inputs of mean 1e3 with unit
    noise and per-channel offsets; batch of 3, and sample 1 alone gives the same bits"""
    dev = cuda_device
    g = _g(C * 7 + HW)
    N, J = 3, 512 // C
    x = 1e3 + torch.randn(1, 1, C, generator=g) + torch.randn(N, HW, C, generator=g)
    xd = x.view(N, HW, 1, C).to(dev)
    m = x.double().mean(1)
    am = x.double().abs().mean(1)
    for i, (C1, C2, biased) in enumerate(GATE_CONFIGS):
        for act1, act2 in (ACTS[(2 * i) % 9], ACTS[(2 * i + 1) % 9]):
            w1 = torch.randn(C1, C, generator=g) / math.sqrt(C) / 1e3
            b1 = torch.randn(C1, generator=g) if biased else None
            w2 = torch.randn(C2, C1, generator=g) / math.sqrt(C1) if C2 else None
            b2 = torch.randn(C2, generator=g) if (biased and C2) else None
            dv = lambda t: None if t is None else t.to(dev)  # noqa: E731
            full, out = _buf((N, C2 or C1), dev)
            ops.faceparse_gate(xd, dv(w1), dv(b1), act1, out, w2=dv(w2), b2=dv(b2), act2=act2)
            torch.cuda.synchronize()
            _tail_ok(full, out.numel())
            h_pre = m @ w1.double().t() + (b1.double() if biased else 0)
            h = _act(h_pre, act1)
            s1 = 0.25 if act1 == 2 else 1.0
            a1 = am @ w1.double().abs().t() + (b1.double().abs() if biased else 0)
            k1 = (math.ceil(HW / J) + J + math.ceil(C / 32) + 16) * U
            if w2 is None:
                want, bound = h, s1 * k1 * a1 + 4 * U
            else:
                want = _act(h @ w2.double().t() + (b2.double() if biased else 0), act2)
                s2 = 0.25 if act2 == 2 else 1.0
                a2 = a1 @ w2.double().abs().t()
                hb = (h.abs() @ w2.double().abs().t()) + (b2.double().abs() if biased else 0)
                bound = s2 * (s1 * (k1 + C1 * U) * a2 + (C1 + 4) * U * hb + 4 * U * w2.double().abs().sum(1)) + 4 * U
            _within("gate", (out.double().cpu() - want).abs(), bound, f"C={C} HW={HW} C1={C1} C2={C2} "
                    f"bias={biased} act={act1},{act2}")
            if i == 0 or (C2 == 512 and biased):
                one = torch.empty_like(out[:1])
                ops.faceparse_gate(xd[1:2], dv(w1), dv(b1), act1, one, w2=dv(w2), b2=dv(b2), act2=act2)
                assert torch.equal(one, out[1:2]), "a sample's gate depends on its batch"


# ------------------------------------------------------------------------------------------------------------------
# upsample-argmax: labels and agreement bit for bit against the fp32 restatement
# ------------------------------------------------------------------------------------------------------------------
def _clamp_pair():
    """an (in, out) pair where the fp32 source coordinate (out - 1) * ((in - 1) / (out - 1)) rounds above in - 1,
    so the last output's second tap is clamped with a non-zero weight"""
    for i in range(48, 70):
        for o in range(300, 700):
            sc = np.float32(i - 1) / np.float32(o - 1)
            if np.float32(o - 1) * sc > i - 1:
                return i, o
    raise AssertionError("no pair found")


def _near_ties(lg, g, ncls):
    """sample 0: classes 1 and 2 equal everywhere and the largest; sample 1 (if any): class 2 one ulp above class 1"""
    N, Hi, Wi, _ = lg.shape
    top = 30 + torch.rand(Hi, Wi, generator=g)  # above every N(0, 9) logit
    if ncls >= 3:
        lg[0, ..., 1] = lg[0, ..., 2] = top
        if N > 1:
            lg[1, ..., 1] = top
            lg[1, ..., 2] = torch.nextafter(top, torch.tensor(float("inf")))
    return lg


CLAMP = _clamp_pair()
# (N, Hi, Wi, ld, ncls, Ho, Wo)
LABEL_CASES = {
    "wi_ncls_12288": (2, 3, 192, 64, 64, 5, 700),
    "ncls_1": (2, 4, 5, 3, 1, 9, 11),
    "ncls_64_network": (2, 64, 64, 64, 64, 512, 512),
    "ho_wo_1": (3, 7, 9, 8, 5, 1, 1),
    "hi_1": (2, 1, 6, 8, 7, 33, 17),
    "downsample": (2, 40, 50, 20, 19, 13, 7),
    "clamp_pair": (2, CLAMP[0], CLAMP[0], 19, 19, CLAMP[1], CLAMP[1]),
    "n_65535": (65535, 2, 2, 3, 3, 2, 3),
}


@pytest.mark.parametrize("case", list(LABEL_CASES))
def test_labels_bit_for_bit(cuda_device, case):
    N, Hi, Wi, ld, ncls, Ho, Wo = LABEL_CASES[case]
    g = _g(Hi * 100 + Wi + ncls)
    lg = _near_ties(torch.randn(N, Hi, Wi, ld, generator=g) * 3, g, ncls)
    lg[..., ncls:] = 1e9  # padding classes are never read
    full, out = _buf((N, Ho, Wo), cuda_device, torch.uint8)
    ops.faceparse_labels(lg.to(cuda_device), ncls, out)
    torch.cuda.synchronize()
    _tail_ok(full, out.numel())
    want = _labels_ref(lg, ncls, Ho, Wo)
    bad = out.cpu() != want
    assert not bad.any(), f"{case}: {int(bad.sum())} labels differ, first at {bad.nonzero()[0].tolist()}"
    if ncls >= 3:
        assert (want[0] == 1).all(), "the tie goes to the first class"
        assert (want[1] == 2).any(), "one ulp apart"


# (n, B, row0, Hi, Wi, ncls, Ho, Wo): Wi ncls from 6141 (the first size whose launch passes the default 48 KB with the
# kernel's static array) to 6144, the admitted limit; row0 >= B and n > B (the pairing wraps more than once); 4096^2
# outputs (16.7 M pixels a row, still exact)
AGREE_CASES = {
    "wi_ncls_6141": (3, 2, 0, 2, 267, 23, 3, 300),
    "wi_ncls_6142": (3, 2, 1, 2, 166, 37, 3, 300),
    "wi_ncls_6143": (3, 2, 0, 2, 6143, 1, 3, 300),
    "wi_ncls_6144": (3, 2, 3, 2, 96, 64, 5, 700),
    "wraps_twice": (8, 3, 7, 9, 11, 19, 41, 37),
    "downsample_hi_1": (4, 2, 5, 1, 30, 7, 1, 13),
    "out_4096": (3, 2, 1, 3, 3, 3, 4096, 4096),
}


@pytest.mark.parametrize("case", list(AGREE_CASES))
def test_agreement_at_the_shared_memory_limit(cuda_device, case):
    n, B, row0, Hi, Wi, ncls, Ho, Wo = AGREE_CASES[case]
    g = _g(n * 1000 + Wi)
    src = _near_ties(torch.randn(B, Hi, Wi, ncls, generator=g) * 3, g, ncls)
    edited = src[(row0 + torch.arange(n)) % B] + 0.3 * torch.arange(n).view(n, 1, 1, 1) * torch.randn(
        n, Hi, Wi, ncls, generator=g)
    full, agree = _buf((n,), cuda_device, torch.int32)
    ops.faceparse_agreement(src.to(cuda_device), edited.to(cuda_device), ncls, (Ho, Wo), agree, row0=row0)
    torch.cuda.synchronize()
    _tail_ok(full, n)
    want = _agreement_ref(src, edited, ncls, Ho, Wo, row0)
    assert torch.equal(agree.cpu().long(), want), (agree.cpu().tolist(), want.tolist())
    assert agree[0].item() == Ho * Wo  # row 0 is its own source
    if ncls > 1 and Ho * Wo >= 100:
        assert len(set(want.tolist())) > 1, "the counts do not tell the rows apart"


# ------------------------------------------------------------------------------------------------------------------
# pack, max-pool, apply
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,S", [(1, 1, 1), (1, 1, 3), (1, 1000, 3), (1000, 1, 1024), (1, 1000, 1024),
                                   (1024, 1024, 512), (3, 5, 1024)])
def test_pack_sizes(cuda_device, H, W, S):
    """within the first-order fp32 error: the source coordinate (Y + 1/2) H / S - 1/2 is off by at most 3 u H, which
    moves the blend by that times the largest step between neighbouring pixels (at most 1); six roundings of the
    blend, the subtraction of the mean and the division by std (>= 0.224)"""
    x = torch.rand(2, 3, H, W, generator=_g(H + W + S)) * 4 - 2  # half of it outside [-1, 1]: clamped
    full, out = _buf((2, S, S, 4), cuda_device)
    ops.faceparse_pack(x.to(cuda_device), out)
    torch.cuda.synchronize()
    _tail_ok(full, out.numel())
    ref = _pack_ref(x, S)
    bound = (3 * (H + W) + 10) * U / 0.224 + 4 * U * ref.abs()
    _within("pack", (out[..., :3].double().cpu() - ref).abs(), bound, f"{H}x{W} -> {S}")
    assert torch.equal(out[..., 3], torch.zeros_like(out[..., 3]))


@pytest.mark.parametrize("H", [1, 2, 3])
def test_maxpool_smallest_maps(cuda_device, H):
    for W in (1, 2, 3):
        x = torch.randn(2, H, W, 4, generator=_g(H * 3 + W))
        full, out = _buf((2, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 4), cuda_device)
        ops.faceparse_maxpool(x.to(cuda_device), out)
        torch.cuda.synchronize()
        _tail_ok(full, out.numel())
        want = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
        assert torch.equal(out.cpu(), want), (H, W)


@pytest.mark.parametrize("H,W", [(1, 1), (3, 5), (7, 3)])
def test_apply_up2_with_a_map_on_odd_sizes(cuda_device, H, W):
    g = _g(H * W)
    f, gate, add = torch.randn(2, H, W, 4, generator=g), torch.rand(2, 4, generator=g), torch.randn(2, H, W, 4,
                                                                                                      generator=g)
    full, out = _buf((2, 2 * H, 2 * W, 4), cuda_device)
    ops.faceparse_apply(f.to(cuda_device), gate.to(cuda_device), add.to(cuda_device), out, up=2)
    torch.cuda.synchronize()
    _tail_ok(full, out.numel())
    want = (f * gate[:, None, None, :] + add).repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(out.cpu(), want)


# ------------------------------------------------------------------------------------------------------------------
# outputs past 2^31 elements
# ------------------------------------------------------------------------------------------------------------------
def _samples(N, k):
    return sorted({0, N - 1, *range(k, N - 1, k)})


def test_pack_past_2_to_the_31_elements(cuda_device):
    """2049 samples of 512^2 x 4 floats (8 GiB) from 1x1 images at +-2 (clamped to 0 or 1, which the blend keeps
    exactly): each sample's pixels are its three normalised values and 0"""
    B, S = 2049, 512
    assert B * S * S * 4 > 2 ** 31
    _need_memory(B * S * S * 16, "pack past 2^31 elements")
    n, c = torch.arange(B).view(B, 1), torch.arange(3).view(1, 3)
    p = ((n * 5 + c * 3) % 7 < 3).float()  # 0 or 1 after the clamp
    x = (4 * p - 2).view(B, 3, 1, 1).to(cuda_device)
    out = torch.empty(B, S, S, 4, device=cuda_device)
    out.view(-1)[-8:].fill_(NAN)
    ops.faceparse_pack(x, out)
    torch.cuda.synchronize()
    want = torch.cat([(p - torch.tensor(MEAN)) / torch.tensor(STD), torch.zeros(B, 1)], 1).to(cuda_device)
    for s in _samples(B, 64):
        assert torch.equal(out[s], want[s].expand(S, S, 4)), f"sample {s} of {B}"
    del out
    torch.cuda.empty_cache()


def test_labels_past_2_to_the_31_elements(cuda_device):
    """8193 samples of 512^2 uint8 labels (2.1 GB) from 1x1 logits whose class n % 64 is 1, every other 0"""
    N, S, ncls = 8193, 512, 64
    assert N * S * S > 2 ** 31
    _need_memory(N * S * S, "labels past 2^31 elements")
    lg = torch.zeros(N, 1, 1, ncls, device=cuda_device)
    nn = torch.arange(N, device=cuda_device)
    lg.view(N, ncls)[nn, nn % ncls] = 1.0
    out = torch.empty(N, S, S, dtype=torch.uint8, device=cuda_device)
    out.view(-1)[-8:].fill_(255)
    ops.faceparse_labels(lg, ncls, out)
    torch.cuda.synchronize()
    for s in _samples(N, 64):
        assert (out[s] == s % ncls).all(), f"sample {s} of {N}"
    del out
    torch.cuda.empty_cache()


def test_apply_past_2_to_the_31_elements(cuda_device):
    """513 samples of 128^2 x 64 upsampled twice: 2^31 + 2^22 output floats (8 GiB) from integer maps, gates in
    {1/2, 1, 2, -1} and integer vectors, all exact"""
    N, H, C = 513, 128, 64
    assert N * (2 * H) ** 2 * C > 2 ** 31
    _need_memory(5 * N * H * H * C * 4, "apply past 2^31 elements")
    dev = cuda_device
    f = torch.empty(N, H, H, C, device=dev)
    hh = torch.arange(H, device=dev).view(H, 1, 1) * 5 + torch.arange(H, device=dev).view(1, H, 1) * 3 + torch.arange(
        C, device=dev).view(1, 1, C) * 7
    for n0 in range(0, N, 64):
        nn = torch.arange(n0, min(N, n0 + 64), device=dev).view(-1, 1, 1, 1)
        f[n0:n0 + 64] = ((hh + 11 * nn) % 61 - 30).float()
    nn, cc = torch.arange(N, device=dev).view(N, 1), torch.arange(C, device=dev).view(1, C)
    gate = torch.tensor([0.5, 1.0, 2.0, -1.0], device=dev)[(nn + cc) % 4].contiguous()
    add = ((nn * 3 + cc) % 9 - 4).float().contiguous()
    out = torch.empty(N, 2 * H, 2 * H, C, device=dev)
    out.view(-1)[-8:].fill_(NAN)
    ops.faceparse_apply(f, gate, add, out, up=2)
    torch.cuda.synchronize()
    for s in _samples(N, 16):
        want = (f[s] * gate[s] + add[s]).repeat_interleave(2, 0).repeat_interleave(2, 1)
        assert torch.equal(out[s], want), f"sample {s} of {N}"
    del f, out
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    """the file's wall time, peak device memory and worst err / bound per kernel, printed at the end (pytest -s)"""
    t0 = time.perf_counter()
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated() / GiB if torch.cuda.is_available() else 0.0
    worst = ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items()))
    print(f"\ntest_face_parsing_limits_gpu: {time.perf_counter() - t0:.1f} s, peak device memory {peak:.2f} GiB; "
          f"worst err / bound: {worst}")
