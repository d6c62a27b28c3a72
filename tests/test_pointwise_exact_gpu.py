"""Exact and derived-bound tests of the UNet's pointwise kernels, the sampler updates and the attention glue, at the shapes
the four bench.WORKLOADS plans launch (SHAPES below) plus edge shapes.

test_kernels_gpu.py, test_conv_coverage_gpu.py and test_plans_gpu.py check these kernels against fp64 with flat
tolerances of about one fp16 ulp relative to max|ref|, which a rounding-mode or 1-ulp defect passes.  Here:

  * operands are integers or dyadics wherever the result can be exact, and the output is compared with `==` against fp64
    (gn_finalize through an exact emulation of its fp64/fp32 operation order, apply with act = 0, pack_input, unpack,
    transpose_tc, axpby, ddim_update, ddpm_update with mask 0);
  * elsewhere each element gets a bound beta on the kernel's fp32 value before its final rounding, derived in the test's
    docstring from the kernel's own operation order with u = 2^-24 and the CUDA Programming Guide's ulp tables (expf,
    sinf, cosf, acosf: 2 ulp; sqrtf and IEEE division: correctly rounded; __expf: 2 + floor(1.173 |x|) ulp).  An ulp of
    an fp32 value v is at most 2u|v|;
  * fp16 outputs use the rounding criterion: with r the fp64 value of the operation on the kernel's actual inputs, the
    output must lie in [RN16(r - beta), RN16(r + beta)].  Where both ends agree (the interval holds no fp16 rounding
    boundary) that is RN16(r) bit for bit: the "strict" class, which must be most of the elements and whose share is
    printed.  A round-toward-zero store or a 1-ulp defect fails it;
  * every output is NaN-filled with one guard sample (or row) behind it that must stay NaN, every element must be
    written, and a second launch must give the same bits.  Mismatches are reported by (sample, pixel, channel) or by
    (row, column).

The default GroupNorm path (conv epilogue tile statistics -> gn_finalize) is checked at |mean|/std ~ 30 against a bound
derived from the epilogue's summation order (test_default_groupnorm_path_at_large_mean).

The whole file takes about 37 s on an NVIDIA H100 80GB HBM3 at a 700 W power limit, 15 s of it building the four plans
for the shape table.
"""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
NAN = float("nan")
FULL_REF_ELEMS = 1 << 26  # larger outputs: the fp64 reference covers samples 0, B/2 and B-1
STRICT_MIN = 0.5          # least share of fp16 outputs in the strict class

# ------------------------------------------------------------------------------------------------------------------
# every (kernel, shape) the four bench.WORKLOADS plans launch at their benchmark batch sizes (one edit evaluation, the
# explicit-delta_h path and the sampler step).  test_plans_reach_only_tabled_shapes fails when a plan launches a shape
# missing here.  Keys:
#   gn_finalize (N, Ca, Ta, Cb, Tb, HW, ss_stride, eps)     apply (N, Hi, Wi, Ca, Cb, act, resample, Caff, off)
#   pack_input (N, Cin, H, W)        timestep_embedding (N, dim, variant)
#   linear (N, I, O, in_stride, out_stride, act_in, act_out)   attention (N, T, heads, d)   softmax_rows (rows, T)
#   transpose_tc (N, T, C, ld)       slerp_h (N, H, W, C, T)   ddim_update / ddpm_update (N, Cx, H, W, Ce)
#   unpack_nchw (N, C, H, W)
# ------------------------------------------------------------------------------------------------------------------
SHAPES = {
    'apply': {
        (4, 8, 8, 1024, 0, 0, 0, 1024, 0), (4, 8, 8, 1024, 0, 1, 0, 1024, 0), (4, 8, 8, 1024, 0, 1, 0, 2048, 0),
        (4, 8, 8, 1024, 0, 1, 0, 2048, 1024), (4, 8, 8, 1024, 0, 1, 2, 1024, 0), (4, 16, 16, 1024, 0, 1, 1, 1024, 0),
        (4, 32, 32, 512, 0, 1, 1, 512, 0), (4, 64, 64, 512, 0, 1, 1, 512, 0), (4, 128, 128, 256, 0, 1, 1, 256, 0),
        (4, 256, 256, 256, 0, 1, 1, 256, 0), (8, 8, 8, 512, 0, 0, 0, 512, 0), (8, 8, 8, 512, 0, 1, 0, 512, 0),
        (8, 8, 8, 512, 0, 1, 0, 1024, 0), (8, 8, 8, 512, 0, 1, 0, 1024, 512), (8, 8, 8, 512, 0, 1, 2, 512, 0),
        (8, 16, 16, 512, 0, 1, 1, 512, 0), (8, 32, 32, 256, 0, 1, 1, 256, 0), (8, 64, 64, 256, 0, 1, 1, 256, 0),
        (8, 128, 128, 128, 0, 1, 1, 128, 0), (8, 256, 256, 128, 0, 1, 1, 128, 0), (16, 8, 8, 512, 0, 0, 0, 512, 0),
        (16, 8, 8, 512, 0, 0, 2, 0, 0), (16, 8, 8, 512, 0, 1, 0, 512, 0), (16, 8, 8, 512, 0, 1, 0, 1024, 0),
        (16, 8, 8, 512, 0, 1, 0, 1024, 512), (32, 8, 8, 512, 0, 0, 0, 512, 0), (32, 8, 8, 512, 0, 0, 2, 0, 0),
        (32, 8, 8, 512, 0, 1, 0, 512, 0), (32, 8, 8, 512, 0, 1, 0, 1024, 0), (32, 8, 8, 512, 0, 1, 0, 1024, 512),
    },
    'attention': {
        (4, 64, 16, 64), (8, 64, 8, 64), (16, 64, 1, 512), (32, 64, 1, 512),
    },
    'ddim_update': {
        (4, 3, 256, 256, 6), (8, 3, 256, 256, 6), (16, 3, 256, 256, 3), (32, 3, 256, 256, 3),
    },
    'ddpm_update': {
        (4, 3, 256, 256, 6), (8, 3, 256, 256, 6), (16, 3, 256, 256, 3), (32, 3, 256, 256, 3),
    },
    'gn_finalize': {
        (4, 256, 32, 0, 0, 4096, 0, 1e-05), (4, 256, 32, 0, 0, 4096, 52736, 1e-05),
        (4, 256, 128, 0, 0, 16384, 0, 1e-05), (4, 256, 128, 0, 0, 16384, 52736, 1e-05),
        (4, 256, 128, 256, 128, 16384, 0, 1e-05), (4, 256, 512, 0, 0, 65536, 0, 1e-05),
        (4, 256, 512, 0, 0, 65536, 52736, 1e-05), (4, 256, 512, 256, 512, 65536, 0, 1e-05),
        (4, 512, 2, 0, 0, 256, 0, 1e-05), (4, 512, 2, 0, 0, 256, 52736, 1e-05), (4, 512, 8, 0, 0, 1024, 0, 1e-05),
        (4, 512, 8, 0, 0, 1024, 52736, 1e-05), (4, 512, 8, 512, 8, 1024, 0, 1e-05), (4, 512, 32, 0, 0, 4096, 0, 1e-05),
        (4, 512, 32, 0, 0, 4096, 52736, 1e-05), (4, 512, 32, 256, 32, 4096, 0, 1e-05),
        (4, 512, 32, 512, 32, 4096, 0, 1e-05), (4, 512, 128, 0, 0, 16384, 52736, 1e-05),
        (4, 512, 128, 256, 128, 16384, 0, 1e-05), (4, 1024, 2, 0, 0, 256, 0, 1e-05),
        (4, 1024, 2, 0, 0, 256, 52736, 1e-05), (4, 1024, 2, 512, 2, 256, 0, 1e-05),
        (4, 1024, 2, 1024, 2, 256, 0, 1e-05), (4, 1024, 4, 0, 0, 64, 0, 1e-05), (4, 1024, 4, 0, 0, 64, 52736, 1e-05),
        (4, 1024, 4, 1024, 4, 64, 0, 1e-05), (4, 1024, 8, 0, 0, 1024, 52736, 1e-05),
        (4, 1024, 8, 512, 8, 1024, 0, 1e-05), (8, 128, 32, 0, 0, 4096, 0, 1e-05),
        (8, 128, 32, 0, 0, 4096, 19200, 1e-05), (8, 128, 128, 0, 0, 16384, 0, 1e-05),
        (8, 128, 128, 0, 0, 16384, 19200, 1e-05), (8, 128, 128, 128, 128, 16384, 0, 1e-05),
        (8, 128, 512, 0, 0, 65536, 0, 1e-05), (8, 128, 512, 0, 0, 65536, 19200, 1e-05),
        (8, 128, 512, 128, 512, 65536, 0, 1e-05), (8, 256, 2, 0, 0, 256, 0, 1e-05),
        (8, 256, 2, 0, 0, 256, 19200, 1e-05), (8, 256, 8, 0, 0, 1024, 0, 1e-05), (8, 256, 8, 0, 0, 1024, 19200, 1e-05),
        (8, 256, 8, 256, 8, 1024, 0, 1e-05), (8, 256, 32, 0, 0, 4096, 0, 1e-05), (8, 256, 32, 0, 0, 4096, 19200, 1e-05),
        (8, 256, 32, 128, 32, 4096, 0, 1e-05), (8, 256, 32, 256, 32, 4096, 0, 1e-05),
        (8, 256, 128, 0, 0, 16384, 19200, 1e-05), (8, 256, 128, 128, 128, 16384, 0, 1e-05),
        (8, 512, 2, 0, 0, 256, 0, 1e-05), (8, 512, 2, 0, 0, 256, 19200, 1e-05), (8, 512, 2, 256, 2, 256, 0, 1e-05),
        (8, 512, 2, 512, 2, 256, 0, 1e-05), (8, 512, 4, 0, 0, 64, 0, 1e-05), (8, 512, 4, 0, 0, 64, 19200, 1e-05),
        (8, 512, 4, 512, 4, 64, 0, 1e-05), (8, 512, 8, 0, 0, 1024, 19200, 1e-05), (8, 512, 8, 256, 8, 1024, 0, 1e-05),
        (16, 128, 32, 0, 0, 4096, 0, 1e-06), (16, 128, 128, 0, 0, 16384, 0, 1e-06),
        (16, 128, 128, 128, 128, 16384, 0, 1e-06), (16, 128, 512, 0, 0, 65536, 0, 1e-06),
        (16, 128, 512, 128, 512, 65536, 0, 1e-06), (16, 256, 2, 0, 0, 256, 0, 1e-06),
        (16, 256, 8, 0, 0, 1024, 0, 1e-06), (16, 256, 8, 256, 8, 1024, 0, 1e-06), (16, 256, 32, 0, 0, 4096, 0, 1e-06),
        (16, 256, 32, 128, 32, 4096, 0, 1e-06), (16, 256, 32, 256, 32, 4096, 0, 1e-06),
        (16, 256, 128, 128, 128, 16384, 0, 1e-06), (16, 512, 2, 0, 0, 256, 0, 1e-06),
        (16, 512, 2, 256, 2, 256, 0, 1e-06), (16, 512, 2, 512, 2, 256, 0, 1e-06), (16, 512, 4, 0, 0, 64, 0, 1e-06),
        (16, 512, 4, 512, 4, 64, 0, 1e-06), (16, 512, 8, 256, 8, 1024, 0, 1e-06), (32, 128, 32, 0, 0, 4096, 0, 1e-06),
        (32, 128, 128, 0, 0, 16384, 0, 1e-06), (32, 128, 128, 128, 128, 16384, 0, 1e-06),
        (32, 128, 512, 0, 0, 65536, 0, 1e-06), (32, 128, 512, 128, 512, 65536, 0, 1e-06),
        (32, 256, 2, 0, 0, 256, 0, 1e-06), (32, 256, 8, 0, 0, 1024, 0, 1e-06), (32, 256, 8, 256, 8, 1024, 0, 1e-06),
        (32, 256, 32, 0, 0, 4096, 0, 1e-06), (32, 256, 32, 128, 32, 4096, 0, 1e-06),
        (32, 256, 32, 256, 32, 4096, 0, 1e-06), (32, 256, 128, 128, 128, 16384, 0, 1e-06),
        (32, 512, 2, 0, 0, 256, 0, 1e-06), (32, 512, 2, 256, 2, 256, 0, 1e-06), (32, 512, 2, 512, 2, 256, 0, 1e-06),
        (32, 512, 4, 0, 0, 64, 0, 1e-06), (32, 512, 4, 512, 4, 64, 0, 1e-06), (32, 512, 8, 256, 8, 1024, 0, 1e-06),
    },
    'linear': {
        (4, 256, 1024, 256, 1024, 0, 1), (4, 1024, 1024, 1024, 1024, 0, 0), (4, 1024, 52736, 1024, 52736, 1, 0),
        (8, 128, 512, 128, 512, 0, 1), (8, 512, 512, 512, 512, 0, 0), (8, 512, 19200, 512, 19200, 1, 0),
        (16, 128, 512, 128, 512, 0, 1), (16, 512, 512, 512, 512, 0, 0), (16, 512, 10496, 512, 10496, 1, 0),
        (32, 128, 512, 128, 512, 0, 1), (32, 512, 512, 512, 512, 0, 0), (32, 512, 10496, 512, 10496, 1, 0),
    },
    'pack_input': {
        (4, 3, 256, 256), (8, 3, 256, 256), (16, 3, 256, 256), (32, 3, 256, 256),
    },
    'slerp_h': {
        (4, 8, 8, 1024, 4), (8, 8, 8, 512, 4), (16, 8, 8, 512, 4), (32, 8, 8, 512, 4),
    },
    'softmax_rows': {
        (4096, 256), (8192, 256), (16384, 256), (32768, 1024),
    },
    'timestep_embedding': {
        (4, 256, 1), (8, 128, 1), (16, 128, 0), (32, 128, 0),
    },
    'transpose_tc': {
        (4, 256, 1024, 3072), (4, 1024, 512, 1536), (8, 256, 512, 1536), (16, 256, 512, 1536), (32, 256, 512, 1536),
    },
    'unpack_nchw': {
        (4, 1024, 8, 8), (8, 512, 8, 8), (16, 512, 8, 8), (32, 512, 8, 8),
    },
}


def _ops():
    from asyrp_official_b200 import ops
    return ops


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _rows(kernel):
    return sorted(SHAPES.get(kernel, ()))


def _pick(N, numel):
    """the samples the fp64 reference covers"""
    return list(range(N)) if N * numel <= FULL_REF_ELEMS else sorted({0, N // 2, N - 1})


# ------------------------------------------------------------------------------------------------------------------
# fp16 rounding and the criterion
# ------------------------------------------------------------------------------------------------------------------
def rn16(r):
    """round-to-nearest-even of fp64 values to fp16, exactly (no double rounding through fp32), as fp64"""
    a = r.abs()
    _, ex = torch.frexp(a)  # a = m * 2^ex, m in [0.5, 1)
    e = (ex.long() - 11).clamp_min(-24)
    ulp = ((e + 1023) << 52).view(torch.float64)  # 2^e built from its bits: exact
    q = torch.round(r / ulp) * ulp  # r / ulp is exact (ulp is a power of two); torch.round is half-to-even
    return torch.where(q.abs() > 65504.0, torch.sign(r) * math.inf, q)


def _half_ulp16(r):
    """half the fp16 spacing at |r| (fp64): the most the final fp16 rounding can add"""
    _, ex = torch.frexp(r.abs())
    h = (((ex.long() - 12).clamp_min(-25) + 1023) << 52).view(torch.float64)
    return torch.where(r == 0, torch.full_like(h, 2.0 ** -25), h)


class Fp16Check:
    """accumulates the rounding criterion over the launches of one test, and the worst |out - r| / (beta + half an fp16
    ulp at r): how much of the bound plus the final rounding the kernel used"""

    def __init__(self, what):
        self.what, self.n, self.strict, self.worst = what, 0, 0, 0.0

    def __call__(self, got, r, beta, locate, label=""):
        g = got.double()
        lo, hi = rn16(r - beta), rn16(r + beta)
        ok = (g >= lo) & (g <= hi)
        bad = ~ok
        nbad = int(bad.sum())
        if nbad:
            lines = []
            for idx in bad.nonzero()[:8].tolist():
                i = tuple(idx)
                lines.append(f"{locate(*i)}: got {g[i].item()!r}, r {r[i].item()!r}, beta {beta[i].item():.3e}, "
                             f"accepted [{lo[i].item()!r}, {hi[i].item()!r}]")
            pytest.fail(f"{self.what} {label}: {nbad} of {g.numel()} fp16 outputs outside the rounding criterion; "
                        "first:\n  " + "\n  ".join(lines))
        self.n += g.numel()
        self.strict += int((lo == hi).sum())
        self.worst = max(self.worst, float(((g - r).abs() / (beta + _half_ulp16(r))).max()))

    def report(self):
        share = self.strict / max(self.n, 1)
        print(f"\n{self.what}: {self.n} fp16 outputs, {100 * share:.2f}% in the strict class, worst |out - r| / "
              f"(beta + half ulp) {self.worst:.3f}")
        assert share >= STRICT_MIN, f"{self.what}: only {100 * share:.1f}% of the outputs in the strict class"
        return share


class Worst:
    """the largest |error| / bound seen by a test, for its printed summary"""

    def __init__(self, what):
        self.what, self.v = what, 0.0

    def __call__(self, err, beta, locate, label=""):
        frac = err / beta.clamp_min(1e-300)
        bad = ~(err <= beta)
        if bad.any():
            lines = [f"{locate(*tuple(i))}: |err| {err[tuple(i)].item():.3e}, bound {beta[tuple(i)].item():.3e}"
                     for i in bad.nonzero()[:8].tolist()]
            pytest.fail(f"{self.what} {label}: {int(bad.sum())} of {err.numel()} elements exceed the bound; "
                        "first:\n  " + "\n  ".join(lines))
        self.v = max(self.v, float(frac.max()))

    def report(self):
        print(f"\n{self.what}: worst |error| / bound {self.v:.3f}")


def _loc_nhwc(samples):
    return lambda n, y, x, c: f"(sample {samples[n]}, pixel ({y}, {x}), channel {c})"


def _loc_rc(r, c):
    return f"(row {r}, column {c})"


def _launch(full, fn):
    """NaN-fill `full` (the output plus one guard sample / row), run fn twice: guard untouched, every element written,
    same bits both times.  Returns the output (all but the last entry)."""
    bits = {2: torch.int16, 4: torch.int32}[full.element_size()]
    full.fill_(NAN)
    fn()
    torch.cuda.synchronize()
    assert torch.isnan(full[-1]).all(), "the guard behind the output was written"
    first = full.clone()
    full.fill_(NAN)
    fn()
    torch.cuda.synchronize()
    assert torch.equal(first.view(bits), full.view(bits)), "a second launch gives different bits"
    out = full[:-1]
    nw = int(torch.isnan(out).sum())
    assert nw == 0, f"{nw} of {out.numel()} output elements not written"
    return out


# ------------------------------------------------------------------------------------------------------------------
# gn_finalize: exact
# ------------------------------------------------------------------------------------------------------------------
def _fma32(x, y, z):
    """fp32 fma(x, y, z) with one rounding, exactly: x*y is exact in fp64, TwoSum gives the error of the fp64 sum, and
    only an fp64 sum lying exactly on an fp32 midpoint needs that error to decide the direction"""
    x, y, z = (np.asarray(v, dtype=np.float32) for v in (x, y, z))
    p = x.astype(np.float64) * y.astype(np.float64)
    zd = z.astype(np.float64)
    s = p + zd
    bb = s - p
    e = (p - (s - bb)) + (zd - bb)
    r = s.astype(np.float32)
    toward = np.where(s > r.astype(np.float64), np.float32(np.inf), np.float32(-np.inf))
    other = np.nextafter(r, toward)
    mid = (r.astype(np.float64) + other.astype(np.float64)) / 2
    tie = (s == mid) & (e != 0) & (s != r.astype(np.float64))
    pick = np.where(e > 0, np.maximum(r, other), np.minimum(r, other))
    return np.where(tie, pick, r).astype(np.float32)


def _gn_stats(rng, N, Ca, Ta, Cb, Tb, HW, kinds):
    """slot tensors [N][T][C/2][2] whose group totals are exact in fp64 and hit a chosen variance: per group, integer
    filler in every slot, one carrier pair (slot 0, first pair) that fixes sum = m*count and the integer part of the sum
    of squares, and a second carrier holding D, the fp32 value (with at most 28 fractional bits) of var * count"""
    C = Ca + Cb
    cpg = C // 32
    count = HW * cpg
    st = [np.zeros((N, T, c // 2, 2)) for c, T in ((Ca, Ta), (Cb, max(Tb, 1)))]
    for s_ in st:
        s_[..., 0] = rng.integers(-8, 9, s_.shape[:-1])
        s_[..., 1] = rng.integers(0, 65, s_.shape[:-1])
    m_max = int(math.isqrt((1 << 22) // count))
    Ts = (Ta, Tb)
    cell = lambda p: (0, p) if p < Ca // 2 else (1, p - Ca // 2)  # noqa: E731
    pairs = np.concatenate([st[0].sum(1), st[1].sum(1)], 1) if Cb else st[0].sum(1)
    grp = pairs.reshape(N, 32, cpg // 2, 2).sum(2)  # filler totals per group
    for n in range(N):
        for g in range(32):
            p0 = g * cpg // 2
            c0 = cell(p0)
            if cpg // 2 >= 2:
                c1 = (cell(p0 + 1), 0)
            elif Ts[c0[0]] >= 2:
                c1 = (c0, 1)
            else:
                c1 = None
            kind = kinds[(n * 32 + g) % len(kinds)]
            m = int(rng.integers(-m_max, m_max + 1)) if c1 is not None else 0
            if kind == "negative" and m == 0 and c1 is not None and m_max >= 1:
                m = 1
            var = {"zero": 0.0, "eps": 1e-6, "eps5": 1e-5, "1e3eps": 1e-3, "one": 1.0,
                   "negative": -0.5 * m * m - 1e-3}[kind]
            D = float(np.float32(var * count))
            D = math.ldexp(round(math.ldexp(D, 28)), -28)
            assert float(np.float32(D)) == D
            x0 = st[c0[0]][n, 0, c0[1]]
            if c1 is None:
                x0[0], x0[1] = 0.0, D  # the group's only item (m = 0)
                continue
            x1 = st[c1[0][0]][n, c1[1], c1[0][1]]
            x0[0] = m * count - (grp[n, g, 0] - x0[0])
            others = grp[n, g, 1] - x0[1] - x1[1]
            x1[1] = D
            x0[1] = m * m * count - others
    for s_ in st:
        assert np.array_equal(s_.astype(np.float32).astype(np.float64), s_), "slot value not exact in fp32"
    return st[0], (st[1] if Cb else None)


def _gn_expect(sa, sb, Ca, Cb, HW, gamma, beta, eps, ss):
    """candidate (a, b) per (sample, channel) of gn_finalize's operation order: fp64 mean, var (the multiply-subtract
    plain or fused), the clamp, rstd = (float)(1/sqrt(var + (double)eps)), then fp32 a = gamma*rstd and b = beta -
    fmean*a, and with scale_shift a*sc, b*sc + sh, each multiply-add plain or fused"""
    N = sa.shape[0]
    C = Ca + Cb
    cpg = C // 32
    pairs = sa.sum(1) if sb is None else np.concatenate([sa.sum(1), sb.sum(1)], 1)  # exact: dyadics of <= 53 bits
    grp = pairs.reshape(N, 32, cpg // 2, 2).sum(2)
    count = float(np.float32(HW) * np.float32(cpg))
    epsd = float(np.float32(eps))
    cands = []
    for fused in (False, True):
        rstd = np.zeros((N, 32), np.float32)
        fmean = np.zeros((N, 32), np.float32)
        for n in range(N):
            for g in range(32):
                s, q2 = float(grp[n, g, 0]), float(grp[n, g, 1])
                mean = s / count
                q = q2 / count
                var = float(Fraction(q) - Fraction(mean) ** 2) if fused else q - mean * mean
                var = max(var, 0.0)
                rstd[n, g] = np.float32(1.0 / math.sqrt(var + epsd))
                fmean[n, g] = np.float32(mean)
        rs = np.repeat(rstd, cpg, 1)
        fm = np.repeat(fmean, cpg, 1)
        a = (gamma[None] * rs).astype(np.float32)
        bs = [(beta[None] - (fm * a).astype(np.float32)).astype(np.float32), _fma32(-fm, a, np.broadcast_to(beta, a.shape))]
        if ss is not None:
            sc = (np.float32(1.0) + ss[:, :C]).astype(np.float32)
            sh = ss[:, C:2 * C]
            a = (a * sc).astype(np.float32)
            bs = [v for b in bs for v in ((b * sc).astype(np.float32) + sh, _fma32(b, sc, sh))]
        cands.append((a, [np.asarray(b, np.float32) for b in bs]))
    return cands


GN_EDGE = [
    # (N, Ca, Ta, Cb, Tb, HW, ss_stride, eps): seam inside a group (200 + 184, cpg 12), cpg > 32 (C = 2048, the lanes
    # loop twice), one slot, scale_shift with ss_stride > 2C, both eps values
    (3, 200, 2, 184, 3, 64, 0, 1e-6),
    (2, 2048, 2, 0, 0, 16, 0, 1e-5),
    (2, 1024, 1, 1024, 4, 64, 4096 + 96, 1e-5),
    (4, 64, 1, 0, 0, 64, 0, 1e-6),
    (2, 96, 3, 160, 1, 256, 640, 1e-6),
]


@pytest.mark.parametrize("row", [pytest.param(r, id="edge-" + "-".join(map(str, r))) for r in GN_EDGE] + ["plans"])
def test_gn_finalize_exact(cuda_device, row):
    """gn_finalize from statistics slots filled directly with integers (and one fp32 carrier of var*count per group),
    so that the kernel's fp64 sums are exact whatever their order: mean, var, the clamp, rstd and the fp32 affine (and
    the scale/shift step) are emulated bit for bit, accepting the plain and the fused form of every multiply-add.
    Groups have variance 0, ~eps, ~10 eps, ~1e3 eps and ~1, and negative ss/count - mean^2 (the clamp)."""
    ops = _ops()
    dev = cuda_device
    rows = GN_EDGE if row != "plans" else _rows("gn_finalize")
    rows = [row] if row != "plans" else rows
    if not rows:
        pytest.skip("no production shapes tabled")
    rng = np.random.default_rng(7)
    kinds = ["zero", "eps", "eps5", "1e3eps", "one", "negative"]
    for (N, Ca, Ta, Cb, Tb, HW, ss_stride, eps) in rows:
        C = Ca + Cb
        sa, sb = _gn_stats(rng, N, Ca, Ta, Cb, Tb, HW, kinds)
        gamma = rng.standard_normal(C).astype(np.float32)
        beta = rng.standard_normal(C).astype(np.float32)
        ss = None
        ss_dev = None
        if ss_stride:
            off = 7
            emb = rng.standard_normal((N, ss_stride)).astype(np.float32)  # rows of emb_total floats, as the engine
            ss = emb[:, off:off + 2 * C]
            ss_dev = torch.from_numpy(emb).to(dev)[:, off:off + 2 * C]
        full = torch.empty(N + 1, C, 2, dtype=torch.float32, device=dev)
        ta = torch.from_numpy(sa).float().to(dev)
        tb = torch.from_numpy(sb).float().to(dev) if sb is not None else None
        g_d, b_d = torch.from_numpy(gamma).to(dev), torch.from_numpy(beta).to(dev)
        out = _launch(full, lambda: ops.gn_finalize(ta, Ca, tb, Cb, g_d, b_d, eps, N, HW, full[:-1], ss_dev,
                                                    ss_stride)).cpu().numpy()
        ok = np.zeros((N, C), bool)
        for a, bs in _gn_expect(sa, sb, Ca, Cb, HW, gamma, beta, eps, ss):
            okb = np.zeros((N, C), bool)
            for b in bs:
                okb |= out[..., 1] == b
            ok |= (out[..., 0] == a) & okb
        if not ok.all():
            bad = np.argwhere(~ok)[:8]
            a0, b0 = _gn_expect(sa, sb, Ca, Cb, HW, gamma, beta, eps, ss)[0]
            pytest.fail(f"gn_finalize {(N, Ca, Ta, Cb, Tb, HW, ss_stride, eps)}: {int((~ok).sum())} of {ok.size} (a, b) "
                        "wrong; first:\n  " + "\n  ".join(
                            f"(sample {n}, channel {c}, group {c // (C // 32)}): got ({out[n, c, 0]!r}, {out[n, c, 1]!r}),"
                            f" want ({a0[n, c]!r}, {b0[0][n, c]!r})" for n, c in bad))


def _gamma(d):
    return d * U / (1 - d * U)


@pytest.mark.parametrize("N,H,W,C", [(2, 32, 32, 128), (2, 64, 64, 256)])
def test_default_groupnorm_path_at_large_mean(cuda_device, N, H, W, C):
    """The default GroupNorm path: a 1x1 conv writes its fp32 tile statistics, gn_finalize turns them into (a, b).
    Operands are integers (inputs in [-3, 3], 16 weights of +-1 per output channel, integer bias), so every conv output
    is an integer the fp16 output holds exactly, and the fp64 GroupNorm of that output is the exact reference.  Group 5's
    bias of 250 against a spread of ~8 puts |mean|/std near 30.

    Bound, from conv_gemm.cu's epilogue order (NB = 1 tiles): a slot's channel-pair sum adds the two channels (1
    addition), folds the quarter's 32 rows as a 5-level tree (tree_add, rowgroup_sum), adds the MT sub-tiles in order
    (MT - 1 additions) and the 4 quarters from 0 (3 additions): every term passes at most d_s = 8 + MT roundings, so
    |s' - s| <= gamma(d_s) sum|v|.
    The sum of squares adds the rounding of each square: gamma(d_s + 1) sum v^2.  gn_finalize sums the slots in fp64
    (2^-52 per slot and term, negligible but counted).  Then with S, Q the group sums and count = HW*cpg:
      dm = dS/count,  dvar = dQ/count + (2|mean| + dm) dm: the E[x^2] - mean^2 cancellation turns the relative error
      gamma(d) of Q into gamma(d) (mean^2 + var)/var of var, ~900 gamma(d) at |mean|/std = 30;
      rstd' = (float)(1/sqrt(var' + eps)) lies in [1/sqrt(var + eps + dvar), 1/sqrt(max(var + eps - dvar, eps))], plus u;
      a' = RN(gamma rstd'): da = |gamma| drstd + u|gamma| (rstd + drstd);
      fmean = RN32(mean'): dfm = dm + u(|mean| + dm);
      b' = beta - fmean a' (plain or fused): db = (|mean| da + (|a| + da) dfm)(1 + 2u) + 2u (|mean| + dfm)(|a| + da)
      + 2u|b|.
    The consumer applies y' = a' x + b'.  Writing b' = beta - fmean a' + e_b with |e_b| <= 2u(|fmean a'| + |b'|) (the
    product and the subtraction, or one fused rounding), y' - y = (a' - a)(x - mean) - a'(fmean - mean) + e_b, so
      |y' - y| <= da |x - mean| + (|a| + da) dfm + 2u (2 (|mean| + dfm)(|a| + da) + |b|):
    the errors of a and b cancel against each other at x ~ mean.  The worst error of the large-mean group is printed as
    a fraction of that bound."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(21)
    BN, MT = ops.conv_tile_config(H, W, C, False)
    assert W >= 16 and H >= 16  # NB = 1 tiles: the order above
    cpg = C // 32
    x = torch.randint(-3, 4, (N, H, W, 64), generator=g).half()
    w = torch.zeros(C, 64)
    for o in range(C):
        w[o, torch.randperm(64, generator=g)[:16]] = torch.randint(0, 2, (16,), generator=g).float() * 2 - 1
    bias = torch.randint(-20, 21, (C,), generator=g).float()
    bias[5 * cpg:6 * cpg] = 250.0
    out = torch.empty(N, H, W, C, dtype=torch.float16, device=dev)
    st = ops.new_stats(N, H, W, C, dev, False)
    ops.ConvOp([(x.to(dev), ops.MODE_1x1)], ops.pack_conv_weight(w).to(dev), out=out, ebias=bias.to(dev),
               stats=st).launch()
    torch.cuda.synchronize()
    v = out.double().cpu()
    exact = torch.einsum("nhwi,oi->nhwo", x.double(), w.double()) + bias.double()
    assert torch.equal(v, exact), "conv output not the exact integer"
    gam = torch.randn(C, generator=g) + 1.0
    bet = torch.randn(C, generator=g)
    eps = 1e-6
    full = torch.empty(N + 1, C, 2, device=dev)
    aff = _launch(full, lambda: ops.gn_finalize(st, C, None, 0, gam.to(dev), bet.to(dev), eps, N, H * W,
                                                full[:-1])).double().cpu()
    vg = v.reshape(N, H * W, 32, cpg)
    count = H * W * cpg
    S = vg.sum((1, 3))
    Q = (vg * vg).sum((1, 3))
    A1 = vg.abs().sum((1, 3))
    mean = S / count
    var = Q / count - mean * mean
    ds = 8 + MT
    nterm = st.shape[1] * cpg / 2 + 1
    dS = _gamma(ds) * A1 + 2.0 ** -52 * nterm * A1
    dQ = _gamma(ds + 1) * Q + 2.0 ** -52 * nterm * Q
    dm = dS / count
    dvar = dQ / count + (2 * mean.abs() + dm) * dm + 4 * 2.0 ** -53 * Q / count
    epsd = float(np.float32(eps))
    r = 1 / torch.sqrt(var + epsd)
    lo = 1 / torch.sqrt(var + epsd + dvar)
    hi = 1 / torch.sqrt(torch.clamp(var + epsd - dvar, min=epsd))
    dr = torch.maximum(hi - r, r - lo) + U * hi
    rep = lambda t: t.repeat_interleave(cpg, 1)  # noqa: E731
    gd, bd = gam.double(), bet.double()
    a = gd * rep(r)
    b = bd - rep(mean) * a
    da = gd.abs() * rep(dr) + U * gd.abs() * rep(r + dr)
    dfm = rep(dm + U * (mean.abs() + dm))
    db = (rep(mean.abs()) * da + (a.abs() + da) * dfm) * (1 + 2 * U) + 2 * U * (rep(mean.abs()) + dfm) * \
        (a.abs() + da) + 2 * U * b.abs()
    worst = Worst(f"default GroupNorm path {N}x{H}x{W}x{C}")
    loc = lambda n, c: f"(sample {n}, channel {c}, group {c // cpg})"  # noqa: E731
    worst((aff[..., 0] - a).abs(), da, loc, "a")
    worst((aff[..., 1] - b).abs(), db, loc, "b")
    # the normalised output of group 5, per element
    xs = v[..., 5 * cpg:6 * cpg]
    sl = slice(5 * cpg, 6 * cpg)
    y_err = ((aff[:, None, None, sl, 0] - a[:, None, None, sl]) * xs + aff[:, None, None, sl, 1]
             - b[:, None, None, sl]).abs()
    bx = lambda t: t[:, None, None, sl]  # noqa: E731
    mc = rep(mean)
    y_beta = bx(da) * (xs - bx(mc)).abs() + bx((a.abs() + da) * dfm) + \
        2 * U * bx(2 * (mc.abs() + dfm) * (a.abs() + da) + b.abs())
    yw = Worst("normalised output of the large-mean group")
    yw(y_err, y_beta, lambda n, yy, xx, c: f"(sample {n}, pixel ({yy}, {xx}), channel {5 * cpg + c})")
    ratio = float((mean[:, 5].abs() / var[:, 5].sqrt()).min())
    print(f"\ndefault GroupNorm path {N}x{H}x{W}x{C} (BN={BN}, MT={MT}): |mean|/std of group 5 >= {ratio:.1f}; worst "
          f"normalised-output error {float(y_err.max()):.3e} ({yw.v:.3f} of its bound), worst a/b error "
          f"{worst.v:.3f} of the bound")


# ------------------------------------------------------------------------------------------------------------------
# apply
# ------------------------------------------------------------------------------------------------------------------
def _silu_beta(t):
    """bound on |silu_f(t') - silu(t)| for t' = RN32(t) (the kernel's fmaf), silu_f(x) = x / (1 + __expf(-x)):
       |silu(t') - silu(t)| <= (|silu'(t)| + u|t|/2) u|t|  (|silu''| <= 1/2 between t and t');
       e' = __expf(-t') within k = 2 + floor(1.173|t'|) ulp, |e' - e| <= 2uk e;  d' = RN(1 + e'):
       |d' - (1 + e)| <= 2uk e + u(1 + e)(1 + 2uk), so |d'/(1+e) - 1| <= delta = 2uk e/(1+e) + u(1 + 2uk);
       q = RN(t'/d'):  |q - silu(t')| <= |silu(t')| (delta/(1 - delta) + u).
     Where e overflows fp32 (t < -87) the kernel returns -0 (t'/inf): the bound adds |silu(t)|."""
    k = 2.0 + torch.floor(1.173 * (t.abs() * (1 + U)))
    e = torch.exp(-t)
    s = t * torch.sigmoid(t)
    delta = 2 * U * k * (e / (1 + e)) + U * (1 + 2 * U * k)
    sg = torch.sigmoid(t)
    d1 = (sg * (1 + t * (1 - sg))).abs() + 0.5 * U * t.abs()
    beta = d1 * U * t.abs() + s.abs() * (delta / (1 - delta) + U) * (1 + 1e-9)
    return torch.where(t < -87.0, beta + s.abs(), beta), s


def _apply_case(ops, dev, g, N, Hi, Wi, Ca, Cb, act, resample, Caff, off, chk, exact):
    """one apply launch at (N, Hi, Wi, Ca, Cb) with the given affine layout, checked per element"""
    C = Ca + Cb
    Ho, Wo = (Hi // 2, Wi // 2) if resample == 1 else ((2 * Hi, 2 * Wi) if resample == 2 else (Hi, Wi))
    kw = dict(generator=g, device=dev)
    if act == 0:   # integers: a*x + b and the 2x2 sum exact in fp32
        xs = [torch.randint(-1024, 1025, (N, Hi, Wi, c), **kw).half() for c in (Ca, Cb)]
        ab = torch.stack([torch.randint(-127, 128, (N, max(Caff, 1)), **kw) / 64.0,
                          torch.randint(-32768, 32769, (N, max(Caff, 1)), **kw) / 64.0], -1).float()
    else:          # t = a*x + b spans [-90, 90]: __expf overflows for t < -88
        xs = [(torch.rand(N, Hi, Wi, c, **kw) * 180 - 90).half() for c in (Ca, Cb)]
        ab = torch.stack([torch.rand(N, max(Caff, 1), **kw) * 0.5 + 0.75,
                          torch.rand(N, max(Caff, 1), **kw) * 4 - 2], -1).float()
    xa = xs[0]
    xb = xs[1] if Cb else None
    aff = ab if Caff else None
    full = torch.empty(N + 1, Ho, Wo, C, dtype=torch.float16, device=dev)
    out = _launch(full, lambda: ops.apply(xa, xb, aff, full[:-1], act, resample, off))
    sm = _pick(N, Ho * Wo * C)
    idx = torch.tensor(sm, device=dev)
    x = torch.cat([xa[idx]] + ([xb[idx]] if Cb else []), -1).double()
    if Caff:
        a = aff[idx, off:off + C, 0].double()[:, None, None]
        b = aff[idx, off:off + C, 1].double()[:, None, None]
        t = x * a + b
    else:
        t = x
    if act:
        beta, s = _silu_beta(t)
    else:
        beta, s = torch.zeros_like(t), t
    if resample == 1:
        q = [s[:, i::2, j::2] for i in (0, 1) for j in (0, 1)]
        bq = [beta[:, i::2, j::2] for i in (0, 1) for j in (0, 1)]
        r = 0.25 * (q[0] + q[1] + q[2] + q[3])
        mag = q[0].abs() + q[1].abs() + q[2].abs() + q[3].abs()
        # ((s0 + s1) + s2) + s3 in fp32 (three roundings, each <= u * partial sum magnitude), then * 0.25 (exact)
        beta = 0.25 * (bq[0] + bq[1] + bq[2] + bq[3] + (3 * U * mag if act else 0.0))
    elif resample == 2:
        r = s.repeat_interleave(2, 1).repeat_interleave(2, 2)
        beta = beta.repeat_interleave(2, 1).repeat_interleave(2, 2)
    else:
        r = s
    got = out[idx]
    label = f"N={N} {Hi}x{Wi} C={Ca}+{Cb} act={act} resample={resample} affine={'None' if not Caff else f'{off} of {Caff}'}"
    if exact:
        want = rn16(r)
        bad = got.double() != want
        if bad.any():
            i = tuple(bad.nonzero()[0].tolist())
            pytest.fail(f"apply {label}: {int(bad.sum())} of {got.numel()} outputs not RN16 of the exact value; first "
                        f"{_loc_nhwc(sm)(*i)}: got {got[i].item()!r}, want {want[i].item()!r}")
        chk.n += got.numel()
        chk.strict += got.numel()
        chk.worst = max(chk.worst, float(((got.double() - r).abs() / _half_ulp16(r)).max()))
    else:
        chk(got, r, beta, _loc_nhwc(sm), label)


def _apply_edge(dev):
    sms = _sms(dev)
    big_n = 8 * sms + 5  # max_gx = 1
    rows = []
    for C in (64, 192, 384, 768, 1536, 2048):
        rows.append((3, 12, 12, C, 0, C, 0))
    rows += [
        (16, 60, 60, 192, 0, 192, 0),   # gx capped at 8*SMs/N; npix not a multiple of stride*U
        (big_n, 4, 4, 64, 0, 64, 0),    # N > 8*SMs: one block column per sample
        (2, 8, 8, 96, 160, 512, 256),   # two sources, affine_offset into a wider table
        (2, 8, 8, 128, 0, 0, 0),        # affine = None
    ]
    return rows


@pytest.mark.parametrize("act", [0, 1])
def test_apply_edges(cuda_device, act):
    """apply at edge shapes: every channel count class (octets not dividing 256, one pixel per block, C = 2048), a
    capped grid with a ragged tail, N > 8*SMs, two sources with affine_offset, affine = None; all three resample modes.
    act = 0: integer x, dyadic (a, b): RN16 of the exact value, bit for bit.  act = 1: the rounding criterion with
    beta from _silu_beta (and for the 2x2 average the three fp32 additions)."""
    ops = _ops()
    g = torch.Generator(device=cuda_device).manual_seed(11)
    chk = Fp16Check(f"apply edges act={act}")
    for (N, H, W, Ca, Cb, Caff, off) in _apply_edge(cuda_device):
        for resample in (0, 1, 2):
            _apply_case(ops, cuda_device, g, N, H, W, Ca, Cb, act, resample, Caff, off, chk, exact=act == 0)
    chk.report()


@pytest.mark.parametrize("act", [0, 1])
def test_apply_plans(cuda_device, act):
    """apply at every tabled production shape, with both activations (the table's own act is one of them)"""
    ops = _ops()
    rows = _rows("apply")
    if not rows:
        pytest.skip("no production shapes tabled")
    g = torch.Generator(device=cuda_device).manual_seed(12)
    chk = Fp16Check(f"apply production act={act}")
    for (N, Hi, Wi, Ca, Cb, _act, resample, Caff, off) in rows:
        _apply_case(ops, cuda_device, g, N, Hi, Wi, Ca, Cb, act, resample, Caff, off, chk, exact=act == 0)
        torch.cuda.empty_cache()
    chk.report()


# ------------------------------------------------------------------------------------------------------------------
# pack_input, unpack_nchw, transpose_tc, axpby: exact
# ------------------------------------------------------------------------------------------------------------------
def test_pack_unpack_transpose_axpby_exact(cuda_device):
    """pack_input: RN16 of each fp32 input (torch's float -> half is one round-to-nearest-even), zero channels >= Cin;
    unpack_nchw: exact widening; transpose_tc: exact copy, including the v slice of qkv (ld = 3C); axpby: integer fp16
    operands and dyadic coefficients, so alpha*a + beta*b is exact in fp32 (plain or fused) and the output is its
    RN16.  Production shapes from the table, plus grids capped at 16 resp. 8 blocks per SM."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(13)
    sms = _sms(dev)
    packs = _rows("pack_input") + [(3, 3, 33, 35), (2 * sms, 3, 64, 64)]
    for (N, Cin, H, W) in packs:
        x = (torch.randn(N, Cin, H, W, generator=g) * 300).to(dev)
        full = torch.empty(N + 1, H, W, 64, dtype=torch.float16, device=dev)
        out = _launch(full, lambda: ops.pack_input(x, full[:-1]))
        want = torch.zeros_like(out)
        want[..., :Cin] = x.permute(0, 2, 3, 1).half()
        bad = out.view(torch.int16) != want.view(torch.int16)
        if bad.any():
            i = tuple(bad.nonzero()[0].tolist())
            pytest.fail(f"pack_input {(N, Cin, H, W)}: {int(bad.sum())} wrong; first {_loc_nhwc(list(range(N)))(*i)}: "
                        f"got {out[i].item()!r}, want {want[i].item()!r}")
        del x, full, out, want
    for (N, C, H, W) in _rows("unpack_nchw") + [(3, 136, 7, 9)]:
        h = (torch.randn(N, H, W, C, generator=g) * 100).half().to(dev)
        full = torch.empty(N + 1, C, H, W, dtype=torch.float32, device=dev)
        out = _launch(full, lambda: ops.unpack_nchw(h, full[:-1]))
        assert torch.equal(out, h.permute(0, 3, 1, 2).float()), f"unpack_nchw {(N, C, H, W)}"
    for (N, T, C, ld) in _rows("transpose_tc") + [(2, 64, 512, 1536), (3, 256, 64, 192), (1, 1024, 256, 768),
                                                  (2, 200, 96, 96)]:
        qkv = torch.randn(N, T, ld, generator=g).half().to(dev)
        src = qkv[:, :, ld - C:]
        full = torch.empty(N + 1, C, T, dtype=torch.float16, device=dev)
        out = _launch(full, lambda: ops.transpose_tc(src, full[:-1]))
        bad = out.view(torch.int16) != src.transpose(1, 2).contiguous().view(torch.int16)
        if bad.any():
            n, c, t = bad.nonzero()[0].tolist()
            pytest.fail(f"transpose_tc {(N, T, C, ld)}: {int(bad.sum())} wrong; first (sample {n}, channel {c}, t {t})")
    gd = torch.Generator(device=dev).manual_seed(13)
    for numel in (8, 8 * 1000 + 8, 16 * 64 * 64 * 128, 8 * sms * 256 * 8 * 3 + 24):
        a = torch.randint(-2048, 2049, (numel + 8,), generator=gd, device=dev).half()
        b = torch.randint(-2048, 2049, (numel + 8,), generator=gd, device=dev).half()
        full = torch.empty(numel + 8, dtype=torch.float16, device=dev).view(-1, 8)
        out = _launch(full, lambda: ops.axpby(a[:numel], b[:numel], full[:-1], 0.8125, -1.375)).reshape(-1)
        want = rn16(0.8125 * a[:numel].double() - 1.375 * b[:numel].double())
        bad = out.double() != want
        if bad.any():
            i = int(bad.nonzero()[0])
            pytest.fail(f"axpby numel={numel}: {int(bad.sum())} wrong; first element {i}: got {out[i].item()!r}, "
                        f"want {want[i].item()!r}")


# ------------------------------------------------------------------------------------------------------------------
# sampler updates
# ------------------------------------------------------------------------------------------------------------------
def _schedules():
    from asyrp_official_b200.schedule import Schedule, make_sequences
    from asyrp_official_b200.utils.diffusion_utils import get_beta_schedule
    b64 = get_beta_schedule(beta_start=1e-4, beta_end=0.02, num_diffusion_timesteps=1000)
    betas = torch.from_numpy(b64).float()
    ac = np.cumprod(1.0 - b64)
    logvar = np.log(np.maximum(b64 * (1.0 - np.append(1.0, ac[:-1])) / (1.0 - ac), 1e-20))
    out = []
    for n_step in (40, 50):
        seq, seq_next = make_sequences(999, n_step)
        out.append(Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=200))
        out.append(Schedule(betas, seq, seq_next, t_edit=500, t_addnoise=200, dt_lambda=0.9985, dt_end=950))
        out.append(Schedule(betas, seq, seq_next, t_edit=500, sample_type="ddpm", logvars=logvar))
    return out


def _sampler_rows():
    return sorted(set(_rows("ddim_update")) | {(2, 3, 17, 19, 6), (3, 3, 8, 8, 3)})


def test_ddim_update_bit_for_bit(cuda_device):
    """ddim_update against torch fp32 on the CPU in the reference's order (utils/diffusion_utils.py:84-100):
    x0 = (x - em*sqrt(1-at)) / sqrt(at), next = sqrt(an)*x0 + c2*et (+ c1*z), each operation one IEEE rounding, so the
    kernel must match bit for bit for eta = 0 and eta > 0 alike.  The coefficients are those Schedule passes (eta = 1
    below t_addnoise, the last step's an = 1, dt_lambda != 1 at t >= dt_end).  With dt_lambda the reference computes
    (sqrt(1-an)*et)*dt_lambda where the engine passes c2 = sqrt(1-an)*dt_lambda: the two differ by at most one rounding
    of each product, bounded separately.  Production N x 3 x S^2 with the learned-sigma split (Ce = 6), x_next aliasing
    x as the engine calls it, and x0_out."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(14)
    steps = [s for sch in _schedules() for s in sch.steps if s.kind == "ddim"]
    # dt_lambda steps: eta = 0 (c1 = 0), yet c2 is not the fp32 sqrt(1 - an) of a plain eta = 0 step
    is_dt = [s.c1 == 0 and s.c2 != float((1 - torch.tensor(s.an)).sqrt()) for s in steps]
    dt_steps = [s for s, d in zip(steps, is_dt) if d]
    assert dt_steps, "the dt_lambda schedules pass no step with c2 = sqrt(1-an)*dt_lambda"
    sel = [steps[i] for i in sorted({0, 1, 20, 25, 36, 38, 39, len(steps) // 2, len(steps) - 1})] + \
        [s for s in steps if s.c1 != 0][:2] + [s for s in steps if s.an == 1.0][:1]
    rows = _sampler_rows()
    # production rows cycle through the selected steps; every selected step and every dt_lambda step also runs at a
    # small ragged shape
    cases = [(row, alias, sel[(2 * i + j) % len(sel)])
             for i, row in enumerate(rows) for j, alias in enumerate((True, False))]
    cases += [((2, 3, 17, 19, 6), True, s) for s in sel + dt_steps] + [(rows[-1], True, dt_steps[0])]
    n_dt = 0
    for (N, Cx, H, W, Ce), alias, s in cases:
        x = torch.randn(N, Cx, H, W, generator=g) * 3
        et = torch.randn(N, Ce, H, W, generator=g)
        em = torch.randn(N, Ce, H, W, generator=g)
        z = torch.randn(N, Cx, H, W, generator=g) if s.c1 != 0 else None
        xd, etd, emd = x.to(dev), et.to(dev), em.to(dev)
        zd = z.to(dev) if z is not None else None
        x0f = torch.full((N + 1, Cx, H, W), NAN, device=dev)
        if alias:
            ops.ddim_update(xd, etd, emd, zd, xd, x0f[:-1], s.at, s.an, s.c1, s.c2)
            torch.cuda.synchronize()
            got = xd.cpu()
            assert torch.isnan(x0f[-1]).all()
            x0g = x0f[:-1].cpu()
        else:
            full = torch.empty(N + 1, Cx, H, W, device=dev)
            got = _launch(full, lambda: ops.ddim_update(xd, etd, emd, zd, full[:-1], x0f[:-1], s.at, s.an, s.c1,
                                                       s.c2)).cpu()
            x0g = x0f[:-1].cpu()
        at, an = torch.tensor(s.at), torch.tensor(s.an)
        e, m = et[:, :Cx], em[:, :Cx]
        x0 = (x - m * (1 - at).sqrt()) / at.sqrt()
        want = an.sqrt() * x0 + torch.tensor(s.c2) * e
        if z is not None:
            want = want + torch.tensor(s.c1) * z
        for name, gg, ww in (("x0_t", x0g, x0), ("x_next", got, want)):
            bad = gg.view(torch.int32) != ww.view(torch.int32)
            if bad.any():
                n, c, y, xx = bad.nonzero()[0].tolist()
                pytest.fail(f"ddim_update {(N, Cx, H, W, Ce)} t={s.t} c1={s.c1} alias={alias} {name}: "
                            f"{int(bad.sum())} of {gg.numel()} differ; first (sample {n}, channel {c}, pixel "
                            f"({y}, {xx})): got {gg[n, c, y, xx].item()!r}, want {ww[n, c, y, xx].item()!r}")
        if s.c1 == 0 and s.c2 != float((1 - an).sqrt()):  # dt_lambda step: the reference's own order
            lam = 0.9985
            n_dt += 1
            ref = an.sqrt() * x0 + (1 - an).sqrt() * e * lam
            # the two product terms differ by at most two roundings each, the two sums by one each
            beta = 4 * U * (torch.tensor(s.c2).abs() * e.abs()).double() * 1.01 + 2 * U * ref.abs().double() * 1.01
            assert ((got.double() - ref.double()).abs() <= beta).all(), "dt_lambda reassociation bound"
    assert n_dt >= len(dt_steps) + 1, (n_dt, len(dt_steps))


def test_ddpm_update(cuda_device):
    """ddpm_update against torch fp32 in the reference's order (utils/diffusion_utils.py:74-82): weight, 1/sqrt(1-bt),
    mean and the final add are IEEE operations in the same order; only expf(0.5*lv) may differ from the exact exp, by
    at most 2 ulp <= 4u e.  So with mask 0 the output is the mean bit for bit, and with mask 1
       |out - (mean + e z)| <= 4u e|z| + u e|z|(1 + 4u) + u(|mean| + e|z|)(1 + 5u)  (product rounding, final add),
    where mean and e are computed in fp64 from the kernel's own fp32 mean.  Learned logvar spans [-40, 4] (where
    __expf would be off by up to 25 ulp) and the fixed table's entries are used as Schedule passes them; in place."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(15)
    steps = [s for sch in _schedules() for s in sch.steps if s.kind == "ddpm"]
    few = [steps[5], steps[-1]]  # the last step has mask 0
    steps = [steps[i] for i in (0, 5, 20, len(steps) - 2, len(steps) - 1)]
    worst = Worst("ddpm_update")
    for (N, Cx, H, W, Ce) in _sampler_rows():
        for learned in ((False, True) if Ce >= 2 * Cx else (False,)):
            for s in (few if N * Cx * H * W > (1 << 20) else steps):
                x = torch.randn(N, Cx, H, W, generator=g) * 3
                et = torch.randn(N, Ce, H, W, generator=g)
                if learned:
                    et[:, Cx:2 * Cx] = torch.rand(N, Cx, H, W, generator=g) * 44 - 40
                x[::2] = 0.0  # mean exactly 0: the output is the rounded e*z alone
                et[::2, :Cx] = 0.0
                z = torch.randn(N, Cx, H, W, generator=g)
                xd = x.to(dev)
                ops.ddpm_update(xd, et.to(dev), z.to(dev), xd, s.at, s.bt, s.logvar, learned, s.mask)
                torch.cuda.synchronize()
                got = xd.cpu()
                at, bt = torch.tensor(s.at), torch.tensor(s.bt)
                weight = bt / torch.sqrt(1 - at)
                mean = 1 / torch.sqrt(1.0 - bt) * (x - weight * et[:, :Cx])
                lv = et[:, Cx:2 * Cx] if learned else torch.full_like(x, s.logvar)
                loc = lambda n, c, y, xx: f"(sample {n}, channel {c}, pixel ({y}, {xx}))"  # noqa: E731
                if s.mask == 0.0:
                    bad = got.view(torch.int32) != mean.view(torch.int32)
                    assert not bad.any(), f"ddpm_update mask 0 t={s.t}: {int(bad.sum())} differ from the mean"
                    continue
                e = torch.exp(0.5 * lv.double())
                ez = (e * z.double()).abs()
                r = mean.double() + e * z.double()
                beta = 4 * U * ez + U * ez * (1 + 4 * U) + U * (mean.double().abs() + ez) * (1 + 5 * U)
                worst((got.double() - r).abs(), beta, loc, f"t={s.t} learned={learned}")
    worst.report()


# ------------------------------------------------------------------------------------------------------------------
# timestep embedding and the linears
# ------------------------------------------------------------------------------------------------------------------
def _f32(v):
    return float(np.float32(v))


def test_timestep_embedding(cuda_device):
    """every integer t in 0..999 and every t of the schedules, both variants, the production dims.  The reference is
    sin / cos (fp64) of t * exp(arg), arg the reference's fp32 argument (torch: arange * -(ln 1e4/(half-1)), resp.
    -ln 1e4 * arange / half).  The kernel's argument differs from it only through logf(1e4) (1 ulp) and its own
    roundings: |darg| is computed exactly for each candidate of logf.  Then
      fr' = expf(arg'): |fr' - fr| <= fr |darg| (1 + |darg|) + 4u fr'  (2 ulp)
      a' = RN(t fr'):   |a' - t fr| <= t |fr' - fr| + u t fr'
      sinf / cosf(a') within 2 ulp <= 4u |result|, and |sin(a') - sin(a)| <= |a' - a|.
    The existing absolute 2e-4 is looser than this bound for small t and tighter than it at t ~ 1000 and large a.
    This bound does not separate expf from __expf: __expf's extra error here stays inside it (test_ddpm_update does)."""
    ops = _ops()
    dev = cuda_device
    ts = set(range(1000))
    for sch in _schedules():
        ts |= {s.t for s in sch.steps}
    t = torch.tensor(sorted(ts), dtype=torch.float32)
    dims = sorted({d for (_, d, _) in _rows("timestep_embedding")} | {128, 192})
    worst = Worst("timestep_embedding")
    for variant in (0, 1):
        for dim in dims:
            half = dim // 2
            N = t.numel()
            td = t.to(dev)
            full = torch.empty(N + 1, dim, device=dev)
            out = _launch(full, lambda: ops.timestep_embedding(td, full[:-1], variant)).cpu().double()
            i = torch.arange(half, dtype=torch.float32)
            arg_ref = i * -(math.log(10000) / (half - 1)) if variant == 0 else -math.log(10000) * i / half
            darg = torch.zeros(half, dtype=torch.float64)
            L0 = np.float32(math.log(10000.0))
            for L in (np.nextafter(L0, np.float32(0)), L0, np.nextafter(L0, np.float32(100))):
                if variant == 0:
                    c = np.float32(-(L / np.float32(half - 1)))
                    a_k = (i.numpy() * c).astype(np.float32)
                else:
                    a_k = ((-L * i.numpy()).astype(np.float32) / np.float32(half)).astype(np.float32)
                darg = torch.maximum(darg, (torch.from_numpy(a_k).double() - arg_ref.double()).abs())
            fr = torch.exp(arg_ref.double())
            dfr = fr * darg * (1 + darg) + 4 * U * fr * (1 + darg) * 1.0001
            a = t.double()[:, None] * fr[None]
            da = t.double()[:, None] * dfr[None] + U * (a + t.double()[:, None] * dfr[None])
            s, c = torch.sin(a), torch.cos(a)
            want = torch.cat([s, c] if variant == 0 else [c, s], 1)
            beta = da.repeat(1, 2) + 4 * U * (want.abs() + da.repeat(1, 2))
            worst((out - want).abs(), beta, lambda n, j: f"(t {int(t[n])}, column {j})", f"variant={variant} dim={dim}")
    worst.report()


def _linear_rows():
    rows = [r for r in _rows("linear")]
    return rows + [(5, 192, 96, 200, 130, 1, 1), (3, 100, 40, 100, 40, 0, 1), (40, 128, 33, 128, 33, 1, 0)]


def test_linear(cuda_device):
    """linear_rows_kernel (I in {128, 256, 512, 1024}) and linear_kernel (any other I), at the temb MLP's and emb_cat's
    real (N, I, O) and the engine's strides.  Per output: lane l sums its I/32 products in order (acc += w*v, plain or
    fused), then a 5-level xor butterfly, then + bias: with n = I/32 + 6 additions on any path,
       |acc' - sum w v'| <= n u (1 + nu) (sum |w v'| + |bias|)
    and v' = act_in ? v/(1 + expf(-v)) : v carries |v' - silu(v)| <= |silu(v)| (4u e/(1+e) + 2u)(1 + 1e-6) (expf 2 ulp,
    one addition, one division).  act_out adds |silu'| <= 1.1 times the bound before it and |silu(r)|(4u + 2u) after."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(16)
    worst = Worst("linear")
    for (N, I, O, in_stride, out_stride, act_in, act_out) in _linear_rows():
        inp_full = torch.randn(N, in_stride, generator=g) * 3
        w = torch.randn(O, I, generator=g) / math.sqrt(I)
        b = torch.randn(O, generator=g)
        ind = inp_full.to(dev)[:, :I]
        wd, bd = w.to(dev), b.to(dev)
        full = torch.empty(N + 1, out_stride, device=dev)
        keep = torch.randn(N, out_stride - O, generator=g).to(dev)

        def run():
            full[:-1, O:] = keep
            ops.linear(ind, wd, bd, full[:-1], act_in=bool(act_in), act_out=bool(act_out))
        out = _launch(full, run)
        assert torch.equal(out[:, O:], keep), "linear wrote past its O columns"
        x = inp_full[:, :I].double()
        if act_in:
            e = torch.exp(-x)
            v = x * torch.sigmoid(x)
            dv = v.abs() * (4 * U * e / (1 + e) + 2 * U) * (1 + 1e-6)
        else:
            v, dv = x, torch.zeros_like(x)
        wd64 = w.double()
        y = v @ wd64.t() + b.double()
        n = -(-I // 32) + 6
        beta = n * U * (1 + n * U) * ((v.abs() + dv) @ wd64.abs().t() + b.double().abs()) + dv @ wd64.abs().t()
        if act_out:
            y2 = y * torch.sigmoid(y)
            beta = 1.1 * beta + y2.abs() * 6 * U
            y = y2
        worst((out[:, :O].cpu().double() - y).abs(), beta.cpu(), _loc_rc, f"{(N, I, O, in_stride, out_stride)}")
    worst.report()


# ------------------------------------------------------------------------------------------------------------------
# slerp_h
# ------------------------------------------------------------------------------------------------------------------
def _slerp_rows():
    rows = _rows("slerp_h")
    return rows + [(2, 16, 12, 512, 3)]


def test_slerp_h(cuda_device):
    """slerp_h with and without the mask.  Outside the masked window (rows 4..H-2, columns 3..4) h2 must equal h bit
    for bit; stats slots 1.. must be exactly 0.  Inside it the rounding criterion with a bound propagated from the
    kernel's order: each fp32 sum of squares / products has m = HW*C/256 sequential terms per thread then 5 + 8
    additions (block_sum), so |S' - S| <= (m + 13) u sum|terms|; nh = sqrtf, cos = shd/(nh nd) add u each and half the
    relative error of the squares; th0 = acosf(cos) within |dcos|/sin th0 + 2 ulp; s0, s1 are enclosed by evaluating
    them at th0 +- dth (plus 2 ulp per sinf and a division); v = s0 a + s1 dscale b adds 3u(|s0 a| + |s1 dscale b|).
    The bound grows as 1/sin th0: a pair with th0 ~ 1e-3 is included; below th0 ~ 1e-5 it exceeds |v| and is useless.
    Slot 0's statistics (fp32 sum over HW pixels) within HW u sum|v|, + the propagated bound."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(17)
    chk = Fp16Check("slerp_h")
    worst = Worst("slerp_h statistics")
    for (N, H, W, C, T) in _slerp_rows():
        for use_mask in (False, True):
            for near in (False, True):
                h = (torch.randn(N, H, W, C, generator=g) * 2).half()
                dh = torch.randn(N, C, H, W, generator=g)
                if near:  # dh nearly parallel to h: th0 ~ 1e-3
                    dh = (h.float().permute(0, 3, 1, 2) * 1.7 + 3.4e-3 * dh).contiguous()
                hd, dhd = h.to(dev), dh.to(dev)
                h2f = torch.empty(N + 1, H, W, C, dtype=torch.float16, device=dev)
                stf = torch.empty(N + 1, T, C // 2, 2, device=dev)
                tt = 0.3

                def run():
                    stf.fill_(NAN)
                    ops.slerp_h(hd, dhd, h2f[:-1], stf[:-1], tt, use_mask)
                h2 = _launch(h2f, run).cpu()
                st = stf.cpu()
                assert torch.isnan(st[-1]).all() and not torch.isnan(st[:-1]).any()
                assert not st[:-1, 1:].any(), "slerp_h: stats slots other than 0 not zero"
                a = h.double().permute(0, 3, 1, 2)
                b = dh.double()
                m = torch.zeros(H, W, dtype=torch.float64)
                if use_mask:
                    m[4:H - 1, 3:5] = 1
                else:
                    m[:] = 1
                am, bm = a * m, b * m
                shh = (am * am).flatten(1).sum(1)
                sdd = (bm * bm).flatten(1).sum(1)
                shd = (am * bm).flatten(1).sum(1)
                nt = H * W * C / 256 + 13
                eh, ed = nt * U, nt * U
                ehd = nt * U * (am.abs() * bm.abs()).flatten(1).sum(1) / shd.abs()
                nh, nd = shh.sqrt(), sdd.sqrt()
                cos = (shd / (nh * nd)).clamp(-1, 1)
                dcos = cos.abs() * (ehd + eh / 2 + ed / 2 + 4 * U) * 1.001
                th = torch.acos(cos)
                # enclosure of acos over [cos - dcos, cos + dcos] (not first order: near th0 = 0 acos is sqrt-like)
                dth = torch.maximum(th - torch.acos((cos + dcos).clamp(-1, 1)),
                                    torch.acos((cos - dcos).clamp(-1, 1)) - th) + 4 * U * th
                s0, s1 = torch.sin(th * (1 - tt)) / torch.sin(th), torch.sin(th * tt) / torch.sin(th)
                ds0, ds1 = torch.zeros_like(s0), torch.zeros_like(s1)
                for sg in (-1, 1):
                    thp = (th + sg * dth).clamp_min(1e-30)
                    ds0 = torch.maximum(ds0, (torch.sin(thp * (1 - tt)) / torch.sin(thp) - s0).abs())
                    ds1 = torch.maximum(ds1, (torch.sin(thp * tt) / torch.sin(thp) - s1).abs())
                ds0 = ds0 + s0.abs() * 12 * U
                ds1 = ds1 + s1.abs() * 12 * U
                dsc = torch.ones_like(nh) if use_mask else nh / nd
                ddsc = torch.zeros_like(nh) if use_mask else dsc * (eh / 2 + ed / 2 + 3 * U)
                bx = lambda v: v[:, None, None, None]  # noqa: E731
                v = bx(s0) * a + bx(s1 * dsc) * b
                beta = bx(ds0) * a.abs() + (bx(ds1 * dsc) + bx(s1.abs() * ddsc)) * b.abs() + \
                    3 * U * (bx(s0.abs()) * a.abs() + bx((s1 * dsc).abs()) * b.abs())
                inside = m.bool()[None, None].expand_as(v)
                r = torch.where(inside, v, a)
                beta = torch.where(inside, beta, torch.zeros_like(beta))
                got = h2.permute(0, 3, 1, 2)
                out_bad = (~inside) & (got.double() != a)
                assert not out_bad.any(), f"slerp_h mask={use_mask}: h2 differs from h outside the window at " \
                    f"(sample, channel, y, x) {tuple(out_bad.nonzero()[0].tolist())}"
                chk(got, r, beta, lambda n, c, y, x: f"(sample {n}, pixel ({y}, {x}), channel {c})",
                    f"{(N, H, W, C)} mask={use_mask} near={near}")
                gv = got.double()
                pair = gv.reshape(N, C // 2, 2, -1)
                want = torch.stack([pair.sum((2, 3)), (pair * pair).sum((2, 3))], -1)
                mag = torch.stack([pair.abs().sum((2, 3)), (pair * pair).sum((2, 3))], -1)
                # kernel sums its fp32 v (before fp16 rounding): v within beta + half an fp16 ulp of h2
                bv = (gv.abs() * 2.0 ** -11 + 2.0 ** -25).reshape(N, C // 2, 2, -1)
                vb = torch.stack([bv.sum((2, 3)), (2 * pair.abs() * bv + bv * bv).sum((2, 3))], -1)
                sbeta = 2 * H * W * U * mag * 1.01 + vb
                worst((st[:-1, 0].double() - want).abs(), sbeta, lambda n, p, k: f"(sample {n}, pair {p}, {k})",
                      f"{(N, H, W, C)} mask={use_mask}")
    chk.report()
    worst.report()


# ------------------------------------------------------------------------------------------------------------------
# softmax_rows and attention
# ------------------------------------------------------------------------------------------------------------------
def _softmax_rows():
    return _rows("softmax_rows") + [(37, 1), (45, 33), (19, 1000), (16, 1024)]


def test_softmax_rows(cuda_device):
    """P = softmax(scale * S) per row, logits spanning +-100.  With x = scale*S exact in fp64, the kernel's
    v = RN(S*scale) (u|x|), z = RN(v - mx) (u|z|), e' = __expf(z) within k = 2 + floor(1.173|z|) ulp, so
    |e'/e^{x - M} - 1| <= eps_j = u(|x_j| + |x_M|) + u|z| + 2uk (first order, x 1.001); the lane sums (32 terms) and the
    butterfly (5) give |sum' - sum e'| <= 37u sum e'; 1/sum and e*inv add 2u.  beta = p (eps_j + sum_j p_j eps_j + 39u),
    plus 2^-126/sum where __expf flushes to zero; then the rounding criterion."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(18)
    chk = Fp16Check("softmax_rows")
    for (rows, T) in _softmax_rows():
        scale = 1.0 / math.sqrt(64.0) if T != 1000 else 0.0441941738241592
        S = (torch.rand(rows, T, generator=g) * 2 - 1) * (100.0 / scale)
        S[::3] *= 0.02  # rows of moderate range too
        Sd = S.to(dev)
        full = torch.empty(rows + 1, T, dtype=torch.float16, device=dev)
        out = _launch(full, lambda: ops.softmax_rows(Sd, full[:-1], scale))
        x = Sd.double() * float(np.float32(scale))
        M = x.max(1, keepdim=True).values
        z = x - M
        p = torch.softmax(x, 1)
        k = 2 + torch.floor(1.173 * z.abs() * (1 + 4 * U))
        eps = (U * (x.abs() + M.abs()) + U * z.abs() + 2 * U * k) * 1.001
        beta = p * (eps + (p * eps).sum(1, keepdim=True) + 39 * U) * 1.001 + 2.0 ** -126
        chk(out, p, beta, _loc_rc, f"rows={rows} T={T}")
        del Sd, full, out, x, z, p, eps, beta
        torch.cuda.empty_cache()
    chk.report()


def _attn_rows():
    rows = [(N, T, h, d) for (N, T, h, d) in _rows("attention")]
    return rows + [(2, 17, 3, 64), (1, 33, 1, 128), (2, 200, 2, 64), (1, 200, 1, 512), (3, 64, 16, 64)]


def test_attention_kernel(cuda_device):
    """attention_kernel<D> against fp64 softmax(q k^T scale) v, with the rounding criterion.  Derivation (per query,
    head): q and k are small integers, so the fma chain of the logit over D channels is exact (every partial sum an
    integer below 2^24) and only * scale rounds: |x'_j - x_j| <= dx_j = u|x_j|.  The kernel's running max m' enters every
    weight and l alike and cancels, so key j's weight carries a relative error eps_j <= dx_j + u|x_j - m|
    (argument rounding)
    + 2u(2 + 1.173|x_j - m|) (__expf) + sum over the later key tiles of the corr factor's error
    (u R + 2u(2 + 1.173 R), R = max_j x_j - min_j x_j); the common rescaling of acc and l by the same corr cancels.
    The fp32 accumulation adds (T + tiles) u sum w|v| to acc and 7 tiles u sum w to l; the final acc * (1/l) 2u.
    With O = sum w v / sum w:  |O' - O| <= (sum w eps |v - O| + (T + nt) u sum w |v| + |O| 7 nt u sum w)/(sum w (1 - e))
    + 2u|O|, e = max eps + 7 nt u.  Ragged T (17, 33, 200) and N > 1 with heads > 1 exercise the tile and offset logic."""
    ops = _ops()
    dev = cuda_device
    g = torch.Generator().manual_seed(19)
    chk = Fp16Check("attention_kernel")
    for (N, T, heads, d) in _attn_rows():
        C = heads * d
        qkv = torch.randn(N, T, 3 * C, generator=g).half()
        qkv[:, :, :2 * C] = torch.randint(-3, 4, (N, T, 2 * C), generator=g).half()  # q, k: exact logits
        qkv = qkv.to(dev)
        scale = 1.0 / math.sqrt(d)
        full = torch.empty(N + 1, T, C, dtype=torch.float16, device=dev)
        out = _launch(full, lambda: ops.attention(qkv, full[:-1], heads, d, scale))
        q, k, v = (qkv.double()[:, :, i * C:(i + 1) * C].reshape(N, T, heads, d).transpose(1, 2) for i in range(3))
        sc = float(np.float32(scale))
        x = q @ k.transpose(-1, -2) * sc
        assert 9 * d < 2 ** 24  # every partial sum of q.k an exact fp32 integer
        dx = U * x.abs()
        M = x.max(-1, keepdim=True).values
        R = M - x.min(-1, keepdim=True).values
        nt = -(-T // 32)
        z = (x - M).abs()
        eps = dx + U * z + 2 * U * (2 + 1.173 * z) + \
            (nt - 1) * (U * R + 2 * U * (2 + 1.173 * R))
        eps = eps * 1.001
        w = torch.softmax(x, -1)
        O = w @ v
        e = eps.max(-1, keepdim=True).values + 7 * nt * U
        dev_v = (v[..., None, :, :] - O[..., :, None, :]).abs()  # |v_j - O| per (query, key, channel)
        num = ((w * eps)[..., None] * dev_v).sum(-2) + (T + nt) * U * (w @ v.abs()) + O.abs() * 7 * nt * U
        del dev_v
        beta = num / (1 - e) + 2 * U * O.abs() * 1.001
        r = O.transpose(1, 2).reshape(N, T, C)
        beta = beta.transpose(1, 2).reshape(N, T, C)
        chk(out, r, beta, lambda n, t, c: f"(sample {n}, query {t}, head {c // d}, channel {c % d})",
            f"N={N} T={T} heads={heads} d={d}")
    chk.report()


# ------------------------------------------------------------------------------------------------------------------
# the shape table against the plans
# ------------------------------------------------------------------------------------------------------------------
def _record_plan(workload, dev, monkeypatch):
    """(kernel, shape) of every pointwise / attention-glue launch of one edit evaluation of the workload's plan at its
    benchmark batch and of the explicit-delta_h path (mask off and on), recorded through the wrapped entry points.  The
    sampler step's ddim_update / ddpm_update and the middle_h / delta_h unpack_nchw are not driven here: their shapes are
    derived from the plan buffers UNetEngine passes them (P.x, P.et, P.middle_h), so a sampler that launched them on
    other tensors would go unnoticed."""
    import bench
    from asyrp_official_b200 import engine, ops
    family, key, B, _, ckpt, _ = bench.WORKLOADS[workload]
    m, _ = bench.build_model(family, key, dev, ckpt)
    seen = set()

    def wrap(name, keyf):
        orig = getattr(ops, name)

        def f(*a, **k):
            seen.add((name, keyf(*a, **k)))
            return orig(*a, **k)
        monkeypatch.setattr(ops, name, f)

    wrap("gn_finalize", lambda sa, Ca, sb, Cb, gm, bt, eps, N, HW, aff, ss=None, sst=0:
         (N, Ca, sa.shape[1], Cb, sb.shape[1] if sb is not None else 0, HW, sst if ss is not None else 0,
          round(float(eps), 12)))
    wrap("apply", lambda sa, sb, aff, out, act, resample=0, off=0:
         (*sa.shape[:3], sa.shape[3], sb.shape[3] if sb is not None else 0, int(act), int(resample),
          aff.shape[1] if aff is not None else 0, off))
    wrap("pack_input", lambda x, out: tuple(x.shape))
    wrap("timestep_embedding", lambda t, out, variant: (out.shape[0], out.shape[1], variant))
    wrap("linear", lambda inp, w, b, out, act_in=False, act_out=False:
         (inp.shape[0], inp.shape[1], w.shape[0], inp.stride(0), out.stride(0), int(act_in), int(act_out)))
    wrap("attention", lambda qkv, out, heads, d, scale: (qkv.shape[0], qkv.shape[1], heads, d))
    wrap("softmax_rows", lambda S, P, scale: (S.numel() // S.shape[-1], S.shape[-1]))
    wrap("transpose_tc", lambda inp, out: (inp.shape[0], inp.shape[1], inp.shape[2], inp.stride(1)))
    wrap("slerp_h", lambda h, dh, h2, st, t, use_mask=False: (*h.shape[:3], h.shape[3], st.shape[1]))
    eng = engine.UNetEngine(m.arch, m.state_dict(), dev, n_delta=1)
    P = eng.plan(B)
    P.t.fill_(700.0)
    eng.state.update(ignore_timestep=False, slerp_t=0.3, use_mask=False)
    for L in P.launches(edit=True):
        L()
    for use_mask in (False, True):
        eng.state["use_mask"] = use_mask
        for L in P.slerp_ops:
            L()
    torch.cuda.synchronize()
    N, Cx, H, W = P.x.shape
    samp = (N, Cx, H, W, P.et.shape[1])
    seen |= {("ddim_update", samp), ("ddpm_update", samp)}
    mh = P.middle_h.t
    seen.add(("unpack_nchw", (mh.shape[0], mh.shape[3], mh.shape[1], mh.shape[2])))
    monkeypatch.undo()
    del P, eng, m
    torch.cuda.empty_cache()
    return seen


def test_plans_reach_only_tabled_shapes(cuda_device, monkeypatch):
    """every (kernel, shape) the four benchmark plans launch is in SHAPES, and every SHAPES row is launched by a plan"""
    import bench
    seen = set()
    for w in bench.WORKLOADS:
        seen |= _record_plan(w, cuda_device, monkeypatch)
    table = {(k, r) for k, rows in SHAPES.items() for r in rows}
    missing = sorted(seen - table)
    stale = sorted(table - seen)
    if missing:
        by = {}
        for k, r in missing:
            by.setdefault(k, []).append(r)
        pytest.fail(f"{len(missing)} (kernel, shape) pairs the plans launch are missing from SHAPES:\n" +
                    "\n".join(f"    {k!r}: {rows!r}," for k, rows in sorted(by.items())))
    assert not stale, f"SHAPES rows no plan launches: {stale}"
