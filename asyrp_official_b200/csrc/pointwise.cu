// HBM-bound kernels of the Asyrp path: GroupNorm finalise / apply (+SiLU, +2x resample, +concat), input
// packing, timestep embedding + small linears, and the DDIM update.  All activations NHWC fp16; statistics,
// affine tables, embeddings and the sampler state x_t are fp32.
#include <climits>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {

// ---------------------------------------------------------------------------------------------
// GroupNorm finalise: partial (sum, sumsq) per (sample, tile, channel pair) -> per-(sample, channel)
// affine (a, b) with y = a*x + b  ==  GroupNorm(32 groups, eps) [* (1+scale) + shift].
// Reference: torch.nn.GroupNorm in Normalize (ddpm/diffusion.py:68-69, eps 1e-6) and GroupNorm32
// (improved_ddpm/nn.py:17-19, eps 1e-5); scale/shift: improved_ddpm/unet.py:290-294.
// The input may be the channel concatenation of two tensors (decoder skip concat, ddpm/diffusion.py:549,567):
// groups are formed over the virtual concatenated channel axis and may straddle the seam.
// ---------------------------------------------------------------------------------------------
__global__ void gn_finalize_kernel(const float* __restrict__ st_a, int Ca, int Ta, const float* __restrict__ st_b,
                                   int Cb, int Tb, const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float eps, float count, const float* __restrict__ scale_shift, int ss_stride,
                                   float* __restrict__ affine) {
  pdl_trigger();
  pdl_wait();
  const int g = blockIdx.x, n = blockIdx.y;
  const int C = Ca + Cb, cpg = C / 32;
  const int c_lo = g * cpg;
  double s = 0.0, ss = 0.0;
  // channel pairs of this group inside source a and inside source b (a group may straddle the seam); per source
  // the (tile slot, pair) items are flattened so that consecutive threads read consecutive pairs of one slot
  const int p_lo = c_lo / 2, p_hi = (c_lo + cpg) / 2;  // pair range on the concatenated axis
  for (int src = 0; src < 2; ++src) {
    const int Cs = src == 0 ? Ca : Cb, T = src == 0 ? Ta : Tb;
    if (Cs == 0) continue;
    const int off = src == 0 ? 0 : Ca / 2;
    const int lo = (p_lo > off ? p_lo : off) - off;
    const int hi = (p_hi < off + Cs / 2 ? p_hi : off + Cs / 2) - off;
    const int np = hi - lo;
    if (np <= 0) continue;
    const float2* base = reinterpret_cast<const float2*>(src == 0 ? st_a : st_b) +
                         static_cast<size_t>(n) * T * (Cs / 2) + lo;
    const int items = np * T;
#pragma unroll 4
    for (int idx = threadIdx.x; idx < items; idx += blockDim.x) {
      const int t = idx / np, pi = idx - t * np;
      const float2 v = base[static_cast<size_t>(t) * (Cs / 2) + pi];
      s += v.x;
      ss += v.y;
    }
  }
  __shared__ double sh_s[32], sh_ss[32];
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sh_s[w] = s; sh_ss[w] = ss; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    s = l < nw ? sh_s[l] : 0.0;
    ss = l < nw ? sh_ss[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    const double mean = s / count;
    double var = ss / count - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    const float fmean = static_cast<float>(mean);
    for (int i = l; i < cpg; i += 32) {
      const int c = c_lo + i;
      float a = gamma[c] * rstd;
      float b = beta[c] - fmean * a;
      if (scale_shift != nullptr) {
        const float sc = 1.0f + scale_shift[static_cast<size_t>(n) * ss_stride + c];
        const float sh = scale_shift[static_cast<size_t>(n) * ss_stride + C + c];
        a = a * sc;
        b = b * sc + sh;
      }
      affine[(static_cast<size_t>(n) * C + c) * 2] = a;
      affine[(static_cast<size_t>(n) * C + c) * 2 + 1] = b;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Pointwise apply: out = resample(act(a*x + b)) over the channel concat of up to two sources.
//   act: 0 identity, 1 SiLU (nonlinearity ddpm/diffusion.py:63-65 / nn.SiLU)
//   resample: 0 none, 1 2x2 average pool (improved_ddpm/unet.py Downsample use_conv=False :173-181),
//             2 nearest x2 (F.interpolate, ddpm/diffusion.py:83-84, improved_ddpm/unet.py:142-150)
// One thread = 8 channels (16 B) of one output pixel.
// ---------------------------------------------------------------------------------------------
struct ApplyParams {
  const __half* src_a; int Ca;
  const __half* src_b; int Cb;
  const float* affine;  // (a, b) pairs of the source channels, row n at affine + n*aff_stride floats; nullptr = identity
  int aff_stride;
  __half* out;
  int N, Hi, Wi, Ho, Wo;
  int act, resample;
};

__device__ __forceinline__ void load8(const __half* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 t = __half22float2(h[k]);
    f[2 * k] = t.x;
    f[2 * k + 1] = t.y;
  }
}
__device__ __forceinline__ void store8(__half* p, const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(f[2 * k], f[2 * k + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

// Thread mapping: a thread owns ONE channel octet (its affine coefficients stay in registers) and walks output
// pixels; consecutive threads cover consecutive octets of a pixel, so a warp reads/writes whole 128B+ lines.
template <int RESAMPLE>
__global__ void __launch_bounds__(256) apply_kernel(const ApplyParams p) {
  pdl_trigger();
  pdl_wait();
  const int C = p.Ca + p.Cb;
  const int octs = C >> 3;                 // octets per pixel
  const int lanes = blockDim.x / octs;     // pixels processed concurrently by a block (host guarantees octs | 256)
  const int oc = threadIdx.x % octs, pl = threadIdx.x / octs;
  const int n = blockIdx.y;
  const int c = oc * 8;
  const __half* src;
  int Cs, cs;
  if (c < p.Ca) { src = p.src_a; Cs = p.Ca; cs = c; }
  else { src = p.src_b; Cs = p.Cb; cs = c - p.Ca; }
  src += static_cast<size_t>(n) * p.Hi * p.Wi * Cs + cs;
  __half* dst = p.out + static_cast<size_t>(n) * p.Ho * p.Wo * C + c;
  float a[8], b[8];
  if (p.affine != nullptr) {
    const float4* ap = reinterpret_cast<const float4*>(p.affine + static_cast<size_t>(n) * p.aff_stride + c * 2);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float4 t = ap[k];
      a[2 * k] = t.x; b[2 * k] = t.y; a[2 * k + 1] = t.z; b[2 * k + 1] = t.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) { a[k] = 1.f; b[k] = 0.f; }
  }
  const int npix = p.Ho * p.Wo;
  const int stride = gridDim.x * lanes;
  constexpr int U = RESAMPLE == 1 ? 1 : 4;  // output pixels in flight per thread
  for (int base = blockIdx.x * lanes + pl; base < npix; base += stride * U) {
    float v[U][RESAMPLE == 1 ? 4 : 1][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pix = base + u * stride;
      if (pix < npix) {
        if (RESAMPLE == 0) {
          load8(src + static_cast<size_t>(pix) * Cs, v[u][0]);
        } else {
          const int yo = pix / p.Wo, xo = pix - yo * p.Wo;
          if (RESAMPLE == 2) {
            load8(src + (static_cast<size_t>(yo >> 1) * p.Wi + (xo >> 1)) * Cs, v[u][0]);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              load8(src + (static_cast<size_t>(2 * yo + (q >> 1)) * p.Wi + 2 * xo + (q & 1)) * Cs,
                    v[u][RESAMPLE == 1 ? q : 0]);
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int pix = base + u * stride;
      if (pix < npix) {
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = 0.f;
#pragma unroll
        for (int q = 0; q < (RESAMPLE == 1 ? 4 : 1); ++q)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            float t = fmaf(a[k], v[u][q][k], b[k]);
            if (p.act) t = silu_f(t);
            o[k] += t;
          }
        if (RESAMPLE == 1) {
#pragma unroll
          for (int k = 0; k < 8; ++k) o[k] *= 0.25f;
        }
        store8(dst + static_cast<size_t>(pix) * C, o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// x_t fp32 NCHW [N][Cin][H][W] -> fp16 NHWC [N][H][W][64], channels >= Cin zero (conv_in operand)
// ---------------------------------------------------------------------------------------------
__global__ void pack_input_kernel(const float* __restrict__ x, __half* __restrict__ out, int N, int Cin, int H,
                                  int W) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * H * W * 8;  // 8 octets of 8 channels
  for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int oc = static_cast<int>(idx & 7);
    const size_t pix = idx >> 3;
    const size_t hw = static_cast<size_t>(H) * W;
    const size_t n = pix / hw, r = pix % hw;
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = oc * 8 + k;
      f[k] = c < Cin ? x[(n * Cin + c) * hw + r] : 0.f;
    }
    store8(out + pix * 64 + oc * 8, f);
  }
}

// ---------------------------------------------------------------------------------------------
// Sinusoidal timestep embedding.  variant 0: DDPM [sin | cos], freq_i = exp(-i*ln(1e4)/(half-1))
// (ddpm/diffusion.py:42-60); variant 1: ADM [cos | sin], freq_i = exp(-i*ln(1e4)/half) (improved_ddpm/nn.py:103-121)
// ---------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int N, int dim,
                                          int variant) {
  pdl_trigger();
  pdl_wait();
  const int half = dim / 2;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < N * half; idx += gridDim.x * blockDim.x) {
    const int n = idx / half, i = idx % half;
    const float denom = variant == 0 ? static_cast<float>(half - 1) : static_cast<float>(half);
    // same fp32 expression order as the reference: exp(arange * -(ln(1e4)/denom))
    const float fr = variant == 0 ? expf(static_cast<float>(i) * -(logf(10000.0f) / denom))
                                  : expf(-logf(10000.0f) * static_cast<float>(i) / denom);
    const float a = t[n] * fr;
    const float s = sinf(a), c = cosf(a);
    out[n * dim + i] = variant == 0 ? s : c;
    out[n * dim + half + i] = variant == 0 ? c : s;
  }
}

// out[n][o] = bias[o] + sum_i W[o][i] * f(in[n][i]),  f = SiLU when act_in.
// Generic fallback: one warp per (n, o).
__global__ void linear_kernel(const float* __restrict__ in, int in_stride, const float* __restrict__ Wt,
                              const float* __restrict__ bias, float* __restrict__ out, int out_stride, int N, int I,
                              int O, int act_in, int act_out) {
  pdl_trigger();
  pdl_wait();
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp_global >= N * O) return;
  const int n = warp_global / O, o = warp_global % O;
  const float* x = in + static_cast<size_t>(n) * in_stride;
  const float* w = Wt + static_cast<size_t>(o) * I;
  float acc = 0.f;
  for (int i = lane; i < I; i += 32) {
    float v = x[i];
    if (act_in) v = v / (1.0f + expf(-v));
    acc += w[i] * v;
  }
  for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
  if (lane == 0) {
    float r = acc + (bias ? bias[o] : 0.f);
    if (act_out) r = r / (1.0f + expf(-r));
    out[static_cast<size_t>(n) * out_stride + o] = r;
  }
}

// Fast path (I = 32*KI): the block stages f(in) of up to `nc` samples in shared memory once, then each warp keeps
// one weight row in registers and produces that output for all staged samples — the weight matrix (the 10-20 MB of
// concatenated timestep-embedding projections) is read once instead of once per sample.  Per (n, o) the summation
// order is the generic kernel's (lane-strided partial sums, xor-shuffle tree), so both give identical bits.
constexpr int kLinOutPerWarp = 4;
template <int KI>
__global__ void __launch_bounds__(256) linear_rows_kernel(const float* __restrict__ in, int in_stride,
                                                          const float* __restrict__ Wt, const float* __restrict__ bias,
                                                          float* __restrict__ out, int out_stride, int N, int O,
                                                          int nc, int act_in, int act_out) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float xs[];  // [nc][32*KI]
  constexpr int I = 32 * KI;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o0 = (blockIdx.x * 8 + warp) * kLinOutPerWarp;
  for (int n0 = 0; n0 < N; n0 += nc) {
    const int nn = N - n0 < nc ? N - n0 : nc;
    __syncthreads();
    for (int idx = threadIdx.x; idx < nn * I; idx += 256) {
      const int n = idx / I, i = idx - n * I;
      float v = in[static_cast<size_t>(n0 + n) * in_stride + i];
      if (act_in) v = v / (1.0f + expf(-v));
      xs[idx] = v;
    }
    __syncthreads();
    for (int oo = 0; oo < kLinOutPerWarp; ++oo) {
      const int o = o0 + oo;
      if (o >= O) break;
      float w[KI];
#pragma unroll
      for (int k = 0; k < KI; ++k) w[k] = Wt[static_cast<size_t>(o) * I + lane + 32 * k];
      const float b = bias ? bias[o] : 0.f;
      for (int n = 0; n < nn; ++n) {
        const float* x = xs + n * I + lane;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < KI; ++k) acc += w[k] * x[32 * k];
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) {
          float r = acc + b;
          if (act_out) r = r / (1.0f + expf(-r));
          out[static_cast<size_t>(n0 + n) * out_stride + o] = r;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// DDIM update (utils/diffusion_utils.py:84-100), fp32, same operation order as the reference:
//   x0   = (x - em*sqrt(1-at)) / sqrt(at)
//   next = sqrt(an)*x0 + c2*et (+ c1*z)            c2 = sqrt(1-an) for eta=0
// et / em are planar fp32 [N][Ce][H][W] of which channels [0,3) are epsilon (learn_sigma split :47-51).
// ---------------------------------------------------------------------------------------------
__global__ void ddim_update_kernel(const float* __restrict__ x, const float* __restrict__ et,
                                   const float* __restrict__ em, const float* __restrict__ z,
                                   float* __restrict__ x_next, float* __restrict__ x0_out, int N, int Cx, int Ce,
                                   int HW, float at, float an, float c1, float c2, int use_z) {
  pdl_trigger();
  pdl_wait();
  const float sq1 = sqrtf(1.0f - at), sqa = sqrtf(at), sqn = sqrtf(an);
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = idx / (static_cast<size_t>(Cx) * HW), r = idx % (static_cast<size_t>(Cx) * HW);
    const size_t eidx = n * Ce * HW + r;
    const float e = et[eidx], m = em[eidx];
    const float x0 = __fdiv_rn(__fsub_rn(x[idx], __fmul_rn(m, sq1)), sqa);
    float nx = __fadd_rn(__fmul_rn(sqn, x0), __fmul_rn(c2, e));
    if (use_z) nx = __fadd_rn(nx, __fmul_rn(c1, z[idx]));
    x_next[idx] = nx;
    if (x0_out) x0_out[idx] = x0;
  }
}

// Per-row DDIM update: the kernel above with (c1, c2) read per sample from c12 [N][2], so that the rows of one batch can
// follow different eta schedules (an attribute sweep: every row its own t_addnoise).  Per row the operations, their
// order and their rounding are those of ddim_update_kernel with that row's scalars; z is read only by rows whose c1 is
// non-zero (the scalar kernel is launched without z for eta = 0 steps).
__global__ void ddim_update_rows_kernel(const float* __restrict__ x, const float* __restrict__ et,
                                        const float* __restrict__ em, const float* __restrict__ z,
                                        float* __restrict__ x_next, float* __restrict__ x0_out, int N, int Cx, int Ce,
                                        int HW, float at, float an, const float* __restrict__ c12) {
  pdl_trigger();
  pdl_wait();
  const float sq1 = sqrtf(1.0f - at), sqa = sqrtf(at), sqn = sqrtf(an);
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = idx / (static_cast<size_t>(Cx) * HW), r = idx % (static_cast<size_t>(Cx) * HW);
    const size_t eidx = n * Ce * HW + r;
    const float c1 = c12[2 * n], c2 = c12[2 * n + 1];
    const float e = et[eidx], m = em[eidx];
    const float x0 = __fdiv_rn(__fsub_rn(x[idx], __fmul_rn(m, sq1)), sqa);
    float nx = __fadd_rn(__fmul_rn(sqn, x0), __fmul_rn(c2, e));
    if (z != nullptr && c1 != 0.0f) nx = __fadd_rn(nx, __fmul_rn(c1, z[idx]));
    x_next[idx] = nx;
    if (x0_out) x0_out[idx] = x0;
  }
}

// ---------------------------------------------------------------------------------------------
// DDPM ancestral update (utils/diffusion_utils.py:74-82, sampling_type='ddpm'):
//   mean = 1/sqrt(1-bt) * (x - bt/sqrt(1-at) * et);  x_next = mean + mask * exp(0.5*logvar) * z
// logvar: the fixed table entry (learn_sigma=False) or, with learn_sigma, channels [Cx, 2Cx) of the model output
// (the reference uses the raw learned channels as log-variance, :47-51).  mask = 0 at t == 0.
// ---------------------------------------------------------------------------------------------
__global__ void ddpm_update_kernel(const float* __restrict__ x, const float* __restrict__ et, const float* __restrict__ z,
                                   float* __restrict__ x_next, int N, int Cx, int Ce, int HW, float at, float bt,
                                   float logvar, int learned, float mask) {
  pdl_trigger();
  pdl_wait();
  const float weight = __fdiv_rn(bt, sqrtf(1.0f - at));
  const float inv = __fdiv_rn(1.0f, sqrtf(1.0f - bt));
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = idx / (static_cast<size_t>(Cx) * HW), r = idx % (static_cast<size_t>(Cx) * HW);
    const size_t eidx = n * Ce * HW + r;
    const float mean = __fmul_rn(inv, __fsub_rn(x[idx], __fmul_rn(weight, et[eidx])));
    const float lv = learned ? et[eidx + static_cast<size_t>(Cx) * HW] : logvar;
    x_next[idx] = __fadd_rn(mean, __fmul_rn(__fmul_rn(mask, expf(0.5f * lv)), z[idx]));
  }
}

// out = alpha*a + beta*b on fp16 tensors (fp32 math): h2 = c0*h + c_i*delta_h_i  (ddpm/diffusion.py:512-516)
__global__ void axpby_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ out,
                             float alpha, float beta, size_t n8) {
  pdl_trigger();
  pdl_wait();
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float fa[8], fb[8], o[8];
    load8(a + i * 8, fa);
    load8(b + i * 8, fb);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = alpha * fa[k] + beta * fb[k];
    store8(out + i * 8, o);
  }
}

// NHWC fp16 -> NCHW fp32 (API-visible copies of delta_h / middle_h)
__global__ void unpack_nchw_kernel(const __half* __restrict__ in, float* __restrict__ out, int N, int C, int HW) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * C * HW;
  for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = idx / (static_cast<size_t>(C) * HW), r = idx % (static_cast<size_t>(C) * HW);
    const size_t c = r / HW, p = r % HW;
    out[idx] = __half2float(in[(n * HW + p) * C + c]);
  }
}

// ---------------------------------------------------------------------------------------------
// Explicit delta_h injection (DiffStyle / raw-delta_h checkpoints): h2 = slerp(t, h, |h| * dh / |dh|), per sample
// over all C*H*W elements (models/ddpm/diffusion.py:6-40,528-539); with use_mask the interpolation is restricted to
// rows 4..H-2, columns 3..4 without norm matching and h is kept elsewhere (:519-527).
// One block per sample.  h: fp16 NHWC; dh: fp32 NCHW (sample stride dh_stride, 0 = shared); writes h2 (fp16 NHWC)
// and its GroupNorm partial sums into tile slot 0 of `stats` ([N][T][C/2][2]; other slots zeroed).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) t += sh[i];
  return t;
}

// The body of both slerp kernels: sample n = blockIdx.x with slerp weight t.  The per-row kernel only reads t from
// device memory, so row n performs exactly the scalar kernel's operations.
__device__ __forceinline__ void slerp_h_sample(const __half* __restrict__ h, const float* __restrict__ dh,
                                               long long dh_stride, __half* __restrict__ h2, float* __restrict__ stats,
                                               int T, int C, int H, int W, float t, int use_mask, float* sh) {
  const int n = blockIdx.x, HW = H * W;
  const __half* hn = h + static_cast<size_t>(n) * HW * C;
  const float* dn = dh + static_cast<size_t>(n) * dh_stride;
  __half* on = h2 + static_cast<size_t>(n) * HW * C;
  float shh = 0.f, sdd = 0.f, shd = 0.f;
  for (int i = threadIdx.x; i < HW * C; i += blockDim.x) {
    const int pix = i / C, c = i - pix * C;
    const int y = pix / W, x = pix - y * W;
    const float m = use_mask ? ((y >= 4 && y < H - 1 && x >= 3 && x < 5) ? 1.f : 0.f) : 1.f;
    const float a = __half2float(hn[i]) * m, b = dn[static_cast<size_t>(c) * HW + pix] * m;
    shh += a * a; sdd += b * b; shd += a * b;
  }
  shh = block_sum(shh, sh); sdd = block_sum(sdd, sh); shd = block_sum(shd, sh);
  const float nh = sqrtf(shh), nd = sqrtf(sdd);
  const float th0 = acosf(shd / (nh * nd));
  const float s0 = sinf(th0 - th0 * t) / sinf(th0), s1 = sinf(th0 * t) / sinf(th0);
  const float dscale = use_mask ? 1.f : nh / nd;  // v1 = |h| * dh / |dh| (norm-matched) unless masked
  // second pass: h2 and its channel-pair statistics; a thread owns channel pairs, pixels in the inner loop
  float* st = stats + static_cast<size_t>(n) * T * (C / 2) * 2;
  for (int pr = threadIdx.x; pr < C / 2; pr += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int pix = 0; pix < HW; ++pix) {
      const int y = pix / W, x = pix - y * W;
      const bool in = !use_mask || (y >= 4 && y < H - 1 && x >= 3 && x < 5);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int c = pr * 2 + k;
        const float a = __half2float(hn[static_cast<size_t>(pix) * C + c]);
        const float b = dn[static_cast<size_t>(c) * HW + pix];
        const float v = in ? s0 * a + s1 * dscale * b : a;
        on[static_cast<size_t>(pix) * C + c] = __float2half_rn(v);
        s += v; ss += v * v;
      }
    }
    st[pr * 2] = s; st[pr * 2 + 1] = ss;
    for (int tt = 1; tt < T; ++tt) { st[(tt * (C / 2) + pr) * 2] = 0.f; st[(tt * (C / 2) + pr) * 2 + 1] = 0.f; }
  }
}

__global__ void __launch_bounds__(256) slerp_h_kernel(const __half* __restrict__ h, const float* __restrict__ dh,
                                                      long long dh_stride, __half* __restrict__ h2,
                                                      float* __restrict__ stats, int T, int C, int H, int W, float t,
                                                      int use_mask) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sh[8];
  slerp_h_sample(h, dh, dh_stride, h2, stats, T, C, H, W, t, use_mask, sh);
}

// per-sample slerp weight t_rows[n] (a graph input: one captured graph serves every weight table)
__global__ void __launch_bounds__(256) slerp_h_rows_kernel(const __half* __restrict__ h, const float* __restrict__ dh,
                                                           long long dh_stride, __half* __restrict__ h2,
                                                           float* __restrict__ stats, int T, int C, int H, int W,
                                                           const float* __restrict__ t_rows, int use_mask) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sh[8];
  slerp_h_sample(h, dh, dh_stride, h2, stats, T, C, H, W, t_rows[blockIdx.x], use_mask, sh);
}

// Additive direction (h-space directions found from the bottleneck's statistics): h2[n] = c0[n] * h[n] + alpha[n] * d
// with one fp32 NCHW direction d [C][H][W] shared by every sample and (c0, alpha) = coef[n] (fp32 [N][2], a graph
// input like slerp's t_rows).  Each element is v = fmaf(alpha, d, __fmul_rn(c0, h)) in fp32, stored rounded to fp16.
// One block per sample, h2's GroupNorm partial sums written as slerp_h_sample writes them: a thread owns channel pairs,
// sums v and v * v of the fp32 values over the pixels in order into tile slot 0, and zeroes slots 1..T-1.
__global__ void __launch_bounds__(256) add_h_rows_kernel(const __half* __restrict__ h, const float* __restrict__ dir,
                                                         __half* __restrict__ h2, float* __restrict__ stats, int T,
                                                         int C, int HW, const float* __restrict__ coef) {
  pdl_trigger();
  pdl_wait();
  const int n = blockIdx.x;
  const float c0 = coef[2 * n], alpha = coef[2 * n + 1];
  const __half* hn = h + static_cast<size_t>(n) * HW * C;
  __half* on = h2 + static_cast<size_t>(n) * HW * C;
  float* st = stats + static_cast<size_t>(n) * T * (C / 2) * 2;
  for (int pr = threadIdx.x; pr < C / 2; pr += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int pix = 0; pix < HW; ++pix) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int c = pr * 2 + k;
        const float a = __half2float(hn[static_cast<size_t>(pix) * C + c]);
        const float v = fmaf(alpha, dir[static_cast<size_t>(c) * HW + pix], __fmul_rn(c0, a));
        on[static_cast<size_t>(pix) * C + c] = __float2half_rn(v);
        s += v; ss += v * v;
      }
    }
    st[pr * 2] = s; st[pr * 2 + 1] = ss;
    for (int tt = 1; tt < T; ++tt) { st[(tt * (C / 2) + pr) * 2] = 0.f; st[(tt * (C / 2) + pr) * 2 + 1] = 0.f; }
  }
}

}  // namespace asyrp

using namespace asyrp;

static inline int grid_for(size_t total, int block, int cap_mult = 8) {
  size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * cap_mult;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

extern "C" {

ASYRP_API int asyrp_gn_finalize(const float* st_a, int Ca, int Ta, const float* st_b, int Cb, int Tb,
                                const float* gamma, const float* beta, float eps, int N, int HW,
                                const float* scale_shift, int ss_stride, float* affine, void* stream) {
  const int C = Ca + Cb;
  ASYRP_REQUIRE(C % 64 == 0, "asyrp_gn_finalize: C=%d must be a multiple of 64", C);
  ASYRP_REQUIRE(N >= 1 && N <= kMaxGridYZ, "asyrp_gn_finalize: N=%d out of range (1..%d: the grid's y dimension)", N,
                kMaxGridYZ);
  const float count = static_cast<float>(HW) * (C / 32);
  ASYRP_LAUNCH(gn_finalize_kernel, dim3(dim3(32, N)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      st_a, Ca, Ta, st_b, Cb, Tb, gamma, beta, eps, count, scale_shift, ss_stride, affine);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_apply(const void* src_a, int Ca, const void* src_b, int Cb, const float* affine,
                          int affine_stride, void* out, int N, int Hi, int Wi, int act, int resample, void* stream) {
  ASYRP_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "asyrp_apply: channels must be multiples of 8");
  ASYRP_REQUIRE(resample >= 0 && resample <= 2, "asyrp_apply: resample=%d (0 none, 1 avg-pool 2x2, 2 nearest x2)",
                resample);
  ASYRP_REQUIRE(act == 0 || act == 1, "asyrp_apply: act=%d (0 none, 1 SiLU)", act);
  ASYRP_REQUIRE(N >= 1 && N <= kMaxGridYZ, "asyrp_apply: N=%d out of range (1..%d: the grid's y dimension)", N,
                kMaxGridYZ);
  ApplyParams p;
  p.src_a = static_cast<const __half*>(src_a); p.Ca = Ca;
  p.src_b = static_cast<const __half*>(src_b); p.Cb = Cb;
  p.affine = affine; p.aff_stride = affine_stride > 0 ? affine_stride : (Ca + Cb) * 2;
  p.out = static_cast<__half*>(out);
  p.N = N; p.Hi = Hi; p.Wi = Wi;
  p.Ho = resample == 1 ? Hi / 2 : (resample == 2 ? Hi * 2 : Hi);
  p.Wo = resample == 1 ? Wi / 2 : (resample == 2 ? Wi * 2 : Wi);
  p.act = act; p.resample = resample;
  const int octs = (Ca + Cb) / 8;
  ASYRP_REQUIRE(octs >= 1 && octs <= 256, "asyrp_apply: unsupported channel count %d (max 2048)", Ca + Cb);
  // block = lanes * octs threads (<= 256): `lanes` pixels at a time, one channel octet per thread
  const int lanes = 256 / octs;
  const int threads = lanes * octs;
  const int npix = p.Ho * p.Wo;
  int gx = (npix + lanes * 4 - 1) / (lanes * 4);
  const int cap = (sm_count() > 0 ? sm_count() : 132) * 8;
  const int max_gx = cap / N > 0 ? cap / N : 1;
  if (gx > max_gx) gx = max_gx;
  if (gx < 1) gx = 1;
  const dim3 grid(gx, N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (resample == 0) ASYRP_LAUNCH(apply_kernel<0>, dim3(grid), dim3(threads), 0, st, p);
  else if (resample == 1) ASYRP_LAUNCH(apply_kernel<1>, dim3(grid), dim3(threads), 0, st, p);
  else ASYRP_LAUNCH(apply_kernel<2>, dim3(grid), dim3(threads), 0, st, p);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_pack_input(const float* x, void* out, int N, int Cin, int H, int W, void* stream) {
  ASYRP_REQUIRE(Cin <= 64, "asyrp_pack_input: Cin=%d > 64", Cin);
  const size_t total = static_cast<size_t>(N) * H * W * 8;
  ASYRP_LAUNCH(pack_input_kernel, dim3(grid_for(total, 256, 16)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      x, static_cast<__half*>(out), N, Cin, H, W);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_timestep_embedding(const float* t, float* out, int N, int dim, int variant, void* stream) {
  ASYRP_REQUIRE(dim % 2 == 0, "asyrp_timestep_embedding: odd dim %d", dim);
  const int total = N * (dim / 2);
  ASYRP_LAUNCH(timestep_embedding_kernel, dim3((total + 127) / 128), dim3(128), 0, static_cast<cudaStream_t>(stream), t, out, N, dim,
                                                                                               variant);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_linear(const float* in, int in_stride, const float* W, const float* bias, float* out,
                           int out_stride, int N, int I, int O, int act_in, int act_out, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (I == 128 || I == 256 || I == 512 || I == 1024) {
    int nc = (32 * 1024) / (I * 4);  // samples staged per pass: 32 KB of shared memory
    if (nc > N) nc = N;
    const int grid = (O + 8 * kLinOutPerWarp - 1) / (8 * kLinOutPerWarp);
    const size_t smem = static_cast<size_t>(nc) * I * 4;
#define ASYRP_LIN(KI_) \
  ASYRP_LAUNCH(linear_rows_kernel<KI_>, dim3(grid), dim3(256), smem, st, in, in_stride, W, bias, out, out_stride, N, O, nc, act_in, act_out)
    if (I == 128) ASYRP_LIN(4);
    else if (I == 256) ASYRP_LIN(8);
    else if (I == 512) ASYRP_LIN(16);
    else ASYRP_LIN(32);
#undef ASYRP_LIN
  } else {
    const size_t warps = static_cast<size_t>(N) * O;
    const int block = 256;
    const int grid = static_cast<int>((warps * 32 + block - 1) / block);
    ASYRP_LAUNCH(linear_kernel, dim3(grid), dim3(block), 0, st, in, in_stride, W, bias, out, out_stride, N, I, O, act_in, act_out);
  }
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_ddim_update(const float* x, const float* et, const float* em, const float* z, float* x_next,
                                float* x0_out, int N, int Cx, int Ce, int HW, float at, float an, float c1, float c2,
                                void* stream) {
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  ASYRP_LAUNCH(ddim_update_kernel, dim3(grid_for(total, 256, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      x, et, em, z, x_next, x0_out, N, Cx, Ce, HW, at, an, c1, c2, z != nullptr);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_ddim_update_rows(const float* x, const float* et, const float* em, const float* z, float* x_next,
                                     float* x0_out, int N, int Cx, int Ce, int HW, float at, float an, const float* c12,
                                     void* stream) {
  ASYRP_REQUIRE(c12 != nullptr, "asyrp_ddim_update_rows: c12 is NULL");
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  ASYRP_LAUNCH(ddim_update_rows_kernel, dim3(grid_for(total, 256, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream),
      x, et, em, z, x_next, x0_out, N, Cx, Ce, HW, at, an, c12);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_axpby(const void* a, const void* b, void* out, float alpha, float beta, long long numel,
                          void* stream) {
  ASYRP_REQUIRE(numel % 8 == 0, "asyrp_axpby: numel must be a multiple of 8");
  const size_t n8 = static_cast<size_t>(numel) / 8;
  ASYRP_LAUNCH(axpby_kernel, dim3(grid_for(n8, 256, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __half*>(a), static_cast<const __half*>(b), static_cast<__half*>(out), alpha, beta, n8);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_unpack_nchw(const void* in, float* out, int N, int C, int HW, void* stream) {
  const size_t total = static_cast<size_t>(N) * C * HW;
  ASYRP_LAUNCH(unpack_nchw_kernel, dim3(grid_for(total, 256, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const __half*>(in), out, N, C, HW);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_slerp_h(const void* h, const float* dh, long long dh_sample_stride, void* h2, float* stats,
                            int stats_tiles, int N, int C, int H, int W, float t, int use_mask, void* stream) {
  ASYRP_REQUIRE(C % 2 == 0 && stats_tiles >= 1, "asyrp_slerp_h: bad arguments");
  ASYRP_LAUNCH(slerp_h_kernel, dim3(N), dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const __half*>(h), dh, dh_sample_stride,
                                                                    static_cast<__half*>(h2), stats, stats_tiles, C, H,
                                                                    W, t, use_mask);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_slerp_h_rows(const void* h, const float* dh, long long dh_sample_stride, void* h2, float* stats,
                                 int stats_tiles, int N, int C, int H, int W, const float* t_rows, int use_mask,
                                 void* stream) {
  ASYRP_REQUIRE(C % 2 == 0 && stats_tiles >= 1, "asyrp_slerp_h_rows: bad arguments");
  ASYRP_REQUIRE(t_rows != nullptr, "asyrp_slerp_h_rows: t_rows is NULL");
  ASYRP_LAUNCH(slerp_h_rows_kernel, dim3(N), dim3(256), 0, static_cast<cudaStream_t>(stream),
               static_cast<const __half*>(h), dh, dh_sample_stride, static_cast<__half*>(h2), stats, stats_tiles, C, H,
               W, t_rows, use_mask);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_add_h_rows(const void* h, const float* dir, void* h2, float* stats, int stats_tiles, int N, int C,
                               int H, int W, const float* coef, void* stream) {
  ASYRP_REQUIRE(N >= 1 && C >= 2 && C % 2 == 0 && H >= 1 && W >= 1 && stats_tiles >= 1,
                "asyrp_add_h_rows: bad arguments N=%d C=%d H=%d W=%d stats_tiles=%d", N, C, H, W, stats_tiles);
  // per-sample offsets are size_t; the element index within a sample and the tile-slot index are int
  ASYRP_REQUIRE(static_cast<long long>(C) * H * W <= INT_MAX && static_cast<long long>(stats_tiles) * C <= INT_MAX,
                "asyrp_add_h_rows: C * H * W or stats_tiles * C above 2^31 - 1");
  ASYRP_REQUIRE(h != nullptr && dir != nullptr && h2 != nullptr && stats != nullptr,
                "asyrp_add_h_rows: h, dir, h2 and stats are required");
  ASYRP_REQUIRE(coef != nullptr, "asyrp_add_h_rows: coef is NULL");
  ASYRP_REQUIRE(h != h2, "asyrp_add_h_rows: h2 must not alias h");
  ASYRP_LAUNCH(add_h_rows_kernel, dim3(N), dim3(256), 0, static_cast<cudaStream_t>(stream),
               static_cast<const __half*>(h), dir, static_cast<__half*>(h2), stats, stats_tiles, C, H * W, coef);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_ddpm_update(const float* x, const float* et, const float* z, float* x_next, int N, int Cx, int Ce,
                                int HW, float at, float bt, float logvar, int learned_sigma, float mask, void* stream) {
  ASYRP_REQUIRE(z != nullptr, "asyrp_ddpm_update: noise tensor required");
  ASYRP_REQUIRE(!learned_sigma || Ce >= 2 * Cx, "asyrp_ddpm_update: learned sigma needs 2*Cx model channels");
  const size_t total = static_cast<size_t>(N) * Cx * HW;
  ASYRP_LAUNCH(ddpm_update_kernel, dim3(grid_for(total, 256, 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      x, et, z, x_next, N, Cx, Ce, HW, at, bt, logvar, learned_sigma, mask);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
