// DINO ViT (facebookresearch/dino `VisionTransformer`, backbone only) and the structure distance of Splice /
// Plug-and-Play: the mean squared difference of two images' key self-similarity matrices.  Activations are fp32
// [B][T][D], T = 1 + G^2 tokens, D = 64 * heads.
//
//   patches  = patchify(Normalize_imagenet(Resize_aa((x + 1) / 2)))              dino_pack_kernel
//   x        = [cls_token ; patches @ proj^T + b] + pos_embed                   (clip_linear, clip_image_tokens)
//   blocks:  x += proj(attn(norm1(x)));  x += fc2(gelu(fc1(norm2(x))))           dino_layernorm_kernel,
//                                                                                 dino_attention_kernel, clip_linear
//   D(a, b)  = (1/T^2) sum_ij (ka_i.ka_j - kb_i.kb_j)^2, k^ = k / max(|k|, eps)   dino_selfsim_kernel
//
// Every reduction runs in a fixed order (no float atomics) and no kernel mixes images, so an image's features are the
// same bits whatever batch it is in.
#include <cfloat>

#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kHeadDim = 64;
constexpr int kMaxTokens = 1025;   // 1 + 32^2: ViT-*/8 at 256^2
constexpr int kRowThreads = 256;   // LayerNorm: one warp per row
// attention: a CTA of 4 warps per (query tile of 64 rows, head, image); each warp owns 16 query rows
constexpr int kAttnWarps = 4;
constexpr int kQTile = 16 * kAttnWarps;
constexpr int kKTile = 64;
constexpr int kKvLd = kHeadDim + 4;  // smem row pitch: conflict-free K (rows g, cols t) and V (rows 2t, cols g) reads
constexpr int kKvStageFloats = 2 * kKTile * kKvLd;
constexpr size_t kAttnSmem = 2 * kKvStageFloats * sizeof(float);  // K and V tiles, double-buffered
// self-similarity distance: 64 x 64 tiles of the T x T matrices, columns in chunks of 32
constexpr int kSimTile = 64;
constexpr int kSimChunk = 32;
constexpr int kSimThreads = 256;
constexpr int kSimLd = kSimChunk + 1;
// ImageNet's Normalize
__constant__ float kMean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float kStd[3] = {0.229f, 0.224f, 0.225f};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// PyTorch's antialiased bilinear taps (_upsample_bilinear2d_aa, _compute_indices_min_size_weights_aa) of output index
// i for an input of n pixels at scale = n / out: centre scale (i + 0.5), support max(1, scale), the triangle filter
// 1 - |x| at (j + xmin - centre + 0.5) / max(1, scale); the weights are normalised by their sum.
struct AaTaps {
  float center, invscale, total;
  int xmin, xsize;
  __device__ AaTaps(int i, int n, float scale) {
    const float support = scale >= 1.f ? scale : 1.f;
    center = scale * (static_cast<float>(i) + 0.5f);
    invscale = scale >= 1.f ? 1.f / scale : 1.f;
    xmin = max(static_cast<int>(center - support + 0.5f), 0);
    xsize = min(static_cast<int>(center + support + 0.5f), n) - xmin;
    total = 0.f;
    for (int j = 0; j < xsize; ++j) total += raw(j);
  }
  __device__ float raw(int j) const {
    const float w = fabsf((static_cast<float>(j + xmin) - center + 0.5f) * invscale);
    return w < 1.f ? 1.f - w : 0.f;
  }
  __device__ float operator()(int j) const { return total != 0.f ? raw(j) / total : 0.f; }
};

// out[b*G*G + gy*G + gx][c*P*P + ky*P + kx] = (aa(x[b][c]) at pixel (gy*P + ky, gx*P + kx) of R x R - mean_c) / std_c,
// columns 3*P*P .. kpad-1 zero.  (x + 1) / 2 is applied to every tap; each row of taps is summed first (x order), then
// the rows (y order).  Zero-weight taps are skipped, so S == R copies (x + 1) / 2 exactly.
__global__ void dino_pack_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int S, int G, int P,
                                 int kpad) {
  pdl_trigger();
  pdl_wait();
  const int R = G * P, pp = P * P, kdim = 3 * pp;
  const float scale = static_cast<float>(S) / static_cast<float>(R);
  const size_t total = static_cast<size_t>(B) * G * G * kpad;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t row = i / kpad;
    const int k = static_cast<int>(i - row * kpad);
    if (k >= kdim) {
      out[i] = 0.f;
      continue;
    }
    const size_t b = row / (static_cast<size_t>(G) * G);
    const int tok = static_cast<int>(row - b * G * G);
    const int c = k / pp, ky = (k % pp) / P, kx = k % P;
    const AaTaps ty((tok / G) * P + ky, S, scale), tx((tok % G) * P + kx, S, scale);
    const float* img = x + (b * 3 + c) * static_cast<size_t>(S) * S;
    float v = 0.f;
    for (int a = 0; a < ty.xsize; ++a) {
      const float wy = ty(a);
      if (wy == 0.f) continue;
      const float* line = img + static_cast<size_t>(ty.xmin + a) * S + tx.xmin;
      float h = 0.f;
      for (int e = 0; e < tx.xsize; ++e) {
        const float wx = tx(e);
        if (wx != 0.f) h += (line[e] + 1.f) / 2.f * wx;
      }
      v += h * wy;
    }
    out[i] = (v - kMean[c]) / kStd[c];
  }
}

// y = (x - mean) / sqrt(var + eps) * gamma + beta over row r of in (at in + r * ld) into dense out [rows][w]; biased
// variance, two passes, a warp per row
__global__ void __launch_bounds__(kRowThreads) dino_layernorm_kernel(const float* in, long long ld,
                                                                     const float* __restrict__ gamma,
                                                                     const float* __restrict__ beta, float* out,
                                                                     int rows, int w, float eps) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = in + static_cast<size_t>(row) * ld;
  float* y = out + static_cast<size_t>(row) * w;
  float s = 0.f;
  for (int c = lane; c < w; c += 32) s += x[c];
  const float mean = warp_sum(s) / static_cast<float>(w);
  float q = 0.f;
  for (int c = lane; c < w; c += 32) {
    const float d = x[c] - mean;
    q += d * d;
  }
  const float rstd = 1.f / sqrtf(warp_sum(q) / static_cast<float>(w) + eps);
  for (int c = lane; c < w; c += 32) y[c] = (x[c] - mean) * rstd * gamma[c] + beta[c];
}

// Non-causal softmax attention, head size 64, flash-style.  qkv [B*T][3D] packs q | k | v (head h in columns h*64 ..
// h*64+63 of each); out [B*T][D], the heads concatenated.  A CTA per (query tile, head, image); warp w owns query rows
// q0 + 16w .. +15.  Key tiles of 64 are staged through a two-stage cp.async ring in a fixed order; per tile
// S = Q K^T * scale and O += P V on mma.sync m16n8k8 (TF32 operands rounded to nearest, fp32 accumulation), with the
// online softmax in fp32 (m the running row max, l the running sum of exp(s - m)).  P stays in registers: the C
// fragment holds keys 2t, 2t+1 of each 8-key step, so A column t is taken as key 2t and column t+4 as key 2t+1, and the
// B fragment of V reads the same keys.  Rows past T read zeros; keys past T get p = 0.
__global__ void __launch_bounds__(kAttnWarps * 32) dino_attention_kernel(const float* __restrict__ qkv,
                                                                         float* __restrict__ out, int T, int D,
                                                                         float scale) {
  using tf32gemm::cp_async16;
  using tf32gemm::cp_async_commit;
  using tf32gemm::mma_tf32;
  using tf32gemm::tf32;
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int q0 = blockIdx.x * kQTile, h = blockIdx.y;
  const size_t ld = static_cast<size_t>(3) * D;
  const float* base = qkv + static_cast<size_t>(blockIdx.z) * T * ld + static_cast<size_t>(h) * kHeadDim;
  const int ntiles = (T + kKTile - 1) / kKTile;

  auto load = [&](int stage, int kt) {
    float* Ks = sm + stage * kKvStageFloats;
    float* Vs = Ks + kKTile * kKvLd;
    for (int idx = threadIdx.x; idx < kKTile * (kHeadDim / 4); idx += kAttnWarps * 32) {
      const int r = idx >> 4, c = (idx & 15) * 4, j = kt * kKTile + r;
      const bool ok = j < T;
      const float* src = base + (ok ? static_cast<size_t>(j) * ld : 0) + c;
      cp_async16(smem_u32(Ks + r * kKvLd + c), src + D, ok ? 16 : 0);
      cp_async16(smem_u32(Vs + r * kKvLd + c), src + 2 * static_cast<size_t>(D), ok ? 16 : 0);
    }
  };

  pdl_wait();
  load(0, 0);
  cp_async_commit();

  // Q fragments of this warp's 16 rows (A operand, row-major): a0 (g, t), a1 (g+8, t), a2 (g, t+4), a3 (g+8, t+4)
  uint32_t qa[kHeadDim / 8][4];
  {
    const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
    const float* p0 = base + static_cast<size_t>(r0) * ld;
    const float* p1 = base + static_cast<size_t>(r1) * ld;
#pragma unroll
    for (int kk = 0; kk < kHeadDim / 8; ++kk) {
      qa[kk][0] = tf32(r0 < T ? p0[kk * 8 + t] : 0.f);
      qa[kk][1] = tf32(r1 < T ? p1[kk * 8 + t] : 0.f);
      qa[kk][2] = tf32(r0 < T ? p0[kk * 8 + t + 4] : 0.f);
      qa[kk][3] = tf32(r1 < T ? p1[kk * 8 + t + 4] : 0.f);
    }
  }
  float o[kHeadDim / 8][4];
#pragma unroll
  for (int n = 0; n < kHeadDim / 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[n][e] = 0.f;
  float m[2] = {-FLT_MAX, -FLT_MAX}, l[2] = {0.f, 0.f};  // rows g and g + 8; l is this thread's share

  for (int kt = 0; kt < ntiles; ++kt) {
    if (kt + 1 < ntiles) load((kt + 1) & 1, kt + 1);
    cp_async_commit();
    tf32gemm::cp_async_wait<1>();
    __syncthreads();  // tile kt landed for every thread
    const float* Ks = sm + (kt & 1) * kKvStageFloats;
    const float* Vs = Ks + kKTile * kKvLd;
    float s[kKTile / 8][4];
#pragma unroll
    for (int n = 0; n < kKTile / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[n][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < kHeadDim / 8; ++kk) {
        const float* kr = Ks + (n * 8 + g) * kKvLd + kk * 8 + t;
        const uint32_t b[2] = {tf32(kr[0]), tf32(kr[4])};
        mma_tf32(s[n], qa[kk], b);
      }
    }
    // scale, mask the keys past T, and the row maxima of this tile (rows g: e = 0, 1; g + 8: e = 2, 3)
    float mx[2] = {-FLT_MAX, -FLT_MAX};
#pragma unroll
    for (int n = 0; n < kKTile / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = kt * kKTile + n * 8 + 2 * t + (e & 1);
        s[n][e] = j < T ? s[n][e] * scale : -FLT_MAX;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[n][e]);
      }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);
      corr[r] = expf(m[r] - mn);
      m[r] = mn;
      l[r] *= corr[r];
    }
#pragma unroll
    for (int n = 0; n < kKTile / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = kt * kKTile + n * 8 + 2 * t + (e & 1);
        s[n][e] = j < T ? expf(s[n][e] - m[e >> 1]) : 0.f;
        l[e >> 1] += s[n][e];
      }
#pragma unroll
    for (int n = 0; n < kHeadDim / 8; ++n) {
      o[n][0] *= corr[0];
      o[n][1] *= corr[0];
      o[n][2] *= corr[1];
      o[n][3] *= corr[1];
    }
#pragma unroll
    for (int kk = 0; kk < kKTile / 8; ++kk) {
      const uint32_t pa[4] = {tf32(s[kk][0]), tf32(s[kk][2]), tf32(s[kk][1]), tf32(s[kk][3])};
      const float* v0 = Vs + (kk * 8 + 2 * t) * kKvLd + g;
#pragma unroll
      for (int n = 0; n < kHeadDim / 8; ++n) {
        const uint32_t b[2] = {tf32(v0[n * 8]), tf32(v0[kKvLd + n * 8])};
        mma_tf32(o[n], pa, b);
      }
    }
    __syncthreads();  // every warp is done with this stage before the next iteration overwrites it
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  const int r0 = q0 + warp * 16 + g;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = r0 + 8 * hr;
    if (r >= T) continue;
    float* orow = out + (static_cast<size_t>(blockIdx.z) * T + r) * D + static_cast<size_t>(h) * kHeadDim;
#pragma unroll
    for (int n = 0; n < kHeadDim / 8; ++n)
      *reinterpret_cast<float2*>(orow + n * 8 + 2 * t) =
          make_float2(o[n][2 * hr] / l[hr], o[n][2 * hr + 1] / l[hr]);
  }
}

// Tile (I, J), I <= J, of pair p: sum over i in tile I, j in tile J of (Sa_ij - Sb_ij)^2 in fp64, times 2 off the
// diagonal, into partial[p][tile].  S_ij = k^_i . k^_j with k^ = k / max(|k|, eps): the rows are normalised as they are
// staged, the dot products are fp32 fmaf in column order, and a and b run the same code, so equal rows give 0 exactly.
// A thread owns a 4 x 4 block of entries; the CTA's fp64 sum is each warp's butterfly, then the warps in order.
__global__ void __launch_bounds__(kSimThreads) dino_selfsim_kernel(const float* __restrict__ keys, long long ld,
                                                                   const long long* __restrict__ ia,
                                                                   const long long* __restrict__ ib, int T, int D,
                                                                   float eps, double* __restrict__ partial) {
  pdl_trigger();
  __shared__ float tiles[4][kSimTile][kSimLd];  // a_I, a_J, b_I, b_J
  __shared__ float nrm[4][kSimTile];             // the rows' clamped norms max(|k|, eps)
  __shared__ double red[kSimThreads / 32];
  const int nt = (T + kSimTile - 1) / kSimTile;
  int I = 0, rem = blockIdx.x;
  while (rem >= nt - I) rem -= nt - I, ++I;
  const int J = I + rem, p = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  const long long pa = ia[p], pb = ib[p];
  const int nI = min(kSimTile, T - I * kSimTile), nJ = min(kSimTile, T - J * kSimTile);
  // staged tile `which` (a_I, a_J, b_I, b_J): its first key row and its row count
  auto row0 = [&](int which) {
    return (which < 2 ? pa : pb) + static_cast<long long>(which & 1 ? J : I) * kSimTile;
  };
  auto nrow = [&](int which) { return which & 1 ? nJ : nI; };
  for (int r = warp; r < 4 * kSimTile; r += kSimThreads / 32) {
    const int which = r / kSimTile, rr = r % kSimTile;
    if (rr >= nrow(which)) continue;
    const float* row = keys + static_cast<size_t>(row0(which) + rr) * static_cast<size_t>(ld);
    float q = 0.f;
    for (int c = lane; c < D; c += 32) q = fmaf(row[c], row[c], q);
    q = warp_sum(q);
    if (lane == 0) nrm[which][rr] = fmaxf(sqrtf(q), eps);
  }
  const int ti = (threadIdx.x >> 4) * 4, tj = (threadIdx.x & 15) * 4;
  float sa[4][4], sb[4][4];
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) sa[x][y] = sb[x][y] = 0.f;
  for (int c0 = 0; c0 < D; c0 += kSimChunk) {
    __syncthreads();  // the norms are in; the previous chunk is consumed
    for (int e = threadIdx.x; e < 4 * kSimTile * kSimChunk; e += kSimThreads) {
      const int which = e / (kSimTile * kSimChunk), rr = (e / kSimChunk) % kSimTile, c = e % kSimChunk;
      float v = 0.f;
      if (rr < nrow(which) && c0 + c < D)
        v = keys[static_cast<size_t>(row0(which) + rr) * static_cast<size_t>(ld) + c0 + c] / nrm[which][rr];
      tiles[which][rr][c] = v;
    }
    __syncthreads();
    const int cn = min(kSimChunk, D - c0);
    for (int c = 0; c < cn; ++c) {
      float ai[4], aj[4], bi[4], bj[4];
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        ai[x] = tiles[0][ti + x][c];
        aj[x] = tiles[1][tj + x][c];
        bi[x] = tiles[2][ti + x][c];
        bj[x] = tiles[3][tj + x][c];
      }
#pragma unroll
      for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 4; ++y) {
          sa[x][y] = fmaf(ai[x], aj[y], sa[x][y]);
          sb[x][y] = fmaf(bi[x], bj[y], sb[x][y]);
        }
    }
  }
  double acc = 0.0;
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y)
      if (ti + x < nI && tj + y < nJ) {
        const double d = static_cast<double>(sa[x][y]) - static_cast<double>(sb[x][y]);
        acc += d * d;
      }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kSimThreads / 32; ++w) s += red[w];
    partial[static_cast<size_t>(p) * gridDim.x + blockIdx.x] = I == J ? s : 2.0 * s;
  }
}

// out[p] = (sum of pair p's tile partials in tile order) / T^2
__global__ void dino_selfsim_reduce_kernel(const double* __restrict__ partial, double* __restrict__ out, int P,
                                           int ntp, int T) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double s = 0.0;
  for (int q = 0; q < ntp; ++q) s += partial[static_cast<size_t>(p) * ntp + q];
  out[p] = s / (static_cast<double>(T) * T);
}

inline int grid_cap(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

inline int selfsim_tiles(int T) {
  const int nt = (T + kSimTile - 1) / kSimTile;
  return nt * (nt + 1) / 2;
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_dino_pack(const float* x, float* out, int B, int S, int grid, int patch, int kpad, void* stream) {
  ASYRP_REQUIRE(x != nullptr && out != nullptr, "asyrp_dino_pack: null pointer");
  ASYRP_REQUIRE(B > 0 && S > 0 && S <= 4096 && grid > 0 && patch > 0 && grid * patch <= 4096,
                "asyrp_dino_pack: bad shape B=%d S=%d grid=%d patch=%d (S, grid*patch <= 4096)", B, S, grid, patch);
  const int kdim = 3 * patch * patch;
  ASYRP_REQUIRE(kpad % 32 == 0 && kpad >= kdim && kpad < kdim + 32,
                "asyrp_dino_pack: kpad=%d must be 3*patch^2=%d rounded up to a multiple of 32", kpad, kdim);
  const size_t total = static_cast<size_t>(B) * grid * grid * kpad;
  ASYRP_LAUNCH(dino_pack_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), x, out, B,
               S, grid, patch, kpad);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_dino_layernorm(const float* in, long long ld, const float* gamma, const float* beta, float* out,
                                   int rows, int width, float eps, void* stream) {
  ASYRP_REQUIRE(in != nullptr && gamma != nullptr && beta != nullptr && out != nullptr,
                "asyrp_dino_layernorm: null pointer");
  ASYRP_REQUIRE(rows > 0 && width > 0 && ld >= width, "asyrp_dino_layernorm: bad shape rows=%d width=%d ld=%lld", rows,
                width, ld);
  ASYRP_REQUIRE(eps > 0.f, "asyrp_dino_layernorm: eps=%g must be > 0", eps);
  ASYRP_REQUIRE((out == in && ld == width) || out + static_cast<size_t>(rows) * width <= in ||
                    in + static_cast<size_t>(rows - 1) * ld + width <= out,
                "asyrp_dino_layernorm: out must not overlap in (out == in needs ld == width)");
  const int per = kRowThreads / 32;
  ASYRP_LAUNCH(dino_layernorm_kernel, dim3((rows + per - 1) / per), dim3(kRowThreads), 0,
               static_cast<cudaStream_t>(stream), in, ld, gamma, beta, out, rows, width, eps);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_dino_attention(const float* qkv, float* out, int B, int T, int heads, void* stream) {
  ASYRP_REQUIRE(qkv != nullptr && out != nullptr, "asyrp_dino_attention: null pointer");
  ASYRP_REQUIRE(B > 0 && B <= kMaxGridYZ && heads > 0 && heads <= kMaxGridYZ && T > 0 && T <= kMaxTokens,
                "asyrp_dino_attention: bad shape B=%d T=%d heads=%d (T <= %d)", B, T, heads, kMaxTokens);
  ASYRP_REQUIRE(reinterpret_cast<uintptr_t>(qkv) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 8 == 0,
                "asyrp_dino_attention: qkv must be 16-byte and out 8-byte aligned");
  const int D = heads * kHeadDim;
  const size_t n_qkv = static_cast<size_t>(B) * T * 3 * D, n_out = static_cast<size_t>(B) * T * D;
  ASYRP_REQUIRE(out + n_out <= qkv || qkv + n_qkv <= out, "asyrp_dino_attention: out must not overlap qkv");
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(dino_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kAttnSmem)));
  ASYRP_LAUNCH(dino_attention_kernel, dim3((T + kQTile - 1) / kQTile, heads, B), dim3(kAttnWarps * 32), kAttnSmem,
               static_cast<cudaStream_t>(stream), qkv, out, T, D, 1.f / sqrtf(static_cast<float>(kHeadDim)));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_dino_selfsim_partials(int T) {
  return T > 0 && T <= kMaxTokens ? selfsim_tiles(T) : -1;
}

ASYRP_API int asyrp_dino_selfsim_distance(const float* keys, long long ld, const long long* ia, const long long* ib,
                                          int P, int T, int D, float eps, double* partial, double* out, void* stream) {
  ASYRP_REQUIRE(keys != nullptr && ia != nullptr && ib != nullptr && partial != nullptr && out != nullptr,
                "asyrp_dino_selfsim_distance: null pointer");
  ASYRP_REQUIRE(P > 0 && P <= kMaxGridYZ && T > 0 && T <= kMaxTokens && D > 0 && ld >= D,
                "asyrp_dino_selfsim_distance: bad shape P=%d T=%d D=%d ld=%lld (T <= %d, P <= %d)", P, T, D, ld,
                kMaxTokens, kMaxGridYZ);
  ASYRP_REQUIRE(eps > 0.f, "asyrp_dino_selfsim_distance: eps=%g must be > 0", eps);
  ASYRP_REQUIRE(reinterpret_cast<uintptr_t>(keys) % 4 == 0 && reinterpret_cast<uintptr_t>(ia) % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(ib) % 8 == 0 && reinterpret_cast<uintptr_t>(partial) % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(out) % 8 == 0,
                "asyrp_dino_selfsim_distance: keys must be 4-byte and ia, ib, partial, out 8-byte aligned");
  const int ntp = selfsim_tiles(T);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ASYRP_LAUNCH(dino_selfsim_kernel, dim3(ntp, P), dim3(kSimThreads), 0, st, keys, ld, ia, ib, T, D, eps, partial);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  ASYRP_LAUNCH(dino_selfsim_reduce_kernel, dim3((P + 127) / 128), dim3(128), 0, st, partial, out, P, ntp, T);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
