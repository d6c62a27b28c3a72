// CLIP's text tower (OpenAI CLIP `encode_text`) and the text-direction cosine Asyrp.set_t_edit_t_addnoise takes from
// it (diffusion_latent.py:1319-1329).  The LayerNorm, the residual blocks' linear layers and the attention (full
// rather than causal) also serve the image tower (clip_image.cu).  Activations are fp32 [P][T][width] (P prompts, T = 77 tokens).
//
//   x = token_embedding[id] + positional_embedding
//   layers x:  x = x + out_proj(causal_mha(ln_1(x)));  x = x + c_proj(quick_gelu(c_fc(ln_2(x))))
//   feature  = ln_final(x[eot]) @ text_projection,  eot = first argmax of the ids
//
// The linear layers are the TF32 implicit GEMM of tf32_gemm.cuh (a 1x1 conv over a 1 x P*T image) with the bias,
// QuickGELU and residual epilogues.  LayerNorm, the causal attention, the pooling and the cosine are fp32 kernels
// below.  Every reduction runs in a fixed order (a warp's butterfly over lane partial sums taken in index order; no
// float atomics) and no kernel mixes prompts, so a prompt's features are the same bits whatever batch it is in.
#include <cfloat>
#include <climits>

#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kHeadDim = 64;
constexpr int kMaxTokens = 128;     // text tower: keys per query row, four per lane
constexpr int kAttnWarps = 4;
constexpr int kMaxImageTokens = 257;  // image tower: 1 + G^2 tokens, G <= 16 (ViT-L/14 at 224)
constexpr int kImageAttnSlots = 288;  // kMaxImageTokens rounded up to whole lanes: nine keys per lane
constexpr int kImageAttnWarps = 8;
constexpr int kRowThreads = 256;    // LayerNorm / cosine: one warp per row

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// y = (x - mean) / sqrt(var + 1e-5) * gamma + beta over one row of w floats (biased variance, two passes), by one
// warp; y may be x
__device__ __forceinline__ void layernorm_row(const float* x, const float* __restrict__ gamma,
                                              const float* __restrict__ beta, float* y, int w, int lane) {
  float s = 0.f;
  for (int c = lane; c < w; c += 32) s += x[c];
  const float mean = warp_sum(s) / static_cast<float>(w);
  float q = 0.f;
  for (int c = lane; c < w; c += 32) {
    const float d = x[c] - mean;
    q += d * d;
  }
  const float rstd = 1.f / sqrtf(warp_sum(q) / static_cast<float>(w) + 1e-5f);
  for (int c = lane; c < w; c += 32) y[c] = (x[c] - mean) * rstd * gamma[c] + beta[c];
}

// out[p][t][c] = tok[ids[p][t]][c] + pos[t][c]
__global__ void clip_embed_kernel(const int* __restrict__ ids, const float* __restrict__ tok,
                                  const float* __restrict__ pos, float* __restrict__ out, int rows, int T, int w) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(rows) * w;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / w), c = static_cast<int>(i - static_cast<size_t>(r) * w);
    out[i] = tok[static_cast<size_t>(ids[r]) * w + c] + pos[static_cast<size_t>(r % T) * w + c];
  }
}

// row r of in starts at in + r * ld (ld = w for a dense matrix; the image tower's ln_post reads the class-token rows
// with ld = T * w); out is dense [rows][w]
__global__ void __launch_bounds__(kRowThreads) clip_layernorm_kernel(const float* in, const float* __restrict__ gamma,
                                                                     const float* __restrict__ beta, float* out,
                                                                     int rows, int w, size_t ld) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  layernorm_row(in + static_cast<size_t>(row) * ld, gamma, beta, out + static_cast<size_t>(row) * w, w,
                threadIdx.x & 31);
}

// Multi-head attention of one (head, sample) per CTA, causal (text tower) or full (image tower).  qkv [P*T][3w]
// packs q | k | v as nn.MultiheadAttention's in_proj does, head h in columns h*64 .. h*64+63 of each; out [P*T][w],
// the heads concatenated.  A warp per query row i: lane j scores keys j, j+32, ... <= last (last = i when causal,
// T-1 otherwise; 64-term dot in d order, times scale), softmax with the row max subtracted, then
// out[d] = sum_{j <= last} p_j v_j[d] in j order.
template <bool kCausal, int kSlots, int kWarps>
__global__ void __launch_bounds__(kWarps * 32) clip_attention_kernel(const float* __restrict__ qkv,
                                                                     float* __restrict__ out, int T, int w,
                                                                     float scale) {
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;                                   // [T][65]
  float* Vs = Ks + T * (kHeadDim + 1);              // [T][64]
  float* Qs = Vs + T * kHeadDim;                    // [warps][64]
  float* Ps = Qs + kWarps * kHeadDim;               // [warps][kSlots]
  const int h = blockIdx.x, p = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t ld = static_cast<size_t>(3) * w;
  const float* base = qkv + static_cast<size_t>(p) * T * ld + h * kHeadDim;
  pdl_wait();
  for (int i = threadIdx.x; i < T * kHeadDim; i += blockDim.x) {
    const int j = i / kHeadDim, d = i - j * kHeadDim;
    Ks[j * (kHeadDim + 1) + d] = base[j * ld + w + d];
    Vs[j * kHeadDim + d] = base[j * ld + 2 * w + d];
  }
  __syncthreads();
  float* q = Qs + warp * kHeadDim;
  float* pr = Ps + warp * kSlots;
  for (int i = warp; i < T; i += kWarps) {
    const int last = kCausal ? i : T - 1;
    q[lane] = base[i * ld + lane];
    q[lane + 32] = base[i * ld + lane + 32];
    __syncwarp();
    float s[kSlots / 32];
    float mx = -FLT_MAX;
#pragma unroll
    for (int kk = 0; kk < kSlots / 32; ++kk) {
      const int j = lane + 32 * kk;
      s[kk] = -FLT_MAX;
      if (j <= last) {
        const float* kr = Ks + j * (kHeadDim + 1);
        float dot = 0.f;
#pragma unroll 16
        for (int d = 0; d < kHeadDim; ++d) dot += q[d] * kr[d];
        s[kk] = dot * scale;
        mx = fmaxf(mx, s[kk]);
      }
    }
    mx = warp_max(mx);
    float e[kSlots / 32], sum = 0.f;
#pragma unroll
    for (int kk = 0; kk < kSlots / 32; ++kk) {
      e[kk] = lane + 32 * kk <= last ? expf(s[kk] - mx) : 0.f;
      sum += e[kk];
    }
    sum = warp_sum(sum);
#pragma unroll
    for (int kk = 0; kk < kSlots / 32; ++kk)
      if (lane + 32 * kk <= last) pr[lane + 32 * kk] = e[kk] / sum;
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j <= last; ++j) {
      o0 += pr[j] * Vs[j * kHeadDim + lane];
      o1 += pr[j] * Vs[j * kHeadDim + lane + 32];
    }
    float* orow = out + (static_cast<size_t>(p) * T + i) * w + h * kHeadDim;
    orow[lane] = o0;
    orow[lane + 32] = o1;
    __syncwarp();  // q / pr are rewritten by the next row
  }
}

// out[p] = ln_final(x[p][eot]), eot = the first argmax of ids[p]; a warp per prompt
__global__ void __launch_bounds__(kRowThreads) clip_pool_kernel(const float* __restrict__ x, const int* __restrict__ ids,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta,
                                                                float* __restrict__ out, int P, int T, int w) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= P) return;
  int best = INT_MIN, at = T;
  for (int t = lane; t < T; t += 32) {
    const int v = ids[static_cast<size_t>(p) * T + t];
    if (v > best) best = v, at = t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int ob = __shfl_xor_sync(0xffffffffu, best, o), oa = __shfl_xor_sync(0xffffffffu, at, o);
    if (ob > best || (ob == best && oa < at)) best = ob, at = oa;
  }
  layernorm_row(x + (static_cast<size_t>(p) * T + at) * w, gamma, beta, out + static_cast<size_t>(p) * w, w, lane);
}

// cos[n] = sum_c a[n][c] / max(|a[n]|, eps) * b[n][c] / max(|b[n]|, eps), torch.nn.CosineSimilarity(dim=1, eps)'s
// formula; a warp per row
__global__ void __launch_bounds__(kRowThreads) clip_cosine_kernel(const float* __restrict__ a,
                                                                  const float* __restrict__ b, float* __restrict__ cos,
                                                                  int n, int dim, float eps) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* ar = a + static_cast<size_t>(r) * dim;
  const float* br = b + static_cast<size_t>(r) * dim;
  float sa = 0.f, sb = 0.f;
  for (int c = lane; c < dim; c += 32) {
    sa += ar[c] * ar[c];
    sb += br[c] * br[c];
  }
  const float na = fmaxf(sqrtf(warp_sum(sa)), eps), nb = fmaxf(sqrtf(warp_sum(sb)), eps);
  float s = 0.f;
  for (int c = lane; c < dim; c += 32) s += (ar[c] / na) * (br[c] / nb);
  s = warp_sum(s);
  if (lane == 0) cos[r] = s;
}

inline int grid_cap(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

inline size_t attention_smem(int T, int warps, int slots) {
  return (static_cast<size_t>(T) * (2 * kHeadDim + 1) + warps * (kHeadDim + slots)) * sizeof(float);
}

template <bool kCausal, int kSlots, int kWarps>
int launch_attention(const float* qkv, float* out, int P, int T, int heads, cudaStream_t stream) {
  const size_t smem = attention_smem(T, kWarps, kSlots);
  auto kernel = clip_attention_kernel<kCausal, kSlots, kWarps>;
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  ASYRP_LAUNCH(kernel, dim3(heads, P), dim3(kWarps * 32), smem, stream, qkv, out, T, heads * kHeadDim,
               1.f / sqrtf(static_cast<float>(kHeadDim)));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_clip_embed(const int* ids, const float* token_embedding, const float* positional_embedding,
                               float* out, int P, int T, int width, void* stream) {
  ASYRP_REQUIRE(P > 0 && T > 0 && width > 0, "asyrp_clip_embed: bad shape P=%d T=%d width=%d", P, T, width);
  const size_t total = static_cast<size_t>(P) * T * width;
  ASYRP_LAUNCH(clip_embed_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), ids,
               token_embedding, positional_embedding, out, P * T, T, width);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_layernorm(const float* in, const float* gamma, const float* beta, float* out, int rows,
                                   int width, void* stream) {
  ASYRP_REQUIRE(rows > 0 && width > 0, "asyrp_clip_layernorm: bad shape rows=%d width=%d", rows, width);
  const int per = kRowThreads / 32;
  ASYRP_LAUNCH(clip_layernorm_kernel, dim3((rows + per - 1) / per), dim3(kRowThreads), 0,
               static_cast<cudaStream_t>(stream), in, gamma, beta, out, rows, width, static_cast<size_t>(width));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_layernorm_rows(const float* in, long long ld, const float* gamma, const float* beta,
                                        float* out, int rows, int width, void* stream) {
  ASYRP_REQUIRE(rows > 0 && width > 0 && ld >= width, "asyrp_clip_layernorm_rows: bad shape rows=%d width=%d ld=%lld",
                rows, width, ld);
  ASYRP_REQUIRE(out + static_cast<size_t>(rows) * width <= in || in + static_cast<size_t>(rows - 1) * ld + width <= out,
                "asyrp_clip_layernorm_rows: out must not overlap in");
  const int per = kRowThreads / 32;
  ASYRP_LAUNCH(clip_layernorm_kernel, dim3((rows + per - 1) / per), dim3(kRowThreads), 0,
               static_cast<cudaStream_t>(stream), in, gamma, beta, out, rows, width, static_cast<size_t>(ld));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_linear(const float* in, const float* weight, const float* bias, const float* residual,
                                float* out, int M, int K, int N, int epilogue, void* stream) {
  using namespace tf32gemm;
  ASYRP_REQUIRE(M > 0 && M < (1 << 30), "asyrp_clip_linear: bad row count M=%d", M);
  ASYRP_REQUIRE(K > 0 && K % kBK == 0, "asyrp_clip_linear: K=%d must be a positive multiple of %d", K, kBK);
  ASYRP_REQUIRE(N > 0 && N % kBN == 0, "asyrp_clip_linear: N=%d must be a positive multiple of %d", N, kBN);
  ASYRP_REQUIRE((epilogue >= kEpiBias && epilogue <= kEpiResidual) || epilogue == kEpiGelu,
                "asyrp_clip_linear: unknown epilogue %d", epilogue);
  ASYRP_REQUIRE((epilogue == kEpiResidual) == (residual != nullptr),
                "asyrp_clip_linear: a residual is required by, and only by, the residual epilogue");
  ASYRP_REQUIRE(in != out && (residual == nullptr || residual == out || residual + static_cast<size_t>(M) * N <= out ||
                              out + static_cast<size_t>(M) * N <= residual),
                "asyrp_clip_linear: out must not alias in, and may alias residual only exactly");
  Tf32ConvParams p;
  p.in = in; p.w = weight; p.bias = bias; p.residual = residual; p.out = out;
  p.N = 1; p.H = 1; p.W = M; p.Cin = K; p.Ho = 1; p.Wo = M; p.Cout = N; p.kw = 1; p.stride = 1; p.pad = 0;
  p.K = K; p.Kpad = K; p.M = M;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (epilogue) {
    case kEpiBias: return launch_tf32_conv<kEpiBias>(p, st);
    case kEpiQuickGelu: return launch_tf32_conv<kEpiQuickGelu>(p, st);
    case kEpiGelu: return launch_tf32_conv<kEpiGelu>(p, st);
    default: return launch_tf32_conv<kEpiResidual>(p, st);
  }
}

ASYRP_API int asyrp_clip_attention(const float* qkv, float* out, int P, int T, int heads, void* stream) {
  ASYRP_REQUIRE(P > 0 && heads > 0 && T > 0 && T <= kMaxTokens,
                "asyrp_clip_attention: bad shape P=%d T=%d heads=%d (T <= %d)", P, T, heads, kMaxTokens);
  return launch_attention<true, kMaxTokens, kAttnWarps>(qkv, out, P, T, heads, static_cast<cudaStream_t>(stream));
}

ASYRP_API int asyrp_clip_attention_full(const float* qkv, float* out, int P, int T, int heads, void* stream) {
  ASYRP_REQUIRE(P > 0 && heads > 0 && T > 0 && T <= kMaxImageTokens,
                "asyrp_clip_attention_full: bad shape P=%d T=%d heads=%d (T <= %d)", P, T, heads, kMaxImageTokens);
  return launch_attention<false, kImageAttnSlots, kImageAttnWarps>(qkv, out, P, T, heads,
                                                                   static_cast<cudaStream_t>(stream));
}

ASYRP_API int asyrp_clip_pool(const float* x, const int* ids, const float* gamma, const float* beta, float* out, int P,
                              int T, int width, void* stream) {
  ASYRP_REQUIRE(P > 0 && T > 0 && width > 0, "asyrp_clip_pool: bad shape P=%d T=%d width=%d", P, T, width);
  const int per = kRowThreads / 32;
  ASYRP_LAUNCH(clip_pool_kernel, dim3((P + per - 1) / per), dim3(kRowThreads), 0, static_cast<cudaStream_t>(stream), x,
               ids, gamma, beta, out, P, T, width);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_cosine(const float* a, const float* b, float* cos, int n, int dim, float eps, void* stream) {
  ASYRP_REQUIRE(n > 0 && dim > 0, "asyrp_clip_cosine: bad shape n=%d dim=%d", n, dim);
  const int per = kRowThreads / 32;
  ASYRP_LAUNCH(clip_cosine_kernel, dim3((n + per - 1) / per), dim3(kRowThreads), 0, static_cast<cudaStream_t>(stream),
               a, b, cos, n, dim, eps);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
