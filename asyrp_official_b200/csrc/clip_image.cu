// CLIP's image tower (OpenAI CLIP `VisionTransformer.forward`) and the directional similarity of CLIPLoss
// (losses/clip_loss.py:102-117,170-180).  Activations are fp32 [B][T][width], T = 1 + G^2 tokens.
//
//   patches  = patchify(Normalize_clip(Resize_bicubic((x + 1) / 2)))        clip_image_patches_kernel
//   x        = [class_embedding ; patches @ conv1^T] + positional_embedding  (GEMM in clip_text.cu), clip_tokens_kernel
//   x        = ln_pre(x); residual blocks with full attention (clip_text.cu)
//   feature  = ln_post(x[:, 0]) @ proj                                       (clip_text.cu)
//   dir[g]   = mean_i(trg_i/|trg_i| - src_i/|src_i|) / (|.| + add_eps)     clip_direction_kernel
//
// Every reduction runs in a fixed order (no float atomics) and no kernel mixes images, so an image's features are the
// same bits whatever batch it is in.
#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kDirThreads = 256;
// 48 KB of dynamic shared memory (2 * rows per group + dim floats); with the kernel's static red[] that is past the
// default 48 KB per block, so the launch opts in
constexpr int kDirSmemFloats = 12288;
// CLIP's Normalize
__constant__ float kClipMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float kClipStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// PyTorch's cubic convolution coefficients with A = -0.75 (upsample_bicubic2d's get_cubic_upsample_coefficients)
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
  constexpr float A = -0.75f;
  auto conv1 = [](float x) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };
  auto conv2 = [](float x) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };
  c[0] = conv2(t + 1.f);
  c[1] = conv1(t);
  c[2] = conv1(1.f - t);
  c[3] = conv2(2.f - t);
}

// out[b*G*G + gy*G + gx][c*P*P + ky*P + kx] = Normalize_clip(bicubic(x[b][c], pixel (gy*P + ky, gx*P + kx) of R x R)),
// columns kdim = 3*P*P .. kpad-1 zero.  The resize is F.interpolate(mode="bicubic", align_corners=False) without
// antialiasing: source coordinate (o + 0.5) * S/R - 0.5 (not clamped), taps floor-1 .. floor+2 clamped to the image,
// rows interpolated first, then the column.  (x + 1) / 2 is applied to every tap, as Normalize(-1, 2) precedes the
// resize.
__global__ void clip_image_patches_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int S, int G,
                                          int P, int kpad) {
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
    const int b = static_cast<int>(row / (G * G)), tok = static_cast<int>(row % (G * G));
    const int c = k / pp, ky = (k % pp) / P, kx = k % P;
    const int oy = (tok / G) * P + ky, ox = (tok % G) * P + kx;
    const float ry = scale * (oy + 0.5f) - 0.5f, rx = scale * (ox + 0.5f) - 0.5f;
    const float fy = floorf(ry), fx = floorf(rx);
    float wy[4], wx[4];
    cubic_coeffs(ry - fy, wy);
    cubic_coeffs(rx - fx, wx);
    const int iy = static_cast<int>(fy), ix = static_cast<int>(fx);
    const float* img = x + (static_cast<size_t>(b) * 3 + c) * S * S;
    float v = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const float* line = img + static_cast<size_t>(min(max(iy - 1 + a, 0), S - 1)) * S;
      float h = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) h += (line[min(max(ix - 1 + e, 0), S - 1)] + 1.f) / 2.f * wx[e];
      v += h * wy[a];
    }
    out[i] = (v - kClipMean[c]) / kClipStd[c];
  }
}

// out[b][0][c] = class_embedding[c] + pos[0][c];  out[b][1+p][c] = emb[b*(T-1) + p][c] + pos[1+p][c]
__global__ void clip_tokens_kernel(const float* __restrict__ emb, const float* __restrict__ cls,
                                   const float* __restrict__ pos, float* __restrict__ out, int B, int T, int w) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(B) * T * w;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / w;
    const int c = static_cast<int>(i - r * w), t = static_cast<int>(r % T), b = static_cast<int>(r / T);
    const float e = t == 0 ? cls[c] : emb[(static_cast<size_t>(b) * (T - 1) + t - 1) * w + c];
    out[i] = e + pos[static_cast<size_t>(t) * w + c];
  }
}

// One CTA per group g of n rows: d = (1/n) sum_i (trg_i / |trg_i| - src_i / |src_i|) summed in i order, then
// out[g] = d / (|d| + add_eps).  Row norms: a warp per row; |d|: per-thread partials over a fixed column set, each
// warp's butterfly, the eight warp sums added in warp order.
__global__ void __launch_bounds__(kDirThreads) clip_direction_kernel(const float* __restrict__ src,
                                                                     const float* __restrict__ trg,
                                                                     float* __restrict__ out, int n, int dim,
                                                                     float add_eps) {
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  float* ns = sm;           // [n] |src_i|
  float* nt = ns + n;       // [n] |trg_i|
  float* d = nt + n;        // [dim]
  __shared__ float red[kDirThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t base = static_cast<size_t>(blockIdx.x) * n * dim;
  const float* S = src + base;
  const float* Tr = trg + base;
  pdl_wait();
  for (int r = warp; r < 2 * n; r += kDirThreads / 32) {
    const float* row = (r < n ? S : Tr) + static_cast<size_t>(r % n) * dim;
    float q = 0.f;
    for (int c = lane; c < dim; c += 32) q += row[c] * row[c];
    q = sqrtf(warp_sum(q));
    if (lane == 0) sm[r] = q;
  }
  __syncthreads();
  float part = 0.f;
  for (int c = threadIdx.x; c < dim; c += kDirThreads) {
    float acc = 0.f;
    const float* tp = Tr + c;
    const float* sp = S + c;
    for (int i = 0; i < n; ++i, tp += dim, sp += dim) {
      const float a = *tp / nt[i];
      const float b = *sp / ns[i];
      acc += a - b;
    }
    acc /= static_cast<float>(n);
    d[c] = acc;
    part += acc * acc;
  }
  part = warp_sum(part);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int k = 0; k < kDirThreads / 32; ++k) tot += red[k];
  const float denom = sqrtf(tot) + add_eps;
  float* o = out + static_cast<size_t>(blockIdx.x) * dim;
  for (int c = threadIdx.x; c < dim; c += kDirThreads) o[c] = d[c] / denom;
}

inline int grid_cap(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_clip_image_patches(const float* x, float* out, int B, int S, int grid, int patch, int kpad,
                                       void* stream) {
  ASYRP_REQUIRE(B > 0 && S > 0 && grid > 0 && patch > 0 && grid * patch <= 4096,
                "asyrp_clip_image_patches: bad shape B=%d S=%d grid=%d patch=%d", B, S, grid, patch);
  const int kdim = 3 * patch * patch;
  ASYRP_REQUIRE(kpad % 32 == 0 && kpad >= kdim && kpad < kdim + 32,
                "asyrp_clip_image_patches: kpad=%d must be 3*patch^2=%d rounded up to a multiple of 32", kpad, kdim);
  const size_t total = static_cast<size_t>(B) * grid * grid * kpad;
  ASYRP_LAUNCH(clip_image_patches_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               x, out, B, S, grid, patch, kpad);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_image_tokens(const float* patch_emb, const float* class_embedding,
                                      const float* positional_embedding, float* out, int B, int T, int width,
                                      void* stream) {
  ASYRP_REQUIRE(B > 0 && T > 1 && width > 0, "asyrp_clip_image_tokens: bad shape B=%d T=%d width=%d", B, T, width);
  const size_t total = static_cast<size_t>(B) * T * width;
  ASYRP_LAUNCH(clip_tokens_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               patch_emb, class_embedding, positional_embedding, out, B, T, width);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_clip_direction(const float* src, const float* trg, float* out, int groups, int n, int dim,
                                   float add_eps, void* stream) {
  ASYRP_REQUIRE(groups > 0 && n > 0 && dim > 0 && 2 * n + dim <= kDirSmemFloats,
                "asyrp_clip_direction: bad shape groups=%d n=%d dim=%d (2n + dim <= %d)", groups, n, dim,
                kDirSmemFloats);
  ASYRP_REQUIRE(add_eps >= 0.f, "asyrp_clip_direction: add_eps=%g must be >= 0", add_eps);
  const size_t smem = static_cast<size_t>(2 * n + dim) * sizeof(float);
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(clip_direction_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kDirSmemFloats * static_cast<int>(sizeof(float))));
  ASYRP_LAUNCH(clip_direction_kernel, dim3(groups), dim3(kDirThreads), smem, static_cast<cudaStream_t>(stream), src,
               trg, out, n, dim, add_eps);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
