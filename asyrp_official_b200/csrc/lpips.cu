// LPIPS-AlexNet (the lpips package's LPIPS(net='alex', version='0.1'), spatial=False), as Asyrp.compute_lpips_distance
// evaluates it after every inversion step (diffusion_latent.py:1198-1273): scaling layer, the five conv+ReLU slices of
// torchvision's alexnet().features with the two 3/2 max pools, and the per-layer distance head.
//
// Activations are fp32 NHWC.  The convs are the implicit GEMM of tf32_gemm.cuh (mma.sync m16n8k8, TF32 operands
// rounded to nearest, fp32 accumulation) with the ReLU epilogue: M = N*Ho*Wo output pixels, N = Cout, K = kh*kw*Cin, tap-major /
// channel-minor.  fp32 storage, not the UNet's fp16: x0_t of an exploding trajectory reaches |x| ~ 1e3 and the ReLU
// stack carries that scale through five layers.  Every output element is one thread's fixed-order accumulation and
// the distance reduction is fixed-order too, so a sample's distance does not depend on the batch it is in.
#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kDistPixels = 32;     // pixels per CTA of the distance kernel
constexpr int kDistThreads = 256;
using tf32gemm::kBK;
using tf32gemm::kBN;
using tf32gemm::kBM;

// ScalingLayer + layout: fp32 NCHW [N][3][H][W] -> (x - shift) / scale as fp32 NHWC [N][H][W][4], channel 3 zero
__global__ void lpips_pack_kernel(const float* __restrict__ x, const float* __restrict__ shift_scale,
                                  float* __restrict__ out, int N, int HW) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * HW;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = i / HW, px = i - n * HW;
    const float* src = x + n * 3 * HW + px;
    float4 v;
    v.x = (src[0] - shift_scale[0]) / shift_scale[3];
    v.y = (src[HW] - shift_scale[1]) / shift_scale[4];
    v.z = (src[2 * static_cast<size_t>(HW)] - shift_scale[2]) / shift_scale[5];
    v.w = 0.f;
    reinterpret_cast<float4*>(out)[i] = v;
  }
}

// MaxPool2d(3, stride 2), no padding, floor mode; one thread = 4 channels of one output pixel
__global__ void lpips_maxpool_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W,
                                     int C, int Ho, int Wo) {
  pdl_trigger();
  pdl_wait();
  const int C4 = C / 4;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    size_t r = i / C4;
    const int ox = static_cast<int>(r % Wo);
    r /= Wo;
    const int oy = static_cast<int>(r % Ho);
    const size_t n = r / Ho;
    const float4* base = reinterpret_cast<const float4*>(in) + (n * H * W) * C4 + c4;
    float4 m = base[(static_cast<size_t>(2 * oy) * W + 2 * ox) * C4];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const float4 v = base[(static_cast<size_t>(2 * oy + dy) * W + 2 * ox + dx) * C4];
        m.x = fmaxf(m.x, v.x);
        m.y = fmaxf(m.y, v.y);
        m.z = fmaxf(m.z, v.z);
        m.w = fmaxf(m.w, v.w);
      }
    reinterpret_cast<float4*>(out)[i] = m;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}

// One LPIPS layer term: per pixel f/(|f| + 1e-10) of probe row n and reference row n % B, squared difference, the lin
// weights (1x1 conv C -> 1, no bias), then the mean over H*W, added into d[n] (written when !accumulate).  CTA
// (chunk, n) covers pixels [chunk*32, chunk*32 + 32), a warp per pixel with the channels across its lanes; the
// chunk sums go to partial[n][chunk] and the last CTA of sample n (integer ticket) adds them up in chunk order.  The
// pixel -> warp -> chunk mapping depends on H*W and C only: the result does not depend on the batch.
__global__ void __launch_bounds__(kDistThreads) lpips_distance_kernel(
    const float* __restrict__ probe, const float* __restrict__ ref, int B, int HW, int C,
    const float* __restrict__ lin_w, float* partial, int* counters, float* d, int accumulate) {
  pdl_trigger();
  pdl_wait();
  const int chunk = blockIdx.x, nchunk = gridDim.x, n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = kDistThreads / 32;
  const float* P = probe + static_cast<size_t>(n) * HW * C;
  const float* R = ref + static_cast<size_t>(n % B) * HW * C;
  float part = 0.f;
  const int px_end = min(HW, (chunk + 1) * kDistPixels);
  for (int px = chunk * kDistPixels + warp; px < px_end; px += nw) {
    const float* pp = P + static_cast<size_t>(px) * C;
    const float* rr = R + static_cast<size_t>(px) * C;
    float sp = 0.f, sr = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float a = pp[c], b = rr[c];
      sp += a * a;
      sr += b * b;
    }
    const float dp = sqrtf(warp_sum(sp)) + 1e-10f, dr = sqrtf(warp_sum(sr)) + 1e-10f;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float diff = pp[c] / dp - rr[c] / dr;
      s += lin_w[c] * (diff * diff);
    }
    part += warp_sum(s);
  }
  __shared__ float sh[kDistThreads / 32];
  __shared__ int last;
  if (lane == 0) sh[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int w = 0; w < nw; ++w) v += sh[w];
    partial[static_cast<size_t>(n) * nchunk + chunk] = v;
    __threadfence();
    last = atomicAdd(counters + n, 1) == nchunk - 1;
  }
  __syncthreads();
  if (!last || warp != 0) return;
  __threadfence();
  float v = 0.f;
  for (int c = lane; c < nchunk; c += 32) v += __ldcg(partial + static_cast<size_t>(n) * nchunk + c);
  v = warp_sum(v);
  if (lane == 0) {
    v = v / static_cast<float>(HW);
    d[n] = accumulate ? d[n] + v : v;
    counters[n] = 0;  // ready for the next launch
  }
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

ASYRP_API int asyrp_lpips_pack(const float* x, const float* shift_scale, float* out, int N, int H, int W,
                               void* stream) {
  ASYRP_REQUIRE(N > 0 && H > 0 && W > 0, "asyrp_lpips_pack: bad shape N=%d H=%d W=%d", N, H, W);
  const size_t total = static_cast<size_t>(N) * H * W;
  ASYRP_LAUNCH(lpips_pack_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), x,
               shift_scale, out, N, H * W);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_lpips_conv_kpad(int Cin, int kh, int kw) { return (kh * kw * Cin + kBK - 1) / kBK * kBK; }

ASYRP_API int asyrp_lpips_conv(const float* in, const float* weight, const float* bias, float* out, int N, int H,
                               int W, int Cin, int Cout, int kh, int kw, int stride, int pad, void* stream) {
  ASYRP_REQUIRE(Cin > 0 && Cin % 4 == 0, "asyrp_lpips_conv: Cin=%d must be a positive multiple of 4", Cin);
  ASYRP_REQUIRE(Cout > 0 && Cout % kBN == 0, "asyrp_lpips_conv: Cout=%d must be a positive multiple of %d", Cout, kBN);
  ASYRP_REQUIRE(kh > 0 && kw > 0 && stride > 0 && pad >= 0, "asyrp_lpips_conv: bad kernel geometry");
  ASYRP_REQUIRE(bias != nullptr, "asyrp_lpips_conv: the ReLU epilogue needs a bias");
  ASYRP_REQUIRE(in != out, "asyrp_lpips_conv: out must not alias in");
  tf32gemm::Tf32ConvParams p;
  p.in = in; p.w = weight; p.bias = bias; p.residual = nullptr; p.out = out;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.kw = kw; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - kh) / stride + 1;
  p.Wo = (W + 2 * pad - kw) / stride + 1;
  ASYRP_REQUIRE(N > 0 && H + 2 * pad >= kh && W + 2 * pad >= kw, "asyrp_lpips_conv: input %dx%d smaller than the kernel",
                H, W);
  p.K = kh * kw * Cin;
  p.Kpad = asyrp_lpips_conv_kpad(Cin, kh, kw);
  const long long M = static_cast<long long>(N) * p.Ho * p.Wo;
  ASYRP_REQUIRE(M < (1LL << 31) / kBM * kBM, "asyrp_lpips_conv: too many output pixels");
  p.M = static_cast<int>(M);
  return tf32gemm::launch_tf32_conv<tf32gemm::kEpiRelu>(p, static_cast<cudaStream_t>(stream));
}

ASYRP_API int asyrp_lpips_maxpool(const float* in, float* out, int N, int H, int W, int C, void* stream) {
  ASYRP_REQUIRE(C % 4 == 0 && H >= 3 && W >= 3 && N > 0, "asyrp_lpips_maxpool: bad shape N=%d H=%d W=%d C=%d", N, H,
                W, C);
  const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * (C / 4);
  ASYRP_LAUNCH(lpips_maxpool_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), in,
               out, N, H, W, C, Ho, Wo);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_lpips_distance_chunks(int HW) { return (HW + kDistPixels - 1) / kDistPixels; }

ASYRP_API int asyrp_lpips_distance(const float* probe, const float* ref, int N, int B, int HW, int C,
                                   const float* lin_w, float* partial, int* counters, float* d, int accumulate,
                                   void* stream) {
  ASYRP_REQUIRE(N > 0 && B > 0 && HW > 0 && C > 0, "asyrp_lpips_distance: bad shape N=%d B=%d HW=%d C=%d", N, B, HW,
                C);
  ASYRP_LAUNCH(lpips_distance_kernel, dim3(asyrp_lpips_distance_chunks(HW), N), dim3(kDistThreads), 0,
               static_cast<cudaStream_t>(stream), probe, ref, B, HW, C, lin_w, partial, counters, d, accumulate);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
