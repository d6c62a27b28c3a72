// Content preservation of an edit against its source image: PSNR, SSIM and MS-SSIM of the u8 images save_image writes
// (asyrp_official_b200/preservation.py combines the statistics below on the host).
//
//   q = save_image's u8 of x (SavedPng, common.h); lvl0 = q / 255 (fp64); xq = (2 q - 255) / 255 (fp32)  png_quantize
//   SSE[j] = sum over the 3 H W values of (q_edit[j] - q_src[j % B])^2, an exact 64-bit integer      preserve_sse
//   per channel of row j at one level: the means over the (H - 10) x (W - 10) valid pixels of the SSIM map and of the
//     contrast-structure map cs, from an 11-tap Gaussian (sigma 1.5) applied separably without padding  ssim_level
//   avg_pool2d(kernel 2, stride 2, padding (H mod 2, W mod 2)), the padding counted in the divisor   ssim_pool2
//
// The SSIM arithmetic is fp64: sigma^2 = E[x^2] - mu^2 cancels, and C2 = 9e-4 does not hide an fp32 error.  Every
// product and sum of the map formula is an explicitly rounded operation (no contraction into an fma), and the moments of
// x x and x y are formed by the same operations, so identical planes give cs = ssim = 1 exactly.  One CTA owns one
// (row, channel) plane and sums its pixels in a fixed order, so a row's statistics are the same bits in any launch.
#include <climits>
#include <cmath>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kWin = 11, kRad = kWin / 2;
constexpr double kSigma = 1.5, kC1 = 0.01 * 0.01, kC2 = 0.03 * 0.03;
constexpr int kTX = 32, kTY = 16;                                  // output pixels per tile
constexpr int kInX = kTX + 2 * kRad, kInY = kTY + 2 * kRad;        // the tile with its 5-pixel halo
constexpr int kMoments = 5;                                        // mu_x, mu_y, E[x^2], E[y^2], E[xy]
constexpr int kSsimThreads = 256;
constexpr size_t kSsimSmem = sizeof(double) * (2 * kInY * kInX + kMoments * kInY * kTX);
constexpr int kSseThreads = 512;

struct Window {
  double g[kWin];
};

// the normalised Gaussian exp(-k^2 / (2 sigma^2)) / sum, k = -5 .. 5, in fp64 on the host
Window gaussian_window() {
  Window w;
  double s = 0.0;
  for (int k = 0; k < kWin; ++k) {
    const double d = k - kRad;
    w.g[k] = std::exp(-(d * d) / (2.0 * kSigma * kSigma));
    s += w.g[k];
  }
  for (int k = 0; k < kWin; ++k) w.g[k] /= s;
  return w;
}

__global__ void png_quantize_kernel(const float* __restrict__ x, uint8_t* __restrict__ q, double* __restrict__ lvl0,
                                    float* __restrict__ xq, size_t total) {
  pdl_trigger();
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float v = SavedPng::quantize(x[i]);
    q[i] = static_cast<uint8_t>(v);
    if (lvl0 != nullptr) lvl0[i] = static_cast<double>(v) / 255.0;
    // (2 q - 255) is exact in fp32; one rounding of the quotient
    if (xq != nullptr) xq[i] = __fdiv_rn(__fsub_rn(__fmul_rn(2.f, v), 255.f), 255.f);
  }
}

// one CTA per edited row j: the per-thread sums, then a fixed tree; integer arithmetic, so exact
__global__ void __launch_bounds__(kSseThreads) preserve_sse_kernel(const uint8_t* __restrict__ src,
                                                                   const uint8_t* __restrict__ edited,
                                                                   long long* __restrict__ sse, int B, size_t plane) {
  pdl_trigger();
  __shared__ unsigned long long red[kSseThreads / 32];
  pdl_wait();
  const size_t j = blockIdx.x;
  const uint8_t* a = src + (j % B) * plane;
  const uint8_t* b = edited + j * plane;
  unsigned long long s = 0;
  for (size_t i = threadIdx.x; i < plane; i += kSseThreads) {
    const int d = static_cast<int>(a[i]) - static_cast<int>(b[i]);
    s += static_cast<unsigned long long>(d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kSseThreads / 32; ++w) t += red[w];
    sse[j] = static_cast<long long>(t);
  }
}

// Plane p = blockIdx.x = row j * 3 + channel c of the edited level [n][3][H][W], against plane (j % B) * 3 + c of the
// source level.  Output tiles of kTY x kTX pixels in row-major order: the tile and its halo are staged in shared
// memory, the five moments filtered along x for the kInY rows, then along y; each thread adds the ssim and cs of its
// pixels to its sums in tile order, and the CTA sums the threads in a fixed tree.  stats[p] = (mean ssim, mean cs).
__global__ void __launch_bounds__(kSsimThreads) ssim_level_kernel(const double* __restrict__ src,
                                                                  const double* __restrict__ edited,
                                                                  double* __restrict__ stats, int B, int H, int W,
                                                                  Window win) {
  pdl_trigger();
  extern __shared__ double smem[];
  double* xs = smem;                      // [kInY][kInX]
  double* ys = xs + kInY * kInX;          // [kInY][kInX]
  double* hm = ys + kInY * kInX;          // [kMoments][kInY][kTX]
  const int t = threadIdx.x;
  const size_t p = blockIdx.x, hw = static_cast<size_t>(H) * W;
  const size_t j = p / 3, c = p % 3;
  const double* X = src + ((j % B) * 3 + c) * hw;
  const double* Y = edited + p * hw;
  const int Ho = H - 2 * kRad, Wo = W - 2 * kRad;
  const int tiles_x = (Wo + kTX - 1) / kTX, tiles = tiles_x * ((Ho + kTY - 1) / kTY);
  pdl_wait();
  double s_ssim = 0.0, s_cs = 0.0;
  for (int tile = 0; tile < tiles; ++tile) {
    const int oy0 = (tile / tiles_x) * kTY, ox0 = (tile % tiles_x) * kTX;
    // inputs past the image only feed outputs past the valid region, which are not summed
    for (int e = t; e < kInY * kInX; e += kSsimThreads) {
      const int gy = oy0 + e / kInX, gx = ox0 + e % kInX;
      const bool in = gy < H && gx < W;
      const size_t o = static_cast<size_t>(gy) * W + gx;
      xs[e] = in ? X[o] : 0.0;
      ys[e] = in ? Y[o] : 0.0;
    }
    __syncthreads();
    for (int e = t; e < kInY * kTX; e += kSsimThreads) {
      const int iy = e / kTX, ox = e % kTX;
      const double* xr = xs + iy * kInX + ox;
      const double* yr = ys + iy * kInX + ox;
      double m[kMoments] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double a = xr[k], b = yr[k], g = win.g[k];
        m[0] = fma(g, a, m[0]);
        m[1] = fma(g, b, m[1]);
        m[2] = fma(g, __dmul_rn(a, a), m[2]);
        m[3] = fma(g, __dmul_rn(b, b), m[3]);
        m[4] = fma(g, __dmul_rn(a, b), m[4]);
      }
#pragma unroll
      for (int q = 0; q < kMoments; ++q) hm[(q * kInY + iy) * kTX + ox] = m[q];
    }
    __syncthreads();
    for (int e = t; e < kTY * kTX; e += kSsimThreads) {
      const int oy = e / kTX, ox = e % kTX;
      if (oy0 + oy >= Ho || ox0 + ox >= Wo) continue;
      double m[kMoments] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double g = win.g[k];
#pragma unroll
        for (int q = 0; q < kMoments; ++q) m[q] = fma(g, hm[(q * kInY + oy + k) * kTX + ox], m[q]);
      }
      const double mxy = __dmul_rn(m[0], m[1]), mxx = __dmul_rn(m[0], m[0]), myy = __dmul_rn(m[1], m[1]);
      const double sxx = __dsub_rn(m[2], mxx), syy = __dsub_rn(m[3], myy), sxy = __dsub_rn(m[4], mxy);
      const double cs = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, sxy), kC2), __dadd_rn(__dadd_rn(sxx, syy), kC2));
      const double lum = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, mxy), kC1), __dadd_rn(__dadd_rn(mxx, myy), kC1));
      s_ssim = __dadd_rn(s_ssim, __dmul_rn(lum, cs));
      s_cs = __dadd_rn(s_cs, cs);
    }
    __syncthreads();
  }
  double* red = smem;  // 2 x 256 doubles of the (now idle) staging tiles
  red[t] = s_ssim;
  red[kSsimThreads + t] = s_cs;
  __syncthreads();
  for (int h = kSsimThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      red[t] += red[t + h];
      red[kSsimThreads + t] += red[kSsimThreads + t + h];
    }
    __syncthreads();
  }
  if (t == 0) {
    const double count = static_cast<double>(Ho) * Wo;
    stats[2 * p] = red[0] / count;
    stats[2 * p + 1] = red[kSsimThreads] / count;
  }
}

// out[plane][oy][ox] = (the four taps of rows 2 oy - ph + {0, 1}, columns 2 ox - pw + {0, 1} inside the plane, row-major,
// summed from 0) / 4, ph = H mod 2, pw = W mod 2
__global__ void ssim_pool2_kernel(const double* __restrict__ in, double* __restrict__ out, size_t planes, int H, int W,
                                  int Ho, int Wo) {
  pdl_trigger();
  pdl_wait();
  const int ph = H % 2, pw = W % 2;
  const size_t total = planes * Ho * Wo;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % Wo), oy = static_cast<int>((i / Wo) % Ho);
    const double* pl = in + (i / (static_cast<size_t>(Wo) * Ho)) * (static_cast<size_t>(H) * W);
    double s = 0.0;
    for (int dy = 0; dy < 2; ++dy) {
      const int y = 2 * oy - ph + dy;
      if (y < 0 || y >= H) continue;
      for (int dx = 0; dx < 2; ++dx) {
        const int xx = 2 * ox - pw + dx;
        if (xx >= 0 && xx < W) s += pl[static_cast<size_t>(y) * W + xx];
      }
    }
    out[i] = s * 0.25;
  }
}

inline int grid_for(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

inline bool aligned(const void* p, size_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

// the largest element count of one tensor the kernels index (size_t, below 2^62 so that no offset wraps)
constexpr long long kMaxElems = 1LL << 62;

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_png_quantize(const float* x, uint8_t* q, double* lvl0, float* xq, int B, int H, int W,
                                 void* stream) {
  ASYRP_REQUIRE(B > 0 && H > 0 && W > 0, "asyrp_png_quantize: bad shape B=%d H=%d W=%d", B, H, W);
  ASYRP_REQUIRE(static_cast<long long>(B) * 3 * H <= kMaxElems / W, "asyrp_png_quantize: B * 3 * H * W too large");
  ASYRP_REQUIRE(x != nullptr && q != nullptr, "asyrp_png_quantize: null x or q");
  ASYRP_REQUIRE(aligned(x, 4) && aligned(lvl0, 8) && aligned(xq, 4),
                "asyrp_png_quantize: x / xq must be 4-byte and lvl0 8-byte aligned");
  const size_t total = static_cast<size_t>(B) * 3 * H * W;
  ASYRP_LAUNCH(png_quantize_kernel, dim3(grid_for(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), x, q,
               lvl0, xq, total);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_preserve_sse(const uint8_t* src, const uint8_t* edited, long long* sse, int n, int B,
                                 long long plane, void* stream) {
  ASYRP_REQUIRE(n > 0 && B > 0 && plane > 0, "asyrp_preserve_sse: bad shape n=%d B=%d plane=%lld", n, B, plane);
  // 65025 per element: below 2^63 for any plane up to 2^47 elements
  ASYRP_REQUIRE(plane <= (1LL << 47), "asyrp_preserve_sse: plane=%lld above 2^47 elements", plane);
  ASYRP_REQUIRE(static_cast<long long>(n > B ? n : B) <= kMaxElems / plane,
                "asyrp_preserve_sse: %d rows x %lld elements too large", n > B ? n : B, plane);
  ASYRP_REQUIRE(src != nullptr && edited != nullptr && sse != nullptr, "asyrp_preserve_sse: null buffer");
  ASYRP_REQUIRE(aligned(sse, 8), "asyrp_preserve_sse: sse must be 8-byte aligned");
  ASYRP_LAUNCH(preserve_sse_kernel, dim3(n), dim3(kSseThreads), 0, static_cast<cudaStream_t>(stream), src, edited,
               sse, B, static_cast<size_t>(plane));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_ssim_level(const double* src, const double* edited, double* stats, int n, int B, int H, int W,
                               void* stream) {
  ASYRP_REQUIRE(n > 0 && B > 0, "asyrp_ssim_level: bad shape n=%d B=%d", n, B);
  ASYRP_REQUIRE(H >= kWin && W >= kWin, "asyrp_ssim_level: H=%d W=%d below the %d x %d window", H, W, kWin, kWin);
  // the grid holds one CTA per plane; the tile count and the in-tile coordinates are int
  ASYRP_REQUIRE(3LL * n <= INT_MAX, "asyrp_ssim_level: 3 n=%lld planes above 2^31 - 1", 3LL * n);
  ASYRP_REQUIRE(H <= INT_MAX - kInY && W <= INT_MAX - kInX, "asyrp_ssim_level: H=%d or W=%d too large", H, W);
  ASYRP_REQUIRE(((H - 2LL * kRad + kTY - 1) / kTY) * ((W - 2LL * kRad + kTX - 1) / kTX) <= INT_MAX,
                "asyrp_ssim_level: too many tiles for H=%d W=%d", H, W);
  ASYRP_REQUIRE(3LL * (n > B ? n : B) * H <= kMaxElems / W, "asyrp_ssim_level: rows x 3 H W too large");
  ASYRP_REQUIRE(src != nullptr && edited != nullptr && stats != nullptr, "asyrp_ssim_level: null buffer");
  ASYRP_REQUIRE(aligned(src, 8) && aligned(edited, 8) && aligned(stats, 8),
                "asyrp_ssim_level: src, edited and stats must be 8-byte aligned");
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(ssim_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kSsimSmem)));
  ASYRP_LAUNCH(ssim_level_kernel, dim3(3 * n), dim3(kSsimThreads), kSsimSmem, static_cast<cudaStream_t>(stream), src,
               edited, stats, B, H, W, gaussian_window());
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_ssim_pool2(const double* in, double* out, int rows, int H, int W, void* stream) {
  ASYRP_REQUIRE(rows > 0 && H > 0 && W > 0, "asyrp_ssim_pool2: bad shape rows=%d H=%d W=%d", rows, H, W);
  ASYRP_REQUIRE(H < INT_MAX && W < INT_MAX, "asyrp_ssim_pool2: H=%d or W=%d too large", H, W);
  ASYRP_REQUIRE(3LL * rows * H <= kMaxElems / W, "asyrp_ssim_pool2: rows x 3 H W too large");
  ASYRP_REQUIRE(in != nullptr && out != nullptr && in != out, "asyrp_ssim_pool2: null or aliased buffers");
  ASYRP_REQUIRE(aligned(in, 8) && aligned(out, 8), "asyrp_ssim_pool2: in and out must be 8-byte aligned");
  const int Ho = H / 2 + H % 2, Wo = W / 2 + W % 2;
  const size_t planes = 3 * static_cast<size_t>(rows);
  ASYRP_LAUNCH(ssim_pool2_kernel, dim3(grid_for(planes * Ho * Wo, 256)), dim3(256), 0,
               static_cast<cudaStream_t>(stream), in, out, planes, H, W, Ho, Wo);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
