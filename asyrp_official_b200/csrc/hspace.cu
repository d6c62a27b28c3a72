// Statistics of the UNet bottleneck h over many samples, for editing directions found without training.
//
//   G[i][j] = sum_k (x[i][k] - mu[k]) (x[j][k] - mu[k])          the centred sample Gram, fp64 [n][n]   h_gram_kernel
//   out[k][j] = sum_r w[k][r] (x[r][j] - mu[j])  (mu optional)     weighted column sums, fp64 [K][d]      h_combine_kernel
//
// The Gram is the dual of the d x d covariance: with d = C * 64 = 32768 or 65536 features and a few thousand samples,
// its eigenvectors u give the principal directions as X_c^T u (h_combine with w = u / sqrt(lambda)).  Every sum runs in
// fp64 over its index in order from 0 with one fma per term, so results do not depend on the launch, and G[i][j] and
// G[j][i] are the same bits.
#include <climits>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kHTile = 64;      // Gram tile: 64 x 64 outputs per CTA
constexpr int kHK = 16;         // feature slice staged in shared memory
constexpr int kHThreads = 256;  // each thread 4 x 4 outputs: rows ty + 16 a, columns tx + 16 b
constexpr int kCombK = 8;       // combine: weight rows per thread
constexpr int kCombThreads = 256;

// One 64 x 64 tile of G.  Staging: 16 consecutive features of 64 samples per slice, centred in fp64; features past d
// and samples past n stage as 0 (adding fma(0, 0, acc) leaves acc unchanged).
__global__ void __launch_bounds__(kHThreads) h_gram_kernel(const float* __restrict__ x, const double* __restrict__ mu,
                                                          double* __restrict__ G, int n, int d) {
  pdl_trigger();
  __shared__ double xs[kHK][kHTile];
  __shared__ double ys[kHK][kHTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kHTile, j0 = blockIdx.x * kHTile;
  pdl_wait();
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < d; k0 += kHK) {
#pragma unroll
    for (int q = 0; q < kHK * kHTile / kHThreads; ++q) {
      const int e = t + kHThreads * q;
      const int ii = e / kHK, kk = e % kHK, k = k0 + kk;
      const double m = k < d ? mu[k] : 0.0;
      xs[kk][ii] = i0 + ii < n && k < d ? static_cast<double>(x[static_cast<size_t>(i0 + ii) * d + k]) - m : 0.0;
      ys[kk][ii] = j0 + ii < n && k < d ? static_cast<double>(x[static_cast<size_t>(j0 + ii) * d + k]) - m : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kHK; ++kk) {
      double xa[4], yb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xa[a] = xs[kk][ty + 16 * a];
#pragma unroll
      for (int b = 0; b < 4; ++b) yb[b] = ys[kk][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(xa[a], yb[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
      if (i < n && j < n) G[static_cast<size_t>(i) * n + j] = acc[a][b];
    }
}

// out[k][j] for one column j per thread and up to kCombK weight rows k = blockIdx.y * kCombK + kk; the rows r in
// order from 0, acc = fma(w[k][r], x[r][j] - mu[j], acc).  x is read coalesced along j; w[k][r] is one broadcast load.
__global__ void __launch_bounds__(kCombThreads) h_combine_kernel(const float* __restrict__ x,
                                                                const double* __restrict__ w,
                                                                const double* __restrict__ mu, double* __restrict__ out,
                                                                int n, int d, int K) {
  pdl_trigger();
  pdl_wait();
  const int j = blockIdx.x * kCombThreads + threadIdx.x;
  if (j >= d) return;
  const int k0 = blockIdx.y * kCombK;
  const int kn = min(kCombK, K - k0);
  const double m = mu != nullptr ? mu[j] : 0.0;
  double acc[kCombK];
#pragma unroll
  for (int kk = 0; kk < kCombK; ++kk) acc[kk] = 0.0;
  for (int r = 0; r < n; ++r) {
    const double v = static_cast<double>(x[static_cast<size_t>(r) * d + j]) - m;
#pragma unroll
    for (int kk = 0; kk < kCombK; ++kk)
      if (kk < kn) acc[kk] = fma(w[static_cast<size_t>(k0 + kk) * n + r], v, acc[kk]);
  }
#pragma unroll
  for (int kk = 0; kk < kCombK; ++kk)
    if (kk < kn) out[static_cast<size_t>(k0 + kk) * d + j] = acc[kk];
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_h_gram(const float* x, const double* mu, double* G, int n, int d, void* stream) {
  ASYRP_REQUIRE(n >= 2 && d > 0, "asyrp_h_gram: bad shape n=%d d=%d (n >= 2, d > 0)", n, d);
  // the element index r * d + k is formed in size_t, but the staging loop steps k by 16 in int and one call is
  // limited to fewer than 2^31 elements like the other row kernels
  ASYRP_REQUIRE(static_cast<long long>(n) * d < (1LL << 31), "asyrp_h_gram: n * d = %lld not below 2^31",
                static_cast<long long>(n) * d);
  ASYRP_REQUIRE(d <= INT_MAX - kHK + 1, "asyrp_h_gram: d=%d above %d", d, INT_MAX - kHK + 1);
  ASYRP_REQUIRE(x != nullptr && mu != nullptr && G != nullptr, "asyrp_h_gram: x, mu and G are required");
  const unsigned tiles = static_cast<unsigned>((static_cast<long long>(n) + kHTile - 1) / kHTile);
  ASYRP_REQUIRE(tiles <= static_cast<unsigned>(kMaxGridYZ), "asyrp_h_gram: n=%d above %d rows", n,
                kMaxGridYZ * kHTile);
  ASYRP_LAUNCH(h_gram_kernel, dim3(tiles, tiles), dim3(kHThreads), 0, static_cast<cudaStream_t>(stream), x, mu, G, n,
               d);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_h_combine(const float* x, const double* w, const double* mu, double* out, int n, int d, int K,
                              void* stream) {
  ASYRP_REQUIRE(n > 0 && d > 0 && K > 0, "asyrp_h_combine: bad shape n=%d d=%d K=%d (all positive)", n, d, K);
  ASYRP_REQUIRE(static_cast<long long>(n) * d < (1LL << 31), "asyrp_h_combine: n * d = %lld not below 2^31",
                static_cast<long long>(n) * d);
  ASYRP_REQUIRE(static_cast<long long>(K) * n < (1LL << 31) && static_cast<long long>(K) * d < (1LL << 31),
                "asyrp_h_combine: K * n = %lld or K * d = %lld not below 2^31", static_cast<long long>(K) * n,
                static_cast<long long>(K) * d);
  ASYRP_REQUIRE(d <= INT_MAX - kCombThreads + 1, "asyrp_h_combine: d=%d above %d", d, INT_MAX - kCombThreads + 1);
  ASYRP_REQUIRE(x != nullptr && w != nullptr && out != nullptr, "asyrp_h_combine: x, w and out are required");
  const long long kb = (static_cast<long long>(K) + kCombK - 1) / kCombK;
  ASYRP_REQUIRE(kb <= kMaxGridYZ, "asyrp_h_combine: K=%d above %d weight rows", K, kMaxGridYZ * kCombK);
  ASYRP_LAUNCH(h_combine_kernel, dim3((d + kCombThreads - 1) / kCombThreads, static_cast<unsigned>(kb)),
               dim3(kCombThreads), 0, static_cast<cudaStream_t>(stream), x, w, mu, out, n, d, K);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
