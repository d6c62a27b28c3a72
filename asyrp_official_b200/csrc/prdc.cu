// k-nearest-neighbour balls of feature sets for improved precision / recall (Kynkaanniemi et al. 2019) and density /
// coverage (Naeem et al. 2020), without materialising the distance matrix.
//
//   D(u, v) = sum_c (u_c - v_c)^2 over the d features, each difference and the sum in fp64, the sum in feature order
//     from 0 (one fma per feature), so identical rows give exactly 0 and a pair's D does not depend on the launch
//   r_k(i) = the (k + 1)-th smallest D(x_i, x_j) over every row j of x, j = i included      knn_tile_kernel, knn_merge
//   per pair of a [n][d] and b [m][d]: D < ra[i], D < rb[j] counted per row of a and of b    knn_counts_kernel
//
// A CTA computes a 64 x 64 tile of D exactly as fid_gram_kernel computes its gram tile (16 features staged in shared
// memory, 4 x 4 outputs per thread), with the feature index bounds-checked so that any d works.  The radii keep a
// sorted list of the k + 1 smallest values of each row in shared memory; a row's columns may be split over several CTAs,
// whose lists a second kernel merges.  The (k + 1)-th smallest value of a multiset does not depend on the order its
// members arrive in, so the radii are the same bits for any split.  The counts are integer atomics, so they are exact.
#include <cmath>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kTile = 64;      // 64 x 64 distances per CTA
constexpr int kSlice = 16;     // features staged in shared memory per step
constexpr int kThreads = 256;  // each thread 4 x 4 distances: rows ty + 16 a, columns tx + 16 b
constexpr int kMaxK = 32;
// row pitch in doubles of the staging slices and the distance tile: with 65, the staging stores (16 features of two
// rows per warp) and the distance tile's row-wise reads hit distinct banks; with 64 both would be 16-way conflicts
constexpr int kPitch = kTile + 1;
constexpr int kMergeThreads = 64;

// acc[a][b] = D(x[i0 + ty + 16 a], y[j0 + tx + 16 b]) for the rows below n and the columns below m (0 elsewhere)
__device__ __forceinline__ void distance_tile(const float* __restrict__ x, const float* __restrict__ y, int n, int m,
                                              int d, int i0, int j0, double (*xs)[kPitch], double (*ys)[kPitch],
                                              double (&acc)[4][4]) {
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < d; k0 += kSlice) {
#pragma unroll
    for (int q = 0; q < kSlice * kTile / kThreads; ++q) {  // 16 consecutive features of 64 rows
      const int e = t + kThreads * q, ii = e / kSlice, kk = e % kSlice, k = k0 + kk;
      const bool kin = k < d;
      xs[kk][ii] = kin && i0 + ii < n ? static_cast<double>(x[static_cast<size_t>(i0 + ii) * d + k]) : 0.0;
      ys[kk][ii] = kin && j0 + ii < m ? static_cast<double>(y[static_cast<size_t>(j0 + ii) * d + k]) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kSlice; ++kk) {
      double xa[4], yb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) xa[a] = xs[kk][ty + 16 * a];
#pragma unroll
      for (int b = 0; b < 4; ++b) yb[b] = ys[kk][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const double diff = xa[a] - yb[b];
          acc[a][b] = fma(diff, diff, acc[a][b]);
        }
    }
    __syncthreads();
  }
}

// Insert v into the ascending list list[0], list[stride], ..., list[(len - 1) stride] of the len smallest values seen,
// dropping the largest; a v not below the largest leaves the list as it is (its (len)-th value would not change).
__device__ __forceinline__ void list_insert(double* list, int stride, int len, double v) {
  if (!(v < list[(len - 1) * stride])) return;
  int s = len - 1;
  for (; s > 0 && list[(s - 1) * stride] > v; --s) list[s * stride] = list[(s - 1) * stride];
  list[s * stride] = v;
}

// Row block blockIdx.x (64 rows of x), column part blockIdx.y of `parts`: the column tiles
// [p * tiles / parts, (p + 1) * tiles / parts).  Writes the ascending k + 1 smallest D of each row over the part's
// columns (+inf past the part's column count) to work[p][row][0 .. k].
// Dynamic shared memory: the staging slices, the 64 x kPitch distance tile and the lists [k + 1][64].
__global__ void __launch_bounds__(kThreads) knn_tile_kernel(const float* __restrict__ x, double* __restrict__ work,
                                                            int n, int d, int kp1, int parts) {
  pdl_trigger();
  extern __shared__ double smem[];
  double(*xs)[kPitch] = reinterpret_cast<double(*)[kPitch]>(smem);
  double(*ys)[kPitch] = reinterpret_cast<double(*)[kPitch]>(smem + kSlice * kPitch);
  double* dt = smem + 2 * kSlice * kPitch;
  double* list = dt + kTile * kPitch;
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.x * kTile, tiles = (n + kTile - 1) / kTile, p = blockIdx.y;
  const int first = static_cast<int>(static_cast<long long>(p) * tiles / parts);
  const int last = static_cast<int>(static_cast<long long>(p + 1) * tiles / parts);
  for (int s = t; s < kp1 * kTile; s += kThreads) list[s] = INFINITY;
  pdl_wait();
  for (int jt = first; jt < last; ++jt) {
    const int j0 = jt * kTile;
    double acc[4][4];
    distance_tile(x, x, n, n, d, i0, j0, xs, ys, acc);
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) dt[(ty + 16 * a) * kPitch + tx + 16 * b] = acc[a][b];
    __syncthreads();
    if (t < kTile) {
      const int cols = min(kTile, n - j0);
      for (int c = 0; c < cols; ++c) list_insert(list + t, kTile, kp1, dt[t * kPitch + c]);
    }
    __syncthreads();
  }
  if (t < kTile && i0 + t < n) {
    double* out = work + (static_cast<size_t>(p) * n + i0 + t) * kp1;
    for (int s = 0; s < kp1; ++s) out[s] = list[s * kTile + t];
  }
}

// radii[i] = the kp1-th smallest of the parts' lists of row i (work[p][i][0 .. kp1), each ascending)
__global__ void __launch_bounds__(kMergeThreads) knn_merge_kernel(const double* __restrict__ work,
                                                                  double* __restrict__ radii, int n, int kp1,
                                                                  int parts) {
  pdl_trigger();
  __shared__ double list[(kMaxK + 1) * kMergeThreads];
  const int t = threadIdx.x, i = blockIdx.x * kMergeThreads + t;
  for (int s = 0; s < kp1; ++s) list[s * kMergeThreads + t] = INFINITY;
  pdl_wait();
  if (i >= n) return;
  for (int p = 0; p < parts; ++p) {
    const double* in = work + (static_cast<size_t>(p) * n + i) * kp1;
    for (int s = 0; s < kp1; ++s) {
      const double v = in[s];
      if (!(v < list[(kp1 - 1) * kMergeThreads + t])) break;  // the rest of this ascending list is no smaller
      list_insert(list + t, kMergeThreads, kp1, v);
    }
  }
  radii[i] = list[(kp1 - 1) * kMergeThreads + t];
}

// Tile (blockIdx.y: 64 rows of a, blockIdx.x: 64 rows of b): adds to b_in_a[j] #{i : D < ra[i]}, to a_in_b[i]
// #{j : D < rb[j]} and to a_covered[i] #{j : D < ra[i]} over the tile's pairs (one atomic per row / column and output)
__global__ void __launch_bounds__(kThreads) knn_counts_kernel(const float* __restrict__ a,
                                                              const double* __restrict__ ra, int n,
                                                              const float* __restrict__ b,
                                                              const double* __restrict__ rb, int m, int d,
                                                              unsigned* __restrict__ b_in_a,
                                                              unsigned* __restrict__ a_in_b,
                                                              unsigned* __restrict__ a_covered) {
  pdl_trigger();
  __shared__ double xs[kSlice][kPitch];
  __shared__ double ys[kSlice][kPitch];
  __shared__ unsigned col_in[kTile], row_in[kTile], row_cov[kTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kTile, j0 = blockIdx.x * kTile;
  if (t < kTile) col_in[t] = row_in[t] = row_cov[t] = 0u;
  pdl_wait();
  double acc[4][4];
  distance_tile(a, b, n, m, d, i0, j0, xs, ys, acc);
  double rai[4], rbj[4];
  unsigned colv[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + ty + 16 * q, j = j0 + tx + 16 * q;
    // no D is below -inf: rows past n add nothing to b_in_a, columns past m nothing to a_in_b; colv keeps columns past
    // m out of a_covered.  The counts of rows and columns past the sets are never stored.
    rai[q] = i < n ? ra[i] : -INFINITY;
    rbj[q] = j < m ? rb[j] : -INFINITY;
    colv[q] = j < m;
  }
  unsigned rin[4] = {0u, 0u, 0u, 0u}, rcov[4] = {0u, 0u, 0u, 0u}, cin[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const unsigned in_a = acc[p][q] < rai[p];
      rcov[p] += in_a & colv[q];
      cin[q] += in_a;
      rin[p] += acc[p][q] < rbj[q];
    }
#pragma unroll
  for (int q = 0; q < 4; ++q) {  // the 16 threads of a half warp share rows ty + 16 q
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      rin[q] += __shfl_xor_sync(0xffffffffu, rin[q], o);
      rcov[q] += __shfl_xor_sync(0xffffffffu, rcov[q], o);
    }
  }
  if (tx == 0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      row_in[ty + 16 * q] = rin[q];
      row_cov[ty + 16 * q] = rcov[q];
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
    if (cin[q]) atomicAdd(&col_in[tx + 16 * q], cin[q]);
  __syncthreads();
  if (t < kTile) {
    if (j0 + t < m && col_in[t]) atomicAdd(&b_in_a[j0 + t], col_in[t]);
    if (i0 + t < n && row_in[t]) atomicAdd(&a_in_b[i0 + t], row_in[t]);
    if (i0 + t < n && row_cov[t]) atomicAdd(&a_covered[i0 + t], row_cov[t]);
  }
}

inline size_t knn_tile_smem(int kp1) {
  return sizeof(double) * (2 * kSlice * kPitch + kTile * kPitch + static_cast<size_t>(kp1) * kTile);
}

// column parts per row block, at most one per column tile: about 16 CTAs per SM, so that with three resident per SM
// the last of the five or more waves is short (at n = 30000 a single part would be 1.2 waves of 469 CTAs)
inline int knn_parts(int n) {
  const int tiles = (n + kTile - 1) / kTile;
  const int want = 16 * (sm_count() > 0 ? sm_count() : 132);
  const int parts = (want + tiles - 1) / tiles;
  return parts < tiles ? parts : tiles;
}

inline bool aligned(const void* p, size_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API long long asyrp_fid_knn_radii_workspace(int n, int k) {
  if (n < 1 || k < 1 || k > kMaxK) return -1;
  return static_cast<long long>(knn_parts(n)) * n * (k + 1);
}

ASYRP_API int asyrp_fid_knn_radii(const float* x, double* radii, double* work, int n, int d, int k, void* stream) {
  ASYRP_REQUIRE(k >= 1 && k <= kMaxK, "asyrp_fid_knn_radii: k=%d not in 1..%d", k, kMaxK);
  ASYRP_REQUIRE(n >= k + 1, "asyrp_fid_knn_radii: n=%d rows, needs at least k + 1 = %d", n, k + 1);
  ASYRP_REQUIRE(d >= 1, "asyrp_fid_knn_radii: d=%d must be positive", d);
  ASYRP_REQUIRE(x != nullptr && radii != nullptr && work != nullptr, "asyrp_fid_knn_radii: null buffer");
  ASYRP_REQUIRE(aligned(x, 4) && aligned(radii, 8) && aligned(work, 8),
                "asyrp_fid_knn_radii: x must be 4-byte and radii / work 8-byte aligned");
  ASYRP_REQUIRE(static_cast<void*>(radii) != static_cast<void*>(work), "asyrp_fid_knn_radii: radii must not alias work");
  const int parts = knn_parts(n), kp1 = k + 1;
  const size_t smem = knn_tile_smem(kp1);
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(knn_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(knn_tile_smem(kMaxK + 1))));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ASYRP_LAUNCH(knn_tile_kernel, dim3((n + kTile - 1) / kTile, parts), dim3(kThreads), smem, st, x, work, n, d, kp1,
               parts);
  ASYRP_LAUNCH(knn_merge_kernel, dim3((n + kMergeThreads - 1) / kMergeThreads), dim3(kMergeThreads), 0, st,
               static_cast<const double*>(work), radii, n, kp1, parts);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_knn_counts(const float* a, const double* ra, int n, const float* b, const double* rb, int m,
                                   int d, unsigned* b_in_a, unsigned* a_in_b, unsigned* a_covered, void* stream) {
  ASYRP_REQUIRE(n >= 1 && m >= 1 && d >= 1, "asyrp_fid_knn_counts: bad shape n=%d m=%d d=%d", n, m, d);
  ASYRP_REQUIRE(n <= kMaxGridYZ * kTile, "asyrp_fid_knn_counts: n=%d above %d rows", n, kMaxGridYZ * kTile);
  ASYRP_REQUIRE(a != nullptr && ra != nullptr && b != nullptr && rb != nullptr && b_in_a != nullptr &&
                    a_in_b != nullptr && a_covered != nullptr,
                "asyrp_fid_knn_counts: null buffer");
  ASYRP_REQUIRE(aligned(a, 4) && aligned(b, 4) && aligned(ra, 8) && aligned(rb, 8) && aligned(b_in_a, 4) &&
                    aligned(a_in_b, 4) && aligned(a_covered, 4),
                "asyrp_fid_knn_counts: a / b / counts must be 4-byte and ra / rb 8-byte aligned");
  ASYRP_REQUIRE(b_in_a != a_in_b && b_in_a != a_covered && a_in_b != a_covered,
                "asyrp_fid_knn_counts: b_in_a, a_in_b and a_covered must be distinct buffers");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ASYRP_CHECK_CUDA(cudaMemsetAsync(b_in_a, 0, sizeof(unsigned) * m, st));
  ASYRP_CHECK_CUDA(cudaMemsetAsync(a_in_b, 0, sizeof(unsigned) * n, st));
  ASYRP_CHECK_CUDA(cudaMemsetAsync(a_covered, 0, sizeof(unsigned) * n, st));
  ASYRP_LAUNCH(knn_counts_kernel, dim3((m + kTile - 1) / kTile, (n + kTile - 1) / kTile), dim3(kThreads), 0, st, a,
               ra, n, b, rb, m, d, b_in_a, a_in_b, a_covered);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
