// Region-restricted edits: a soft mask per image from face-parsing labels, and the per-step blend of the edit pass
// back into the unedited trajectory outside it.
//
//   blend      x[n][c][p] = fmaf(m, x, (1 - m) * r),  m = mask[n % B][p], r = ref[n % B][c][p]   blend_rows_kernel{,4}
//   compose    rows n = k B + j of K attributes x B images: s = M_1 + .. + M_K (fp32, in order); w_k = M_k and
//              w_0 = 1 - s if s <= 1, else w_k = M_k / s and w_0 = 0; acc = w_0 r, then acc = fmaf(w_k, x[k B + j],
//              acc) for k = 1..K; acc is written to all K rows of image j           compose_rows_kernel{,4}<K>
//   select     mask[n][y][x] = 1 if a label of the footprint rows [ceil(y 512 / S), ceil((y + 1) 512 / S)) (columns
//              likewise) is in class_bits, else 0                                                  region_mask_kernel
//   dilate     out = max of in over [i - r, i + r] along one axis, indices outside the image left out  mask_dilate_kernel
//   blur       out = sum_{k=-R..R} taps[k + R] in[clamp(i + k)] along one axis, fp32 fmaf in tap order;
//              a window whose inputs are all equal returns that value                             mask_blur_kernel
//
// The blend and the compose are the hot paths: each runs once per step inside the trajectory graph over N * C * HW
// fp32.  With HW a multiple of 4 each thread moves one float4 of x, ref and mask; otherwise one element.  m = 1 gives
// x exactly and m = 0 gives r exactly (for finite x and r).  The compose computes its weights in registers from the K
// masks of a pixel, once for all C channels; with K = 1 it is the blend operation for operation.  Every kernel
// indexes in 64 bits where a count can pass 2^31.
#include <cstdint>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kRegionThreads = 256;
constexpr int kLabelSize = 512;      // the face parser's label maps are 512 x 512
constexpr int kMaxDilate = 32;
constexpr int kMaxBlurRadius = 48;   // ceil(3 sigma) for sigma <= 16
constexpr int kMaxComposeRows = 8;   // attributes of one composite: their masks stay in registers

__device__ __forceinline__ float blend1(float m, float x, float r) {
  return fmaf(m, x, __fmul_rn(__fsub_rn(1.f, m), r));
}

// one float4 of one (n, c) plane per thread: grid (ceil(HW / 4 / 256), planes), planes n * C + c strided by gridDim.y
__global__ void __launch_bounds__(kRegionThreads) blend_rows_kernel4(float4* __restrict__ x,
                                                                    const float4* __restrict__ ref,
                                                                    const float4* __restrict__ mask, int N, int B,
                                                                    int C, int HW4) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kRegionThreads + threadIdx.x;
  if (p >= HW4) return;
  for (long long plane = blockIdx.y; plane < static_cast<long long>(N) * C; plane += gridDim.y) {
    const int n = static_cast<int>(plane / C), c = static_cast<int>(plane % C), b = n % B;
    float4* xp = x + plane * HW4 + p;
    const float4 m = __ldg(mask + static_cast<long long>(b) * HW4 + p);
    const float4 r = __ldg(ref + (static_cast<long long>(b) * C + c) * HW4 + p);
    float4 v = *xp;
    v.x = blend1(m.x, v.x, r.x);
    v.y = blend1(m.y, v.y, r.y);
    v.z = blend1(m.z, v.z, r.z);
    v.w = blend1(m.w, v.w, r.w);
    *xp = v;
  }
}

__global__ void __launch_bounds__(kRegionThreads) blend_rows_kernel(float* __restrict__ x, const float* __restrict__ ref,
                                                                   const float* __restrict__ mask, int N, int B, int C,
                                                                   int HW) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kRegionThreads + threadIdx.x;
  if (p >= HW) return;
  for (long long plane = blockIdx.y; plane < static_cast<long long>(N) * C; plane += gridDim.y) {
    const int n = static_cast<int>(plane / C), c = static_cast<int>(plane % C), b = n % B;
    float* xp = x + plane * HW + p;
    *xp = blend1(__ldg(mask + static_cast<long long>(b) * HW + p), *xp,
                 __ldg(ref + (static_cast<long long>(b) * C + c) * HW + p));
  }
}

// compose: the K masks of one pixel -> the weights, in place (w[k] replaces m[k]); returns w0
template <int K>
__device__ __forceinline__ float compose_weights(float (&m)[K]) {
  float s = m[0];
#pragma unroll
  for (int k = 1; k < K; ++k) s = __fadd_rn(s, m[k]);
  if (s <= 1.f) return __fsub_rn(1.f, s);
#pragma unroll
  for (int k = 0; k < K; ++k) m[k] = __fdiv_rn(m[k], s);
  return 0.f;
}

// one float4 of pixels of image j per thread: grid (ceil(HW / 4 / 256), images j strided by gridDim.y).  The K mask
// float4s are loaded once, turned into weights, and reused for the C channels.
template <int K>
__global__ void __launch_bounds__(kRegionThreads) compose_rows_kernel4(float4* __restrict__ x,
                                                                      const float4* __restrict__ ref,
                                                                      const float4* __restrict__ masks, int B, int C,
                                                                      int HW4) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kRegionThreads + threadIdx.x;
  if (p >= HW4) return;
  for (int j = blockIdx.y; j < B; j += gridDim.y) {
    float mx[K], my[K], mz[K], mw[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float4 m = __ldg(masks + (static_cast<long long>(k) * B + j) * HW4 + p);
      mx[k] = m.x;
      my[k] = m.y;
      mz[k] = m.z;
      mw[k] = m.w;
    }
    const float w0x = compose_weights<K>(mx), w0y = compose_weights<K>(my), w0z = compose_weights<K>(mz),
                w0w = compose_weights<K>(mw);
    for (int c = 0; c < C; ++c) {
      const float4 r = __ldg(ref + (static_cast<long long>(j) * C + c) * HW4 + p);
      float4 acc = make_float4(__fmul_rn(w0x, r.x), __fmul_rn(w0y, r.y), __fmul_rn(w0z, r.z), __fmul_rn(w0w, r.w));
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float4 v = x[((static_cast<long long>(k) * B + j) * C + c) * HW4 + p];
        acc.x = fmaf(mx[k], v.x, acc.x);
        acc.y = fmaf(my[k], v.y, acc.y);
        acc.z = fmaf(mz[k], v.z, acc.z);
        acc.w = fmaf(mw[k], v.w, acc.w);
      }
#pragma unroll
      for (int k = 0; k < K; ++k) x[((static_cast<long long>(k) * B + j) * C + c) * HW4 + p] = acc;
    }
  }
}

template <int K>
__global__ void __launch_bounds__(kRegionThreads) compose_rows_kernel(float* __restrict__ x,
                                                                     const float* __restrict__ ref,
                                                                     const float* __restrict__ masks, int B, int C,
                                                                     int HW) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kRegionThreads + threadIdx.x;
  if (p >= HW) return;
  for (int j = blockIdx.y; j < B; j += gridDim.y) {
    float w[K];
#pragma unroll
    for (int k = 0; k < K; ++k) w[k] = __ldg(masks + (static_cast<long long>(k) * B + j) * HW + p);
    const float w0 = compose_weights<K>(w);
    for (int c = 0; c < C; ++c) {
      float acc = __fmul_rn(w0, __ldg(ref + (static_cast<long long>(j) * C + c) * HW + p));
#pragma unroll
      for (int k = 0; k < K; ++k) acc = fmaf(w[k], x[((static_cast<long long>(k) * B + j) * C + c) * HW + p], acc);
#pragma unroll
      for (int k = 0; k < K; ++k) x[((static_cast<long long>(k) * B + j) * C + c) * HW + p] = acc;
    }
  }
}

template <int K>
int launch_compose(float* x, const float* ref, const float* masks, int B, int C, int HW, bool vec, cudaStream_t st) {
  const int per = vec ? HW / 4 : HW;
  const dim3 grid((per + kRegionThreads - 1) / kRegionThreads, B < kMaxGridYZ ? B : kMaxGridYZ);
  if (vec) {
    ASYRP_LAUNCH(compose_rows_kernel4<K>, grid, dim3(kRegionThreads), 0, st, reinterpret_cast<float4*>(x),
                 reinterpret_cast<const float4*>(ref), reinterpret_cast<const float4*>(masks), B, C, per);
  } else {
    ASYRP_LAUNCH(compose_rows_kernel<K>, grid, dim3(kRegionThreads), 0, st, x, ref, masks, B, C, HW);
  }
  return ASYRP_OK;
}

// one output pixel per thread: grid (ceil(S^2 / 256), N)
__global__ void __launch_bounds__(kRegionThreads) region_mask_kernel(const unsigned char* __restrict__ labels,
                                                                    unsigned class_bits, float* __restrict__ mask,
                                                                    int S) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * kRegionThreads + threadIdx.x;
  if (i >= S * S) return;
  const int y = i / S, xo = i % S;
  const int y0 = (y * kLabelSize + S - 1) / S, y1 = ((y + 1) * kLabelSize + S - 1) / S;
  const int x0 = (xo * kLabelSize + S - 1) / S, x1 = ((xo + 1) * kLabelSize + S - 1) / S;
  const unsigned char* lab = labels + static_cast<size_t>(blockIdx.y) * kLabelSize * kLabelSize;
  bool hit = false;
  for (int yy = y0; yy < y1 && !hit; ++yy)
    for (int xx = x0; xx < x1; ++xx) {
      const unsigned l = lab[yy * kLabelSize + xx];
      if (l < 32 && ((class_bits >> l) & 1u)) {
        hit = true;
        break;
      }
    }
  mask[static_cast<size_t>(blockIdx.y) * S * S + i] = hit ? 1.f : 0.f;
}

// axis 0: along a row (x), axis 1: along a column (y)
__global__ void __launch_bounds__(kRegionThreads) mask_dilate_kernel(const float* __restrict__ in,
                                                                    float* __restrict__ out, int S, int r, int axis) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * kRegionThreads + threadIdx.x;
  if (i >= S * S) return;
  const int y = i / S, xo = i % S;
  const float* img = in + static_cast<size_t>(blockIdx.y) * S * S;
  const int pos = axis == 0 ? xo : y, stride = axis == 0 ? 1 : S;
  const float* line = img + (axis == 0 ? y * S : xo);
  const int lo = max(pos - r, 0), hi = min(pos + r, S - 1);
  float v = line[lo * stride];
  for (int k = lo + 1; k <= hi; ++k) v = fmaxf(v, line[k * stride]);
  out[static_cast<size_t>(blockIdx.y) * S * S + i] = v;
}

__global__ void __launch_bounds__(kRegionThreads) mask_blur_kernel(const float* __restrict__ in,
                                                                  const float* __restrict__ taps,
                                                                  float* __restrict__ out, int S, int R, int axis) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * kRegionThreads + threadIdx.x;
  if (i >= S * S) return;
  const int y = i / S, xo = i % S;
  const float* img = in + static_cast<size_t>(blockIdx.y) * S * S;
  const int pos = axis == 0 ? xo : y, stride = axis == 0 ? 1 : S;
  const float* line = img + (axis == 0 ? y * S : xo);
  const float first = line[min(max(pos - R, 0), S - 1) * stride];
  float acc = 0.f;
  bool flat = true;
  for (int k = -R; k <= R; ++k) {
    const float v = line[min(max(pos + k, 0), S - 1) * stride];
    flat = flat && v == first;
    acc = fmaf(__ldg(taps + k + R), v, acc);
  }
  out[static_cast<size_t>(blockIdx.y) * S * S + i] = flat ? first : acc;
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

int check_mask_args(const char* fn, const void* in, const float* out, int N, int S) {
  ASYRP_REQUIRE(in != nullptr && out != nullptr, "%s: in and out are required", fn);
  ASYRP_REQUIRE(N > 0 && N <= kMaxGridYZ, "%s: N=%d outside 1..%d", fn, N, kMaxGridYZ);
  ASYRP_REQUIRE(S > 0 && S <= kLabelSize, "%s: S=%d outside 1..%d", fn, S, kLabelSize);
  ASYRP_REQUIRE(aligned(out, 4), "%s: out is not 4-byte aligned", fn);
  return ASYRP_OK;
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_blend_rows(float* x, const float* ref, const float* mask, int N, int B, int C, int HW,
                               void* stream) {
  ASYRP_REQUIRE(x != nullptr && ref != nullptr && mask != nullptr, "asyrp_blend_rows: x, ref and mask are required");
  ASYRP_REQUIRE(N > 0 && B > 0 && C > 0 && HW > 0, "asyrp_blend_rows: bad shape N=%d B=%d C=%d HW=%d (all positive)",
                N, B, C, HW);
  ASYRP_REQUIRE(N % B == 0, "asyrp_blend_rows: N=%d is not a multiple of B=%d", N, B);
  const bool vec = HW % 4 == 0;
  const uintptr_t a = vec ? 16 : 4;
  ASYRP_REQUIRE(aligned(x, a) && aligned(ref, a) && aligned(mask, a),
                "asyrp_blend_rows: x, ref and mask must be %d-byte aligned (HW=%d)", static_cast<int>(a), HW);
  const int per = vec ? HW / 4 : HW;
  const unsigned gy = static_cast<unsigned>(
      static_cast<long long>(N) * C < kMaxGridYZ ? static_cast<long long>(N) * C : kMaxGridYZ);
  const dim3 grid((per + kRegionThreads - 1) / kRegionThreads, gy);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (vec) {
    ASYRP_LAUNCH(blend_rows_kernel4, grid, dim3(kRegionThreads), 0, st, reinterpret_cast<float4*>(x),
                 reinterpret_cast<const float4*>(ref), reinterpret_cast<const float4*>(mask), N, B, C, per);
  } else {
    ASYRP_LAUNCH(blend_rows_kernel, grid, dim3(kRegionThreads), 0, st, x, ref, mask, N, B, C, HW);
  }
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_compose_rows(float* x, const float* ref, const float* masks, int K, int B, int C, int HW,
                                 void* stream) {
  ASYRP_REQUIRE(x != nullptr && ref != nullptr && masks != nullptr,
                "asyrp_compose_rows: x, ref and masks are required");
  ASYRP_REQUIRE(K >= 1 && K <= kMaxComposeRows, "asyrp_compose_rows: K=%d outside 1..%d", K, kMaxComposeRows);
  ASYRP_REQUIRE(B > 0 && C > 0 && HW > 0, "asyrp_compose_rows: bad shape B=%d C=%d HW=%d (all positive)", B, C, HW);
  const bool vec = HW % 4 == 0;
  const uintptr_t a = vec ? 16 : 4;
  ASYRP_REQUIRE(aligned(x, a) && aligned(ref, a) && aligned(masks, a),
                "asyrp_compose_rows: x, ref and masks must be %d-byte aligned (HW=%d)", static_cast<int>(a), HW);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = ASYRP_OK;
  switch (K) {
    case 1: rc = launch_compose<1>(x, ref, masks, B, C, HW, vec, st); break;
    case 2: rc = launch_compose<2>(x, ref, masks, B, C, HW, vec, st); break;
    case 3: rc = launch_compose<3>(x, ref, masks, B, C, HW, vec, st); break;
    case 4: rc = launch_compose<4>(x, ref, masks, B, C, HW, vec, st); break;
    case 5: rc = launch_compose<5>(x, ref, masks, B, C, HW, vec, st); break;
    case 6: rc = launch_compose<6>(x, ref, masks, B, C, HW, vec, st); break;
    case 7: rc = launch_compose<7>(x, ref, masks, B, C, HW, vec, st); break;
    default: rc = launch_compose<8>(x, ref, masks, B, C, HW, vec, st); break;
  }
  if (rc != ASYRP_OK) return rc;
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_region_mask(const unsigned char* labels, unsigned class_bits, float* mask, int N, int S,
                                void* stream) {
  const int rc = check_mask_args("asyrp_region_mask", labels, mask, N, S);
  if (rc != ASYRP_OK) return rc;
  ASYRP_LAUNCH(region_mask_kernel, dim3((S * S + kRegionThreads - 1) / kRegionThreads, N), dim3(kRegionThreads), 0,
               static_cast<cudaStream_t>(stream), labels, class_bits, mask, S);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_mask_dilate(const float* in, float* out, int N, int S, int r, int axis, void* stream) {
  const int rc = check_mask_args("asyrp_mask_dilate", in, out, N, S);
  if (rc != ASYRP_OK) return rc;
  ASYRP_REQUIRE(aligned(in, 4) && in != out, "asyrp_mask_dilate: in must be 4-byte aligned and distinct from out");
  ASYRP_REQUIRE(r >= 0 && r <= kMaxDilate, "asyrp_mask_dilate: r=%d outside 0..%d", r, kMaxDilate);
  ASYRP_REQUIRE(axis == 0 || axis == 1, "asyrp_mask_dilate: axis=%d is not 0 or 1", axis);
  ASYRP_LAUNCH(mask_dilate_kernel, dim3((S * S + kRegionThreads - 1) / kRegionThreads, N), dim3(kRegionThreads), 0,
               static_cast<cudaStream_t>(stream), in, out, S, r, axis);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_mask_blur(const float* in, const float* taps, float* out, int N, int S, int R, int axis,
                              void* stream) {
  const int rc = check_mask_args("asyrp_mask_blur", in, out, N, S);
  if (rc != ASYRP_OK) return rc;
  ASYRP_REQUIRE(aligned(in, 4) && in != out, "asyrp_mask_blur: in must be 4-byte aligned and distinct from out");
  ASYRP_REQUIRE(taps != nullptr && aligned(taps, 4), "asyrp_mask_blur: taps are required, 4-byte aligned");
  ASYRP_REQUIRE(R >= 0 && R <= kMaxBlurRadius, "asyrp_mask_blur: R=%d outside 0..%d", R, kMaxBlurRadius);
  ASYRP_REQUIRE(axis == 0 || axis == 1, "asyrp_mask_blur: axis=%d is not 0 or 1", axis);
  ASYRP_LAUNCH(mask_blur_kernel, dim3((S * S + kRegionThreads - 1) / kRegionThreads, N), dim3(kRegionThreads), 0,
               static_cast<cudaStream_t>(stream), in, taps, out, S, R, axis);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
