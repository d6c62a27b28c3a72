// Exact inversion: the DDIM update of an edit pass anchored to the recorded DDIM inversion of its input images.
//
//   anchored   y  = Phi(x, em, et)                    the DDIM update of ddim_update_kernel without the c1 z term
//              yr = Phi(A_cur[b], E_cur[b], E_cur[b])  the same operations on the anchor of image b = n % B
//              x_next = A_next[b] + (y - yr)           __fsub_rn, then __fadd_rn
//   with Phi(x, m, e) = sqrt(an) x0 + c2 e, x0 = (x - m sqrt(1 - at)) / sqrt(at), in ddim_update_kernel's order.
//
// A row that does not edit reads x = A_cur and em = et = E_cur, so y and yr are the same bits and x_next is A_next
// exactly.  Stochastic steps keep their c2 in both terms and draw no noise: the same c1 z in y and yr would cancel.
// c2 is a scalar, or per row from c12 [N][2] (the c2 column; c1 is not read).  x0_out, when given, receives the edit's
// x0.  This replaces ddim_update / ddim_update_rows one for one in an anchored trajectory and reads six tensors where
// they read three.  With HW a multiple of 4 each thread moves one float4 of every tensor; otherwise one element.
// 64-bit offsets throughout.
#include <cstdint>

#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace {

constexpr int kAnchorThreads = 256;

struct Coef {
  float sq1, sqa, sqn;
};

// ddim_update_kernel's operations: x0 = (x - m sq1) / sqa; sqn x0 + c2 e
__device__ __forceinline__ float phi(const Coef& k, float c2, float x, float m, float e) {
  const float x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(m, k.sq1)), k.sqa);
  return __fadd_rn(__fmul_rn(k.sqn, x0), __fmul_rn(c2, e));
}

__device__ __forceinline__ float anchored1(const Coef& k, float c2, float x, float e, float m, float a, float an,
                                           float ea, float* x0) {
  *x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(m, k.sq1)), k.sqa);
  const float y = __fadd_rn(__fmul_rn(k.sqn, *x0), __fmul_rn(c2, e));
  return __fadd_rn(an, __fsub_rn(y, phi(k, c2, a, ea, ea)));
}

// one float4 of one (n, c) plane per thread: grid (ceil(HW / 4 / 256), planes), planes n * Cx + c strided by gridDim.y
__global__ void __launch_bounds__(kAnchorThreads) anchored_kernel4(const float4* x, const float4* __restrict__ et,
                                                                  const float4* __restrict__ em,
                                                                  const float4* __restrict__ a_cur,
                                                                  const float4* __restrict__ a_next,
                                                                  const float4* __restrict__ e_cur, float4* x_next,
                                                                  float4* __restrict__ x0_out, int N, int B, int Cx,
                                                                  int Ce, int HW4, float at, float an, float c2,
                                                                  const float* __restrict__ c12) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kAnchorThreads + threadIdx.x;
  if (p >= HW4) return;
  const Coef k{sqrtf(1.0f - at), sqrtf(at), sqrtf(an)};
  for (long long plane = blockIdx.y; plane < static_cast<long long>(N) * Cx; plane += gridDim.y) {
    const int n = static_cast<int>(plane / Cx), c = static_cast<int>(plane % Cx), b = n % B;
    const float cc = c12 != nullptr ? c12[2 * n + 1] : c2;
    const long long xi = plane * HW4 + p;
    const long long ei = (static_cast<long long>(n) * Ce + c) * HW4 + p;
    const long long ai = (static_cast<long long>(b) * Cx + c) * HW4 + p;
    const float4 xv = x[xi], e = __ldg(et + ei), m = __ldg(em + ei);
    const float4 a = __ldg(a_cur + ai), na = __ldg(a_next + ai), ea = __ldg(e_cur + ai);
    float4 o, x0;
    o.x = anchored1(k, cc, xv.x, e.x, m.x, a.x, na.x, ea.x, &x0.x);
    o.y = anchored1(k, cc, xv.y, e.y, m.y, a.y, na.y, ea.y, &x0.y);
    o.z = anchored1(k, cc, xv.z, e.z, m.z, a.z, na.z, ea.z, &x0.z);
    o.w = anchored1(k, cc, xv.w, e.w, m.w, a.w, na.w, ea.w, &x0.w);
    x_next[xi] = o;
    if (x0_out != nullptr) x0_out[xi] = x0;
  }
}

__global__ void __launch_bounds__(kAnchorThreads) anchored_kernel(const float* x, const float* __restrict__ et,
                                                                 const float* __restrict__ em,
                                                                 const float* __restrict__ a_cur,
                                                                 const float* __restrict__ a_next,
                                                                 const float* __restrict__ e_cur, float* x_next,
                                                                 float* __restrict__ x0_out, int N, int B, int Cx,
                                                                 int Ce, int HW, float at, float an, float c2,
                                                                 const float* __restrict__ c12) {
  pdl_trigger();
  pdl_wait();
  const int p = blockIdx.x * kAnchorThreads + threadIdx.x;
  if (p >= HW) return;
  const Coef k{sqrtf(1.0f - at), sqrtf(at), sqrtf(an)};
  for (long long plane = blockIdx.y; plane < static_cast<long long>(N) * Cx; plane += gridDim.y) {
    const int n = static_cast<int>(plane / Cx), c = static_cast<int>(plane % Cx), b = n % B;
    const float cc = c12 != nullptr ? c12[2 * n + 1] : c2;
    const long long xi = plane * HW + p;
    const long long ei = (static_cast<long long>(n) * Ce + c) * HW + p;
    const long long ai = (static_cast<long long>(b) * Cx + c) * HW + p;
    float x0;
    const float o = anchored1(k, cc, x[xi], __ldg(et + ei), __ldg(em + ei), __ldg(a_cur + ai), __ldg(a_next + ai),
                              __ldg(e_cur + ai), &x0);
    x_next[xi] = o;
    if (x0_out != nullptr) x0_out[xi] = x0;
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_ddim_update_anchored(const float* x, const float* et, const float* em, const float* a_cur,
                                         const float* a_next, const float* e_cur, float* x_next, float* x0_out, int N,
                                         int B, int Cx, int Ce, int HW, float at, float an, float c2, const float* c12,
                                         void* stream) {
  ASYRP_REQUIRE(x != nullptr && et != nullptr && em != nullptr && a_cur != nullptr && a_next != nullptr &&
                    e_cur != nullptr && x_next != nullptr,
                "asyrp_ddim_update_anchored: x, et, em, A_cur, A_next, E_cur and x_next are required");
  ASYRP_REQUIRE(N > 0 && B > 0 && Cx > 0 && Ce > 0 && HW > 0,
                "asyrp_ddim_update_anchored: bad shape N=%d B=%d Cx=%d Ce=%d HW=%d (all positive)", N, B, Cx, Ce, HW);
  ASYRP_REQUIRE(N % B == 0, "asyrp_ddim_update_anchored: N=%d is not a multiple of B=%d", N, B);
  ASYRP_REQUIRE(Ce >= Cx, "asyrp_ddim_update_anchored: Ce=%d below Cx=%d", Ce, Cx);
  const bool vec = HW % 4 == 0;
  const uintptr_t a = vec ? 16 : 4;
  ASYRP_REQUIRE(aligned(x, a) && aligned(et, a) && aligned(em, a) && aligned(a_cur, a) && aligned(a_next, a) &&
                    aligned(e_cur, a) && aligned(x_next, a) && (x0_out == nullptr || aligned(x0_out, a)),
                "asyrp_ddim_update_anchored: every tensor must be %d-byte aligned (HW=%d)", static_cast<int>(a), HW);
  ASYRP_REQUIRE(c12 == nullptr || aligned(c12, 4), "asyrp_ddim_update_anchored: c12 must be 4-byte aligned");
  const int per = vec ? HW / 4 : HW;
  const unsigned gy = static_cast<unsigned>(
      static_cast<long long>(N) * Cx < kMaxGridYZ ? static_cast<long long>(N) * Cx : kMaxGridYZ);
  const dim3 grid((per + kAnchorThreads - 1) / kAnchorThreads, gy);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (vec) {
    ASYRP_LAUNCH(anchored_kernel4, grid, dim3(kAnchorThreads), 0, st, reinterpret_cast<const float4*>(x),
                 reinterpret_cast<const float4*>(et), reinterpret_cast<const float4*>(em),
                 reinterpret_cast<const float4*>(a_cur), reinterpret_cast<const float4*>(a_next),
                 reinterpret_cast<const float4*>(e_cur), reinterpret_cast<float4*>(x_next),
                 reinterpret_cast<float4*>(x0_out), N, B, Cx, Ce, per, at, an, c2, c12);
  } else {
    ASYRP_LAUNCH(anchored_kernel, grid, dim3(kAnchorThreads), 0, st, x, et, em, a_cur, a_next, e_cur, x_next, x0_out,
                 N, B, Cx, Ce, HW, at, an, c2, c12);
  }
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
