// Thin inline-PTX wrappers for the sm_90a features the Asyrp kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait), proxy fences.
// Only what the kernels in this directory need; everything is __device__ __forceinline__.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace asyrp {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// Warp index as a value the compiler can prove warp-uniform (so role branches are uniform branches and everything
// computed inside them from uniform inputs lives in uniform registers).
__device__ __forceinline__ int uniform_warp_id() { return __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0); }

// elect.sync: true in exactly one lane of a converged warp.  The single-thread TMA instructions take uniform-register
// operands: issued from warp-uniform control flow under this predicate they compile to a plain predicated
// instruction; issued from an `if (lane == 0)` branch the compiler wraps every one of them in a vote / R2UR /
// BRA.U.ANY "waterfall" loop.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// explicit shared-state-space 16-byte accesses on a 32-bit shared address (a generic pointer costs an S2R + LEA
// address-space conversion per access inside hot loops)
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// try_wait with a suspend-time hint (ns): the waiting thread may stay suspended until the phase completes instead
// of re-issuing the poll every ~14 cycles (three issue slots each, taken from the epilogue warps of the same SMSP).
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_suspend(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait_hint(bar, parity, 20000u)) {
  }
}

// ---------------------------------------------------------------- proxy fences
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, sm_90a)
// D[64 x N registers of the warpgroup] (+)= A[smem desc, 64 x 16] * B[smem desc, N x 16]^T, fp16 operands (both
// K-major), fp32 accumulators.  Accumulator fragment of thread t (warp w = t/32 of the warpgroup, lane l):
// d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e].
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across wgmma_fence / wgmma_wait
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_f16_n16(float (&d)[8], uint64_t desc_a, uint64_t desc_b,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (rows of 128 B, 8-row atoms).
// Field layout follows the PTX ISA "matrix descriptor format": start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// base_offset [49,52) (0: every operand stage is 1024B-aligned), layout_type [62,64) (1 = SWIZZLE_128B).
// sbo_bytes: distance between consecutive 8-row groups (1024 for a dense tile; (TW+2)*128 when the rows are the
// pixels of a halo tile whose image rows are TW+2 pixels apart).  The 128B swizzle is a function of the shared
// memory ADDRESS bits (chunk ^= (addr >> 7) & 7), so start addresses need only be 16B-aligned as long as the data
// was written with the same address-based pattern (TMA does, given a 1024B-aligned box base).
// lo word = start address field (+ LBO), hi word = SBO / swizzle mode: the K loop only ever changes lo.
__device__ __forceinline__ uint32_t gmma_desc_lo(uint32_t smem_addr) {
  return ((smem_addr & 0x3FFFF) >> 4) | (1u << 16);
}
__device__ __forceinline__ uint32_t gmma_desc_hi(uint32_t sbo_bytes) { return (sbo_bytes >> 4) | (1u << 30); }
__device__ __forceinline__ uint64_t gmma_desc(uint32_t lo, uint32_t hi) {
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

// ---------------------------------------------------------------- programmatic dependent launch
// launch_dependents: the next kernel in the stream may be scheduled once every CTA of this grid has executed it;
// wait: block until the preceding grid has completed and its memory operations are visible (no-op without PDL).
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- per-warpgroup register budget
// setmaxnreg: every warp of a warpgroup executes the same instruction.  dec returns registers above N to the CTA's
// pool; inc blocks until the pool (what the launch allocated, minus what other warpgroups hold) can raise this
// warpgroup to N.  N is a multiple of 8 in [24, 256]; ptxas allocates the code that follows under the new limit.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }
// branch-free SiLU on the SFU: x * rcp(1 + 2^(-x*log2e)); relative error ~2^-21 (the result is rounded to fp16).
// x -> -inf gives x*0 = -0, x -> +inf gives x*1.
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// SiLU from ONE special-function op: with h = x/2, x*sigmoid(x) = h + h*tanh(h).  tanh.approx.f32 carries 11 bits
// (max relative error 2^-11): the error is <= 2^-12 |x|, absolute in |x| and not relative to the result, so in the
// negative tail it is far above the result's fp16 rounding (x = -6: up to 1.5e-3 on silu = -0.0148).  Takes h, not x:
// callers fold the 1/2 into the affine that precedes the activation.
__device__ __forceinline__ float silu_tanh_half(float h) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

}  // namespace asyrp
