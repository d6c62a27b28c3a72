// Micro-benchmark: TMA ingest rate per SM (bytes/clk) for (a) all CTAs streaming the same matrix (weights),
// (b) every CTA its own rows (activations, L2-resident), (c) as (a) with cluster-of-2 multicast halves.
// Build + run: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/probe_tma scripts/probe_tma.cu && /tmp/probe_tma
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdint>
#include <vector>
#include <algorithm>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); return 1; } } while (0)

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* b, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(s32(b)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(ra) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t ph) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(s32(b)), "r"(ph) : "memory");
  }
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* b, uint32_t ph) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(s32(b)), "r"(ph) : "memory");
  }
}
__device__ __forceinline__ void tma2d(void* dst, const void* tm, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(s32(dst)), "l"((uint64_t)tm), "r"(s32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma2d_mc(void* dst, const void* tm, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(s32(dst)), "l"((uint64_t)tm), "r"(s32(bar)), "r"(c0), "r"(c1), "h"(mask) : "memory");
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }

constexpr int kStageBytes = 16384;  // box 64 (K) x 128 rows fp16

// mode 0: same rows for every CTA; mode 1: CTA-private rows
template <int MC>
__global__ void __launch_bounds__(64, 1) ingest_kernel(const __grid_constant__ CUtensorMap tm, int mode, int kboxes, int reps, int stages, long long* cycles) {
  extern __shared__ uint8_t raw[];
  uint8_t* smem = raw + ((1024u - (s32(raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + stages * kStageBytes);
  uint64_t* empty = full + stages;
  const uint32_t rank = MC ? cluster_rank() : 0;
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], MC ? 2 : 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (MC) cluster_sync();
  const int row0 = mode == 1 ? (MC ? blockIdx.x / 2 : blockIdx.x) * 128 : 0;
  const long long t0 = clock64();
  const int total = kboxes * reps;
  if (threadIdx.x == 0) {
    int s = 0; uint32_t ph = 0;
    for (int i = 0; i < total; ++i) {
      if (MC) mbar_wait_cluster(&empty[s], ph ^ 1); else mbar_wait(&empty[s], ph ^ 1);
      mbar_expect(&full[s], kStageBytes);
      const int kb = i % kboxes;
      if (MC) tma2d_mc(smem + s * kStageBytes + rank * (kStageBytes / 2), &tm, &full[s], kb * 64, row0 + rank * 64, 3);
      else tma2d(smem + s * kStageBytes, &tm, &full[s], kb * 64, row0);
      if (++s == stages) { s = 0; ph ^= 1; }
    }
  } else if (threadIdx.x == 32) {
    int s = 0; uint32_t ph = 0;
    for (int i = 0; i < total; ++i) {
      mbar_wait(&full[s], ph);
      if (MC) { mbar_arrive_remote(&empty[s], 0); mbar_arrive_remote(&empty[s], 1); }
      else mbar_arrive(&empty[s]);
      if (++s == stages) { s = 0; ph ^= 1; }
    }
  }
  __syncthreads();
  const long long t1 = clock64();
  if (MC) cluster_sync();
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

typedef CUresult (*PFN_enc)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
  void* fp = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
  PFN_enc enc = (PFN_enc)fp;
  const int K = 2304, rows = 132 * 128;
  __half* w; CK(cudaMalloc(&w, (size_t)rows * K * 2)); CK(cudaMemset(w, 0, (size_t)rows * K * 2));
  long long* cyc; CK(cudaMalloc(&cyc, 132 * 8));
  auto make = [&](int boxrows, CUtensorMap* tm) {
    cuuint64_t gd[2] = {(cuuint64_t)K, (cuuint64_t)rows}; cuuint64_t gs[1] = {(cuuint64_t)K * 2};
    cuuint32_t bx[2] = {64, (cuuint32_t)boxrows}, es[2] = {1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUtensorMap tm128, tm64;
  if (make(128, &tm128) != CUDA_SUCCESS || make(64, &tm64) != CUDA_SUCCESS) { printf("encode failed\n"); return 1; }
  const int stages = 12;
  const size_t smem = 1024 + stages * kStageBytes + stages * 16;
  CK(cudaFuncSetAttribute(ingest_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(ingest_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int kboxes = K / 64, reps = 40;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int mc = 0; mc < 2; ++mc)
    for (int mode = 0; mode < 2; ++mode)
      for (int grid : {132, 66, 33}) {
        if (mc && mode == 1) continue;
        for (int it = 0; it < 2; ++it) {  // second run timed (L2 warm)
          cudaEventRecord(e0);
          if (!mc) {
            ingest_kernel<0><<<grid, 64, smem>>>(tm128, mode, kboxes, reps, stages, cyc);
          } else {
            cudaLaunchConfig_t cfg = {}; cfg.gridDim = dim3(grid); cfg.blockDim = dim3(64); cfg.dynamicSmemBytes = smem;
            cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            cfg.attrs = at; cfg.numAttrs = 1;
            CK(cudaLaunchKernelEx(&cfg, ingest_kernel<1>, tm64, mode, kboxes, reps, stages, cyc));
          }
          cudaEventRecord(e1);
          CK(cudaDeviceSynchronize());
        }
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        std::vector<long long> h(grid); cudaMemcpy(h.data(), cyc, grid * 8, cudaMemcpyDeviceToHost);
        std::sort(h.begin(), h.end());
        const double bytes = (double)kboxes * reps * kStageBytes;
        printf("%s mode=%s grid=%3d: %.3f ms  per-SM smem fill %.1f B/clk (median CTA), %.1f (slowest)  chip %.2f TB/s into smem\n",
               mc ? "multicast2" : "unicast   ", mode ? "private" : "shared ", grid, ms, bytes / h[grid / 2], bytes / h[grid - 1], bytes * grid / ms / 1e9);
      }
  return 0;
}
