// Self-attention over the spatial positions of one feature map (softmax(q k^T / sqrt(d)) v), fp16 in/out,
// fp32 logits / softmax / accumulation.  Reference: AttnBlock.forward (ddpm/diffusion.py:200-225, one head,
// d = C) and QKVAttentionLegacy.forward (improved_ddpm/unet.py:379-396, heads of 64 channels, q and k each
// scaled by d^-1/4, softmax in fp32).  The q/k/v projections and proj_out run on the wgmma GEMM kernel
// (conv_gemm.cu); this kernel is the T x T part with a warp-level online softmax.
//
// Layout: qkv [N][T][3*C] with C = heads*D: q at [0,C), k at [C,2C), v at [2C,3C), head h at h*D.
// Block = 8 warps; each warp owns 2 queries; keys/values streamed through shared memory 32 at a time.
#include "common.h"
#include "ptx.cuh"

namespace asyrp {

template <int D>
__global__ void __launch_bounds__(256) attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ out,
                                                        int T, int heads, float scale) {
  pdl_trigger();
  pdl_wait();
  constexpr int QT = 16, KT = 32, KS = D + 8;  // padded key row stride (halves): conflict-free 16B reads
  extern __shared__ __align__(16) uint8_t smem_attn[];
  __half* sq = reinterpret_cast<__half*>(smem_attn);  // [QT][D]
  __half* sk = sq + QT * D;                           // [KT][KS]
  __half* sv = sk + KT * KS;                          // [KT][D]

  const int n = blockIdx.z, head = blockIdx.y, q0 = blockIdx.x * QT;
  const int C = heads * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* base = qkv + static_cast<size_t>(n) * T * 3 * C;

  // stage the query tile
  for (int i = threadIdx.x; i < QT * (D / 8); i += blockDim.x) {
    const int r = i / (D / 8), c8 = i % (D / 8);
    uint4 u = make_uint4(0, 0, 0, 0);
    if (q0 + r < T) u = *reinterpret_cast<const uint4*>(base + static_cast<size_t>(q0 + r) * 3 * C + head * D + c8 * 8);
    *reinterpret_cast<uint4*>(sq + r * D + c8 * 8) = u;
  }

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float2 acc[2][D / 64];
#pragma unroll
  for (int qi = 0; qi < 2; ++qi)
#pragma unroll
    for (int j = 0; j < D / 64; ++j) acc[qi][j] = make_float2(0.f, 0.f);

  for (int k0 = 0; k0 < T; k0 += KT) {
    __syncthreads();  // previous tile fully consumed (also covers the sq staging on the first pass)
    for (int i = threadIdx.x; i < KT * (D / 8); i += blockDim.x) {
      const int r = i / (D / 8), c8 = i % (D / 8);
      uint4 uk = make_uint4(0, 0, 0, 0), uv = make_uint4(0, 0, 0, 0);
      if (k0 + r < T) {
        const __half* row = base + static_cast<size_t>(k0 + r) * 3 * C + head * D + c8 * 8;
        uk = *reinterpret_cast<const uint4*>(row + C);
        uv = *reinterpret_cast<const uint4*>(row + 2 * C);
      }
      *reinterpret_cast<uint4*>(sk + r * KS + c8 * 8) = uk;
      *reinterpret_cast<uint4*>(sv + r * D + c8 * 8) = uv;
    }
    __syncthreads();

#pragma unroll
    for (int qi = 0; qi < 2; ++qi) {
      const __half* qrow = sq + (warp * 2 + qi) * D;
      const __half* krow = sk + lane * KS;
      float s = 0.f;
#pragma unroll 4
      for (int c8 = 0; c8 < D / 8; ++c8) {
        const uint4 uq = *reinterpret_cast<const uint4*>(qrow + c8 * 8);
        const uint4 uk = *reinterpret_cast<const uint4*>(krow + c8 * 8);
        const __half2* hq = reinterpret_cast<const __half2*>(&uq);
        const __half2* hk = reinterpret_cast<const __half2*>(&uk);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = __half22float2(hq[k]), b = __half22float2(hk[k]);
          s = fmaf(a.x, b.x, s);
          s = fmaf(a.y, b.y, s);
        }
      }
      s = (k0 + lane < T) ? s * scale : -INFINITY;
      float mx = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float m_new = fmaxf(m_run[qi], mx);
      const float corr = __expf(m_run[qi] - m_new);
      const float pr = __expf(s - m_new);
      float ps = pr;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
      l_run[qi] = l_run[qi] * corr + ps;
      m_run[qi] = m_new;
#pragma unroll
      for (int j = 0; j < D / 64; ++j) {
        acc[qi][j].x *= corr;
        acc[qi][j].y *= corr;
      }
#pragma unroll 8
      for (int kk = 0; kk < KT; ++kk) {
        const float pk = __shfl_sync(0xffffffffu, pr, kk);
        const __half* vrow = sv + kk * D + 2 * lane;
#pragma unroll
        for (int j = 0; j < D / 64; ++j) {
          const float2 vv = __half22float2(*reinterpret_cast<const __half2*>(vrow + 64 * j));
          acc[qi][j].x = fmaf(pk, vv.x, acc[qi][j].x);
          acc[qi][j].y = fmaf(pk, vv.y, acc[qi][j].y);
        }
      }
    }
  }

#pragma unroll
  for (int qi = 0; qi < 2; ++qi) {
    const int t = q0 + warp * 2 + qi;
    if (t < T) {
      const float inv = 1.0f / l_run[qi];
      __half* orow = out + (static_cast<size_t>(n) * T + t) * C + head * D + 2 * lane;
#pragma unroll
      for (int j = 0; j < D / 64; ++j)
        *reinterpret_cast<__half2*>(orow + 64 * j) = __floats2half2_rn(acc[qi][j].x * inv, acc[qi][j].y * inv);
    }
  }
}

template <int D>
static int launch_attention(const void* qkv, void* out, int N, int T, int heads, float scale, cudaStream_t st) {
  constexpr int QT = 16, KT = 32, KS = D + 8;
  const size_t smem = (QT * D + KT * KS + KT * D) * sizeof(__half);
  static bool attr_set = false;
  if (!attr_set) {
    ASYRP_CHECK_CUDA(
        cudaFuncSetAttribute(attention_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    attr_set = true;
  }
  dim3 grid((T + QT - 1) / QT, heads, N);
  ASYRP_LAUNCH(attention_kernel<D>, dim3(grid), dim3(256), smem, st, static_cast<const __half*>(qkv), static_cast<__half*>(out), T, heads,
                                              scale);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Tensor-core attention helpers: the two GEMMs (q k^T, P v) run on conv_gemm_kernel in batched-weight mode;
// these two kernels are the glue: v -> v^T (the P v GEMM wants K-major rows) and the fp32 row softmax.
// ---------------------------------------------------------------------------------------------------------
// in: [N][T][ld] (C channels from `in`), out: [N][C][T]
__global__ void __launch_bounds__(256) transpose_tc_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                                           int T, int C, int ld) {
  pdl_trigger();
  pdl_wait();
  __shared__ __half tile[32][34];
  const int n = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8)
    if (t0 + i < T) tile[i][tx] = in[(static_cast<size_t>(n) * T + t0 + i) * ld + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (t0 + tx < T) out[(static_cast<size_t>(n) * C + c0 + i) * T + t0 + tx] = tile[tx][i];
}

// P[r][:] = softmax(scale * S[r][:]) over T columns, fp32 math (th.softmax(weight.float()), unet.py:393); one warp per row
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ S, __half* __restrict__ P,
                                                           int rows, int T, float scale) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + static_cast<size_t>(row) * T;
  __half* o = P + static_cast<size_t>(row) * T;
  float v[32];  // T <= 1024
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int c = lane + i * 32;
    v[i] = c < T ? s[c] * scale : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
  for (int of = 16; of > 0; of >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, of));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    v[i] = __expf(v[i] - mx);
    sum += v[i];
  }
  for (int of = 16; of > 0; of >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, of);
  const float inv = 1.0f / sum;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int c = lane + i * 32;
    if (c < T) o[c] = __float2half_rn(v[i] * inv);
  }
}

}  // namespace asyrp

using namespace asyrp;

extern "C" ASYRP_API int asyrp_transpose_tc(const void* in, void* out, int N, int T, int C, int ld, void* stream) {
  ASYRP_REQUIRE(C % 32 == 0, "asyrp_transpose_tc: C=%d must be a multiple of 32", C);
  dim3 grid((T + 31) / 32, C / 32, N);
  ASYRP_LAUNCH(transpose_tc_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), static_cast<const __half*>(in),
                                                                           static_cast<__half*>(out), T, C, ld);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

extern "C" ASYRP_API int asyrp_softmax_rows(const void* S, void* P, long long rows, int T, float scale, void* stream) {
  ASYRP_REQUIRE(T >= 1 && T <= 1024, "asyrp_softmax_rows: T=%d out of range (<= 1024)", T);
  ASYRP_LAUNCH(softmax_rows_kernel, dim3(static_cast<unsigned>((rows + 7) / 8)), dim3(256), 0, static_cast<cudaStream_t>(stream), 
      static_cast<const float*>(S), static_cast<__half*>(P), static_cast<int>(rows), T, scale);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

extern "C" ASYRP_API int asyrp_attention(const void* qkv, void* out, int N, int T, int heads, int head_dim,
                                         float scale, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (head_dim) {
    case 64: return launch_attention<64>(qkv, out, N, T, heads, scale, st);
    case 128: return launch_attention<128>(qkv, out, N, T, heads, scale, st);
    case 256: return launch_attention<256>(qkv, out, N, T, heads, scale, st);
    case 512: return launch_attention<512>(qkv, out, N, T, heads, scale, st);
    default:
      set_error("asyrp_attention: unsupported head_dim %d (supported 64/128/256/512)", head_dim);
      return ASYRP_ERR_INVALID;
  }
}
