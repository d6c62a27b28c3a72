// The fp32-in / fp32-out implicit GEMM on the tensor cores shared by the LPIPS convs (lpips.cu), the CLIP towers'
// linear layers (clip_text.cu, a linear layer being a 1x1 conv over a 1 x M image), the ArcFace IR-SE50 convs
// (arcface.cu), the face-parsing BiSeNet convs (face_parsing.cu) and the Inception-v3 convs (fid.cu): mma.sync m16n8k8, TF32
// operands rounded to nearest, fp32 accumulation, M = N*Ho*Wo output pixels, N = Cout, K = kh*kw*Cin tap-major /
// channel-minor.  The epilogue is a template parameter; the main loop is the same code for every epilogue, so an
// output element is the same fixed-order accumulation whichever layer or batch it belongs to.
#pragma once
#include "common.h"
#include "ptx.cuh"

namespace asyrp {
namespace tf32gemm {

constexpr int kBM = 128;            // output pixels per CTA tile
constexpr int kBN = 64;             // output channels per CTA tile
constexpr int kBK = 32;             // K slice per pipeline stage
constexpr int kLd = kBK + 4;        // shared-memory row pitch (floats): conflict-free fragment loads
constexpr int kStages = 3;
constexpr int kThreads = 256;       // 8 warps: 4 along M (32 pixels each) x 2 along N (32 channels each)
constexpr int kStageFloats = (kBM + kBN) * kLd;
constexpr size_t kConvSmem = static_cast<size_t>(kStages) * kStageFloats * sizeof(float);

// epilogues: v = acc + bias, then
enum Epilogue : int {
  kEpiRelu = 0,       // max(v, 0)                  (LPIPS convs)
  kEpiBias = 1,       // v                          (bias may be null: v = acc)
  kEpiQuickGelu = 2,  // v * sigmoid(1.702 v)       (CLIP's QuickGELU)
  kEpiResidual = 3,   // residual + v               (residual may be out: read and written by the same thread)
  kEpiPrelu = 4,      // v > 0 ? v : prelu[c] * v   (ArcFace's per-channel PReLU; bias may be null)
  kEpiResidualRelu = 5,  // max(residual + v, 0)    (BiSeNet's BasicBlock end; bias may be null)
  // max(v, 0) stored to channels [0, cstore) of output rows of pitch ldo, the horizontal padding padw (p.pad is then
  // the vertical one): an Inception branch of any even width writes its slice of the block output.  The other
  // epilogues ignore padw / ldo / cstore (pad both ways, pitch and bound Cout).
  kEpiReluSlice = 6,
  kEpiGelu = 7,       // 0.5 v (1 + erf(v / sqrt(2)))  (DINO's exact GELU)
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ uint32_t tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

struct Tf32ConvParams {
  const float* in;        // [N][H][W][Cin]
  const float* w;         // [Cout][Kpad], K = kh*kw*Cin tap-major / channel-minor, zero columns past K
  const float* bias;      // [Cout]
  const float* residual;  // [M][Cout] (kEpiResidual, kEpiResidualRelu)
  const float* prelu;     // [Cout] PReLU slopes (kEpiPrelu only)
  float* out;             // [N][Ho][Wo][Cout]
  int N, H, W, Cin, Ho, Wo, Cout, kw, stride, pad, K, Kpad, M;
  int padw, ldo, cstore;  // kEpiReluSlice only
};

__device__ __forceinline__ float quick_gelu(float z) { return z * (1.f / (1.f + expf(-(1.702f * z)))); }
__device__ __forceinline__ float gelu_erf(float z) { return 0.5f * z * (1.f + erff(z * 0.70710678118654752f)); }

// out = epilogue(conv(in) + bias).  CTA tile 128 pixels x 64 channels, K in slices of 32 through a 3-stage cp.async
// ring; the im2col gather is 16-byte chunks (4 channels of one tap: Cin % 4 == 0), zero-filled outside the image, so
// the padding is zeros of the operand as stored.  The weight rows n0 .. n0 + 63 are read without a bound: w and bias
// hold Cout rows (zero rows past a narrower branch's width).
template <int kEpi>
__global__ void __launch_bounds__(kThreads) tf32_conv_kernel(const Tf32ConvParams p) {
  pdl_trigger();
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;

  // A loader: this thread gathers chunk column `col` of rows row0 + 32*i
  const int col = tid & 7, row0 = tid >> 3;
  const float* a_base[4];
  int a_iy[4], a_ix[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + row0 + 32 * i;
    a_base[i] = p.in;
    a_iy[i] = -(1 << 28);  // rows past M: every tap out of range -> zeros
    a_ix[i] = 0;
    if (m < p.M) {
      const int hw = p.Ho * p.Wo;
      const int n = m / hw, r = m - n * hw;
      const int oy = r / p.Wo, ox = r - oy * p.Wo;
      a_base[i] = p.in + static_cast<size_t>(n) * p.H * p.W * p.Cin;
      a_iy[i] = oy * p.stride - p.pad;
      a_ix[i] = ox * p.stride - (kEpi == kEpiReluSlice ? p.padw : p.pad);
    }
  }

  auto load = [&](int stage, int kc) {
    float* As = smem + stage * kStageFloats;
    float* Bs = As + kBM * kLd;
    const int k = kc * kBK + col * 4;
    const bool kval = k < p.K;
    int ci = 0, ky = 0, kx = 0;
    if (kval) {
      const int tap = k / p.Cin;
      ci = k - tap * p.Cin;
      ky = tap / p.kw;
      kx = tap - ky * p.kw;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int iy = a_iy[i] + ky, ix = a_ix[i] + kx;
      const bool ok = kval && static_cast<unsigned>(iy) < static_cast<unsigned>(p.H) &&
                      static_cast<unsigned>(ix) < static_cast<unsigned>(p.W);
      const float* src = ok ? a_base[i] + (static_cast<size_t>(iy) * p.W + ix) * p.Cin + ci : p.in;
      cp_async16(smem_u32(As + (row0 + 32 * i) * kLd + col * 4), src, ok ? 16 : 0);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int idx = tid + kThreads * j, r = idx >> 3, c = idx & 7;
      cp_async16(smem_u32(Bs + r * kLd + c * 4), p.w + static_cast<size_t>(n0 + r) * p.Kpad + kc * kBK + c * 4, 16);
    }
  };

  const int nk = p.Kpad / kBK;
  pdl_wait();
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nk) load(s, s);
    cp_async_commit();
  }

  float acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.f;

  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int g = lane >> 2, t = lane & 3;
  for (int kc = 0; kc < nk; ++kc) {
    cp_async_wait<kStages - 2>();
    __syncthreads();  // slice kc landed for every thread; slice kc-1's stage is free
    {
      const int nx = kc + kStages - 1;
      if (nx < nk) load(nx % kStages, nx);
      cp_async_commit();
    }
    const float* As = smem + (kc % kStages) * kStageFloats;
    const float* Bs = As + kBM * kLd;
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 8) {
      uint32_t a[2][4], b[4][2];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const float* ar = As + (wm + mi * 16 + g) * kLd + kk + t;
        a[mi][0] = tf32(ar[0]);
        a[mi][1] = tf32(ar[8 * kLd]);
        a[mi][2] = tf32(ar[4]);
        a[mi][3] = tf32(ar[8 * kLd + 4]);
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float* br = Bs + (wn + ni * 8 + g) * kLd + kk + t;
        b[ni][0] = tf32(br[0]);
        b[ni][1] = tf32(br[4]);
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) mma_tf32(acc[mi][ni], a[mi], b[ni]);
    }
  }

#pragma unroll
  for (int ni = 0; ni < 4; ++ni) {
    const int c = n0 + wn + ni * 8 + 2 * t;
    float b0 = 0.f, b1 = 0.f;
    if (kEpi == kEpiRelu || kEpi == kEpiReluSlice || p.bias != nullptr) {
      b0 = p.bias[c];
      b1 = p.bias[c + 1];
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + wm + mi * 16 + g + 8 * h;
        if (m < p.M && (kEpi != kEpiReluSlice || c < p.cstore)) {
          const size_t o = static_cast<size_t>(m) * (kEpi == kEpiReluSlice ? p.ldo : p.Cout) + c;
          float2 v = make_float2(acc[mi][ni][2 * h] + b0, acc[mi][ni][2 * h + 1] + b1);
          if (kEpi == kEpiRelu || kEpi == kEpiReluSlice) {
            v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
          } else if (kEpi == kEpiQuickGelu) {
            v = make_float2(quick_gelu(v.x), quick_gelu(v.y));
          } else if (kEpi == kEpiGelu) {
            v = make_float2(gelu_erf(v.x), gelu_erf(v.y));
          } else if (kEpi == kEpiResidual) {
            const float2 r = *reinterpret_cast<const float2*>(p.residual + o);
            v = make_float2(r.x + v.x, r.y + v.y);
          } else if (kEpi == kEpiResidualRelu) {
            const float2 r = *reinterpret_cast<const float2*>(p.residual + o);
            v = make_float2(fmaxf(r.x + v.x, 0.f), fmaxf(r.y + v.y, 0.f));
          } else if (kEpi == kEpiPrelu) {
            v = make_float2(v.x > 0.f ? v.x : p.prelu[c] * v.x, v.y > 0.f ? v.y : p.prelu[c + 1] * v.y);
          }
          *reinterpret_cast<float2*>(p.out + o) = v;
        }
      }
  }
}

// launch over the grid of p (p.M pixels, p.Cout channels).  The channel tiles sit in grid y; in and w are read with
// 16-byte cp.async, out and the residual with 8-byte float2 accesses.  The pixel tile count is formed in 64 bits: p.M
// may be up to 2^31 - 1.
template <int kEpi>
inline int launch_tf32_conv(const Tf32ConvParams& p, cudaStream_t stream) {
  ASYRP_REQUIRE(p.Cout / kBN <= kMaxGridYZ, "tf32 conv: Cout=%d above %d channel tiles of %d", p.Cout, kMaxGridYZ,
                kBN);
  ASYRP_REQUIRE(reinterpret_cast<uintptr_t>(p.in) % 16 == 0 && reinterpret_cast<uintptr_t>(p.w) % 16 == 0,
                "tf32 conv: in and weight must be 16-byte aligned");
  ASYRP_REQUIRE(reinterpret_cast<uintptr_t>(p.out) % 8 == 0 && reinterpret_cast<uintptr_t>(p.residual) % 8 == 0,
                "tf32 conv: out and residual must be 8-byte aligned");
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(tf32_conv_kernel<kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(kConvSmem)));
  const unsigned pixel_tiles = static_cast<unsigned>((static_cast<long long>(p.M) + kBM - 1) / kBM);
  ASYRP_LAUNCH(tf32_conv_kernel<kEpi>, dim3(pixel_tiles, p.Cout / kBN), dim3(kThreads), kConvSmem, stream, p);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // namespace tf32gemm
}  // namespace asyrp
