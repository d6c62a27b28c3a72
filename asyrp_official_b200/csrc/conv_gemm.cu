// Implicit-GEMM convolution / batched GEMM on Hopper tensor cores (wgmma, sm_90a), TMA-fed.
//
// One kernel serves every dense contraction of the Asyrp UNet path:
//   * 3x3 stride-1 pad-1 convs        (ResnetBlock.conv1/conv2, Upsample.conv; ddpm/diffusion.py:122-133,77-81)
//   * 3x3 stride-2 convs, pad (0,1,0,1) (Downsample.conv; ddpm/diffusion.py:96-107)
//   * 1x1 convs                        (nin_shortcut :145-149, AttnBlock q/k/v/proj :179-198, DeltaBlock :236-249,
//                                       improved_ddpm/unet.py qkv/proj_out :333-336, skip_connection :264)
//   * plain GEMMs (rows = "pixels" of an H=1 image)
//
// Data layout: activations NHWC fp16, weights [Cout][K] fp16 with K = sum over segments of taps*C_seg
// (tap-major, channel-minor), accumulation fp32 in registers, epilogue fp32.
//
// The K loop walks "segments": each segment is one source tensor (so a channel-concat input is two
// segments and never materialised; a fused 1x1 shortcut is one more segment accumulated into the same
// accumulators).  For a 3x3/s1 segment the producer loads, per 64-channel chunk, ONE (TH+2) x (8+2)-pixel halo tile
// and the nine taps are start-address offsets into it (the 128B swizzle is a function of the shared-memory
// address, the descriptor's stride-byte-offset is the halo pitch); layers narrower than 8x16 pixels use three
// dx-shifted copies whose dy taps are 1024B-aligned row offsets.  TMA's out-of-bounds zero fill is the padding.
//
// Warp roles (576 threads): warps 0..7 = two consumer warpgroups (wgmma into register accumulators, then the
// epilogue: accumulators -> shared-memory staging tile -> bias/residual -> fp16 NHWC store + GroupNorm partial sums),
// warps 8..15 = in-place operand transform (fused GroupNorm-apply + SiLU), warp 16 = activation TMA producer,
// warp 17 = weight TMA producer (whole-warp uniform control flow, one elected lane issues).  Persistent: each CTA
// loops over output tiles; the producers run ahead across tile boundaries, so the loads of tile i+1 overlap the
// epilogue of tile i.
#include "common.h"
#include "ptx.cuh"
#include <cstring>
#include <memory>

namespace asyrp {

static constexpr int kMaxSeg = 3;
static constexpr int kNumConsumerWarps = 8;   // two warpgroups
static constexpr int kNumTransformWarps = 8;
static constexpr int kWarpT = kNumConsumerWarps;                // first transform warp
static constexpr int kWarpA = kWarpT + kNumTransformWarps;      // activation (A operand) producer warp
static constexpr int kWarpB = kWarpA + 1;                       // weight (B operand) producer warp
static constexpr int kNumThreads = 32 * (kWarpB + 1);

struct ConvSegDev {
  int nchunks;  // C / 64
  int mode;     // 0: 1x1, 1: 3x3 stride 1 (three dx-shifted copies), 2: 3x3 stride 2 (parity view),
                // 3: 3x3 stride 1 from ONE halo tile (TW == 8: every tap is an address offset into it)
  int kbase;    // first K column of this segment in the weight matrix
  int C;        // channels of the source
  // optional in-place operand transform  x -> act(a*x + b)  (GroupNorm apply + SiLU), applied to the A tile in
  // shared memory between the TMA load and the MMA; out-of-image pixels stay exactly zero (the conv's padding)
  const float* affine;  // [N][aff_stride] floats: (a, b) pairs of this segment's channels, or nullptr
  int aff_stride;
  int act;              // 1: SiLU after the affine
  // In-kernel GroupNorm finalise (replaces the affine table and the gn_finalize launch that fills it): the transform
  // threads compute (a, b) of their 8 channels from per-(sample, channel pair) sums that the PRODUCERS' epilogues
  // accumulated with 64-bit integer atomics (fixed point, kStatScale): integer addition commutes, so the statistics —
  // and everything downstream — stay bit-reproducible whatever order the tiles finish in.
  const long long* gn_sums[2];  // [N][C_i/2][2] (sum, sum of squares) of the two sources of the (virtual) concat
  int gn_C[2];                  // their channel counts (gn_C[1] == 0: single source)
  const float* gn_gamma;        // [C_total] GroupNorm weight / bias on the concatenated axis; nullptr = mode off
  const float* gn_beta;
  const float* gn_ss;           // ADM: (scale | shift) rows [N][gn_ss_stride] (improved_ddpm/unet.py:290-294) or nullptr
  int gn_ss_stride;
  float gn_eps, gn_inv_count;   // 1 / (H*W * channels per group)
  int gn_off;                   // first channel of this segment on the concatenated axis
};
static constexpr float kStatScale = 262144.0f;  // 2^18: resolution 3.8e-6 per tile sum, range +-3.5e13

struct ConvParams {
  CUtensorMap tmA[kMaxSeg];
  CUtensorMap tmB;
  ConvSegDev seg[kMaxSeg];
  int nseg;
  int N, H, W, Cout;      // output geometry
  int TW, TH, NB;         // pixel sub-tile: TW x TH pixels of NB samples, TW*TH*NB == 128
  int MT;                 // sub-tiles (stacked in y) per CTA tile: 1 or 2; all share every weight tile
  int tiles_x, tiles_y, tiles_n, m_tiles, n_tiles;
  // exact division by m_tiles / tiles_x / tiles_x*tiles_y as __umulhi(x, mul): mul = 2^32/d + 1, valid while
  // x*d < 2^32; d == 1 is encoded as mul == 0, "range too large, divide in hardware" as mul == 1
  uint32_t mul_m, mul_x, mul_xy;
  int a_stages, b_stages;
  uint32_t a_stage_bytes;  // ring slot size for A copies
  // Optional second activation ring for the 1x1 ("light") stages of a halo-tile conv.  A light stage is consumed in
  // 4 MMAs; a heavy (3x3 halo) stage needs load + in-place transform + 36 MMAs.  In one shared ring the light stages
  // of tile i occupy the slots the first heavy stage of tile i+1 should already be loading / transforming into, and
  // the tensor pipe idles for that latency at every tile boundary.  l_stages == 0: single ring.
  int l_stages;
  uint32_t l_stage_bytes;
  uint32_t row_bytes;      // NB*TW*128 : bytes of one tile row (all samples) of one 64-channel chunk
  const float* ebias;      // fp32 bias (+ timestep-embedding projection): row n at ebias + n*ebias_stride
  int ebias_stride;        // 0: one row shared by all samples
  const __half* res;       // residual, NHWC like out, or nullptr
  // res_mode 1: the residual is nearest-x2 upsampled on the fly (source [N][H/2][W/2][Cout]); 2: 2x2 average-pooled
  // (source [N][2H][2W][Cout]) — the skip branch of the ADM up / down ResBlocks (improved_ddpm/unet.py:279-284,297)
  int res_mode;
  float res_scale, acc_scale;
  // optional device-side copy of (acc_scale, res_scale): when set it overrides the two by-value fields, so that one
  // captured CUDA graph serves every hs_coeff tuple (the DeltaBlock coefficients are per-call arguments of forward())
  const float* scales;
  __half* out;             // [N][H][W][Cout] fp16, or nullptr when out_planar is used
  float* out_planar;       // optional fp32 planar [N][planar_c][H][W] holding output channels [0, planar_c)
  int planar_c;
  float* stats;            // [N][tiles_y*tiles_x][Cout/2][2] partial (sum, sumsq) or nullptr
  long long* sums_out;     // [N][Cout/2][2] fixed-point (sum, sumsq) accumulated with integer atomics, or nullptr
  int b_batched;           // weights have a per-sample batch dimension (attention GEMMs)
  // multi-head attention GEMMs: the batch index ns of a tile is (sample, head).  a_heads > 1: the activation map has
  // a head dimension (64-channel slices of one tensor); b_heads likewise for the per-sample weights; out_heads > 1:
  // the Cout columns of batch entry ns = n*out_heads + head go to channels [head*Cout, (head+1)*Cout) of sample n
  int a_heads, b_heads, out_heads;
  int out_ld;              // elements between consecutive output pixels (Cout * out_heads)
  int out_f32;             // `out` is fp32 (attention logits keep fp32 precision for the softmax)
  int any_transform;       // some segment has an affine: the MMA warp then waits on readyA instead of fullA
  int any_gn;              // some segment finalises its GroupNorm in the kernel (per-tile group statistics in smem)
  // up2: this conv is "3x3 conv of the nearest-x2 upsampled input" (Upsample.conv, ddpm/diffusion.py:77-87) evaluated
  // on the SOURCE image as four sub-pixel phases: output pixel (2i+a, 2j+b) only ever sees the 2x2 source
  // neighbourhood rows {i-1+a, i+a} x cols {j-1+b, j+b}, with the 3x3 taps that fall on the same source pixel summed
  // on the host.  N/H/W are the source geometry, the output is [N][2H][2W][Cout]; the channel-tile index carries the
  // phase (n_tiles = 4 * Cout/BN, weight rows phase-major, K = 4*C): 4 of 9 tap MMAs, no upsampled tensor in HBM.
  int up2;
  // K-loop order: entries (segment << 6 | 64-channel chunk), see asyrp_conv_create().
  int n_sched;
  uint8_t sched[64];
#ifdef ASYRP_TRACE
  long long* trace;  // diagnostic build only: [CTA][kTraceRoles][kTraceLen] clock64() stamps, see scripts/conv_trace.py
#endif
};
// Pipeline timeline of a diagnostic build (-DASYRP_TRACE, scripts/conv_trace.py): one elected lane per role stamps
// clock64() at its hand-off points; compiled out of the product library.
#ifdef ASYRP_TRACE
static constexpr int kTraceRoles = 10, kTraceLen = 128;
#define ASYRP_TRACE_STAMP(role, idx)                                                                    \
  do {                                                                                                  \
    if (p.trace != nullptr && lane == 0 && (idx) < kTraceLen)                                           \
      p.trace[(static_cast<size_t>(blockIdx.x) * kTraceRoles + (role)) * kTraceLen + (idx)] = clock64(); \
  } while (0)
#else
#define ASYRP_TRACE_STAMP(role, idx) do { } while (0)
#endif

__device__ __forceinline__ int fast_div(int x, uint32_t mul, int d) {
  // mul == 0: d == 1; mul == 1: range too large for the 32-bit multiply-high (huge batches) -> hardware division
  return mul > 1u ? static_cast<int>(__umulhi(static_cast<uint32_t>(x), mul)) : (mul == 0u ? x : x / d);
}
// tile index -> (pixel tile column, row, sample-group, channel tile); a runtime integer division costs ~20
// dependent instructions and every role needs these five at each tile start
struct TileCoord { int mt, nt, tx, ty, tn; };
__device__ __forceinline__ TileCoord tile_coord(const ConvParams& p, int tile) {
  TileCoord c;
  c.nt = fast_div(tile, p.mul_m, p.m_tiles);
  c.mt = tile - c.nt * p.m_tiles;
  c.tn = fast_div(c.mt, p.mul_xy, p.tiles_x * p.tiles_y);
  const int rem = c.mt - c.tn * (p.tiles_x * p.tiles_y);
  c.ty = fast_div(rem, p.mul_x, p.tiles_x);
  c.tx = rem - c.ty * p.tiles_x;
  return c;
}

// In-place operand transform of U pixels per thread (pixels px, px+lanes, ...; 8 threads per pixel, one 16-byte
// chunk = 8 channels each) of a SWIZZLE_128B stage:  x -> act(a*x + b), out-of-image pixels -> 0 (the conv padding).
template <int U>
__device__ __forceinline__ void transform_pixels(uint8_t* stage, int px, int jl, int lanes, int npix, int& hy, int& r,
                                                 int dhy, int dr, int prow, int xb, int yb, int W, int H, bool n_ok,
                                                 const float (&ca)[8], const float (&cb)[8], int act) {
  uint4 u[U];
  bool ok[U], inimg[U];
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const int pk = px + k * lanes;
    ok[k] = pk < npix;
    const int x = xb + r, y = yb + hy;
    inimg[k] = ok[k] && x >= 0 && x < W && y >= 0 && y < H && n_ok;
    u[k] = make_uint4(0u, 0u, 0u, 0u);
    if (ok[k]) u[k] = *reinterpret_cast<const uint4*>(stage + pk * 128 + ((jl ^ (pk & 7)) << 4));
    hy += dhy;
    r += dr;
    if (r >= prow) { r -= prow; ++hy; }
  }
#pragma unroll
  for (int k = 0; k < U; ++k) {
    __half2* h2 = reinterpret_cast<__half2*>(&u[k]);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = __half22float2(h2[e]);
      f.x = fmaf(ca[2 * e], f.x, cb[2 * e]);
      f.y = fmaf(ca[2 * e + 1], f.y, cb[2 * e + 1]);
      if (act == 2) { f.x = silu_tanh_half(f.x); f.y = silu_tanh_half(f.y); }  // (ca, cb) already halved
      else if (act) { f.x = silu_fast(f.x); f.y = silu_fast(f.y); }
      h2[e] = inimg[k] ? __floats2half2_rn(f.x, f.y) : __floats2half2_rn(0.f, 0.f);
    }
  }
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const int pk = px + k * lanes;
    if (ok[k]) *reinterpret_cast<uint4*>(stage + pk * 128 + ((jl ^ (pk & 7)) << 4)) = u[k];
  }
}

// The same with everything per-pixel hoisted out: `base` already points at this thread's 16-byte chunk of its first
// pixel (pixel lane * 128 B + swizzled chunk; pixel lanes are 32 apart = 4096 B, which leaves the swizzle phase
// pk & 7 unchanged), bit k of `vld` / `img` says whether pixel k exists in the stage / lies inside the image.
// CHK = false: every pixel exists and lies inside the image (all but the last group of an interior tile).
template <int U, bool CHK>
__device__ __forceinline__ void transform_fast(uint32_t base, uint32_t vld, uint32_t img, const float (&ca)[8],
                                               const float (&cb)[8], int act) {
  uint4 u[U];
#pragma unroll
  for (int k = 0; k < U; ++k) {
    if (CHK) {
      u[k] = make_uint4(0u, 0u, 0u, 0u);
      if ((vld >> k) & 1u) u[k] = lds128(base + k * 4096);
    } else {
      u[k] = lds128(base + k * 4096);
    }
  }
  if (act == 2) {  // one-MUFU SiLU, (ca, cb) already halved: 4 instead of 7.5 instructions per element
#pragma unroll
    for (int k = 0; k < U; ++k) {
      __half2* h2 = reinterpret_cast<__half2*>(&u[k]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h2[e]);
        f.x = silu_tanh_half(fmaf(ca[2 * e], f.x, cb[2 * e]));
        f.y = silu_tanh_half(fmaf(ca[2 * e + 1], f.y, cb[2 * e + 1]));
        h2[e] = __floats2half2_rn(f.x, f.y);
      }
      if (CHK && !((img >> k) & 1u)) u[k] = make_uint4(0u, 0u, 0u, 0u);
    }
  } else {
#pragma unroll
    for (int k = 0; k < U; ++k) {
      __half2* h2 = reinterpret_cast<__half2*>(&u[k]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h2[e]);
        f.x = fmaf(ca[2 * e], f.x, cb[2 * e]);
        f.y = fmaf(ca[2 * e + 1], f.y, cb[2 * e + 1]);
        if (act) { f.x = silu_fast(f.x); f.y = silu_fast(f.y); }
        h2[e] = __floats2half2_rn(f.x, f.y);
      }
      if (CHK && !((img >> k) & 1u)) u[k] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
#pragma unroll
  for (int k = 0; k < U; ++k)
    if (!CHK || ((vld >> k) & 1u)) sts128(base + k * 4096, u[k]);
}

// (a, b) of 8 consecutive channels [c0, c0+8) of segment `sg` for sample n:  GroupNorm(32 groups over the concatenated
// channel axis, eps) [* (1 + scale) + shift] as y = a*x + b.  Same arithmetic as gn_finalize_kernel (fp64 mean / var),
// evaluated by every transform thread for its own channels once per (tile, 64-channel chunk): a group's sums are
// 1..24 16-byte loads that all threads of the CTA share through L1.  The 8 channels touch at most 4 groups (2 channels
// per group at C = 64).  Everything is statically indexed: ca / cb must stay in registers for the transform loop.
__device__ __forceinline__ void gn_group_stats(const ConvSegDev& sg, int n, int g, int cpg, double inv, float& mean,
                                               float& rstd) {
  long long s1 = 0, s2 = 0;
  const int pa = sg.gn_C[0] >> 1, pb = sg.gn_C[1] >> 1;
  const int p_lo = (g * cpg) >> 1, p_hi = p_lo + (cpg >> 1);
#pragma unroll 1
  for (int pi = p_lo; pi < p_hi; ++pi) {
    const long long* q = pi < pa ? sg.gn_sums[0] + (static_cast<size_t>(n) * pa + pi) * 2
                                 : sg.gn_sums[1] + (static_cast<size_t>(n) * pb + (pi - pa)) * 2;
    const longlong2 v = *reinterpret_cast<const longlong2*>(q);
    s1 += v.x;
    s2 += v.y;
  }
  const double m = static_cast<double>(s1) * inv;
  double var = static_cast<double>(s2) * inv - m * m;
  if (var < 0.0) var = 0.0;
  rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(sg.gn_eps)));
  mean = static_cast<float>(m);
}
// (a, b) of this thread's 8 channels from the tile's group statistics `gs` ([32] (mean, rstd) in shared memory, written
// once per tile by 32 lanes, see the transform role): everything statically indexed, ca / cb stay in registers.
__device__ __forceinline__ void gn_affine8(const ConvSegDev& sg, const float2* gs, int n, int c0, float (&ca)[8],
                                           float (&cb)[8]) {
  const int C = sg.gn_C[0] + sg.gn_C[1], cpg = C >> 5;
  const int cg0 = sg.gn_off + c0;
  const int g0 = cg0 / cpg;  // the 8 channels touch at most 4 groups (2 channels per group at C = 64)
  const float2 s0 = gs[g0], s1 = gs[min(g0 + 1, 31)], s2 = gs[min(g0 + 2, 31)], s3 = gs[min(g0 + 3, 31)];
  const float4* gp = reinterpret_cast<const float4*>(sg.gn_gamma + cg0);
  const float4* bp = reinterpret_cast<const float4*>(sg.gn_beta + cg0);
  const float4 g_lo = gp[0], g_hi = gp[1], b_lo = bp[0], b_hi = bp[1];
  const float gam[8] = {g_lo.x, g_lo.y, g_lo.z, g_lo.w, g_hi.x, g_hi.y, g_hi.z, g_hi.w};
  const float bet[8] = {b_lo.x, b_lo.y, b_lo.z, b_lo.w, b_hi.x, b_hi.y, b_hi.z, b_hi.w};
  int bound = (g0 + 1) * cpg - cg0;  // channels [0, bound) of the 8 belong to group g0, and so on
  int k = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= bound) { ++k; bound += cpg; }
    const float2 st = k == 0 ? s0 : (k == 1 ? s1 : (k == 2 ? s2 : s3));
    float a = gam[i] * st.y;
    float b = bet[i] - st.x * a;
    if (sg.gn_ss != nullptr) {
      const float* ssp = sg.gn_ss + static_cast<size_t>(n) * sg.gn_ss_stride + cg0 + i;
      const float sc = 1.0f + ssp[0];
      const float sh = ssp[C];
      a = a * sc;
      b = b * sc + sh;
    }
    ca[i] = a;
    cb[i] = b;
  }
}
__device__ __forceinline__ void stat_atomic_add(long long* dst, float v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(dst), static_cast<unsigned long long>(__float2ll_rn(v * kStatScale)));
}

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(BN == 16 || BN == 64 || BN == 128, "wgmma tile widths of this kernel");
  if constexpr (BN == 16) wgmma_f16_n16(d, desc_a, desc_b, accumulate);
  else if constexpr (BN == 64) wgmma_f16_n64(d, desc_a, desc_b, accumulate);
  else wgmma_f16_n128(d, desc_a, desc_b, accumulate);
}

// NV consecutive fp32 values of the staging tile at shared address `addr` (16-byte aligned)
template <int NV>
__device__ __forceinline__ void ld_staged(uint32_t addr, uint32_t (&r)[NV]) {
#pragma unroll
  for (int i = 0; i < NV / 4; ++i) {
    const uint4 v = lds128(addr + 16 * i);
    r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
  }
}

// BN output channels x MT sub-tiles of 128 pixels per CTA tile; each consumer warpgroup accumulates MT x BN/2 fp32
// registers per thread.  MT * BN <= 128 bounds them to 64: ptxas allocates 96 registers per thread to every
// instantiation at 576 threads, and the 64- and 128-channel ones still spill ~100 bytes outside the wgmma chain.
template <int BN, int MT>
__global__ void __launch_bounds__(kNumThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvParams p) {
  pdl_trigger();  // the next kernel of the stream may be scheduled as soon as every CTA of this grid is running
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B operands need 1024B alignment
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  const int warp = uniform_warp_id();
  const int lane = threadIdx.x & 31;
  constexpr uint32_t kBStage = BN * 128;
  constexpr int kCPitch = MT * BN + 4;  // staging row pitch in floats: +16 B per row keeps the row reads conflict-free
  static_assert(MT * BN <= 128, "accumulator registers per consumer thread");

  uint8_t* sA = smem;
  uint8_t* sL = sA + p.a_stages * p.a_stage_bytes;  // light ring (may be empty)
  uint8_t* sB = sL + p.l_stages * p.l_stage_bytes;
  float* sC = reinterpret_cast<float*>(sB + p.b_stages * kBStage);  // [128][kCPitch] accumulator staging tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(sC + 128 * kCPitch);
  const int n_aslots = p.a_stages + p.l_stages;     // barrier index: heavy slots first, then light slots
  uint64_t* fullA = bars;
  uint64_t* emptyA = fullA + n_aslots;
  uint64_t* readyA = emptyA + n_aslots;
  uint64_t* fullB = readyA + n_aslots;
  uint64_t* emptyB = fullB + p.b_stages;
  float* s_stats = reinterpret_cast<float*>(emptyB + p.b_stages);     // [2][4][BN/32][32]
  float2* s_gstat = reinterpret_cast<float2*>(s_stats + 2 * 4 * BN);  // [2][kMaxSeg][32] (mean, rstd), see gn_affine8
  const int THT = MT * p.TH;  // rows of the CTA tile

  if (threadIdx.x == 0) {
    for (int i = 0; i < n_aslots; ++i) {
      mbar_init(&fullA[i], 1);
      mbar_init(&emptyA[i], kNumConsumerWarps);
      mbar_init(&readyA[i], kNumTransformWarps);
    }
    for (int i = 0; i < p.b_stages; ++i) {
      mbar_init(&fullB[i], 1);
      mbar_init(&emptyB[i], kNumConsumerWarps);
    }
    fence_mbar_init();
  }
  if (warp == kWarpA && lane == 0) {
    for (int s = 0; s < p.nseg; ++s) tma_prefetch_desc(&p.tmA[s]);
    tma_prefetch_desc(&p.tmB);
  }
  __syncthreads();
  // everything above (barrier init, descriptor prefetch) overlapped the previous kernel's tail; from here on global
  // memory written by it is read (and buffers it may still read are written)
  pdl_wait();

  const int total_tiles = p.m_tiles * p.n_tiles;

  if (warp == kWarpA) {
    // ======================================================== TMA producer, A operand (activations)
    // A and B have independent rings and independent producer threads, so the activation prefetch (which the
    // transform warps must also touch) runs a full A-ring ahead regardless of the weight ring's depth.
    // Whole warp, uniform control flow; one elected lane issues (see elect_one()).
    int sa = 0, sl = 0;      // heavy / light ring cursors
    uint32_t pa = 0, pl = 0;
    [[maybe_unused]] int tr_n = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord tc = tile_coord(p, tile);
      const int x0 = tc.tx * p.TW, y0 = tc.ty * THT, n0 = tc.tn * p.NB;
      for (int e = 0; e < p.n_sched; ++e) {
        const int s = p.sched[e] >> 6, ch = p.sched[e] & 63;
        const ConvSegDev sg = p.seg[s];
        const bool lt = p.l_stages != 0 && sg.mode == 0;
        const int ncopies = (sg.mode == 0 || sg.mode == 3) ? 1 : (sg.mode == 1 ? 3 : 9);
        const uint32_t a_bytes = sg.mode == 3 ? (THT + 2) * (p.TW + 2) * 128u
                                              : (sg.mode == 1 ? (THT + 2) : THT) * p.row_bytes;
        for (int cp = 0; cp < ncopies; ++cp) {
          const int slot = lt ? p.a_stages + sl : sa;
          mbar_wait_suspend(&emptyA[slot], (lt ? pl : pa) ^ 1);
          ASYRP_TRACE_STAMP(0, tr_n);
          ++tr_n;
          uint8_t* dst = lt ? sL + sl * p.l_stage_bytes : sA + sa * p.a_stage_bytes;
          int c0 = ch * 64, c1, c2 = n0, c3 = 0, c4;
          if (sg.mode == 3) {
            c1 = x0 - 1; c4 = y0 - 1;
          } else if (sg.mode == 0) {
            c1 = x0; c2 = n0 / p.a_heads; c3 = n0 % p.a_heads; c4 = y0;
          } else if (sg.mode == 1) {
            c1 = x0 + cp - 1; c4 = y0 - 1;
          } else {
            const int ky = cp / 3, kx = cp % 3;
            c0 += (kx & 1) * sg.C; c1 = x0 + (kx >> 1); c3 = ky & 1; c4 = y0 + (ky >> 1);
          }
          if (elect_one()) {
            mbar_arrive_expect_tx(&fullA[slot], a_bytes);
            tma_load_5d(dst, &p.tmA[s], &fullA[slot], c0, c1, c2, c3, c4);
          }
          if (lt) {
            if (++sl == p.l_stages) { sl = 0; pl ^= 1; }
          } else {
            if (++sa == p.a_stages) { sa = 0; pa ^= 1; }
          }
        }
      }
    }
  } else if (warp == kWarpB) {
    // ======================================================== TMA producer, B operand (weights)
    int sb = 0;
    uint32_t pb = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const TileCoord tc = tile_coord(p, tile);
      const int nt = tc.nt, tn = tc.tn;
      const int bz = p.b_batched ? tn * p.NB : 0;
      const int b_n = bz / p.b_heads, b_h = bz % p.b_heads;
      for (int e = 0; e < p.n_sched; ++e) {
        const int s = p.sched[e] >> 6, ch = p.sched[e] & 63;
        const ConvSegDev sg = p.seg[s];
        const int ncopies = (sg.mode == 0 || sg.mode == 3) ? 1 : (sg.mode == 1 ? 3 : 9);
        const int ntaps = sg.mode == 1 ? 3 : (sg.mode == 3 ? (p.up2 ? 4 : 9) : 1);
        for (int cp = 0; cp < ncopies; ++cp) {
          for (int tp = 0; tp < ntaps; ++tp) {
            // tap index in the weight matrix: ky*3+kx (up2: dy*2+dx of the phase's 2x2 kernel; the weight rows
            // nt*BN already select the phase)
            const int tap = sg.mode == 0 ? 0 : (sg.mode == 1 ? tp * 3 + cp : (sg.mode == 3 ? tp : cp));
            mbar_wait_suspend(&emptyB[sb], pb ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&fullB[sb], kBStage);
              tma_load_4d(sB + sb * kBStage, &p.tmB, &fullB[sb], sg.kbase + tap * sg.C + ch * 64, nt * BN, b_h, b_n);
            }
            if (++sb == p.b_stages) { sb = 0; pb ^= 1; }
          }
        }
      }
    }
  } else if (warp >= kWarpT) {
    // ======================================================== operand transform warps, in place
    if (p.any_transform) {
      constexpr int kLanes = kNumTransformWarps * 4;  // pixels handled concurrently (8 threads per pixel)
      const int tt = threadIdx.x - kWarpT * 32;
      const int jl = tt & 7;                  // logical 16B chunk = channels [jl*8, jl*8+8) of the 64-channel slab
      const int pl = tt >> 3;                 // pixel lane
      const int toff = pl * 128 + ((jl ^ (pl & 7)) << 4);  // this thread's chunk of pixel `pl` inside a stage
      // Pixel masks of this thread, bit m = pixel pl + 32*m.  Halo geometry ((TW+2) x (THT+2) pixels, tiles always
      // whole): which pixels exist, and which sit in the left / right column or top / bottom row of the halo — those
      // are outside the image exactly when the tile touches that image edge.  Plain geometry (1x1 stages): existence.
      uint32_t h_vld = 0, h_l = 0, h_r = 0, h_t = 0, h_b = 0, d_vld = 0;
      {
        const int prow = p.TW + 2, rows = THT + 2;
#pragma unroll 1
        for (int m = 0, pk = pl; pk < rows * prow; ++m, pk += kLanes) {
          const int hy = pk / prow, r = pk - hy * prow;
          h_vld |= 1u << m;
          if (r == 0) h_l |= 1u << m;
          if (r == prow - 1) h_r |= 1u << m;
          if (hy == 0) h_t |= 1u << m;
          if (hy == rows - 1) h_b |= 1u << m;
        }
#pragma unroll 1
        for (int m = 0, pk = pl; pk < THT * p.TW * p.NB; ++m, pk += kLanes) d_vld |= 1u << m;
      }
      int sa = 0, sl = 0;
      uint32_t pa = 0, plt = 0;
      [[maybe_unused]] int tr_n = 0;
      // In-kernel GroupNorm: lane g of transform warp s computes (mean, rstd) of group g of segment s for the sample of a
      // tile, ONE tile ahead (the buffer of tile i+1 is written while tile i is transformed; the named barrier at the
      // top of tile i+1 publishes it).  fp64 like gn_finalize_kernel; 32 x nseg threads per tile, not every thread.
      auto group_stats = [&](int tile_next, int buf) {
        const int s = tt >> 5;
        if (s < p.nseg && p.seg[s].gn_gamma != nullptr) {
          const ConvSegDev& sg = p.seg[s];
          const TileCoord tcn = tile_coord(p, tile_next);
          const int n = tcn.tn < p.N ? tcn.tn : 0;  // NB == 1
          const int cpg = (sg.gn_C[0] + sg.gn_C[1]) >> 5;
          float m, r;
          gn_group_stats(sg, n, tt & 31, cpg,
                         static_cast<double>(sg.gn_inv_count) * (1.0 / static_cast<double>(kStatScale)), m, r);
          s_gstat[(buf * kMaxSeg + s) * 32 + (tt & 31)] = make_float2(m, r);
        }
      };
      if (p.any_gn && static_cast<int>(blockIdx.x) < total_tiles) group_stats(blockIdx.x, 0);
      int git = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++git) {
        const TileCoord tc = tile_coord(p, tile);
        const int x0 = tc.tx * p.TW, y0 = tc.ty * THT, n0 = tc.tn * p.NB;
        if (p.any_gn) {
          named_bar_sync(2, kNumTransformWarps * 32);
          if (tile + static_cast<int>(gridDim.x) < total_tiles) group_stats(tile + gridDim.x, (git + 1) & 1);
        }
        for (int e = 0; e < p.n_sched; ++e) {
          const int s = p.sched[e] >> 6, ch = p.sched[e] & 63;
          const ConvSegDev sg = p.seg[s];
          const bool lt = p.l_stages != 0 && sg.mode == 0;
          const int ncopies = (sg.mode == 0 || sg.mode == 3) ? 1 : (sg.mode == 1 ? 3 : 9);
          const int pw = sg.mode == 3 ? p.TW + 2 : p.TW;      // pixels per (row, sample) in the stage
          const int prow = pw * p.NB;                          // pixels per tile row
          const int rows = (sg.mode == 1 || sg.mode == 3) ? THT + 2 : THT;
          const int npix = rows * prow;
          const int yoff = (sg.mode == 1 || sg.mode == 3) ? -1 : 0;
          {
            float ca[8], cb[8];
            if (sg.affine != nullptr && p.NB == 1) {
              const float4* ap = reinterpret_cast<const float4*>(
                  sg.affine + static_cast<size_t>(n0 < p.N ? n0 : 0) * sg.aff_stride + (ch * 64 + jl * 8) * 2);
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float4 t4 = ap[k];
                ca[2 * k] = t4.x; cb[2 * k] = t4.y; ca[2 * k + 1] = t4.z; cb[2 * k + 1] = t4.w;
              }
            } else if (sg.gn_gamma != nullptr) {  // GroupNorm finalise in place of the table (NB == 1 by construction)
              gn_affine8(sg, s_gstat + ((git & 1) * kMaxSeg + s) * 32, n0 < p.N ? n0 : 0, ch * 64 + jl * 8, ca, cb);
            }
            if (sg.act == 2) {
#pragma unroll
              for (int k = 0; k < 8; ++k) { ca[k] *= 0.5f; cb[k] *= 0.5f; }
            }
            for (int cp = 0; cp < ncopies; ++cp) {
              const int slot = lt ? p.a_stages + sl : sa;
              mbar_wait_suspend(&fullA[slot], lt ? plt : pa);
              if (warp == kWarpT) ASYRP_TRACE_STAMP(1, tr_n);
              if (sg.affine != nullptr || sg.gn_gamma != nullptr) {
                uint8_t* stage = lt ? sL + sl * p.l_stage_bytes : sA + sa * p.a_stage_bytes;
                const int xoff = sg.mode == 3 ? -1 : (sg.mode == 1 ? cp - 1 : 0);
                // whole tile inside the image (always true for halo tiles; 1x1 stages of ragged layers fall back)
                const bool whole = x0 + p.TW <= p.W && y0 + THT <= p.H && n0 < p.N;
                if (p.NB == 1 && whole && (sg.mode == 3 || sg.mode == 0)) {
                  // Up to 4 pixels in flight per thread (all shared-memory loads first, branch-free math, then the
                  // stores); the last groups of a stage use the 2- and 1-wide variants instead of idle lanes (a
                  // 180-pixel halo tile is 1.4 four-wide passes).  No per-pixel index arithmetic: see the masks above.
                  uint32_t m_vld = d_vld, m_img = d_vld;
                  bool m_plain = true;
                  if (sg.mode == 3) {
                    const bool el = x0 == 0, er = x0 + p.TW >= p.W, et = y0 == 0, eb = y0 + THT >= p.H;
                    m_vld = h_vld;
                    m_img = h_vld & ~((el ? h_l : 0u) | (er ? h_r : 0u) | (et ? h_t : 0u) | (eb ? h_b : 0u));
                    m_plain = !(el || er || et || eb);
                  }
                  const uint32_t tb = smem_u32(stage) + toff;
                  const int ng = (npix + kLanes - 1) / kLanes;  // 32-pixel groups of the stage (<= 11)
                  int m = 0;
                  if (m_plain)  // interior tile: only the last group (partial) needs the masks
                    for (; m + 4 < ng; m += 4) transform_fast<4, false>(tb + m * 4096, 0u, 0u, ca, cb, sg.act);
                  for (; m + 4 <= ng; m += 4)
                    transform_fast<4, true>(tb + m * 4096, m_vld >> m, m_img >> m, ca, cb, sg.act);
                  if (m + 2 <= ng) {
                    transform_fast<2, true>(tb + m * 4096, m_vld >> m, m_img >> m, ca, cb, sg.act);
                    m += 2;
                  }
                  if (m < ng) transform_fast<1, true>(tb + m * 4096, m_vld >> m, m_img >> m, ca, cb, sg.act);
                } else if (p.NB == 1) {
                  // three dx-shifted copies (mode 1): the in-image test depends on the copy
                  // (hy, r) = (tile row, position inside the row) of pixel px, advanced incrementally (no divisions)
                  int hy = pl / prow, r = pl - hy * prow;
                  const int dhy = kLanes / prow, dr = kLanes - dhy * prow;
                  const bool n_ok = n0 < p.N;
                  int px = pl;
                  for (; px - pl + 3 * kLanes < npix; px += 4 * kLanes)
                    transform_pixels<4>(stage, px, jl, kLanes, npix, hy, r, dhy, dr, prow, x0 + xoff, y0 + yoff, p.W,
                                        p.H, n_ok, ca, cb, sg.act);
                  if (px - pl + kLanes < npix) {
                    transform_pixels<2>(stage, px, jl, kLanes, npix, hy, r, dhy, dr, prow, x0 + xoff, y0 + yoff, p.W,
                                        p.H, n_ok, ca, cb, sg.act);
                    px += 2 * kLanes;
                  }
                  if (px - pl < npix)
                    transform_pixels<1>(stage, px, jl, kLanes, npix, hy, r, dhy, dr, prow, x0 + xoff, y0 + yoff, p.W,
                                        p.H, n_ok, ca, cb, sg.act);
                } else {
                  // tiles spanning several samples (layers below 16x16 when fused): per-pixel sample lookup
                  for (int px = pl; px < npix; px += kLanes) {
                    const int hy = px / prow, r = px - hy * prow;
                    const int nn = r / pw, xx = r - nn * pw;
                    const int x = x0 + xx + xoff, y = y0 + hy + yoff, n = n0 + nn;
                    uint4* slot = reinterpret_cast<uint4*>(stage + px * 128 + ((jl ^ (px & 7)) << 4));
                    uint4 u = make_uint4(0u, 0u, 0u, 0u);
                    if (x >= 0 && x < p.W && y >= 0 && y < p.H && n < p.N) {
                      const float4* ap = reinterpret_cast<const float4*>(
                          sg.affine + static_cast<size_t>(n) * sg.aff_stride + (ch * 64 + jl * 8) * 2);
#pragma unroll
                      for (int k = 0; k < 4; ++k) {
                        const float4 t4 = ap[k];
                        ca[2 * k] = t4.x; cb[2 * k] = t4.y; ca[2 * k + 1] = t4.z; cb[2 * k + 1] = t4.w;
                      }
                      u = *slot;
                      __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
                      for (int k = 0; k < 4; ++k) {
                        float2 f = __half22float2(h2[k]);
                        f.x = fmaf(ca[2 * k], f.x, cb[2 * k]);
                        f.y = fmaf(ca[2 * k + 1], f.y, cb[2 * k + 1]);
                        if (sg.act == 2) { f.x = silu_tanh_half(0.5f * f.x); f.y = silu_tanh_half(0.5f * f.y); }
                        else if (sg.act) { f.x = silu_fast(f.x); f.y = silu_fast(f.y); }
                        h2[k] = __floats2half2_rn(f.x, f.y);
                      }
                    }
                    *slot = u;
                  }
                }
                fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
              }
              __syncwarp();
              if (warp == kWarpT) ASYRP_TRACE_STAMP(2, tr_n);
              ++tr_n;
              if (lane == 0) mbar_arrive(&readyA[slot]);
              if (lt) {
                if (++sl == p.l_stages) { sl = 0; plt ^= 1; }
              } else {
                if (++sa == p.a_stages) { sa = 0; pa ^= 1; }
              }
            }
          }
        }
      }
    }
  } else {
    // ======================================================== consumers (warps 0..7): wgmma, then the epilogue
    // Warpgroup wg accumulates rows [64 wg, 64 wg + 64) of every 128-pixel sub-tile in registers.  The epilogue works
    // on the staging tile in shared memory (row = pixel of the sub-tile, column = sub * BN + channel): warp (q, half)
    // owns pixel rows [32q, 32q+32) and drains the 32-channel column chunks half, half+2, ...
    const int wg = warp >> 2;
    const uint32_t b_lo0 = gmma_desc_lo(smem_u32(sB));
    const uint32_t sC_addr = smem_u32(sC);
    const int q = warp & 3;
    const int half = warp >> 2;
    const int ep_tid = warp * 32 + lane;
    const int row = q * 32 + lane;
    const int xx = row % p.TW, nn = (row / p.TW) % p.NB, yy = row / (p.TW * p.NB);
    const int tiles_per_sample = p.tiles_x * p.tiles_y * (p.up2 ? 4 : 1);  // statistics slots per sample
    constexpr int kEpThreads = kNumConsumerWarps * 32;
    float acc_scale = p.acc_scale, res_scale = p.res_scale;
    if (p.scales != nullptr) {
      acc_scale = __ldg(p.scales);
      res_scale = __ldg(p.scales + 1);
    }
    // ring slots whose last reader is a wgmma group: handed back to the producers once that group has completed
    auto release = [&](int b, int a) {
      __syncwarp();
      if (lane == 0) {
        if (b >= 0) mbar_arrive(&emptyB[b]);
        if (a >= 0) mbar_arrive(&emptyA[a]);
      }
    };
    int sa = 0, sl = 0, sb = 0;
    uint32_t pa = 0, pl = 0, pb = 0;
    int it = 0;
    [[maybe_unused]] int tr_n = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++it) {
      ASYRP_TRACE_STAMP(5, it);
      float acc[MT][BN / 2];
#pragma unroll
      for (int sub = 0; sub < MT; ++sub)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[sub][i] = 0.f;
      int up_a = 0, up_b = 0;  // up2: sub-pixel phase of this tile = first tap (ky, kx) of its 2x2 kernel
      if (p.up2) {
        const int ph = fast_div(tile, p.mul_m, p.m_tiles) / (p.Cout / BN);
        up_a = ph >> 1;
        up_b = ph & 1;
      }
      uint32_t accumulate = 0;
      int rel_b = -1, rel_a = -1;  // slots read by the wgmma group in flight
      for (int e = 0; e < p.n_sched; ++e) {
        const int s = p.sched[e] >> 6;
        const ConvSegDev sg = p.seg[s];
        const bool lt = p.l_stages != 0 && sg.mode == 0;
        const int ncopies = (sg.mode == 0 || sg.mode == 3) ? 1 : (sg.mode == 1 ? 3 : 9);
        const int ntaps = sg.mode == 1 ? 3 : (sg.mode == 3 ? (p.up2 ? 4 : 9) : 1);
        // byte strides inside the A stage: between 8-row groups, between sub-tiles, per ky / kx tap step
        const uint32_t halo_pitch = (p.TW + 2) * 128u;
        const uint32_t sbo = sg.mode == 3 ? halo_pitch : 1024u;
        const uint32_t sub_stride = sg.mode == 3 ? p.TH * halo_pitch : p.TH * p.row_bytes;
        // descriptors as (lo, hi) words: only the start-address field (16-byte units) changes inside the loop
        const uint32_t a_hi = gmma_desc_hi(sbo), b_hi = gmma_desc_hi(1024u);
        const uint32_t sub16 = sub_stride >> 4;
        // this warpgroup's 64 rows start 8 row groups into the sub-tile
        const uint32_t wg16 = (8u * wg * sbo) >> 4;
        // tap step in 16-byte units.  mode 1: dy tap = row shift inside the dx copy; mode 3: (ky, kx) = pixel
        // offset inside the halo tile: +128 B per kx, and from kx=2 to the next ky row +halo_pitch-256 B
        // (up2: 2x2 taps starting at (up_a, up_b): +128 B per kx, +halo_pitch-128 B to the next ky row)
        const uint32_t step16 = sg.mode == 3 ? 8u : (p.row_bytes >> 4);
        const int kxn = p.up2 ? 2 : 3;
        const uint32_t wrap16 = sg.mode == 3 ? ((halo_pitch - 128u * (kxn - 1)) >> 4) : step16;
        const uint32_t first16 = (sg.mode == 3 && p.up2) ? ((up_a * halo_pitch + up_b * 128u) >> 4) : 0u;
        for (int cp = 0; cp < ncopies; ++cp) {
          const int slot = lt ? p.a_stages + sl : sa;
          ASYRP_TRACE_STAMP(3, tr_n);
          mbar_wait(p.any_transform ? &readyA[slot] : &fullA[slot], lt ? pl : pa);
          ASYRP_TRACE_STAMP(4, tr_n);
          ++tr_n;
          uint32_t a_lo =
              gmma_desc_lo(smem_u32(lt ? sL + sl * p.l_stage_bytes : sA + sa * p.a_stage_bytes)) + first16 + wg16;
          int kx = 0;
          for (int tp = 0; tp < ntaps; ++tp) {
            mbar_wait(&fullB[sb], pb);
            const uint32_t b_lo = b_lo0 + sb * (kBStage >> 4);
            wgmma_fence();
#pragma unroll
            for (int sub = 0; sub < MT; ++sub) {
#pragma unroll
              for (int k = 0; k < 4; ++k)
                wgmma_bn<BN>(acc[sub], gmma_desc(a_lo + sub * sub16 + 2 * k, a_hi), gmma_desc(b_lo + 2 * k, b_hi),
                             (accumulate | k) ? 1u : 0u);
            }
            wgmma_commit();
            // the group before this one has completed: its weight stage (and the activation stage it finished) go back
            wgmma_wait<1>();
            release(rel_b, rel_a);
            rel_b = sb;
            rel_a = tp == ntaps - 1 ? slot : -1;
            accumulate = 1;
            if (++sb == p.b_stages) { sb = 0; pb ^= 1; }
            if (++kx == kxn) { kx = 0; a_lo += wrap16; } else { a_lo += step16; }
          }
          ASYRP_TRACE_STAMP(9, tr_n - 1);
          if (lt) {
            if (++sl == p.l_stages) { sl = 0; pl ^= 1; }
          } else {
            if (++sa == p.a_stages) { sa = 0; pa ^= 1; }
          }
        }
      }
      wgmma_wait<0>();
      release(rel_b, rel_a);
#pragma unroll
      for (int sub = 0; sub < MT; ++sub) wgmma_fence_operands(acc[sub]);

      // accumulators -> staging tile; the barrier before makes sure every consumer has drained the previous tile
      named_bar_sync(3, kEpThreads);
      if (warp == 0) ASYRP_TRACE_STAMP(7, it);
      {
        const int r0 = 64 * wg + 16 * q + (lane >> 2);
#pragma unroll
        for (int sub = 0; sub < MT; ++sub)
#pragma unroll
          for (int j = 0; j < BN / 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              *reinterpret_cast<float2*>(sC + (r0 + 8 * h) * kCPitch + sub * BN + 8 * j + 2 * (lane & 3)) =
                  make_float2(acc[sub][4 * j + 2 * h], acc[sub][4 * j + 2 * h + 1]);
      }
      named_bar_sync(3, kEpThreads);
      const uint32_t c_row = sC_addr + static_cast<uint32_t>(row * kCPitch) * 4u;

      const TileCoord tc = tile_coord(p, tile);
      const int tx = tc.tx, ty = tc.ty, tn = tc.tn;
      // up2: the channel-tile index carries the sub-pixel phase (a, b); outputs land on the (2H, 2W) grid
      int nt = tc.nt, ph = 0;
      if (p.up2) {
        const int cts = p.Cout / BN;
        ph = nt / cts;
        nt -= ph * cts;
      }
      const int ps = p.up2 ? 2 : 1, OH = p.H * ps, OW = p.W * ps, pa_ = ph >> 1, pb_ = ph & 1;
      const int x = tx * p.TW + xx, n = tn * p.NB + nn;
      const int tile_in_sample = (ty * p.tiles_x + tx) * (p.up2 ? 4 : 1) + ph;
      float* st = s_stats + (it & 1) * (4 * BN);
      if constexpr (BN == 16) {
        // narrow-N tile of conv_out (3 / 6 real output channels, fp32 planar store): one 16-column load per sub-tile,
        // warps of the second half have nothing to drain
        if (half == 0) {
#pragma unroll 1
          for (int sub = 0; sub < MT; ++sub) {
            const int y = ty * THT + sub * p.TH + yy;
            const bool valid = (x < p.W) && (y < p.H) && (n < p.N);
            uint32_t r[16];
            ld_staged<16>(c_row + sub * BN * 4, r);
            if (valid) {
              const float* eb = p.ebias != nullptr ? p.ebias + static_cast<size_t>(n) * p.ebias_stride : nullptr;
              const size_t hw = static_cast<size_t>(p.H) * p.W;
              float* pp = p.out_planar + static_cast<size_t>(n) * p.planar_c * hw + static_cast<size_t>(y) * p.W + x;
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (i < p.planar_c) pp[i * hw] = (__uint_as_float(r[i]) + (eb != nullptr ? eb[i] : 0.f)) * acc_scale;
            }
          }
        }
      } else {
#pragma unroll 1
      for (int cc = half; cc < BN / 32; cc += 2) {
        const int c0 = nt * BN + cc * 32;
        // statistics of this chunk: slot `lane` (see below) summed over the sub-tiles.  Reduced across the lanes once per
        // sub-tile: per-lane partial sums kept alive across the sub-tile loop (32 more registers next to r[] and v[])
        // would spill
        float wtot = 0.f;
#pragma unroll 1
        for (int sub = 0; sub < MT; ++sub) {
          float ws[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) ws[j] = 0.f;
          const int y = ty * THT + sub * p.TH + yy;
          const bool valid = (x < p.W) && (y < p.H) && (n < p.N);
          // output row of this pixel: batch entry n may be a (sample, head) pair writing a channel slice
          const size_t pix = ((static_cast<size_t>(n / p.out_heads) * OH + y * ps + pa_) * OW + x * ps + pb_) * p.out_ld +
                             static_cast<size_t>(n % p.out_heads) * p.Cout;
          uint32_t r[32];
          ld_staged<32>(c_row + (sub * BN + cc * 32) * 4, r);
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
          if (p.ebias != nullptr) {
            const float* eb = p.ebias + static_cast<size_t>(valid ? n : 0) * p.ebias_stride + c0;
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 b4 = *reinterpret_cast<const float4*>(eb + i);
              v[i] += b4.x; v[i + 1] += b4.y; v[i + 2] += b4.z; v[i + 3] += b4.w;
            }
          }
          if (acc_scale != 1.0f) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] *= acc_scale;
          }
          if (p.res != nullptr && valid) {
            if (p.res_mode == 2) {
              // skip branch of a down ResBlock: 2x2 average of the double-resolution tensor, fp32
              const size_t rW = static_cast<size_t>(p.W) * 2;
              const __half* r0 = p.res + ((static_cast<size_t>(n) * p.H * 2 + y * 2) * rW + x * 2) * p.Cout + c0;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float a8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) {
                  const uint4 u = *reinterpret_cast<const uint4*>(r0 + ((q4 >> 1) * rW + (q4 & 1)) * p.Cout + j * 8);
                  const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    const float2 f = __half22float2(h2[k]);
                    a8[2 * k] += f.x;
                    a8[2 * k + 1] += f.y;
                  }
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) v[j * 8 + k] += res_scale * (0.25f * a8[k]);
              }
            } else {
              // res_mode 1: nearest-x2 of the half-resolution tensor (skip branch of an up ResBlock)
              const size_t rpix = p.res_mode == 1 ? ((static_cast<size_t>(n) * (p.H >> 1) + (y >> 1)) * (p.W >> 1) + (x >> 1)) *
                                                        p.Cout
                                                  : pix;
              const uint4* rp = reinterpret_cast<const uint4*>(p.res + rpix + c0);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const uint4 u = rp[j];
                const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const float2 f = __half22float2(h2[k]);
                  v[j * 8 + k * 2] += res_scale * f.x;
                  v[j * 8 + k * 2 + 1] += res_scale * f.y;
                }
              }
            }
          }
          if (p.out_planar != nullptr) {
            if (valid && c0 == 0) {
              const size_t hw = static_cast<size_t>(p.H) * p.W;
              float* pp = p.out_planar + static_cast<size_t>(n) * p.planar_c * hw + static_cast<size_t>(y) * p.W + x;
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (i < p.planar_c) pp[i * hw] = v[i];
            }
          } else if (p.out_f32) {
            if (valid) {
              float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + pix + c0);
#pragma unroll
              for (int j = 0; j < 8; ++j) op[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
          } else if (valid) {
            uint4* op = reinterpret_cast<uint4*>(p.out + pix + c0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              uint4 u;
              __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
              for (int k = 0; k < 4; ++k) h2[k] = __floats2half2_rn(v[j * 8 + k * 2], v[j * 8 + k * 2 + 1]);
              op[j] = u;
            }
          }
          if (p.stats != nullptr) {
            if (p.NB == 1) {
              // slot j<16 : sum of channel pair j ; slot j>=16 : sum of squares of pair j-16 (this lane's pixel)
              if (valid) {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                  ws[j] += v[2 * j] + v[2 * j + 1];
                  ws[16 + j] += v[2 * j] * v[2 * j] + v[2 * j + 1] * v[2 * j + 1];
                }
              }
            } else {
              // tiles spanning several samples (tiny layers): one masked warp reduction per sample
              for (int sn = 0; sn < p.NB; ++sn) {
                const bool mine = valid && (nn == sn);
                float w[32];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                  const float a = mine ? v[2 * j] : 0.f, b = mine ? v[2 * j + 1] : 0.f;
                  w[j] = a + b;
                  w[16 + j] = a * a + b * b;
                }
#pragma unroll
                for (int h = 16; h >= 1; h >>= 1) {
                  const bool up = (lane & h) != 0;
#pragma unroll
                  for (int i = 0; i < h; ++i) {
                    const float send = up ? w[i] : w[i + h];
                    const float keep = up ? w[i + h] : w[i];
                    w[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
                  }
                }
                const int ns = tn * p.NB + sn;
                if (ns < p.N) {  // one slot per (sample, tile, lane quarter): deterministic, no atomics
                  float* g = p.stats + (((static_cast<size_t>(ns) * tiles_per_sample + tile_in_sample) * 4 + q) *
                                            (p.Cout / 2) + (c0 / 2) + (lane & 15)) * 2 + (lane >> 4);
                  *g = w[0];
                }
              }
            }
          }
          if (p.stats != nullptr && p.NB == 1) {
            // recursive-halving reduce-scatter over the 32 lanes: afterwards ws[0] on lane L is the total of slot L
#pragma unroll
            for (int h = 16; h >= 1; h >>= 1) {
              const bool up = (lane & h) != 0;
#pragma unroll
              for (int i = 0; i < h; ++i) {
                const float send = up ? ws[i] : ws[i + h];
                const float keep = up ? ws[i + h] : ws[i];
                ws[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
              }
            }
            wtot += ws[0];
          }
        }  // sub
        if (p.stats != nullptr && p.NB == 1) st[(q * (BN / 32) + cc) * 32 + lane] = wtot;
      }  // cc
      }
      if (warp == 0) ASYRP_TRACE_STAMP(8, it);

      if (BN >= 32 && p.stats != nullptr && p.NB == 1) {
        named_bar_sync(1, kEpThreads);
        for (int e = ep_tid; e < BN; e += kEpThreads) {
          const int cc = e >> 5, j = e & 31;
          float tot = 0.f;
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) tot += st[(qq * (BN / 32) + cc) * 32 + j];
          float* g = p.stats + ((static_cast<size_t>(tn) * tiles_per_sample + tile_in_sample) * (p.Cout / 2) +
                                (nt * BN + cc * 32) / 2 + (j & 15)) * 2 + (j >> 4);
          *g = tot;
          if (p.sums_out != nullptr)
            stat_atomic_add(p.sums_out + (static_cast<size_t>(tn) * (p.Cout / 2) + (nt * BN + cc * 32) / 2 + (j & 15)) * 2 +
                                (j >> 4), tot);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
struct ConvOp {
  ConvParams p;
  int BN;
  int MT;
  int grid;
  size_t smem_bytes;
};

}  // namespace asyrp

using namespace asyrp;

static const void* conv_kernel_ptr(int BN, int MT) {
  if (BN == 16) return MT == 2 ? reinterpret_cast<const void*>(&conv_gemm_kernel<16, 2>)
                               : reinterpret_cast<const void*>(&conv_gemm_kernel<16, 1>);
  if (BN == 128) return reinterpret_cast<const void*>(&conv_gemm_kernel<128, 1>);
  return MT == 2 ? reinterpret_cast<const void*>(&conv_gemm_kernel<64, 2>)
                 : reinterpret_cast<const void*>(&conv_gemm_kernel<64, 1>);
}

extern "C" {

struct AsyrpConvSeg {
  const void* src;  // fp16 NHWC source tensor
  int C;            // its channel count (multiple of 64)
  int mode;         // 0: 1x1, 1: 3x3 s1 p1, 2: 3x3 s2 pad(0,1,0,1) (source is [N][2H][2W][C])
  const float* affine;  // optional fused GroupNorm-apply: (a, b) pairs of this segment's channels, row n at
                        // affine + n*affine_stride floats; the operand becomes act(a*x + b)
  int affine_stride;
  int act;              // 1: SiLU
  int ld;               // elements between consecutive pixels of `src` (0: C) — channel slices of a wider tensor
  // in-kernel GroupNorm finalise (alternative to `affine`): see ConvSegDev
  const long long* gn_sums_a;
  int gn_Ca;
  const long long* gn_sums_b;
  int gn_Cb;
  const float* gn_gamma;
  const float* gn_beta;
  const float* gn_scale_shift;
  int gn_ss_stride;
  float gn_eps;
  int gn_hw;
  int gn_off;
};

struct AsyrpConvDesc {
  int N, H, W, Cout;  // output geometry (NHWC)
  int nseg;
  AsyrpConvSeg seg[3];
  const void* weight;  // fp16 [batch?][Cout][Ktot]
  int weight_batched;  // 1: one weight matrix per sample (requires 128-row tiles within one sample)
  int weight_ld;       // elements between consecutive weight rows (0: Ktot)
  long long weight_batch_stride;  // elements between consecutive samples' matrices (0: Cout*weight_ld)
  // multi-head batched GEMMs (attention): N counts (sample, head) pairs
  int a_heads;         // >1: segment 0 is [N/a_heads][H][W][ld] and head h reads channels [h*C, (h+1)*C)
  int b_heads;         // >1: the weights are [N/b_heads][Cout][weight_ld] and head h reads columns [h*K, (h+1)*K)
  int out_heads;       // >1: out is [N/out_heads][H][W][out_heads*Cout], head h writes channels [h*Cout, ...)
  int out_f32;         // 1: `out` is fp32 NHWC instead of fp16 (no residual / stats)
  const float* ebias;  // fp32, row n at ebias + n*ebias_stride (stride 0: shared row), or null
  int ebias_stride;
  const void* residual;  // fp16 NHWC [N][H][W][Cout] or null
  float res_scale, acc_scale;
  void* out;     // fp16 NHWC (ignored when out_planar is set)
  float* stats;  // partial GroupNorm sums, see asyrp_conv_stats_tiles()
  float* out_planar;  // optional: fp32 NCHW [N][planar_c][H][W] receiving output channels [0, planar_c<=8)
  int planar_c;
  int up2;  // 1: sub-pixel evaluation of conv3x3(nearest-x2 upsample(src)): see ConvParams::up2
  const float* scales;  // optional DEVICE pointer to (acc_scale, res_scale); overrides the two fields above at run time
  int res_mode;         // 0: residual has the output geometry; 1: [N][H/2][W/2][Cout], nearest-x2; 2: [N][2H][2W][Cout], avg-pool 2x2
  long long* sums_out;  // optional [N][Cout/2][2] int64: (sum, sumsq) * 2^18 of the output, accumulated atomically
};

static void conv_tile_shape(int H, int W, int halo, int* TW, int* TH, int* NB);

// The fused operand transform evaluates SiLU with ONE special-function op (tanh.approx.f32, 11 bits: absolute error
// <= 2^-12 |x|, the size of the fp16 rounding the operand receives anyway) instead of ex2 + rcp: 4 instead of 7.5
// instructions per element on the transform warps, whose work per 3x3 stage is comparable to that stage's MMAs.
// ASYRP_SILU_TANH=0 / asyrp_set_silu_tanh(0): the 2-MUFU form.
static int g_silu_tanh = -1;
static int silu_tanh_enabled() {
  if (g_silu_tanh < 0) {
    const char* e = getenv("ASYRP_SILU_TANH");
    g_silu_tanh = (e != nullptr) ? (e[0] != '0') : 1;
  }
  return g_silu_tanh;
}
// A 3x3/s1 conv whose output is at least 8 wide and 16 tall uses 8x16-pixel sub-tiles fed from one halo tile per
// 64-channel chunk ("halo" geometry, segment mode 3); otherwise three dx-shifted copies (mode 1).
static int conv_halo_ok(int H, int W) { return H % 16 == 0 && W % 8 == 0; }

// Tile configuration: BN output channels x MT sub-tiles of 128 pixels per CTA tile.  Larger tiles re-use operands
// better (the accumulators of a consumer warpgroup, MT*BN/2 fp32 registers per thread, bound MT*BN <= 128); small
// layers instead need enough tiles to occupy the 132 SMs of an H100 SXM.  Pick the most efficient configuration that
// still yields ~a full wave of tiles (0.8 x 132) at a NOMINAL batch of 16, else the one with the most tiles.  The choice must not
// depend on the actual batch: the tile partition fixes the summation order of the GroupNorm partial sums, and a
// sample's result has to be bit-identical whatever batch (or batch shard on another GPU) it is part of.
static void conv_config(int H, int W, int Cout, int halo, int* BN, int* MT, int phases = 1) {
  int TW, TH, NB;
  conv_tile_shape(H, W, halo, &TW, &TH, &NB);
  if (NB == 0) {  // no 128-pixel tile fits this geometry
    *BN = 0;
    *MT = 0;
    return;
  }
  constexpr int kNominalBatch = 16;
  if (Cout == 16) {  // conv_out: 3 / 6 real channels in one 16-wide N tile (an N=64 tile spends 4x the operand reads)
    *BN = 16;
    *MT = (NB == 1 && H > 1 && H % (2 * TH) == 0 && W % TW == 0) ? 2 : 1;
    return;
  }
  const int tiles_x = (W + TW - 1) / TW, tiles_n = (kNominalBatch + NB - 1) / NB;
  const int cand[3][2] = {{128, 1}, {64, 2}, {64, 1}};  // by decreasing operand re-use
  int best = -1, best_tiles = -1;
  for (int i = 0; i < 3; ++i) {
    const int bn = cand[i][0], mt = cand[i][1];
    if (Cout % bn != 0) continue;
    // two stacked sub-tiles: whole tiles only
    if (mt == 2 && !(NB == 1 && H > 1 && H % (2 * TH) == 0 && W % TW == 0)) continue;
    const int tiles = tiles_x * ((H + TH * mt - 1) / (TH * mt)) * tiles_n * (Cout / bn) * phases;
    if (tiles >= 106) { best = i; break; }
    if (tiles > best_tiles) { best = i; best_tiles = tiles; }
  }
  *BN = cand[best][0];
  *MT = cand[best][1];
}

// TW x TH pixels of NB samples, TW * TH * NB == 128; NB == 0 (and TH == 0) when no such tile exists: a width that is
// not a power of two below the tile width (e.g. W = 12, or W = 96 for H = 1), or an empty image
static void conv_tile_shape(int H, int W, int halo, int* TW, int* TH, int* NB) {
  int tw, th;
  if (halo) {
    *TW = 8; *TH = 16; *NB = 1;
    return;
  }
  if (H < 1 || W < 1) {
    *TW = 0; *TH = 0; *NB = 0;
    return;
  }
  if (H == 1) {
    tw = W < 128 ? W : 128;
    th = 1;
  } else {
    tw = W < 16 ? W : 16;
    th = 128 / tw;
    if (th > 8) th = 8;
    if (th > H) th = H;
  }
  // largest power-of-two tile that divides 128
  while (th > 0 && 128 % (tw * th) != 0) --th;
  *TW = tw;
  *TH = th;
  *NB = th > 0 ? 128 / (tw * th) : 0;
}

// number of pixel tiles per sample the stats buffer must hold: stats is [N][tiles][Cout/2][2] floats.
// For layers whose tile spans several samples (NB>1) the kernel writes one slot per epilogue warp (4).
// has_3x3: the conv producing the statistics contains a 3x3 stride-1 segment (tile geometry depends on it).
// 0: the geometry cannot be tiled (asyrp_conv_create rejects it)
ASYRP_API int asyrp_conv_stats_tiles(int H, int W, int Cout, int has_3x3) {
  int TW, TH, NB, bn, mt;
  const int halo = has_3x3 && conv_halo_ok(H, W);
  conv_tile_shape(H, W, halo, &TW, &TH, &NB);
  if (NB == 0) return 0;
  conv_config(H, W, Cout, halo, &bn, &mt);
  const int tht = TH * mt;
  const int tiles = ((W + TW - 1) / TW) * ((H + tht - 1) / tht);
  return NB == 1 ? tiles : tiles * 4;
}

// tile configuration of a conv with this output geometry: BN * 16 + MT (e.g. 128 * 16 + 1 = 128 channels x 128 pixels);
// 0: the geometry cannot be tiled
ASYRP_API int asyrp_conv_tile_config(int H, int W, int Cout, int has_3x3) {
  int bn, mt;
  const int halo = has_3x3 && conv_halo_ok(H, W);
  conv_config(H, W, Cout, halo, &bn, &mt);
  return bn * 16 + mt;
}

// statistics slots per sample written by an up2 conv over an H x W SOURCE image (output 2H x 2W)
ASYRP_API int asyrp_conv_stats_tiles_up2(int H, int W, int Cout) {
  int TW, TH, NB, bn, mt;
  if (!conv_halo_ok(H, W)) return 0;
  conv_tile_shape(H, W, 1, &TW, &TH, &NB);
  conv_config(H, W, Cout, 1, &bn, &mt, 4);
  const int tht = TH * mt;
  return ((W + TW - 1) / TW) * ((H + tht - 1) / tht) * 4;
}

ASYRP_API int asyrp_conv_create(const AsyrpConvDesc* d, void** out_op) {
  ASYRP_REQUIRE(d && out_op, "asyrp_conv_create: null argument");
  ASYRP_REQUIRE(d->nseg >= 1 && d->nseg <= kMaxSeg, "asyrp_conv_create: nseg=%d out of range", d->nseg);
  ASYRP_REQUIRE(d->Cout % 64 == 0 || (d->Cout == 16 && d->out_planar != nullptr && d->stats == nullptr &&
                                      d->residual == nullptr && !d->up2 && !d->weight_batched),
                "asyrp_conv_create: Cout=%d must be a multiple of 64 (or 16 with a planar fp32 output)", d->Cout);
  // owned here until it is handed out, so that every rejection below frees it
  std::unique_ptr<ConvOp> op(new ConvOp());
  ConvParams& p = op->p;
  memset(&p, 0, sizeof(p));
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cout = d->Cout;
  bool has3 = false;
  for (int s = 0; s < d->nseg; ++s) has3 = has3 || d->seg[s].mode == 1;
  const int halo = has3 && conv_halo_ok(d->H, d->W);
  conv_tile_shape(d->H, d->W, halo, &p.TW, &p.TH, &p.NB);
  ASYRP_REQUIRE(p.TW * p.TH * p.NB == 128, "asyrp_conv_create: cannot tile H=%d W=%d into 128 pixels", d->H,
                d->W);
  ASYRP_REQUIRE(!(d->weight_batched && p.NB != 1), "asyrp_conv_create: batched weights need NB==1");
  if (d->up2)
    ASYRP_REQUIRE(halo && d->nseg == 1 && !d->weight_batched && !d->out_f32 &&
                      d->out_planar == nullptr && d->out_heads <= 1 && d->a_heads <= 1 && d->residual == nullptr,
                  "asyrp_conv_create: up2 needs one plain 3x3 segment on a source of H %% 16 == 0, W %% 8 == 0");
  p.up2 = d->up2 ? 1 : 0;
  conv_config(d->H, d->W, d->Cout, halo, &op->BN, &op->MT, p.up2 ? 4 : 1);
  p.MT = op->MT;
  const int THT = p.TH * p.MT;
  p.tiles_x = (d->W + p.TW - 1) / p.TW;
  p.tiles_y = (d->H + THT - 1) / THT;
  p.tiles_n = (d->N + p.NB - 1) / p.NB;
  p.m_tiles = p.tiles_x * p.tiles_y * p.tiles_n;
  p.n_tiles = (d->Cout / op->BN) * (p.up2 ? 4 : 1);
  {
    // x / dv == umulhi(x, 2^32/dv + 1) for all x with x*dv < 2^32; the largest dividend is the tile count
    const unsigned long long xmax = static_cast<unsigned long long>(p.m_tiles) * p.n_tiles;
    auto magic = [xmax](uint32_t dv) -> uint32_t {
      if (dv <= 1) return 0u;
      if (xmax * dv >= (1ull << 32)) return 1u;
      return static_cast<uint32_t>((1ull << 32) / dv) + 1u;
    };
    p.mul_m = magic(p.m_tiles);
    p.mul_x = magic(p.tiles_x);
    p.mul_xy = magic(p.tiles_x * p.tiles_y);
    ASYRP_REQUIRE(xmax < (1ull << 31), "asyrp_conv_create: %llu tiles exceed the tile-index range", xmax);
  }
  p.row_bytes = p.NB * p.TW * 128;
  p.nseg = d->nseg;
  bool any3 = false;
  int ktot = 0;
  for (int s = 0; s < d->nseg; ++s) {
    const AsyrpConvSeg& sg = d->seg[s];
    ASYRP_REQUIRE(sg.C % 64 == 0 && sg.C > 0, "asyrp_conv_create: segment channels %d not a multiple of 64", sg.C);
    ASYRP_REQUIRE(sg.mode >= 0 && sg.mode <= 2, "asyrp_conv_create: bad segment mode %d", sg.mode);
    const int mode = (sg.mode == 1 && halo) ? 3 : sg.mode;
    p.seg[s].nchunks = sg.C / 64;
    p.seg[s].mode = mode;
    p.seg[s].kbase = ktot;
    p.seg[s].C = sg.C;
    p.seg[s].affine = sg.affine;
    p.seg[s].aff_stride = sg.affine_stride;
    p.seg[s].act = (sg.act == 1 && silu_tanh_enabled()) ? 2 : sg.act;
    ASYRP_REQUIRE(!(sg.affine != nullptr && sg.mode == 2), "asyrp_conv_create: no fused affine on stride-2 segments");
    if (sg.gn_gamma != nullptr) {
      ASYRP_REQUIRE(sg.affine == nullptr && sg.gn_sums_a != nullptr && sg.gn_beta != nullptr && sg.gn_Ca > 0 &&
                        (sg.gn_Ca + sg.gn_Cb) % 64 == 0 && sg.gn_Ca % 2 == 0 && (sg.gn_Cb == 0 || sg.gn_sums_b != nullptr) &&
                        sg.gn_hw > 0 && sg.mode != 2 && p.NB == 1,
                    "asyrp_conv_create: in-kernel GroupNorm needs sums, gamma / beta, a stride-1 segment and tiles "
                    "inside one sample");
      p.seg[s].gn_sums[0] = sg.gn_sums_a;
      p.seg[s].gn_sums[1] = sg.gn_sums_b;
      p.seg[s].gn_C[0] = sg.gn_Ca;
      p.seg[s].gn_C[1] = sg.gn_Cb;
      p.seg[s].gn_gamma = sg.gn_gamma;
      p.seg[s].gn_beta = sg.gn_beta;
      p.seg[s].gn_ss = sg.gn_scale_shift;
      p.seg[s].gn_ss_stride = sg.gn_ss_stride;
      p.seg[s].gn_eps = sg.gn_eps;
      p.seg[s].gn_inv_count = 1.0f / (static_cast<float>(sg.gn_hw) * static_cast<float>((sg.gn_Ca + sg.gn_Cb) / 32));
      p.seg[s].gn_off = sg.gn_off;
      p.any_transform = 1;
      p.any_gn = 1;
    }
    if (sg.affine != nullptr) p.any_transform = 1;
    ktot += (sg.mode == 0 ? 1 : (p.up2 ? 4 : 9)) * sg.C;
    any3 = any3 || sg.mode == 1;
    uint64_t dims[5], strides[4];
    uint32_t box[5];
    const uint64_t C = sg.C;
    const uint64_t L = sg.ld > 0 ? sg.ld : sg.C;  // pixel pitch
    ASYRP_REQUIRE(L >= C && L % 8 == 0, "asyrp_conv_create: segment ld=%d must be >= C and a multiple of 8", sg.ld);
    ASYRP_REQUIRE(!(sg.mode == 2 && L != C), "asyrp_conv_create: stride-2 segments need a dense source");
    if (sg.mode != 2) {
      const uint64_t H = d->H, W = d->W;
      const uint64_t ah = (s == 0 && d->a_heads > 1) ? d->a_heads : 1;
      ASYRP_REQUIRE(ah == 1 || (sg.mode == 0 && d->nseg == 1 && d->N % ah == 0 && L >= ah * C),
                    "asyrp_conv_create: a_heads needs one 1x1 segment with ld >= heads*C");
      dims[0] = C; dims[1] = W; dims[2] = d->N / ah; dims[3] = ah; dims[4] = H;
      strides[0] = L * 2; strides[1] = H * W * L * 2; strides[2] = (ah > 1 ? C : W * L) * 2; strides[3] = W * L * 2;
      box[0] = 64; box[1] = mode == 3 ? p.TW + 2 : p.TW; box[2] = p.NB; box[3] = 1;
      box[4] = (mode == 1 || mode == 3) ? THT + 2 : THT;
    } else {
      const uint64_t Hi = 2 * d->H, Wi = 2 * d->W;
      dims[0] = 2 * C; dims[1] = Wi / 2; dims[2] = d->N; dims[3] = 2; dims[4] = Hi / 2;
      strides[0] = 2 * C * 2; strides[1] = Hi * Wi * C * 2; strides[2] = Wi * C * 2; strides[3] = 2 * Wi * C * 2;
      box[0] = 64; box[1] = p.TW; box[2] = p.NB; box[3] = 1; box[4] = THT;
    }
    int rc = encode_tensor_map(&p.tmA[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, sg.src, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc != ASYRP_OK) return rc;
  }
  {
    const uint64_t bh = (d->weight_batched && d->b_heads > 1) ? d->b_heads : 1;
    uint64_t dims[4] = {static_cast<uint64_t>(ktot), static_cast<uint64_t>(d->Cout) * (p.up2 ? 4 : 1), bh,
                        static_cast<uint64_t>(d->weight_batched ? d->N / bh : 1)};
    const uint64_t wld = d->weight_ld > 0 ? d->weight_ld : ktot;
    const uint64_t wbs = d->weight_batch_stride > 0 ? static_cast<uint64_t>(d->weight_batch_stride) : wld * d->Cout;
    ASYRP_REQUIRE(wld >= static_cast<uint64_t>(ktot) && wld % 8 == 0 && wbs % 8 == 0,
                  "asyrp_conv_create: weight_ld / weight_batch_stride must cover K and be multiples of 8");
    ASYRP_REQUIRE(bh == 1 || wld >= bh * static_cast<uint64_t>(ktot), "asyrp_conv_create: b_heads needs weight_ld >= heads*K");
    // dim 2 = head (column slices of width K inside a row of weight_ld elements), dim 3 = sample
    uint64_t strides[3] = {wld * 2, (bh > 1 ? static_cast<uint64_t>(ktot) : wbs) * 2, wbs * 2};
    uint32_t box[4] = {64, static_cast<uint32_t>(op->BN), 1, 1};
    int rc = encode_tensor_map(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, d->weight, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc != ASYRP_OK) return rc;
  }
  {
    // K-loop schedule.  Single activation ring: heavy chunks (3x3 taps) in order, then the light chunks (1x1
    // segments).  Separate rings (halo tiles with 1x1 segments): the light chunks are spread evenly behind the heavy
    // ones (H0 L0 L1 H1 L2 L3 ...), so that each pair of light slots is refilled during a heavy stage.
    uint8_t heavy[64], light[64];
    int nh = 0, nl = 0;
    for (int sg_ = 0; sg_ < d->nseg; ++sg_)
      for (int ch = 0; ch < p.seg[sg_].nchunks; ++ch) {
        ASYRP_REQUIRE(nh + nl < 64 && ch < 64, "asyrp_conv_create: more than 64 K chunks (%d channels) per tile", ktot);
        (p.seg[sg_].mode == 0 ? light[nl++] : heavy[nh++]) = static_cast<uint8_t>((sg_ << 6) | ch);
      }
    const bool spread = halo && nl > 0 && nh > 0;
    int il = 0, n = 0;
    for (int ih = 0; ih < nh; ++ih) {
      p.sched[n++] = heavy[ih];
      const int upto = spread ? (nl * (ih + 1) + nh - 1) / nh : ((ih == nh - 1) ? nl : 0);
      while (il < upto) p.sched[n++] = light[il++];
    }
    while (il < nl) p.sched[n++] = light[il++];
    p.n_sched = n;
  }
  p.b_batched = d->weight_batched;
  p.a_heads = d->a_heads > 1 ? d->a_heads : 1;
  p.b_heads = (d->weight_batched && d->b_heads > 1) ? d->b_heads : 1;
  p.out_heads = d->out_heads > 1 ? d->out_heads : 1;
  p.out_ld = d->Cout * p.out_heads;
  p.out_f32 = d->out_f32;
  ASYRP_REQUIRE(!d->out_f32 || (d->residual == nullptr && d->stats == nullptr && d->out_planar == nullptr),
                "asyrp_conv_create: out_f32 excludes residual / stats / planar output");
  ASYRP_REQUIRE(p.out_heads == 1 || (d->N % p.out_heads == 0 && d->stats == nullptr && d->out_planar == nullptr),
                "asyrp_conv_create: out_heads needs N %% heads == 0, no stats / planar output");
  p.a_stage_bytes = halo ? (((THT + 2) * (p.TW + 2) * 128u + 1023u) / 1024u) * 1024u
                         : (any3 ? THT + 2 : THT) * p.row_bytes;
  const uint32_t b_stage = op->BN * 128;
  // accumulator staging tile of the epilogue: 128 pixel rows x (MT*BN + 4) fp32
  const uint32_t staging = 128u * (op->MT * op->BN + 4) * 4u;
  // operand rings: everything the 227 KB of shared memory leaves after the staging tile, barriers and the statistics
  // scratch.  Activations: 3-4 stages; weights: as deep as fits (<= 16 stages) — small-N tiles issue an MMA group
  // every ~100 cycles, so the weight prefetch must run many K steps ahead of the ~1 us TMA latency.
  const uint32_t ring_budget = 227 * 1024 - 1024 /*alignment*/ - 1024 /*barriers*/ - 2 * 4 * op->BN * 4 /*stats*/ -
                               2048 /*per-tile GroupNorm group statistics: 2 x 3 x 32 float2*/ - staging;
  bool has_light = false;
  for (int s = 0; s < d->nseg; ++s) has_light = has_light || d->seg[s].mode == 0;
  p.l_stages = 0;
  p.l_stage_bytes = THT * p.row_bytes;
  p.a_stages = (p.MT == 2 || halo) ? 3 : 4;
  if (halo && has_light) {
    // separate rings: 2 heavy slots (load + transform of one overlap the MMAs of the other; the light MMAs give the
    // slack) + 2 light slots, if at least 3 weight stages still fit
    const uint32_t need = 2 * p.a_stage_bytes + 2 * p.l_stage_bytes;
    if (need + 3 * b_stage <= ring_budget) { p.a_stages = 2; p.l_stages = 2; }
  }
#ifdef ASYRP_TRACE
  if (const char* e = getenv("ASYRP_A_STAGES")) {  // diagnostic build: ring depths from the environment
    const int v = atoi(e);
    if (v >= 2) p.a_stages = v;
  }
  if (const char* e = getenv("ASYRP_L_STAGES")) {
    const int v = atoi(e);
    if (v >= 2 && p.l_stages != 0) p.l_stages = v;
  }
#endif
  const uint32_t a_ring = p.a_stages * p.a_stage_bytes + p.l_stages * p.l_stage_bytes;
  while (p.l_stages == 0 && p.a_stages > 2 && p.a_stages * p.a_stage_bytes + 2 * b_stage > ring_budget) --p.a_stages;
  int bs = static_cast<int>((ring_budget - (p.l_stages ? a_ring : p.a_stages * p.a_stage_bytes)) / b_stage);
  p.b_stages = bs > 16 ? 16 : (bs < 2 ? 2 : bs);
#ifdef ASYRP_TRACE
  if (const char* e = getenv("ASYRP_B_STAGES_MAX")) {  // diagnostic build: cap the weight ring depth
    const int cap = atoi(e);
    if (cap >= 2 && p.b_stages > cap) p.b_stages = cap;
  }
#endif
  p.ebias = d->ebias;
  p.ebias_stride = d->ebias_stride;
  p.out_planar = d->out_planar;
  p.planar_c = d->planar_c;
  ASYRP_REQUIRE(d->out_planar == nullptr || (d->planar_c >= 1 && d->planar_c <= 8),
                "asyrp_conv_create: planar_c=%d out of range", d->planar_c);
  p.res = static_cast<const __half*>(d->residual);
  p.res_scale = d->res_scale;
  p.acc_scale = d->acc_scale;
  p.scales = d->scales;
  p.res_mode = d->residual != nullptr ? d->res_mode : 0;
  ASYRP_REQUIRE(p.res_mode >= 0 && p.res_mode <= 2, "asyrp_conv_create: res_mode %d", d->res_mode);
  ASYRP_REQUIRE(p.res_mode == 0 || (!p.up2 && p.out_heads == 1 && !d->out_f32 && d->out_planar == nullptr &&
                                    (p.res_mode == 2 || (d->H % 2 == 0 && d->W % 2 == 0))),
                "asyrp_conv_create: resampled residual needs a plain NHWC fp16 output (even H, W for nearest-x2)");
  p.out = static_cast<__half*>(d->out);
  p.stats = d->stats;
  p.sums_out = d->sums_out;
  ASYRP_REQUIRE(d->sums_out == nullptr || (d->stats != nullptr && p.NB == 1 && op->BN >= 32),
                "asyrp_conv_create: sums_out needs stats and tiles inside one sample");
  op->smem_bytes = 1024 + static_cast<size_t>(p.a_stages) * p.a_stage_bytes +
                   static_cast<size_t>(p.l_stages) * p.l_stage_bytes + static_cast<size_t>(p.b_stages) * b_stage +
                   staging + (3 * (p.a_stages + p.l_stages) + 2 * p.b_stages) * 8 + 2 * 4 * op->BN * 4 +
                   2 * kMaxSeg * 32 * sizeof(float2);
  ASYRP_REQUIRE(op->smem_bytes <= 227 * 1024, "asyrp_conv_create: smem %zu too large", op->smem_bytes);
  const int sms = sm_count();
  if (sms <= 0) return ASYRP_ERR_NO_DEVICE;
  const int total = p.m_tiles * p.n_tiles;
  op->grid = total < sms ? total : sms;
  cudaError_t e = cudaFuncSetAttribute(conv_kernel_ptr(op->BN, op->MT),
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) {
    set_error("asyrp_conv_create: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    return ASYRP_ERR_CUDA;
  }
  *out_op = op.release();
  return ASYRP_OK;
}

ASYRP_API int asyrp_conv_launch(void* handle, void* stream) {
  ASYRP_REQUIRE(handle, "asyrp_conv_launch: null op");
  ConvOp* op = static_cast<ConvOp*>(handle);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  void* args[] = {&op->p};
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3(op->grid);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = op->smem_bytes;
  cfg.stream = st;
  cfg.attrs = attr;
  if (pdl_enabled()) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg.numAttrs;
  }
  ASYRP_CHECK_CUDA(cudaLaunchKernelExC(&cfg, conv_kernel_ptr(op->BN, op->MT), args));
  return ASYRP_OK;
}

// h2 = c0*h + c_i*delta_h_i (ddpm/diffusion.py:512-516) is evaluated by the last DeltaBlock conv's epilogue;
// the coefficients are per-call arguments of the reference forward(), hence adjustable after creation.
ASYRP_API int asyrp_conv_set_scales(void* handle, float acc_scale, float res_scale) {
  ASYRP_REQUIRE(handle, "asyrp_conv_set_scales: null op");
  ConvOp* op = static_cast<ConvOp*>(handle);
  op->p.acc_scale = acc_scale;
  op->p.res_scale = res_scale;
  return ASYRP_OK;
}

ASYRP_API void asyrp_conv_destroy(void* handle) { delete static_cast<ConvOp*>(handle); }

#ifdef ASYRP_TRACE
// diagnostic build only: device buffer [grid][kTraceRoles][kTraceLen] int64 receiving the pipeline timeline
ASYRP_API int asyrp_conv_set_trace(void* handle, long long* buf) {
  ASYRP_REQUIRE(handle, "asyrp_conv_set_trace: null op");
  static_cast<ConvOp*>(handle)->p.trace = buf;
  return static_cast<ConvOp*>(handle)->grid;
}
#endif
// SiLU of the fused operand transform: 1 = one tanh.approx (default), 0 = ex2 + rcp; negative: back to the default
// (ASYRP_SILU_TANH).  Affects ops created afterwards.
ASYRP_API int asyrp_set_silu_tanh(int enabled) {
  g_silu_tanh = enabled < 0 ? -1 : (enabled ? 1 : 0);
  return ASYRP_OK;
}

}  // extern "C"
