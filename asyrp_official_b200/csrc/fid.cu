// Inception-v3 pool features (the FID variant of pytorch-fid) and the set statistics of FID and KID.
//
//   x299 = 2 * bilinear_299(floor(clamp((x + 1) / 2 * 255 + 1/2, 0, 255)) / 255) - 1 as NHWC, 4 channels
//                                                                                        fid_pack_kernel<SavedPng>
//   the same from the u8 of a decoded image file (u8 NHWC), bit-identical for the same u8  fid_pack_kernel<DecodedU8>
//   BasicConv2d = conv (1x1, 3x3, 5x5, 1x7, 7x1, 1x3, 3x1; separate vertical / horizontal padding) + folded BN + ReLU,
//     written into a channel slice [0, cstore) of rows of pitch ldo                     tf32_gemm.cuh (kEpiReluSlice)
//   max-pool 3x3 / 2 (stem, InceptionB / D), avg-pool 3x3 / 1 pad 1 without the padding (FIDInceptionA / C / E_1),
//     max-pool 3x3 / 1 pad 1 (FIDInceptionE_2), each into a channel slice             fid_pool_kernel
//   pool features = mean over the 8 x 8 pixels of Mixed_7c                             fid_mean_kernel
//   mu, Sigma = column means and (n - 1)-normalised centred covariance, fp64           fid_colmean_kernel, fid_gram
//   sum_ij (x_i . y_j / d + 1)^3, fp64, optionally without i == j                      fid_gram, fid_sum_kernel
//   the same over gathered rows, one sum per index subset (subset KID)                 fid_gram<gather>, fid_sum
//
// Every reduction runs in a fixed order and no kernel uses atomics or mixes samples, so an image's features are the
// same bits whatever batch it is in, and the statistics of a set are the same bits whatever launches produced its rows.
#include <cfloat>
#include <climits>

#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kGramTile = 64;     // fp64 gram tile: 64 x 64 outputs per CTA
constexpr int kGramK = 16;        // contraction slice staged in shared memory
constexpr int kGramThreads = 256; // each thread 4 x 4 outputs: rows ty + 16 a, columns tx + 16 b
constexpr int kSumThreads = 256;

enum PoolMode : int { kPoolMax3s2 = 0, kPoolAvg3s1 = 1, kPoolMax3s1 = 2 };

// The pixel readers of fid_pack_kernel: px(b, c, y, x) = q / 255 (fp32, rounded once) of the u8 value q of channel c
// at (y, x) of image b.
// SavedPng (common.h): x fp32 NCHW [B][3][H][W]; q = the u8 save_image writes for x.
// DecodedU8: q read from u8 NHWC [B][H][W][3], a decoded image file
struct DecodedU8 {
  const uint8_t* __restrict__ x;
  int H, W;
  __device__ float operator()(size_t b, int c, int yy, int xx) const {
    return __fdiv_rn(static_cast<float>(x[((b * H + yy) * W + xx) * 3 + c]), 255.f);
  }
};

// out[b][Y][X] = (2 * bilinear(px)(Y, X) - 1, channels 0..2; 0).  The resize H x W -> S x S is
// F.interpolate(mode='bilinear', align_corners=False) as in faceparse_pack_kernel: source row
// (Y + .5) * H / S - .5 clamped at 0, rows y0 = floor, y1 = min(y0 + 1, H - 1) weighted 1 - l, l; rows blended first.
// The blend sees only px's values, so both readers give the same bits for the same q.
template <class Px>
__global__ void fid_pack_kernel(Px px, float* __restrict__ out, int B, int H, int W, int S) {
  pdl_trigger();
  pdl_wait();
  const float sh = static_cast<float>(H) / static_cast<float>(S), sw = static_cast<float>(W) / static_cast<float>(S);
  const size_t total = static_cast<size_t>(B) * S * S;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int X = static_cast<int>(i % S), Y = static_cast<int>((i / S) % S);
    const size_t b = i / (static_cast<size_t>(S) * S);
    const float fy = fmaxf((Y + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((X + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min(static_cast<int>(fy), H - 1), x0 = min(static_cast<int>(fx), W - 1);
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - y0, lx = fx - x0;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float top = (1.f - lx) * px(b, c, y0, x0) + lx * px(b, c, y0, x1);
      const float bot = (1.f - lx) * px(b, c, y1, x0) + lx * px(b, c, y1, x1);
      v[c] = 2.f * ((1.f - ly) * top + ly * bot) - 1.f;
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], 0.f);
  }
}

// 3 x 3 pooling of in [N][H][W][C4 float4s] into out [N][Ho][Wo] rows of ldo4 float4s (the first C4 written).
// kPoolMax3s2: max over the window at (2 oy, 2 ox), no padding.  kPoolMax3s1: max over the taps inside the image of
// the window centred on (oy, ox) (padding never wins).  kPoolAvg3s1: the sum of those taps in row-major order from 0,
// divided by their count (count_include_pad=False).
template <int kMode>
__global__ void fid_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C4,
                                int Ho, int Wo, int ldo4) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    const size_t pix = i / C4;
    const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho);
    const size_t n = pix / (static_cast<size_t>(Wo) * Ho);
    const int cy = kMode == kPoolMax3s2 ? 2 * oy + 1 : oy, cx = kMode == kPoolMax3s2 ? 2 * ox + 1 : ox;
    const bool avg = kMode == kPoolAvg3s1;
    float4 m = avg ? make_float4(0.f, 0.f, 0.f, 0.f) : make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
    int cnt = 0;
    for (int y = cy - 1; y <= cy + 1; ++y) {
      if (y < 0 || y >= H) continue;
      for (int xx = cx - 1; xx <= cx + 1; ++xx) {
        if (xx < 0 || xx >= W) continue;
        const float4 v = reinterpret_cast<const float4*>(in)[((n * H + y) * W + xx) * C4 + c4];
        if (avg) {
          m = make_float4(m.x + v.x, m.y + v.y, m.z + v.z, m.w + v.w);
        } else {
          m = make_float4(fmaxf(m.x, v.x), fmaxf(m.y, v.y), fmaxf(m.z, v.z), fmaxf(m.w, v.w));
        }
        ++cnt;
      }
    }
    if (avg) {
      const float c = static_cast<float>(cnt);
      m = make_float4(__fdiv_rn(m.x, c), __fdiv_rn(m.y, c), __fdiv_rn(m.z, c), __fdiv_rn(m.w, c));
    }
    reinterpret_cast<float4*>(out)[pix * ldo4 + c4] = m;
  }
}

// out[n][c] = (in[n][0][c] + in[n][1][c] + ... + in[n][HW - 1][c]) / HW, the sum in pixel order from 0
__global__ void fid_mean_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int HW, int C) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = i / C, c = i % C;
    const float* p = in + n * HW * C + c;
    float s = 0.f;
    for (int k = 0; k < HW; ++k) s += p[static_cast<size_t>(k) * C];
    out[i] = __fdiv_rn(s, static_cast<float>(HW));
  }
}

// mu[j] = (x[0][j] + ... + x[n - 1][j]) / n in fp64, the sum in row order from 0
__global__ void fid_colmean_kernel(const float* __restrict__ x, double* __restrict__ mu, int n, int d) {
  pdl_trigger();
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d) return;
  double s = 0.0;
  for (int r = 0; r < n; ++r) s += static_cast<double>(x[static_cast<size_t>(r) * d + j]);
  mu[j] = s / n;
}

// A 64 x 64 tile of a fp64 gram matrix, each output accumulated over the contraction index in order from 0.
//   kKid false (covariance): out[i][j] = sum_r (x[r][i] - mu[i]) (x[r][j] - mu[j]) / (rows - 1), i, j < cols (= d);
//     rows = n, x = y.
//   kKid true (kernel sum): v = (x[i] . y[j]) / d + 1 over the d features, k = v^3, i < n, j < m (rows = n, cols = m);
//     pairs i == j are skipped when exclude_diag; the CTA's sum of its k (each thread's 16 in order, then a fixed
//     tree) goes to partial[blockIdx.y][blockIdx.x].
//   kGather (with kKid, subset z = blockIdx.z): the same with row i of x read from x[idx_x[z][i]] and row j of y from
//     y[idx_y[z][j]], n = m = the subset size; the sum goes to partial[z][blockIdx.y][blockIdx.x].  The tile order and
//     the tree are those of the plain kernel sum, so a subset's partials are those of the gathered matrices.
template <bool kKid, bool kGather>
__global__ void __launch_bounds__(kGramThreads) fid_gram_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ y,
                                                                const double* __restrict__ mu,
                                                                double* __restrict__ out, int n, int m, int d,
                                                                int exclude_diag, const int* __restrict__ idx_x,
                                                                const int* __restrict__ idx_y) {
  static_assert(kKid || !kGather, "fid_gram_kernel: the gather is a kernel-sum mode");
  pdl_trigger();
  __shared__ double xs[kGramK][kGramTile];
  __shared__ double ys[kGramK][kGramTile];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = blockIdx.y * kGramTile, j0 = blockIdx.x * kGramTile;
  const int kdim = kKid ? d : n;  // contraction length
  pdl_wait();
  // kGather: the source rows of this thread's staging loads, sample ii = t / 16 + 16 q of the tile in load q
  int rx[kGramK * kGramTile / kGramThreads], ry[kGramK * kGramTile / kGramThreads];
  if (kGather) {
    const int* ix = idx_x + static_cast<size_t>(blockIdx.z) * n;
    const int* iy = idx_y + static_cast<size_t>(blockIdx.z) * m;
#pragma unroll
    for (int q = 0; q < kGramK * kGramTile / kGramThreads; ++q) {
      const int ii = (t + kGramThreads * q) / kGramK;
      rx[q] = i0 + ii < n ? ix[i0 + ii] : 0;
      ry[q] = j0 + ii < m ? iy[j0 + ii] : 0;
    }
  }
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < kdim; k0 += kGramK) {
#pragma unroll
    for (int q = 0; q < kGramK * kGramTile / kGramThreads; ++q) {
      const int e = t + kGramThreads * q;
      if (kKid) {  // rows of x / y are samples: 16 consecutive features of 64 samples
        const int ii = e / kGramK, kk = e % kGramK, k = k0 + kk;
        const int r = kGather ? rx[q] : i0 + ii, c = kGather ? ry[q] : j0 + ii;
        xs[kk][ii] = i0 + ii < n ? static_cast<double>(x[static_cast<size_t>(r) * d + k]) : 0.0;
        ys[kk][ii] = j0 + ii < m ? static_cast<double>(y[static_cast<size_t>(c) * d + k]) : 0.0;
      } else {  // rows of x are samples, columns features: 64 consecutive features of 16 samples, centred
        const int kk = e / kGramTile, ii = e % kGramTile, r = k0 + kk;
        const bool ok = r < n;
        xs[kk][ii] = ok ? static_cast<double>(x[static_cast<size_t>(r) * d + i0 + ii]) - mu[i0 + ii] : 0.0;
        ys[kk][ii] = ok ? static_cast<double>(x[static_cast<size_t>(r) * d + j0 + ii]) - mu[j0 + ii] : 0.0;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGramK; ++kk) {
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
  if (!kKid) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
        out[static_cast<size_t>(i0 + ty + 16 * a) * d + j0 + tx + 16 * b] = acc[a][b] / (n - 1);
    return;
  }
  double s = 0.0;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
      if (i < n && j < m && !(exclude_diag && i == j)) {
        const double v = acc[a][b] / d + 1.0;
        s += v * v * v;
      }
    }
  double* red = &xs[0][0];  // 256 doubles of the (now idle) staging buffer
  red[t] = s;
  __syncthreads();
  for (int h = kGramThreads / 2; h > 0; h >>= 1) {
    if (t < h) red[t] += red[t + h];
    __syncthreads();
  }
  if (t == 0) out[(static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = red[0];
}

// out[z] = the sum of the `count` partials partial[z][0 .. count), z = blockIdx.x: thread t adds partials t, t + 256,
// ... in order, then a fixed tree
__global__ void __launch_bounds__(kSumThreads) fid_sum_kernel(const double* __restrict__ partial, int count,
                                                              double* __restrict__ out) {
  pdl_trigger();
  __shared__ double red[kSumThreads];
  pdl_wait();
  const int t = threadIdx.x;
  const double* p = partial + static_cast<size_t>(blockIdx.x) * count;
  double s = 0.0;
  for (int i = t; i < count; i += kSumThreads) s += p[i];
  red[t] = s;
  __syncthreads();
  for (int h = kSumThreads / 2; h > 0; h >>= 1) {
    if (t < h) red[t] += red[t + h];
    __syncthreads();
  }
  if (t == 0) out[blockIdx.x] = red[0];
}

inline int fid_grid(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

inline bool aligned(const void* p, size_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

// the 64-row gram tiles of `rows` rows, in 64 bits: rows + 63 overflows int near 2^31
inline long long gram_tiles(int rows) { return (static_cast<long long>(rows) + kGramTile - 1) / kGramTile; }

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_fid_pack(const float* x, float* out, int B, int H, int W, int S, void* stream) {
  ASYRP_REQUIRE(B > 0 && H > 0 && W > 0 && S > 0, "asyrp_fid_pack: bad shape B=%d H=%d W=%d S=%d", B, H, W, S);
  ASYRP_REQUIRE(aligned(out, 16), "asyrp_fid_pack: out must be 16-byte aligned (float4 stores)");
  const size_t total = static_cast<size_t>(B) * S * S;
  ASYRP_LAUNCH(fid_pack_kernel<SavedPng>, dim3(fid_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               SavedPng{x, H, W}, out, B, H, W, S);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_pack_u8(const uint8_t* x, float* out, int B, int H, int W, int S, void* stream) {
  ASYRP_REQUIRE(B > 0 && H > 0 && W > 0 && S > 0, "asyrp_fid_pack_u8: bad shape B=%d H=%d W=%d S=%d", B, H, W, S);
  ASYRP_REQUIRE(aligned(out, 16), "asyrp_fid_pack_u8: out must be 16-byte aligned (float4 stores)");
  const size_t total = static_cast<size_t>(B) * S * S;
  ASYRP_LAUNCH(fid_pack_kernel<DecodedU8>, dim3(fid_grid(total, 256)), dim3(256), 0,
               static_cast<cudaStream_t>(stream), DecodedU8{x, H, W}, out, B, H, W, S);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_conv(const float* in, const float* weight, const float* bias, float* out, int N, int H, int W,
                             int Cin, int Cout, int kh, int kw, int stride, int padh, int padw, int ldo, int cstore,
                             void* stream) {
  using namespace tf32gemm;
  ASYRP_REQUIRE(Cin > 0 && Cin % 4 == 0, "asyrp_fid_conv: Cin=%d must be a positive multiple of 4", Cin);
  ASYRP_REQUIRE(Cout > 0 && Cout % kBN == 0, "asyrp_fid_conv: Cout=%d must be a positive multiple of %d", Cout, kBN);
  // the geometry in 64 bits: the kernel's tap coordinates (oy * stride - padh + ky < H + 2 padh, likewise x), K and the
  // output pixel index are int, so the padded extents, Kpad and N Ho Wo must each fit in one
  const long long Hp = H + 2LL * padh, Wp = W + 2LL * padw;
  ASYRP_REQUIRE(N > 0 && H > 0 && W > 0 && kh > 0 && kw > 0 && stride > 0 && padh >= 0 && padw >= 0 && Hp >= kh &&
                    Wp >= kw,
                "asyrp_fid_conv: bad geometry N=%d H=%d W=%d kh=%d kw=%d stride=%d padh=%d padw=%d", N, H, W, kh, kw,
                stride, padh, padw);
  ASYRP_REQUIRE(Hp <= INT_MAX && Wp <= INT_MAX,
                "asyrp_fid_conv: padded extent H + 2 padh=%lld or W + 2 padw=%lld above 2^31 - 1", Hp, Wp);
  constexpr long long kMaxK = INT_MAX / kBK * kBK;  // the largest Kpad in int
  ASYRP_REQUIRE(static_cast<long long>(kh) * kw <= kMaxK / Cin,
                "asyrp_fid_conv: K = kh * kw * Cin = %d * %d * %d above %lld", kh, kw, Cin, kMaxK);
  ASYRP_REQUIRE(cstore > 0 && cstore % 2 == 0 && cstore <= Cout && ldo >= cstore && ldo % 2 == 0,
                "asyrp_fid_conv: cstore=%d must be even and in (0, Cout=%d], ldo=%d even and >= cstore", cstore, Cout,
                ldo);
  ASYRP_REQUIRE(bias != nullptr && aligned(out, 8), "asyrp_fid_conv: needs a bias and an 8-byte aligned out");
  ASYRP_REQUIRE(in != out, "asyrp_fid_conv: out must not alias in");
  const long long Ho = (Hp - kh) / stride + 1, Wo = (Wp - kw) / stride + 1;
  const long long NHo = N * Ho;  // below 2^62; with NHo < 2^31 the product with Wo is too
  ASYRP_REQUIRE(NHo < (1LL << 31) / kBM * kBM && NHo * Wo < (1LL << 31) / kBM * kBM,
                "asyrp_fid_conv: too many output pixels");
  Tf32ConvParams p;
  p.in = in; p.w = weight; p.bias = bias; p.residual = nullptr; p.prelu = nullptr; p.out = out;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.kw = kw; p.stride = stride; p.pad = padh;
  p.padw = padw; p.ldo = ldo; p.cstore = cstore;
  p.Ho = static_cast<int>(Ho);
  p.Wo = static_cast<int>(Wo);
  p.K = kh * kw * Cin;
  p.Kpad = (p.K + kBK - 1) / kBK * kBK;
  p.M = static_cast<int>(NHo * Wo);
  return launch_tf32_conv<kEpiReluSlice>(p, static_cast<cudaStream_t>(stream));
}

ASYRP_API int asyrp_fid_pool(const float* in, float* out, int N, int H, int W, int C, int mode, int ldo,
                             void* stream) {
  ASYRP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && ldo >= C && ldo % 4 == 0,
                "asyrp_fid_pool: bad shape N=%d H=%d W=%d C=%d ldo=%d", N, H, W, C, ldo);
  ASYRP_REQUIRE(mode >= kPoolMax3s2 && mode <= kPoolMax3s1, "asyrp_fid_pool: mode=%d not in 0..2", mode);
  ASYRP_REQUIRE(mode != kPoolMax3s2 || (H >= 3 && W >= 3), "asyrp_fid_pool: H=%d W=%d below the 3 x 3 window", H, W);
  ASYRP_REQUIRE(aligned(in, 16) && aligned(out, 16), "asyrp_fid_pool: in and out must be 16-byte aligned");
  ASYRP_REQUIRE(in != out, "asyrp_fid_pool: out must not alias in");
  const int Ho = mode == kPoolMax3s2 ? (H - 3) / 2 + 1 : H, Wo = mode == kPoolMax3s2 ? (W - 3) / 2 + 1 : W;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * (C / 4);
  const dim3 grid(fid_grid(total, 256));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (mode == kPoolMax3s2) {
    ASYRP_LAUNCH(fid_pool_kernel<kPoolMax3s2>, grid, dim3(256), 0, st, in, out, N, H, W, C / 4, Ho, Wo, ldo / 4);
  } else if (mode == kPoolAvg3s1) {
    ASYRP_LAUNCH(fid_pool_kernel<kPoolAvg3s1>, grid, dim3(256), 0, st, in, out, N, H, W, C / 4, Ho, Wo, ldo / 4);
  } else {
    ASYRP_LAUNCH(fid_pool_kernel<kPoolMax3s1>, grid, dim3(256), 0, st, in, out, N, H, W, C / 4, Ho, Wo, ldo / 4);
  }
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_mean(const float* in, float* out, int N, int HW, int C, void* stream) {
  ASYRP_REQUIRE(N > 0 && HW > 0 && C > 0, "asyrp_fid_mean: bad shape N=%d HW=%d C=%d", N, HW, C);
  const size_t total = static_cast<size_t>(N) * C;
  ASYRP_LAUNCH(fid_mean_kernel, dim3(fid_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), in, out,
               N, HW, C);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_moments(const float* x, double* mu, double* sigma, int n, int d, void* stream) {
  ASYRP_REQUIRE(n >= 2 && d > 0 && d % kGramTile == 0 && d / kGramTile <= kMaxGridYZ,
                "asyrp_fid_moments: bad shape n=%d d=%d (n >= 2, d a multiple of %d)", n, d, kGramTile);
  ASYRP_REQUIRE(static_cast<long long>(n) * d < (1LL << 40), "asyrp_fid_moments: n * d too large");
  // the gram kernel steps through the n rows 16 at a time in int
  ASYRP_REQUIRE(n <= INT_MAX - kGramK + 1, "asyrp_fid_moments: n=%d above %d rows", n, INT_MAX - kGramK + 1);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ASYRP_LAUNCH(fid_colmean_kernel, dim3((d + 255) / 256), dim3(256), 0, st, x, mu, n, d);
  ASYRP_LAUNCH(fid_gram_kernel<false, false>, dim3(d / kGramTile, d / kGramTile), dim3(kGramThreads), 0, st, x, x,
               static_cast<const double*>(mu), sigma, n, d, d, 0, static_cast<const int*>(nullptr),
               static_cast<const int*>(nullptr));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_kernel_sum_partials(int n, int m) {
  // fid_sum_kernel's threads step through the count by kSumThreads in int: count + kSumThreads - 1 must fit in one
  const long long count = gram_tiles(n) * gram_tiles(m);
  return n > 0 && m > 0 && count <= INT_MAX - kSumThreads + 1 ? static_cast<int>(count) : -1;
}

ASYRP_API int asyrp_fid_kernel_sum(const float* x, const float* y, double* partial, double* out, int n, int m, int d,
                                   int exclude_diag, void* stream) {
  ASYRP_REQUIRE(n > 0 && m > 0 && d > 0 && d % kGramK == 0,
                "asyrp_fid_kernel_sum: bad shape n=%d m=%d d=%d (d a multiple of %d)", n, m, d, kGramK);
  ASYRP_REQUIRE(n <= kMaxGridYZ * kGramTile, "asyrp_fid_kernel_sum: n=%d too large (above %d rows)", n,
                kMaxGridYZ * kGramTile);
  ASYRP_REQUIRE(exclude_diag == 0 || exclude_diag == 1, "asyrp_fid_kernel_sum: exclude_diag=%d must be 0 or 1",
                exclude_diag);
  const int count = asyrp_fid_kernel_sum_partials(n, m);
  ASYRP_REQUIRE(count > 0, "asyrp_fid_kernel_sum: n=%d x m=%d too large (above %d partials)", n, m,
                INT_MAX - kSumThreads + 1);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(static_cast<unsigned>(gram_tiles(m)), static_cast<unsigned>(gram_tiles(n)));
  ASYRP_LAUNCH(fid_gram_kernel<true, false>, grid, dim3(kGramThreads), 0, st, x, y,
               static_cast<const double*>(nullptr), partial, n, m, d, exclude_diag, static_cast<const int*>(nullptr),
               static_cast<const int*>(nullptr));
  ASYRP_LAUNCH(fid_sum_kernel, dim3(1), dim3(kSumThreads), 0, st, static_cast<const double*>(partial), count, out);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_fid_kernel_sum_subsets_partials(int s, int subsets) {
  const long long tiles = gram_tiles(s);
  const long long count = tiles * tiles * subsets;
  return s > 0 && subsets > 0 && count < (1LL << 31) ? static_cast<int>(count) : -1;
}

ASYRP_API int asyrp_fid_kernel_sum_subsets(const float* x, const float* y, const int* idx_x, const int* idx_y,
                                           double* partial, double* out, int n, int m, int s, int subsets, int d,
                                           int exclude_diag, void* stream) {
  ASYRP_REQUIRE(n > 0 && m > 0 && s > 0 && subsets > 0 && d > 0,
                "asyrp_fid_kernel_sum_subsets: bad shape n=%d m=%d s=%d subsets=%d d=%d", n, m, s, subsets, d);
  ASYRP_REQUIRE(d % kGramK == 0, "asyrp_fid_kernel_sum_subsets: d=%d must be a multiple of %d", d, kGramK);
  ASYRP_REQUIRE(subsets <= kMaxGridYZ, "asyrp_fid_kernel_sum_subsets: subsets=%d above %d", subsets, kMaxGridYZ);
  ASYRP_REQUIRE(exclude_diag == 0 || exclude_diag == 1,
                "asyrp_fid_kernel_sum_subsets: exclude_diag=%d must be 0 or 1", exclude_diag);
  ASYRP_REQUIRE(!exclude_diag || s >= 2, "asyrp_fid_kernel_sum_subsets: exclude_diag needs s >= 2 (s=%d)", s);
  ASYRP_REQUIRE(asyrp_fid_kernel_sum_subsets_partials(s, subsets) > 0,
                "asyrp_fid_kernel_sum_subsets: s=%d x subsets=%d too large", s, subsets);
  ASYRP_REQUIRE(idx_x != nullptr && idx_y != nullptr, "asyrp_fid_kernel_sum_subsets: needs idx_x and idx_y");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int tiles = (s + kGramTile - 1) / kGramTile;
  ASYRP_LAUNCH(fid_gram_kernel<true, true>, dim3(tiles, tiles, subsets), dim3(kGramThreads), 0, st, x, y,
               static_cast<const double*>(nullptr), partial, s, s, d, exclude_diag, idx_x, idx_y);
  ASYRP_LAUNCH(fid_sum_kernel, dim3(subsets), dim3(kSumThreads), 0, st, static_cast<const double*>(partial),
               tiles * tiles, out);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
