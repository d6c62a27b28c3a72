// Face-parsing BiSeNet (BiSeNet(n_classes=19), eval mode) and the segmentation consistency of an edit: the fraction of
// output pixels whose argmax label equals the label of the same pixel of its source image.
//
//   x512   = normalise(resize_512(clamp(x, -1, 1) / 2 + 1/2)) as NHWC, 4 channels      faceparse_pack_kernel
//   ResNet-18: conv 7x7/2 + BN + ReLU, max-pool 3x3/2 pad 1, 8 BasicBlocks              tf32_gemm.cuh (kEpiRelu,
//     out = relu(shortcut + BN2(conv2(relu(BN1(conv1(x))))))                            kEpiBias, kEpiResidualRelu),
//                                                                                       faceparse_maxpool_kernel
//   context path: avg = ConvBNReLU1x1(mean_hw(feat32))                                  faceparse_gate_kernel
//     ARM(x)      = f * sigmoid(BN(conv1x1(mean_hw(f)))), f = ConvBNReLU3x3(x)          faceparse_gate_kernel
//     s32, s16    = ARM(feat) + avg | up32, materialised at twice the size (nearest)    faceparse_apply_kernel
//   FFM: f = ConvBNReLU1x1(cat[feat8, up16]) as two GEMMs (the second adds the first),
//        out = f * sigmoid(conv2(relu(conv1(mean_hw(f))))) + f                          faceparse_gate_kernel, _apply
//   head: ConvBNReLU3x3, conv1x1 to n_classes (Cout zero-padded to 64)                  tf32_gemm.cuh
//   labels = argmax_c bilinear_align_corners(logits, 512 x 512)                         faceparse_upsample_argmax_kernel
//   agree[j] = #pixels where labels(edited[j]) == labels(src[(row0 + j) % B])          (kPair: no label map stored)
//
// BatchNorm is folded into the conv weights and biases on the host.  Activations are fp32 NHWC.  Every reduction runs
// in a fixed order; the only atomics are integer adds of the agreement counts, which are exact.  No kernel mixes
// samples, so an image's logits and labels are the same bits whatever batch it is in.
#include <cfloat>

#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kGateThreads = 512;
constexpr int kGateMaxC = 512;
constexpr int kArgmaxThreads = 256;
constexpr int kMaxClasses = 64;
// dynamic shared memory of the upsample-argmax kernel: Wi * ncls blended floats per label map (two maps with kPair);
// with kPair's static warp_same[] the admitted 48 KB is past the default 48 KB per block, so both launches opt in
constexpr int kArgmaxSmemBytes = 48 * 1024;

__device__ __forceinline__ float gate_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float activate(float v, int act) {
  return act == 1 ? fmaxf(v, 0.f) : act == 2 ? 1.f / (1.f + expf(-v)) : v;
}

// out[b][Y][X][c] = (bilinear(clamp(x[b][c], -1, 1) * 0.5 + 0.5)(Y, X) - mean[c]) / std[c], channel 3 zero; the resize
// H x W -> S x S is F.interpolate(mode='bilinear', align_corners=False): source row (Y + .5) * H / S - .5 clamped at
// 0, the two rows y0 = floor, y1 = min(y0 + 1, H - 1) weighted 1 - l, l (likewise columns), rows blended first.
__global__ void faceparse_pack_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int H, int W,
                                      int S) {
  pdl_trigger();
  pdl_wait();
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  const float sh = static_cast<float>(H) / static_cast<float>(S), sw = static_cast<float>(W) / static_cast<float>(S);
  const size_t total = static_cast<size_t>(B) * S * S;
  const size_t plane = static_cast<size_t>(H) * W;
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
      const float* img = x + (b * 3 + c) * plane;
      auto px = [&](int yy, int xx) {
        return fminf(fmaxf(img[static_cast<size_t>(yy) * W + xx], -1.f), 1.f) * 0.5f + 0.5f;
      };
      const float top = (1.f - lx) * px(y0, x0) + lx * px(y0, x1);
      const float bot = (1.f - lx) * px(y1, x0) + lx * px(y1, x1);
      v[c] = ((1.f - ly) * top + ly * bot - mean[c]) / stdv[c];
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], 0.f);
  }
}

// MaxPool2d(3, stride 2, padding 1) over fp32 NHWC: padding taps are skipped (they are -inf in torch)
__global__ void faceparse_maxpool_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W,
                                         int C4, int Ho, int Wo) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    const size_t pix = i / C4;
    const int ox = static_cast<int>(pix % Wo), oy = static_cast<int>((pix / Wo) % Ho);
    const size_t n = pix / (static_cast<size_t>(Wo) * Ho);
    float4 m = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
    for (int dy = -1; dy <= 1; ++dy) {
      const int y = 2 * oy + dy;
      if (y < 0 || y >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int xx = 2 * ox + dx;
        if (xx < 0 || xx >= W) continue;
        const float4 v = reinterpret_cast<const float4*>(in)[((n * H + y) * W + xx) * C4 + c4];
        m = make_float4(fmaxf(m.x, v.x), fmaxf(m.y, v.y), fmaxf(m.z, v.z), fmaxf(m.w, v.w));
      }
    }
    reinterpret_cast<float4*>(out)[i] = m;
  }
}

// The gate of sample n (one CTA per sample): m = mean over the HW pixels of in[n] (thread t sums channel t % C over
// pixels t / C, t / C + 512 / C, ...; the 512 / C partials of a channel are added in order), h = act1(w1 m + b1) (a warp
// per output, lane partials then a butterfly), and, when w2 is given, out = act2(w2 h + b2) (a thread per output, in
// order), else out = h.  w1 [C1][C], w2 [C2][C1]; biases may be null; act 0 none, 1 ReLU, 2 sigmoid.
__global__ void __launch_bounds__(kGateThreads) faceparse_gate_kernel(const float* __restrict__ in,
                                                                      const float* __restrict__ w1,
                                                                      const float* __restrict__ b1, int C1, int act1,
                                                                      const float* __restrict__ w2,
                                                                      const float* __restrict__ b2, int C2, int act2,
                                                                      float* __restrict__ out, int HW, int C) {
  pdl_trigger();
  __shared__ float part[kGateThreads];
  __shared__ float mean[kGateMaxC];
  __shared__ float hidden[kGateMaxC];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int J = kGateThreads / C, c = t % C, j = t / C;
  const float* X = in + static_cast<size_t>(blockIdx.x) * HW * C;
  pdl_wait();
  float s = 0.f;
  for (int p = j; p < HW; p += J) s += X[static_cast<size_t>(p) * C + c];
  part[t] = s;
  __syncthreads();
  if (t < C) {
    float tot = 0.f;
    for (int k = 0; k < J; ++k) tot += part[k * C + t];
    mean[t] = tot / static_cast<float>(HW);
  }
  __syncthreads();
  for (int k = warp; k < C1; k += kGateThreads / 32) {
    const float* w = w1 + static_cast<size_t>(k) * C;
    float v = 0.f;
    for (int i = lane; i < C; i += 32) v += w[i] * mean[i];
    v = gate_warp_sum(v);
    if (lane == 0) hidden[k] = activate(v + (b1 != nullptr ? b1[k] : 0.f), act1);
  }
  __syncthreads();
  if (w2 == nullptr) {
    if (t < C1) out[static_cast<size_t>(blockIdx.x) * C1 + t] = hidden[t];
    return;
  }
  if (t < C2) {
    const float* w = w2 + static_cast<size_t>(t) * C1;
    float z = 0.f;
    for (int k = 0; k < C1; ++k) z += w[k] * hidden[k];
    out[static_cast<size_t>(blockIdx.x) * C2 + t] = activate(z + (b2 != nullptr ? b2[t] : 0.f), act2);
  }
}

// out[n][y][x][c] = f[n][y / up][x / up][c] * gate[n][c] + add, out at up times f's size (nearest upsampling of the
// sum); add = add[n][c] (add_map 0: a per-sample vector broadcast over the map) or add[n][y / up][x / up][c] (add_map
// 1: a map at f's size).  One product, one sum, each rounded once.
__global__ void faceparse_apply_kernel(const float* __restrict__ f, const float* __restrict__ gate,
                                       const float* __restrict__ add, int add_map, float* __restrict__ out, int N,
                                       int H, int W, int C4, int up) {
  pdl_trigger();
  pdl_wait();
  const int Ho = H * up, Wo = W * up;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    const size_t pix = i / C4;
    const int x = static_cast<int>(pix % Wo), y = static_cast<int>((pix / Wo) % Ho);
    const size_t n = pix / (static_cast<size_t>(Wo) * Ho);
    const size_t src = ((n * H + y / up) * W + x / up) * C4 + c4;
    const float4 v = reinterpret_cast<const float4*>(f)[src];
    const float4 g = reinterpret_cast<const float4*>(gate)[n * C4 + c4];
    const float4 a = reinterpret_cast<const float4*>(add)[add_map ? src : n * C4 + c4];
    reinterpret_cast<float4*>(out)[i] =
        make_float4(__fadd_rn(__fmul_rn(v.x, g.x), a.x), __fadd_rn(__fmul_rn(v.y, g.y), a.y),
                    __fadd_rn(__fmul_rn(v.z, g.z), a.z), __fadd_rn(__fmul_rn(v.w, g.w), a.w));
  }
}

__device__ __forceinline__ float lerp_rn(float a, float b, float l) {
  return __fadd_rn(__fmul_rn(1.f - l, a), __fmul_rn(l, b));
}

// Source row (or column) of output index o under align_corners=True: s = o * (in - 1) / (out - 1) in fp32, the two
// taps floor(s) and min(floor(s) + 1, in - 1) with weights 1 - l, l.
__device__ __forceinline__ void ac_taps(int o, float scale, int in, int& i0, int& i1, float& l) {
  const float s = static_cast<float>(o) * scale;
  i0 = min(static_cast<int>(s), in - 1);
  i1 = min(i0 + 1, in - 1);
  l = s - static_cast<float>(i0);
}

// The logits of sample n blended between source rows y0 and y1 with weight ly, into row[x][c] (shared memory)
__device__ __forceinline__ void blend_row(const float* __restrict__ logits, size_t n, int Hi, int Wi, int ld, int ncls,
                                          int y0, int y1, float ly, float* row) {
  const float* r0 = logits + ((n * Hi + y0) * Wi) * static_cast<size_t>(ld);
  const float* r1 = logits + ((n * Hi + y1) * Wi) * static_cast<size_t>(ld);
  for (int k = threadIdx.x; k < Wi * ncls; k += blockDim.x) {
    const int x = k / ncls, c = k - x * ncls;
    row[k] = lerp_rn(r0[static_cast<size_t>(x) * ld + c], r1[static_cast<size_t>(x) * ld + c], ly);
  }
}

// argmax over the classes of row (blended rows, [Wi][ncls]) at output column X: the first class wins a tie
__device__ __forceinline__ int row_argmax(const float* row, int ncls, int x0, int x1, float lx) {
  const float* a = row + x0 * ncls;
  const float* b = row + x1 * ncls;
  float best = lerp_rn(a[0], b[0], lx);
  int arg = 0;
  for (int c = 1; c < ncls; ++c) {
    const float v = lerp_rn(a[c], b[c], lx);
    if (v > best) {
      best = v;
      arg = c;
    }
  }
  return arg;
}

// One CTA per output row Y of sample (or edited row) blockIdx.y: F.interpolate(logits, (Ho, Wo), 'bilinear',
// align_corners=True) then argmax over the ncls classes (channel pitch ld).  Source rows are blended first (once per
// CTA, into shared memory), then columns.  kPair: also the label of source sample (row0 + j) % B at the same pixel;
// the CTA adds the number of equal labels to agree[j].  Otherwise labels[n][Y][X] (uint8) is written.
template <bool kPair>
__global__ void __launch_bounds__(kArgmaxThreads) faceparse_upsample_argmax_kernel(
    const float* __restrict__ logits, const float* __restrict__ src_logits, uint8_t* __restrict__ labels,
    unsigned int* __restrict__ agree, int B, int row0, int Hi, int Wi, int ld, int ncls, int Ho, int Wo, float sh,
    float sw) {
  pdl_trigger();
  extern __shared__ float rows[];
  const int Y = blockIdx.x;
  const size_t j = blockIdx.y;
  int y0, y1;
  float ly;
  ac_taps(Y, sh, Hi, y0, y1, ly);
  pdl_wait();
  blend_row(logits, j, Hi, Wi, ld, ncls, y0, y1, ly, rows);
  if (kPair) blend_row(src_logits, (row0 + j) % B, Hi, Wi, ld, ncls, y0, y1, ly, rows + Wi * ncls);
  __syncthreads();
  int same = 0;
  for (int X = threadIdx.x; X < Wo; X += kArgmaxThreads) {
    int x0, x1;
    float lx;
    ac_taps(X, sw, Wi, x0, x1, lx);
    const int lab = row_argmax(rows, ncls, x0, x1, lx);
    if (kPair) {
      same += lab == row_argmax(rows + Wi * ncls, ncls, x0, x1, lx);
    } else {
      labels[(j * Ho + Y) * Wo + X] = static_cast<uint8_t>(lab);
    }
  }
  if (kPair) {
    __shared__ int warp_same[kArgmaxThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) same += __shfl_xor_sync(0xffffffffu, same, o);
    if ((threadIdx.x & 31) == 0) warp_same[threadIdx.x >> 5] = same;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < kArgmaxThreads / 32; ++w) tot += warp_same[w];
      atomicAdd(agree + j, static_cast<unsigned int>(tot));
    }
  }
}

inline int fp_grid(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

inline float ac_scale(int in, int out) {
  return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_faceparse_pack(const float* x, float* out, int B, int H, int W, int S, void* stream) {
  ASYRP_REQUIRE(B > 0 && H > 0 && W > 0 && S > 0, "asyrp_faceparse_pack: bad shape B=%d H=%d W=%d S=%d", B, H, W, S);
  const size_t total = static_cast<size_t>(B) * S * S;
  ASYRP_LAUNCH(faceparse_pack_kernel, dim3(fp_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), x,
               out, B, H, W, S);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_faceparse_conv(const float* in, const float* weight, const float* bias, const float* residual,
                                   float* out, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                                   int relu, void* stream) {
  using namespace tf32gemm;
  ASYRP_REQUIRE(Cin > 0 && Cin % 4 == 0, "asyrp_faceparse_conv: Cin=%d must be a positive multiple of 4", Cin);
  ASYRP_REQUIRE(Cout > 0 && Cout % kBN == 0, "asyrp_faceparse_conv: Cout=%d must be a positive multiple of %d", Cout,
                kBN);
  ASYRP_REQUIRE(N > 0 && k > 0 && stride > 0 && pad >= 0 && H + 2 * pad >= k && W + 2 * pad >= k,
                "asyrp_faceparse_conv: bad geometry N=%d H=%d W=%d k=%d stride=%d pad=%d", N, H, W, k, stride, pad);
  ASYRP_REQUIRE(relu == 0 || relu == 1, "asyrp_faceparse_conv: relu=%d must be 0 or 1", relu);
  ASYRP_REQUIRE(residual == nullptr || relu == 1, "asyrp_faceparse_conv: a residual is added before the ReLU only");
  ASYRP_REQUIRE(residual != nullptr || relu == 0 || bias != nullptr,
                "asyrp_faceparse_conv: the ReLU epilogue without a residual needs a bias");
  ASYRP_REQUIRE(in != out, "asyrp_faceparse_conv: out must not alias in");
  Tf32ConvParams p;
  p.in = in; p.w = weight; p.bias = bias; p.residual = residual; p.prelu = nullptr; p.out = out;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.kw = k; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - k) / stride + 1;
  p.Wo = (W + 2 * pad - k) / stride + 1;
  p.K = k * k * Cin;
  p.Kpad = (p.K + kBK - 1) / kBK * kBK;
  const long long M = static_cast<long long>(N) * p.Ho * p.Wo;
  ASYRP_REQUIRE(M < (1LL << 31) / kBM * kBM, "asyrp_faceparse_conv: too many output pixels");
  p.M = static_cast<int>(M);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (residual != nullptr) return launch_tf32_conv<kEpiResidualRelu>(p, st);
  return relu ? launch_tf32_conv<kEpiRelu>(p, st) : launch_tf32_conv<kEpiBias>(p, st);
}

ASYRP_API int asyrp_faceparse_maxpool(const float* in, float* out, int N, int H, int W, int C, void* stream) {
  ASYRP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "asyrp_faceparse_maxpool: bad shape N=%d H=%d W=%d C=%d",
                N, H, W, C);
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * (C / 4);
  ASYRP_LAUNCH(faceparse_maxpool_kernel, dim3(fp_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               in, out, N, H, W, C / 4, Ho, Wo);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_faceparse_gate(const float* in, const float* w1, const float* b1, int C1, int act1,
                                   const float* w2, const float* b2, int C2, int act2, float* out, int N, int HW,
                                   int C, void* stream) {
  ASYRP_REQUIRE(N > 0 && HW > 0 && C > 0 && C <= kGateMaxC && kGateThreads % C == 0,
                "asyrp_faceparse_gate: bad shape N=%d HW=%d C=%d (C must divide %d)", N, HW, C, kGateThreads);
  ASYRP_REQUIRE(C1 > 0 && C1 <= kGateMaxC && (w2 == nullptr || (C2 > 0 && C2 <= kGateThreads)),
                "asyrp_faceparse_gate: bad widths C1=%d C2=%d (1 .. %d)", C1, C2, kGateMaxC);
  ASYRP_REQUIRE(act1 >= 0 && act1 <= 2 && act2 >= 0 && act2 <= 2, "asyrp_faceparse_gate: act1=%d act2=%d not in 0..2",
                act1, act2);
  ASYRP_LAUNCH(faceparse_gate_kernel, dim3(N), dim3(kGateThreads), 0, static_cast<cudaStream_t>(stream), in, w1, b1,
               C1, act1, w2, b2, C2, act2, out, HW, C);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_faceparse_apply(const float* f, const float* gate, const float* add, int add_map, float* out,
                                    int N, int H, int W, int C, int up, void* stream) {
  ASYRP_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && (up == 1 || up == 2) && (add_map == 0 || add_map == 1),
                "asyrp_faceparse_apply: bad shape N=%d H=%d W=%d C=%d up=%d add_map=%d", N, H, W, C, up, add_map);
  ASYRP_REQUIRE(out != f && out != add, "asyrp_faceparse_apply: out must not alias f or add");
  const size_t total = static_cast<size_t>(N) * H * up * W * up * (C / 4);
  ASYRP_LAUNCH(faceparse_apply_kernel, dim3(fp_grid(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), f,
               gate, add, add_map, out, N, H, W, C / 4, up);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_faceparse_labels(const float* logits, uint8_t* labels, int N, int Hi, int Wi, int ld, int ncls,
                                     int Ho, int Wo, void* stream) {
  ASYRP_REQUIRE(N > 0 && N <= kMaxGridYZ && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && ncls > 0 && ncls <= kMaxClasses &&
                    ld >= ncls,
                "asyrp_faceparse_labels: bad shape N=%d Hi=%d Wi=%d ld=%d ncls=%d Ho=%d Wo=%d", N, Hi, Wi, ld, ncls, Ho,
                Wo);
  const size_t smem = static_cast<size_t>(Wi) * ncls * sizeof(float);
  ASYRP_REQUIRE(smem <= kArgmaxSmemBytes, "asyrp_faceparse_labels: Wi * ncls = %d * %d too large", Wi, ncls);
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(faceparse_upsample_argmax_kernel<false>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kArgmaxSmemBytes));
  ASYRP_LAUNCH(faceparse_upsample_argmax_kernel<false>, dim3(Ho, N), dim3(kArgmaxThreads), smem,
               static_cast<cudaStream_t>(stream), logits, nullptr, labels, nullptr, 1, 0, Hi, Wi, ld, ncls, Ho, Wo,
               ac_scale(Hi, Ho), ac_scale(Wi, Wo));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_faceparse_agreement(const float* src_logits, const float* edited_logits, unsigned int* agree,
                                        int n, int B, int row0, int Hi, int Wi, int ld, int ncls, int Ho, int Wo,
                                        void* stream) {
  ASYRP_REQUIRE(n > 0 && n <= kMaxGridYZ && B > 0 && row0 >= 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && ncls > 0 &&
                    ncls <= kMaxClasses && ld >= ncls,
                "asyrp_faceparse_agreement: bad shape n=%d B=%d row0=%d Hi=%d Wi=%d ld=%d ncls=%d Ho=%d Wo=%d", n, B,
                row0, Hi, Wi, ld, ncls, Ho, Wo);
  const size_t smem = 2 * static_cast<size_t>(Wi) * ncls * sizeof(float);
  ASYRP_REQUIRE(smem <= kArgmaxSmemBytes, "asyrp_faceparse_agreement: Wi * ncls = %d * %d too large", Wi, ncls);
  ASYRP_CHECK_CUDA(cudaFuncSetAttribute(faceparse_upsample_argmax_kernel<true>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kArgmaxSmemBytes));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  ASYRP_CHECK_CUDA(cudaMemsetAsync(agree, 0, static_cast<size_t>(n) * sizeof(unsigned int), st));
  ASYRP_LAUNCH(faceparse_upsample_argmax_kernel<true>, dim3(Ho, n), dim3(kArgmaxThreads), smem, st, edited_logits,
               src_logits, nullptr, agree, B, row0, Hi, Wi, ld, ncls, Ho, Wo, ac_scale(Hi, Ho), ac_scale(Wi, Wo));
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
