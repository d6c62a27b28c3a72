// ArcFace IR-SE50 (the reference's models/insight_face Backbone(112, 50, 'ir_se')) and IDLoss
// (losses/id_loss.py): crop, AdaptiveAvgPool2d(112), the backbone, l2_norm and the per-row feature dot product.
//
//   x112     = AdaptiveAvgPool2d(112)(x[:, :, 35:223, 32:220]) as NHWC, 4 channels     arcface_preprocess_kernel
//   h        = PReLU(BN(conv3x3(x112)))                                               tf32_gemm.cuh, kEpiPrelu
//   per bottleneck block (in -> depth, stride s):
//     xb     = BN0(x)       (materialised: the conv zero-pads BN0(x), not x)         arcface_affine_kernel (block 0),
//                                                                                     else the previous block's apply
//     t      = PReLU(conv3x3(xb))                                                     kEpiPrelu, no bias
//     r      = BN4(conv3x3/s(t))                                                      kEpiBias (BN folded)
//     sc     = x | x[::2, ::2] | BN(conv1x1/s(x))                                     -, -, kEpiBias (BN folded)
//     out    = r * sigmoid(fc2(relu(fc1(mean_hw(r))))) + sc                           arcface_se_scale_kernel,
//                                                                                     arcface_se_apply_kernel
//   feature  = l2_norm(BN1d(Linear(flatten(BN2d(out)))))  (both BNs folded into the linear layer; clip_text.cu's
//              linear entry point runs it)                                            arcface_l2norm_kernel
//   id[j]    = feature_edit[j] . feature_src[j % B]                                   arcface_dot_kernel
//
// Activations are fp32 NHWC.  Every reduction runs in a fixed order with no float atomics, and no kernel mixes
// samples, so an image's features are the same bits whatever batch it is in.
#include "common.h"
#include "ptx.cuh"
#include "tf32_gemm.cuh"

namespace asyrp {
namespace {

constexpr int kCropY = 35, kCropX = 32, kCrop = 188, kPool = 112;  // IDLoss.extract_feats
constexpr int kSeThreads = 512;
constexpr int kSeMaxHidden = 32;  // C / 16 with C <= 512

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// out[b][i][j][c] = mean of x[b][c] over rows 35 + [floor(188 i / 112), ceil(188 (i+1) / 112)) and columns
// 32 + [floor(188 j / 112), ceil(188 (j+1) / 112)) (AdaptiveAvgPool2d's bins: 2 or 3 pixels, overlapping), summed row
// by row, left to right; channel 3 zero.  x fp32 NCHW [B][3][H][W], out fp32 NHWC [B][112][112][4].
__global__ void arcface_preprocess_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int H, int W) {
  pdl_trigger();
  pdl_wait();
  const size_t total = static_cast<size_t>(B) * kPool * kPool;
  const size_t plane = static_cast<size_t>(H) * W;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % kPool), oy = static_cast<int>((i / kPool) % kPool);
    const size_t b = i / (kPool * kPool);
    const int y0 = kCropY + (kCrop * oy) / kPool, y1 = kCropY + (kCrop * (oy + 1) + kPool - 1) / kPool;
    const int x0 = kCropX + (kCrop * ox) / kPool, x1 = kCropX + (kCrop * (ox + 1) + kPool - 1) / kPool;
    const float inv = 1.f / static_cast<float>((y1 - y0) * (x1 - x0));
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* img = x + (b * 3 + c) * plane;
      float s = 0.f;
      for (int y = y0; y < y1; ++y)
        for (int xx = x0; xx < x1; ++xx) s += img[static_cast<size_t>(y) * W + xx];
      v[c] = s * inv;
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], 0.f);
  }
}

// out = in * scale[c] + shift[c] over fp32 NHWC [rows][C] (an eval-mode BatchNorm2d folded to an affine)
__global__ void arcface_affine_kernel(const float* __restrict__ in, const float* __restrict__ scale,
                                      const float* __restrict__ shift, float* __restrict__ out, size_t total4,
                                      int C4) {
  pdl_trigger();
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    const float4 a = reinterpret_cast<const float4*>(scale)[c4];
    const float4 b = reinterpret_cast<const float4*>(shift)[c4];
    reinterpret_cast<float4*>(out)[i] = make_float4(v.x * a.x + b.x, v.y * a.y + b.y, v.z * a.z + b.z, v.w * a.w + b.w);
  }
}

// SEModule's gate of sample n (one CTA per sample): m = mean over the HW pixels of res[n] (thread t sums channel
// t % C over pixels t / C, t / C + 512 / C, ...; the 512 / C partials of a channel are added in order), hidden =
// relu(fc1 m) (a warp per hidden unit, butterfly over channels), scale[n][c] = sigmoid(fc2[c] . hidden) (in order).
// fc1 [C/16][C], fc2 [C][C/16] (1x1 convs without bias).
__global__ void __launch_bounds__(kSeThreads) arcface_se_scale_kernel(const float* __restrict__ res,
                                                                      const float* __restrict__ fc1,
                                                                      const float* __restrict__ fc2,
                                                                      float* __restrict__ scale, int HW, int C) {
  pdl_trigger();
  __shared__ float part[kSeThreads];
  __shared__ float mean[kSeThreads];
  __shared__ float hidden[kSeMaxHidden];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int J = kSeThreads / C, c = t % C, j = t / C, Cr = C / 16;
  const float* R = res + static_cast<size_t>(blockIdx.x) * HW * C;
  pdl_wait();
  float s = 0.f;
  for (int p = j; p < HW; p += J) s += R[static_cast<size_t>(p) * C + c];
  part[t] = s;
  __syncthreads();
  if (t < C) {
    float tot = 0.f;
    for (int k = 0; k < J; ++k) tot += part[k * C + t];
    mean[t] = tot / static_cast<float>(HW);
  }
  __syncthreads();
  for (int k = warp; k < Cr; k += kSeThreads / 32) {
    const float* w = fc1 + static_cast<size_t>(k) * C;
    float v = 0.f;
    for (int i = lane; i < C; i += 32) v += w[i] * mean[i];
    v = warp_sum(v);
    if (lane == 0) hidden[k] = fmaxf(v, 0.f);
  }
  __syncthreads();
  if (t < C) {
    const float* w = fc2 + static_cast<size_t>(t) * Cr;
    float z = 0.f;
    for (int k = 0; k < Cr; ++k) z += w[k] * hidden[k];
    scale[static_cast<size_t>(blockIdx.x) * C + t] = 1.f / (1.f + expf(-z));
  }
}

// Block end: out = res * scale[n][c] + sc, sc read at pixel (y * ss, x * ss) of the shortcut map [N][Hs][Ws][C]
// (ss = 1: the identity or the conv shortcut's output; ss = 2: MaxPool2d(1, 2) of the block input).  When out2 is not
// null it also gets out * bn_scale[c] + bn_shift[c], the next block's pre-conv BatchNorm.
__global__ void arcface_se_apply_kernel(const float* __restrict__ res, const float* __restrict__ scale,
                                        const float* __restrict__ sc, float* __restrict__ out,
                                        const float* __restrict__ bn_scale, const float* __restrict__ bn_shift,
                                        float* __restrict__ out2, int N, int Ho, int Wo, int C, int Hs, int Ws,
                                        int ss) {
  pdl_trigger();
  pdl_wait();
  const int C4 = C / 4;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(i % C4);
    const size_t pix = i / C4;
    const int x = static_cast<int>(pix % Wo), y = static_cast<int>((pix / Wo) % Ho);
    const size_t n = pix / (static_cast<size_t>(Wo) * Ho);
    const float4 r = reinterpret_cast<const float4*>(res)[i];
    const float4 s = reinterpret_cast<const float4*>(scale)[n * C4 + c4];
    const float4 h = reinterpret_cast<const float4*>(sc)[((n * Hs + static_cast<size_t>(y) * ss) * Ws +
                                                          static_cast<size_t>(x) * ss) * C4 + c4];
    const float4 o = make_float4(__fadd_rn(__fmul_rn(r.x, s.x), h.x), __fadd_rn(__fmul_rn(r.y, s.y), h.y),
                                 __fadd_rn(__fmul_rn(r.z, s.z), h.z), __fadd_rn(__fmul_rn(r.w, s.w), h.w));
    reinterpret_cast<float4*>(out)[i] = o;
    if (out2 != nullptr) {
      const float4 a = reinterpret_cast<const float4*>(bn_scale)[c4];
      const float4 b = reinterpret_cast<const float4*>(bn_shift)[c4];
      reinterpret_cast<float4*>(out2)[i] =
          make_float4(o.x * a.x + b.x, o.y * a.y + b.y, o.z * a.z + b.z, o.w * a.w + b.w);
    }
  }
}

// l2_norm without epsilon: out[r] = in[r] / |in[r]|, a warp per row (lane partials, butterfly)
__global__ void arcface_l2norm_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int dim) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* a = in + static_cast<size_t>(row) * dim;
  float q = 0.f;
  for (int c = lane; c < dim; c += 32) q += a[c] * a[c];
  const float norm = sqrtf(warp_sum(q));
  for (int c = lane; c < dim; c += 32) out[static_cast<size_t>(row) * dim + c] = a[c] / norm;
}

// id[j] = edited[j] . src[j % B], a warp per row
__global__ void arcface_dot_kernel(const float* __restrict__ src, const float* __restrict__ edited,
                                   float* __restrict__ id, int n, int B, int dim) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* e = edited + static_cast<size_t>(row) * dim;
  const float* s = src + static_cast<size_t>(row % B) * dim;
  float q = 0.f;
  for (int c = lane; c < dim; c += 32) q += e[c] * s[c];
  q = warp_sum(q);
  if (lane == 0) id[row] = q;
}

inline int grid_cap(size_t total, int block) {
  const size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count() > 0 ? sm_count() : 132) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace
}  // namespace asyrp

using namespace asyrp;

extern "C" {

ASYRP_API int asyrp_arcface_preprocess(const float* x, float* out, int B, int H, int W, void* stream) {
  ASYRP_REQUIRE(B > 0 && H >= kCropY + kCrop && W >= kCropX + kCrop,
                "asyrp_arcface_preprocess: bad shape B=%d H=%d W=%d (the crop needs H >= %d, W >= %d)", B, H, W,
                kCropY + kCrop, kCropX + kCrop);
  const size_t total = static_cast<size_t>(B) * kPool * kPool;
  ASYRP_LAUNCH(arcface_preprocess_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               x, out, B, H, W);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_arcface_conv(const float* in, const float* weight, const float* bias, const float* prelu,
                                 float* out, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad,
                                 void* stream) {
  using namespace tf32gemm;
  ASYRP_REQUIRE(Cin > 0 && Cin % 4 == 0, "asyrp_arcface_conv: Cin=%d must be a positive multiple of 4", Cin);
  ASYRP_REQUIRE(Cout > 0 && Cout % kBN == 0, "asyrp_arcface_conv: Cout=%d must be a positive multiple of %d", Cout,
                kBN);
  ASYRP_REQUIRE(N > 0 && k > 0 && stride > 0 && pad >= 0 && H + 2 * pad >= k && W + 2 * pad >= k,
                "asyrp_arcface_conv: bad geometry N=%d H=%d W=%d k=%d stride=%d pad=%d", N, H, W, k, stride, pad);
  ASYRP_REQUIRE(in != out, "asyrp_arcface_conv: out must not alias in");
  Tf32ConvParams p;
  p.in = in; p.w = weight; p.bias = bias; p.residual = nullptr; p.prelu = prelu; p.out = out;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.kw = k; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - k) / stride + 1;
  p.Wo = (W + 2 * pad - k) / stride + 1;
  p.K = k * k * Cin;
  p.Kpad = (p.K + kBK - 1) / kBK * kBK;
  const long long M = static_cast<long long>(N) * p.Ho * p.Wo;
  ASYRP_REQUIRE(M < (1LL << 31) / kBM * kBM, "asyrp_arcface_conv: too many output pixels");
  p.M = static_cast<int>(M);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return prelu != nullptr ? launch_tf32_conv<kEpiPrelu>(p, st) : launch_tf32_conv<kEpiBias>(p, st);
}

ASYRP_API int asyrp_arcface_affine(const float* in, const float* scale, const float* shift, float* out, long long rows,
                                   int C, void* stream) {
  ASYRP_REQUIRE(rows > 0 && C > 0 && C % 4 == 0, "asyrp_arcface_affine: bad shape rows=%lld C=%d", rows, C);
  const size_t total4 = static_cast<size_t>(rows) * (C / 4);
  ASYRP_LAUNCH(arcface_affine_kernel, dim3(grid_cap(total4, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream), in,
               scale, shift, out, total4, C / 4);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_arcface_se_scale(const float* res, const float* fc1, const float* fc2, float* scale, int N, int HW,
                                     int C, void* stream) {
  ASYRP_REQUIRE(N > 0 && HW > 0 && C >= 16 && C <= kSeThreads && kSeThreads % C == 0 && C % 16 == 0,
                "asyrp_arcface_se_scale: bad shape N=%d HW=%d C=%d (C: 16 .. %d, dividing %d)", N, HW, C, kSeThreads,
                kSeThreads);
  ASYRP_LAUNCH(arcface_se_scale_kernel, dim3(N), dim3(kSeThreads), 0, static_cast<cudaStream_t>(stream), res, fc1, fc2,
               scale, HW, C);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_arcface_se_apply(const float* res, const float* scale, const float* shortcut, float* out,
                                     const float* bn_scale, const float* bn_shift, float* out2, int N, int Ho, int Wo,
                                     int C, int Hs, int Ws, int ss, void* stream) {
  ASYRP_REQUIRE(N > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 4 == 0 && (ss == 1 || ss == 2),
                "asyrp_arcface_se_apply: bad shape N=%d Ho=%d Wo=%d C=%d ss=%d", N, Ho, Wo, C, ss);
  ASYRP_REQUIRE((Ho - 1) * ss < Hs && (Wo - 1) * ss < Ws, "asyrp_arcface_se_apply: shortcut %dx%d too small", Hs, Ws);
  ASYRP_REQUIRE((out2 == nullptr) == (bn_scale == nullptr) && (out2 == nullptr) == (bn_shift == nullptr),
                "asyrp_arcface_se_apply: out2 needs, and only it needs, bn_scale and bn_shift");
  const size_t total = static_cast<size_t>(N) * Ho * Wo * (C / 4);
  ASYRP_LAUNCH(arcface_se_apply_kernel, dim3(grid_cap(total, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
               res, scale, shortcut, out, bn_scale, bn_shift, out2, N, Ho, Wo, C, Hs, Ws, ss);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_arcface_l2norm(const float* in, float* out, int rows, int dim, void* stream) {
  ASYRP_REQUIRE(rows > 0 && dim > 0, "asyrp_arcface_l2norm: bad shape rows=%d dim=%d", rows, dim);
  ASYRP_LAUNCH(arcface_l2norm_kernel, dim3((rows + 7) / 8), dim3(256), 0, static_cast<cudaStream_t>(stream), in, out,
               rows, dim);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

ASYRP_API int asyrp_arcface_dot(const float* src, const float* edited, float* id, int n, int B, int dim,
                                void* stream) {
  ASYRP_REQUIRE(n > 0 && B > 0 && dim > 0, "asyrp_arcface_dot: bad shape n=%d B=%d dim=%d", n, B, dim);
  ASYRP_LAUNCH(arcface_dot_kernel, dim3((n + 7) / 8), dim3(256), 0, static_cast<cudaStream_t>(stream), src, edited, id,
               n, B, dim);
  ASYRP_CHECK_CUDA(cudaGetLastError());
  return ASYRP_OK;
}

}  // extern "C"
