/* libasyrp_b200.so — C ABI of the Asyrp sampling engine (hand-written CUDA for the H100, sm_90a).
 *
 * The reference (kwonminki/Asyrp_official) has no FFI: its seam for this path is Python call signatures
 * (utils/diffusion_utils.py:24 denoising_step, models/ddpm/diffusion.py:473 DDPM.forward,
 * models/improved_ddpm/unet.py:676 UNetModel.forward).  This header is the boundary a maintainer binds instead
 * of torch's cuDNN/cuBLAS calls; every entry point names the reference operations it replaces.  INTEGRATION.md
 * shows the ctypes stub (asyrp_official_b200/_lib.py is the shipped one).
 *
 * Conventions
 *  - plain pointers and sizes; all pointers are DEVICE pointers unless noted; the caller owns every buffer
 *  - activations: NHWC fp16 ("half"); weights: fp16 [Cout][K] with K = taps*Cin, tap-major / channel-minor;
 *    statistics, affine tables, embeddings, sampler state: fp32
 *  - `stream` is a cudaStream_t; calls only enqueue work, never synchronise, never allocate device memory
 *  - return 0 on success, <0 on error (ASYRP_ERR_*); asyrp_last_error() gives the message (thread local)
 */
#ifndef ASYRP_B200_H
#define ASYRP_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define ASYRP_OK 0
#define ASYRP_ERR_INVALID (-1)   /* bad argument / unsupported shape */
#define ASYRP_ERR_CUDA (-2)      /* CUDA runtime or driver error */
#define ASYRP_ERR_NO_DEVICE (-3) /* no usable device / driver */

const char* asyrp_last_error(void);

/* Programmatic dependent launch: every kernel of the library begins with griddepcontrol.launch_dependents and
 * executes griddepcontrol.wait before its first global-memory access, and is launched with the
 * programmaticStreamSerialization attribute, so consecutive kernels of a stream (or of a captured graph) overlap
 * launch latency and prologue with the predecessor's tail.  Results are unchanged.  Default off: inside the captured
 * trajectory graph it measured neutral (443.0 vs 448.7 ms); ASYRP_PDL=1 in the environment or asyrp_set_pdl(1) turns
 * it on for eager, launch-bound callers.  The reference's equivalent is the implicit stream order of
 * PyTorch's eager launches (one or more library kernels per line of models/ddpm/diffusion.py:473-580). */
int asyrp_set_pdl(int enabled);
int asyrp_get_pdl(void);

/* ---- implicit-GEMM convolution on wgmma tensor cores ---------------------------------------------------
 * Replaces torch.nn.Conv2d / Conv1d(k=1) / bmm call sites of the UNets:
 *   ResnetBlock.conv1/conv2/nin_shortcut  models/ddpm/diffusion.py:122-149     (3x3 s1 p1, 1x1)
 *   Downsample.conv (pad (0,1,0,1), s2)   models/ddpm/diffusion.py:96-108
 *   Upsample.conv                         models/ddpm/diffusion.py:77-88
 *   AttnBlock.q/k/v/proj_out              models/ddpm/diffusion.py:179-198
 *   ResBlock in_layers[2]/out_layers[3]/skip_connection, AttentionBlock.qkv/proj_out, DeltaBlock 1x1 convs
 *                                         models/improved_ddpm/unet.py:224-264,333-336,821-834
 *   conv_in / conv_out                    models/ddpm/diffusion.py:357-361,424-428 ; unet.py:522-524,654-658
 * A descriptor lists up to 3 K-segments (sources): a channel concatenation (torch.cat of decoder input and skip,
 * ddpm/diffusion.py:549) is two segments; a fused 1x1 shortcut is one more segment of the same accumulator.
 * Epilogue: out = acc_scale*(acc + ebias[n]) + res_scale*residual, stored fp16 NHWC (or fp32 planar channels),
 * plus per-(sample, tile, channel-pair) partial sums for the GroupNorm that consumes the output. */
#define ASYRP_CONV_1x1 0
#define ASYRP_CONV_3x3 1    /* stride 1, zero pad 1 */
#define ASYRP_CONV_3x3_S2 2 /* stride 2, zero pad right/bottom by 1; source is [N][2H][2W][C] */

typedef struct AsyrpConvSeg {
  const void* src; /* fp16 NHWC source */
  int C;           /* channels, multiple of 64 */
  int mode;        /* ASYRP_CONV_* */
  /* optional fused GroupNorm-apply (+SiLU) on this operand: x -> act(a*x + b), evaluated in shared memory between
   * the TMA load and the MMA (norm1/norm2 + nonlinearity of ResnetBlock, ddpm/diffusion.py:153-161; in_layers /
   * out_layers of ResBlock, improved_ddpm/unet.py:224-228,248-255).  affine: fp32 (a, b) pairs of this segment's
   * channels, row n at affine + n*affine_stride floats (output of asyrp_gn_finalize, offset to the segment's first
   * channel); NULL = raw operand.  Zero padding is applied AFTER the transform, as the reference's convs see it. */
  const float* affine;
  int affine_stride;
  int act;         /* 1: SiLU after the affine */
  int ld;          /* elements between consecutive pixels of src (0: C): lets a segment be a channel slice of a wider
                      tensor, e.g. q = qkv[..., 0:C] */
  /* Alternative to `affine`: GroupNorm finalised INSIDE the kernel (no asyrp_gn_finalize launch, no affine table).
   * gn_sums_a / gn_sums_b: the `sums_out` buffers of the conv(s) that produced the (one or two, virtually concatenated)
   * source tensors of the GroupNorm — [N][C_i/2][2] int64, (sum, sum of squares) * 2^18 per channel pair, accumulated by
   * their epilogues with integer atomics (deterministic) and zeroed by the caller before those convs run; gn_gamma /
   * gn_beta: [Ca+Cb] GroupNorm weight / bias; gn_scale_shift: optional ADM (scale | shift) rows, row n at
   * + n*gn_ss_stride; gn_eps; gn_hw = H*W of the normalised tensor; gn_off: first channel of this segment on the
   * concatenated axis.  Needs tiles inside one sample (H*W >= 128). */
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
} AsyrpConvSeg;

typedef struct AsyrpConvDesc {
  int N, H, W, Cout;     /* output geometry; Cout multiple of 64 (or 16 with out_planar: the conv_out tile) */
  int nseg;              /* 1..3 */
  AsyrpConvSeg seg[3];
  const void* weight;    /* fp16 [Cout][K] ([N][Cout][K] if weight_batched), K = sum_seg taps*C */
  int weight_batched;    /* per-sample weight matrix (batched GEMM, e.g. q k^T) */
  int weight_ld;         /* elements between weight rows (0: K) */
  long long weight_batch_stride; /* elements between per-sample matrices (0: Cout*weight_ld) */
  /* multi-head attention GEMMs (QKVAttentionLegacy, improved_ddpm/unet.py:379-396): N counts (sample, head) pairs.
   * a_heads > 1: segment 0 is [N/a_heads][H][W][ld], head h reads channels [h*C, (h+1)*C);
   * b_heads > 1: weights are [N/b_heads][Cout][weight_ld], head h reads columns [h*K, (h+1)*K);
   * out_heads > 1: out is [N/out_heads][H][W][out_heads*Cout], head h writes channels [h*Cout, (h+1)*Cout). */
  int a_heads, b_heads, out_heads;
  int out_f32;           /* 1: `out` is fp32 NHWC (attention logits); excludes residual / stats / planar */
  const float* ebias;    /* fp32 bias row(s): row n at ebias + n*ebias_stride; NULL = none */
  int ebias_stride;      /* 0: one row shared by all samples (plain bias);
                            >0: per-sample rows (conv bias + timestep-embedding projection) */
  const void* residual;  /* fp16 NHWC [N][H][W][Cout] or NULL */
  float res_scale, acc_scale;
  void* out;             /* fp16 NHWC [N][H][W][Cout] (ignored when out_planar != NULL) */
  float* stats;          /* [N][asyrp_conv_stats_tiles(..)][Cout/2][2] fp32 (sum, sum of squares) or NULL */
  float* out_planar;     /* optional fp32 NCHW [N][planar_c][H][W]: output channels [0, planar_c<=8) only */
  int planar_c;
  /* up2 = 1: the op is Upsample.conv (models/ddpm/diffusion.py:77-87, improved_ddpm/unet.py:142-150), i.e.
   * conv3x3(F.interpolate(src, scale_factor=2, mode="nearest")), evaluated on the SOURCE image as four sub-pixel
   * phases: N/H/W are the source geometry (H%16==0, W%8==0), out is [N][2H][2W][Cout], one ASYRP_CONV_3x3 segment,
   * weight is fp16 [4*Cout][4*C] (phase-major rows, 2x2 taps x C; the 3x3 taps that fall on one source pixel are
   * pre-summed), stats has asyrp_conv_stats_tiles_up2() slots.  4/9 of the MACs, no upsampled tensor.  With a fused
   * affine on the segment this is also in_layers of the ADM ResBlock(up=True): conv(nearest-x2(silu(GN(x)))). */
  int up2;
  /* optional DEVICE pointer to two floats (acc_scale, res_scale) read by the kernel at run time instead of the
   * by-value fields: the DeltaBlock coefficients hs_coeff are per-call arguments of forward()
   * (ddpm/diffusion.py:512-516), so one captured trajectory graph serves every coefficient tuple */
  const float* scales;
  /* residual geometry: 0 = that of the output; 1 = [N][H/2][W/2][Cout], read through nearest-x2 upsampling; 2 =
   * [N][2H][2W][Cout], read through a 2x2 average pool — the skip branch x_upd(x) of the ADM ResBlock(up / down)
   * (improved_ddpm/unet.py:279-284,297), so that the resampled copy of x is never materialised */
  int res_mode;
  /* optional [N][Cout/2][2] int64 accumulators of (sum, sum of squares) * 2^18 of the output, for a consumer's in-kernel
   * GroupNorm (AsyrpConvSeg.gn_*); requires `stats` */
  long long* sums_out;
} AsyrpConvDesc;

/* number of tile slots of the stats buffer of a conv with this output geometry; has_3x3: the conv has an
 * ASYRP_CONV_3x3 segment (selects the 8x16 halo tile geometry when H%16==0 and W%8==0).  0 if the geometry is
 * unsupported (no 128-pixel tile fits it, e.g. W = 12; asyrp_conv_create rejects it with ASYRP_ERR_INVALID) */
int asyrp_conv_stats_tiles(int H, int W, int Cout, int has_3x3);
/* tile configuration the library picks for this output geometry: BN * 16 + MT (BN output channels x MT * 128 pixels per
 * CTA tile); 0 if the geometry is unsupported */
int asyrp_conv_tile_config(int H, int W, int Cout, int has_3x3);
/* the same for an up2 conv over an H x W source image (0 if the geometry is unsupported) */
int asyrp_conv_stats_tiles_up2(int H, int W, int Cout);
/* SiLU inside the fused GroupNorm-apply + SiLU operand transform: 1 (default) = h + h * tanh.approx(h), h = x / 2 (one
 * special-function op, 11-bit tanh), 0 = x * rcp.approx(1 + ex2.approx(-x log2 e)); negative = default (ASYRP_SILU_TANH).
 * Affects ops created afterwards. */
int asyrp_set_silu_tanh(int enabled);
int asyrp_conv_create(const AsyrpConvDesc* desc, void** op); /* encodes TMA descriptors; host only */
int asyrp_conv_launch(void* op, void* stream);
int asyrp_conv_set_scales(void* op, float acc_scale, float res_scale); /* hs_coeff of forward(), diffusion.py:512-516 */
void asyrp_conv_destroy(void* op);

/* ---- GroupNorm(32) statistics -> per-(sample, channel) affine ------------------------------------------
 * Replaces torch.nn.GroupNorm in Normalize (ddpm/diffusion.py:68-69, eps 1e-6) and GroupNorm32
 * (improved_ddpm/nn.py:17-19, eps 1e-5).  The normalised tensor may be the concatenation of two conv outputs
 * (Ca + Cb channels).  scale_shift (optional, [N][>=2C], row stride ss_stride): out = GN(x)*(1+scale)+shift
 * (improved_ddpm/unet.py:290-294).  affine: [N][C][2] with y = a*x + b. */
int asyrp_gn_finalize(const float* stats_a, int Ca, int tiles_a, const float* stats_b, int Cb, int tiles_b,
                      const float* gamma, const float* beta, float eps, int N, int HW, const float* scale_shift,
                      int ss_stride, float* affine, void* stream);

/* ---- out = resample(act(a*x + b)) over the channel concat of up to two NHWC fp16 sources ------------------
 * act: 0 identity, 1 SiLU (x*sigmoid(x), ddpm/diffusion.py:63-65).  resample: 0 none, 1 2x2 average pool
 * (improved_ddpm/unet.py:173-181), 2 nearest x2 (F.interpolate, ddpm/diffusion.py:83-84).  affine: (a, b) pairs of
 * the Ca+Cb channels, row n at affine + n*affine_stride floats (0: rows of (Ca+Cb)*2); NULL = identity. */
int asyrp_apply(const void* src_a, int Ca, const void* src_b, int Cb, const float* affine, int affine_stride,
                void* out, int N, int Hi, int Wi, int act, int resample, void* stream);

/* x_t fp32 NCHW [N][Cin<=64][H][W] -> fp16 NHWC [N][H][W][64] (zero padded channels): operand of conv_in */
int asyrp_pack_input(const float* x, void* out, int N, int Cin, int H, int W, void* stream);

/* sinusoidal timestep embedding, [N] -> [N][dim].  variant 0: get_timestep_embedding (ddpm/diffusion.py:42-60);
 * variant 1: timestep_embedding (improved_ddpm/nn.py:103-121) */
int asyrp_timestep_embedding(const float* t, float* out, int N, int dim, int variant, void* stream);

/* out[n][o] = bias[o] + sum_i W[o][i]*f(in[n][i]); f = SiLU if act_in; SiLU on the result if act_out.
 * Replaces temb.dense / temb_proj (ddpm/diffusion.py:349-354,157) and time_embed / emb_layers (unet.py:513-517,239-245) */
int asyrp_linear(const float* in, int in_stride, const float* W, const float* bias, float* out, int out_stride,
                 int N, int I, int O, int act_in, int act_out, void* stream);

/* DDIM update (utils/diffusion_utils.py:84-97), fp32, same operation order:
 *   x0 = (x - em*sqrt(1-at))/sqrt(at);  x_next = sqrt(an)*x0 + c2*et (+ c1*z)
 * et/em: fp32 planar [N][Ce][HW], channels [0,Cx) are epsilon (learn_sigma split, :47-51); z, x0_out may be NULL;
 * x_next may alias x. */
int asyrp_ddim_update(const float* x, const float* et, const float* em, const float* z, float* x_next,
                      float* x0_out, int N, int Cx, int Ce, int HW, float at, float an, float c1, float c2,
                      void* stream);

/* DDPM ancestral update (utils/diffusion_utils.py:74-82, sampling_type 'ddpm'):
 *   x_next = (x - bt/sqrt(1-at)*et)/sqrt(1-bt) + mask*exp(0.5*logvar)*z;  learned_sigma: logvar = et channels [Cx, 2Cx) */
int asyrp_ddpm_update(const float* x, const float* et, const float* z, float* x_next, int N, int Cx, int Ce, int HW,
                      float at, float bt, float logvar, int learned_sigma, float mask, void* stream);

/* out = alpha*a + beta*b, fp16 tensors of `numel` elements (multiple of 8) */
int asyrp_axpby(const void* a, const void* b, void* out, float alpha, float beta, long long numel, void* stream);

/* Explicit delta_h injection: h2 = slerp(t, h, |h|*dh/|dh|) per sample over C*H*W (models/ddpm/diffusion.py:6-40,
 * 528-539; improved_ddpm/unet.py:720-730); use_mask: interpolate only rows 4..H-2 x columns 3..4 without norm
 * matching, keep h elsewhere (:519-527).  h, h2: fp16 NHWC; dh: fp32 [C][H][W] per sample (stride 0 = shared).
 * stats: [N][stats_tiles][C/2][2] partial sums of h2 (slot 0 filled, the others zeroed). */
int asyrp_slerp_h(const void* h, const float* dh, long long dh_sample_stride, void* h2, float* stats, int stats_tiles,
                  int N, int C, int H, int W, float t, int use_mask, void* stream);

/* NHWC fp16 [N][HW][C] -> NCHW fp32 (API-visible delta_h / middle_h) */
int asyrp_unpack_nchw(const void* in, float* out, int N, int C, int HW, void* stream);

/* softmax(q k^T * scale) v per (sample, head).  qkv: fp16 [N][T][3*heads*head_dim] laid out [q | k | v], head h at
 * h*head_dim; out fp16 [N][T][heads*head_dim].  Replaces the bmm/softmax/bmm of AttnBlock.forward
 * (ddpm/diffusion.py:206-221) and QKVAttentionLegacy.forward (improved_ddpm/unet.py:379-396). */
int asyrp_attention(const void* qkv, void* out, int N, int T, int heads, int head_dim, float scale, void* stream);

/* Tensor-core attention glue (single-head blocks with T >= 128: the q k^T and P v GEMMs run on the conv kernel with
 * weight_batched = 1).  asyrp_transpose_tc: [N][T][ld] (first C channels at `in`) -> [N][C][T].
 * asyrp_softmax_rows: P (fp16) = softmax(scale * S) per row of T <= 1024 fp32 logits, fp32 math. */
int asyrp_transpose_tc(const void* in, void* out, int N, int T, int C, int ld, void* stream);
int asyrp_softmax_rows(const void* S, void* P, long long rows, int T, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ASYRP_B200_H */
