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
  /* layout of `scales`: 0 = one (acc_scale, res_scale) pair for every sample; > 0 = per-sample pairs, that of batch
   * entry n at scales + n*scales_stride floats (requires `scales`; negative is rejected).  Lets one batch carry a
   * different hs_coeff tuple per sample: an edit-strength sweep runs as one batch instead of one trajectory per tuple.
   * Last field, so a zero-initialised descriptor keeps the shared-pair meaning. */
  int scales_stride;
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
/* K-schedule entries of a tile the op's operand-transform warps ready before they run the previous tile's epilogue */
int asyrp_conv_drain_at(void* op);

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

/* asyrp_ddim_update with a (c1, c2) pair per sample: c12 is a DEVICE array [N][2].  Row n gives exactly the bits of
 * asyrp_ddim_update with scalars c12[n]; z (may be NULL) is read only where c1 != 0. */
int asyrp_ddim_update_rows(const float* x, const float* et, const float* em, const float* z, float* x_next,
                           float* x0_out, int N, int Cx, int Ce, int HW, float at, float an, const float* c12,
                           void* stream);

/* Exact inversion (csrc/inversion.cu): the DDIM update of an edit pass anchored to the recorded DDIM inversion of its
 * B input images.  Row n, image b = n % B, in fp32 with the operations of asyrp_ddim_update:
 *   y  = sqrt(an) x0 + c2 et,  x0 = (x - em sqrt(1 - at)) / sqrt(at)
 *   yr = the same operations on (A_cur[b], E_cur[b], E_cur[b])
 *   x_next = A_next[b] + (y - yr)            (subtraction, then addition; never contracted)
 * x, et, em as asyrp_ddim_update ([N][Cx][HW], [N][Ce][HW], Ce >= Cx); A_cur, A_next, E_cur fp32 [B][Cx][HW]; N % B
 * == 0.  x_next may alias x; x0_out (may be NULL) receives the edit's x0.  c12 NULL: c2 for every row; else a DEVICE
 * array [N][2] whose column 1 is row n's c2 (column 0, c1, is not read: no noise is drawn, it would cancel).  A row with
 * x = A_cur and et = em = E_cur gives A_next bit for bit.  With HW % 4 == 0 every pointer must be 16-byte aligned
 * (float4 loads), else 4-byte aligned.  64-bit indexing. */
int asyrp_ddim_update_anchored(const float* x, const float* et, const float* em, const float* a_cur,
                               const float* a_next, const float* e_cur, float* x_next, float* x0_out, int N, int B,
                               int Cx, int Ce, int HW, float at, float an, float c2, const float* c12, void* stream);

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

/* asyrp_slerp_h with the slerp weight of sample n read from t_rows[n] (fp32 [N], device memory); sample n gives the
 * bits of asyrp_slerp_h with t = t_rows[n] (DiffStyle rows with their own hs_coeff in one batch). */
int asyrp_slerp_h_rows(const void* h, const float* dh, long long dh_sample_stride, void* h2, float* stats,
                       int stats_tiles, int N, int C, int H, int W, const float* t_rows, int use_mask, void* stream);

/* Additive direction: h2[n] = c0_n * h[n] + alpha_n * dir, each element v = fmaf(alpha_n, dir, c0_n * h) in fp32
 * (the product rounded first), stored as fp16.  h, h2: fp16 NHWC [N][H][W][C], h2 must not alias h; dir: fp32 NCHW
 * [C][H][W] shared by every sample; coef: fp32 [N][2] = (c0_n, alpha_n) in device memory.  stats:
 * [N][stats_tiles][C/2][2] partial sums of the fp32 v, filled as asyrp_slerp_h fills them (slot 0, the others zeroed).
 * N >= 1, C even, C * H * W and stats_tiles * C at most 2^31 - 1.  Sample n's result does not depend on N. */
int asyrp_add_h_rows(const void* h, const float* dir, void* h2, float* stats, int stats_tiles, int N, int C, int H,
                     int W, const float* coef, void* stream);

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

/* ---- LPIPS-AlexNet: lpips.LPIPS(net='alex', version='0.1'), spatial=False, normalize=False ----------------------
 * Replaces the loss_fn_alex(x, x0) / loss_fn_alex(x0_t, x0) calls of Asyrp.compute_lpips_distance
 * (diffusion_latent.py:1198-1273).  Activations are fp32 NHWC.
 * asyrp_lpips_pack: ScalingLayer, x fp32 NCHW [N][3][H][W] -> (x - shift)/scale as fp32 NHWC [N][H][W][4] (channel 3
 *   zero); shift_scale: 6 floats (shift[3], scale[3]).
 * asyrp_lpips_conv: out = relu(conv(in) + bias), zero padding `pad`, any kh x kw and stride; implicit GEMM on the tensor
 *   cores with TF32 operands (round to nearest) and fp32 accumulation.  in [N][H][W][Cin] (Cin % 4 == 0), out
 *   [N][Ho][Wo][Cout] (Cout % 64 == 0), weight fp32 [Cout][asyrp_lpips_conv_kpad(Cin, kh, kw)]: K = kh*kw*Cin
 *   tap-major / channel-minor, zero columns past K.  bias [Cout] is required; out must not alias in.  The TF32 GEMM's
 *   launcher, shared by every conv and linear layer built on it, refuses Cout above 65535 * 64 (the channel tiles sit
 *   in grid y), in or weight not 16-byte aligned (cp.async) and out or a residual not 8-byte aligned (float2).
 * asyrp_lpips_maxpool: MaxPool2d(3, 2), no padding, floor mode, [N][H][W][C] -> [N][(H-3)/2+1][(W-3)/2+1][C].
 * asyrp_lpips_distance: one layer term of the distance: per pixel, f/(sqrt(sum_c f^2) + 1e-10) of probe row n and of
 *   ref row n % B, squared difference, lin_w [C] (the 1x1 conv C -> 1), mean over the HW pixels; d[n] = term
 *   (+ d[n] when accumulate).  probe [N][HW][C], ref [B][HW][C].  Scratch: partial [N][asyrp_lpips_distance_chunks(HW)]
 *   floats and counters [N] ints, zero before the first call and left zero by every call.  Fixed-order reductions
 *   (integer ticket, no float atomics): d[n] does not depend on N or on the other rows. */
int asyrp_lpips_pack(const float* x, const float* shift_scale, float* out, int N, int H, int W, void* stream);
int asyrp_lpips_conv_kpad(int Cin, int kh, int kw); /* host only */
int asyrp_lpips_conv(const float* in, const float* weight, const float* bias, float* out, int N, int H, int W, int Cin,
                     int Cout, int kh, int kw, int stride, int pad, void* stream);
int asyrp_lpips_maxpool(const float* in, float* out, int N, int H, int W, int C, void* stream);
int asyrp_lpips_distance_chunks(int HW); /* host only */
int asyrp_lpips_distance(const float* probe, const float* ref, int N, int B, int HW, int C, const float* lin_w,
                         float* partial, int* counters, float* d, int accumulate, void* stream);

/* ---- CLIP text tower: OpenAI CLIP's encode_text and the text-direction cosine --------------------------------------
 * Replaces the clip_loss_func.encode_text / CosineSimilarity calls of Asyrp.set_t_edit_t_addnoise
 * (diffusion_latent.py:1319-1329).  Activations are fp32 [P][T][width], P prompts of T tokens, rows = P*T.
 * asyrp_clip_embed: out = token_embedding[ids] + positional_embedding; ids int32 [P][T] (each < the vocabulary),
 *   token_embedding [vocab][width], positional_embedding [T][width].
 * asyrp_clip_layernorm: LayerNorm over width, eps 1e-5, per row of [rows][width]; out may be in.
 * asyrp_clip_linear: out[M][N] = epilogue(in[M][K] @ weight[N][K]^T + bias) (nn.Linear's weight layout), TF32
 *   operands rounded to nearest, fp32 accumulation, the LPIPS conv's GEMM.  K % 32 == 0, N % 64 == 0.  epilogue 1:
 *   identity (bias may be null), 2: QuickGELU z*sigmoid(1.702z), 3: residual + z (residual [M][N], may be out),
 *   7: GELU 0.5 z (1 + erf(z / sqrt 2)) (DINO's MLP).
 * asyrp_clip_attention: causal multi-head attention, head size 64, scale 1/8; qkv [P*T][3*64*heads] as
 *   nn.MultiheadAttention's in_proj packs q | k | v, out [P*T][64*heads] (T <= 128).
 * asyrp_clip_pool: out [P][width] = LayerNorm(x[p][eot]) with eot the first argmax of ids[p].
 * asyrp_clip_cosine: cos[n] = torch.nn.CosineSimilarity(dim=1, eps) of rows a[n], b[n] of [n][dim].
 * Fixed-order reductions, no float atomics, no kernel mixes prompts: a prompt's features do not depend on P. */
int asyrp_clip_embed(const int* ids, const float* token_embedding, const float* positional_embedding, float* out,
                     int P, int T, int width, void* stream);
int asyrp_clip_layernorm(const float* in, const float* gamma, const float* beta, float* out, int rows, int width,
                         void* stream);
int asyrp_clip_linear(const float* in, const float* weight, const float* bias, const float* residual, float* out, int M,
                      int K, int N, int epilogue, void* stream);
int asyrp_clip_attention(const float* qkv, float* out, int P, int T, int heads, void* stream);
int asyrp_clip_pool(const float* x, const int* ids, const float* gamma, const float* beta, float* out, int P, int T,
                    int width, void* stream);
int asyrp_clip_cosine(const float* a, const float* b, float* cos, int n, int dim, float eps, void* stream);

/* ---- CLIP image tower and the directional similarity: OpenAI CLIP's VisionTransformer.forward and CLIPLoss's
 * clip_directional_loss (losses/clip_loss.py:102-117,170-180).  Activations are fp32 [B][T][width], T = 1 + grid^2.
 * asyrp_clip_image_patches: CLIPLoss.preprocess and the patch layout of conv1.  x fp32 [B][3][S][S] in [-1, 1]
 *   (square) -> (x+1)/2 -> F.interpolate(R x R, bicubic, align_corners=False, no antialiasing, A = -0.75, taps clamped
 *   at the edges), R = grid*patch -> (v - mean_c) / std_c with CLIP's mean and std -> out [B*grid^2][kpad]: row
 *   gy*grid + gx of image b, column c*patch^2 + ky*patch + kx (conv1.weight.reshape(width, -1)'s order), columns
 *   3*patch^2 .. kpad-1 zero; kpad = 3*patch^2 rounded up to a multiple of 32.
 * asyrp_clip_image_tokens: out[b][0] = class_embedding + pos[0], out[b][1+p] = patch_emb[b*(T-1) + p] + pos[1+p];
 *   patch_emb [B*(T-1)][width], positional_embedding [T][width].
 * asyrp_clip_layernorm_rows: LayerNorm (eps 1e-5) of rows in + r*ld, r < rows, into dense out [rows][width] (ln_post
 *   of the class token: ld = T*width).  out must not overlap in.
 * asyrp_clip_attention_full: asyrp_clip_attention without the causal mask, T <= 257.
 * asyrp_clip_direction: for each group g of n rows of src and trg [groups*n][dim]:
 *   d = mean_i(trg_i/|trg_i| - src_i/|src_i|), out[g] = d / (|d| + add_eps).  Images: n = 1, add_eps = 1e-7; text
 *   templates: one group, add_eps = 0.  2n + dim <= 12288.
 * Fixed-order reductions, no float atomics, no kernel mixes images or groups. */
int asyrp_clip_image_patches(const float* x, float* out, int B, int S, int grid, int patch, int kpad, void* stream);
int asyrp_clip_image_tokens(const float* patch_emb, const float* class_embedding, const float* positional_embedding,
                            float* out, int B, int T, int width, void* stream);
int asyrp_clip_layernorm_rows(const float* in, long long ld, const float* gamma, const float* beta, float* out,
                              int rows, int width, void* stream);
int asyrp_clip_attention_full(const float* qkv, float* out, int P, int T, int heads, void* stream);
int asyrp_clip_direction(const float* src, const float* trg, float* out, int groups, int n, int dim, float add_eps,
                         void* stream);

/* ---- ArcFace IR-SE50 and the identity similarity: the reference's Backbone(112, 50, 'ir_se') and IDLoss
 * (models/insight_face/model_irse.py, losses/id_loss.py).  Activations are fp32 NHWC.
 * asyrp_arcface_preprocess: IDLoss.extract_feats's crop x[:, :, 35:223, 32:220] and AdaptiveAvgPool2d((112, 112)):
 *   x fp32 NCHW [B][3][H][W] (H >= 223, W >= 220) -> out fp32 NHWC [B][112][112][4], channel 3 zero.  Bin i covers
 *   crop rows [floor(188 i / 112), ceil(188 (i+1) / 112)), likewise columns; summed row by row, left to right.
 * asyrp_arcface_conv: out = epilogue(conv(in) + bias), k x k, zero padding `pad`, any stride, the LPIPS conv's TF32
 *   implicit GEMM; prelu null: bias alone (bias may be null), else PReLU with per-channel slopes prelu [Cout] (bias
 *   may be null).  in [N][H][W][Cin] (Cin % 4 == 0), out [N][Ho][Wo][Cout] (Cout % 64 == 0), weight fp32
 *   [Cout][asyrp_lpips_conv_kpad(Cin, k, k)].
 * asyrp_arcface_affine: out = in * scale[c] + shift[c] over [rows][C] (C % 4 == 0): a folded eval-mode BatchNorm.
 * asyrp_arcface_se_scale: SEModule's gate, one CTA per sample: scale[n][c] = sigmoid(fc2 relu(fc1 mean_hw(res[n])))
 *   with res [N][HW][C], fc1 [C/16][C], fc2 [C][C/16]; C a multiple of 16 that divides 512.
 * asyrp_arcface_se_apply: out = res * scale[n][c] + shortcut[n][y*ss][x*ss][c], res and out [N][Ho][Wo][C], shortcut
 *   [N][Hs][Ws][C], ss 1 (identity, conv shortcut) or 2 (MaxPool2d(1, 2)); out2 (optional, with bn_scale / bn_shift
 *   [C]) = out * bn_scale + bn_shift, the next block's pre-conv BatchNorm.
 * asyrp_arcface_l2norm: out[r] = in[r] / |in[r]| (no epsilon) over [rows][dim]; out must not alias in.
 * asyrp_arcface_dot: id[j] = edited[j] . src[j % B] over rows of dim floats (IDLoss = 1 - id).
 * Fixed-order reductions, no float atomics, no kernel mixes samples. */
int asyrp_arcface_preprocess(const float* x, float* out, int B, int H, int W, void* stream);
int asyrp_arcface_conv(const float* in, const float* weight, const float* bias, const float* prelu, float* out, int N,
                       int H, int W, int Cin, int Cout, int k, int stride, int pad, void* stream);
int asyrp_arcface_affine(const float* in, const float* scale, const float* shift, float* out, long long rows, int C,
                         void* stream);
int asyrp_arcface_se_scale(const float* res, const float* fc1, const float* fc2, float* scale, int N, int HW, int C,
                           void* stream);
int asyrp_arcface_se_apply(const float* res, const float* scale, const float* shortcut, float* out,
                           const float* bn_scale, const float* bn_shift, float* out2, int N, int Ho, int Wo, int C,
                           int Hs, int Ws, int ss, void* stream);
int asyrp_arcface_l2norm(const float* in, float* out, int rows, int dim, void* stream);
int asyrp_arcface_dot(const float* src, const float* edited, float* id, int n, int B, int dim, void* stream);

/* ---- Face-parsing BiSeNet (BiSeNet(n_classes=19), eval mode) and the segmentation consistency of an edit
 * (asyrp_official_b200/face_parsing.py gives the network).  Activations are fp32 NHWC.
 * asyrp_faceparse_pack: x fp32 NCHW [B][3][H][W] -> out fp32 NHWC [B][S][S][4]: clamp to [-1, 1], map to [0, 1],
 *   bilinear resize to S x S (align_corners=False; rows blended first), normalise with ImageNet's mean (0.485, 0.456,
 *   0.406) and std (0.229, 0.224, 0.225); channel 3 zero.
 * asyrp_faceparse_conv: out = epilogue(conv(in) + bias), k x k, zero padding `pad`, any stride, the TF32 implicit GEMM
 *   of asyrp_arcface_conv; relu 0: bias alone (bias may be null); relu 1 without residual: max(v, 0) (bias needed);
 *   residual [N][Ho][Wo][Cout] (relu 1): max(residual + v, 0).  in [N][H][W][Cin] (Cin % 4 == 0), out Cout % 64 == 0,
 *   weight fp32 [Cout][asyrp_lpips_conv_kpad(Cin, k, k)].
 * asyrp_faceparse_maxpool: MaxPool2d(3, 2, padding 1) of [N][H][W][C] (C % 4 == 0) into [N][(H-1)/2+1][(W-1)/2+1][C].
 * asyrp_faceparse_gate: one CTA per sample: m = mean_hw(in[n]) of in [N][HW][C] (C divides 512), h = act1(w1 m + b1)
 *   (w1 [C1][C]), out[n] = act2(w2 h + b2) (w2 [C2][C1]) or h when w2 is null; biases may be null; act 0 identity,
 *   1 ReLU, 2 sigmoid; C1, C2 <= 512.
 * asyrp_faceparse_apply: out[n][y][x][c] = f[n][y/up][x/up][c] * gate[n][c] + add, out [N][H*up][W*up][C], up 1 or 2;
 *   add = add[n][c] (add_map 0) or add[n][y/up][x/up][c] (add_map 1, a map the size of f); C % 4 == 0.
 * asyrp_faceparse_labels: labels uint8 [N][Ho][Wo] = argmax over ncls classes (first wins a tie) of
 *   F.interpolate(logits, (Ho, Wo), 'bilinear', align_corners=True), logits [N][Hi][Wi][ld] (classes 0 .. ncls-1 of a
 *   row of ld floats); ncls <= 64, Wi * ncls <= 12288, N <= 65535.
 * asyrp_faceparse_agreement: agree[j] = number of pixels where the labels of edited row j equal those of source row
 *   (row0 + j) % B (as asyrp_faceparse_labels computes them), label maps never stored; row0 >= 0 lets a chunk of
 *   edited rows starting at row0 keep its pairing; edited_logits [n][Hi][Wi][ld],
 *   src_logits [B][Hi][Wi][ld]; Wi * ncls <= 6144, n <= 65535.
 * Fixed-order reductions, no float atomics, no kernel mixes samples. */
int asyrp_faceparse_pack(const float* x, float* out, int B, int H, int W, int S, void* stream);
int asyrp_faceparse_conv(const float* in, const float* weight, const float* bias, const float* residual, float* out,
                         int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int relu, void* stream);
int asyrp_faceparse_maxpool(const float* in, float* out, int N, int H, int W, int C, void* stream);
int asyrp_faceparse_gate(const float* in, const float* w1, const float* b1, int C1, int act1, const float* w2,
                         const float* b2, int C2, int act2, float* out, int N, int HW, int C, void* stream);
int asyrp_faceparse_apply(const float* f, const float* gate, const float* add, int add_map, float* out, int N, int H,
                          int W, int C, int up, void* stream);
int asyrp_faceparse_labels(const float* logits, unsigned char* labels, int N, int Hi, int Wi, int ld, int ncls, int Ho,
                           int Wo, void* stream);
int asyrp_faceparse_agreement(const float* src_logits, const float* edited_logits, unsigned int* agree, int n, int B,
                              int row0, int Hi, int Wi, int ld, int ncls, int Ho, int Wo, void* stream);

/* ---- Inception-v3 pool features (the FID variant of pytorch-fid) and the set statistics of FID and KID
 * (asyrp_official_b200/fid.py gives the network and the metric).  Activations are fp32 NHWC.
 * asyrp_fid_pack: x fp32 NCHW [B][3][H][W] -> out fp32 NHWC [B][S][S][4]: q = the u8 torchvision's save_image writes
 *   (fp32 (x + 1) * 0.5 * 255 + 0.5, clamped to [0, 255], truncated), q / 255, bilinear resize to S x S
 *   (align_corners=False; rows blended first), 2 v - 1; channel 3 zero; out 16-byte aligned.
 * asyrp_fid_conv: out = max(conv(in) + bias, 0), kh x kw, zero padding padh rows / padw columns, any stride, the TF32
 *   implicit GEMM of asyrp_arcface_conv; in [N][H][W][Cin] (Cin % 4 == 0); weight fp32
 *   [Cout][asyrp_lpips_conv_kpad(Cin, kh, kw)] and bias [Cout] with Cout % 64 == 0 (zero rows past the layer's width);
 *   channels [0, cstore) of out rows [N][Ho][Wo] of pitch ldo are written, the rest untouched: cstore even,
 *   0 < cstore <= Cout, ldo even and >= cstore, out 8-byte aligned (a channel slice of a wider tensor).  The geometry
 *   is checked in 64 bits: H + 2 padh and W + 2 padw at most 2^31 - 1, kh kw Cin at most 2^31 - 32 (Kpad in int),
 *   N Ho Wo below 2^31; the launcher's limits of asyrp_lpips_conv apply.
 * asyrp_fid_pool: mode 0 max-pool 3x3 / 2 without padding (H, W >= 3), 1 avg-pool 3x3 / 1 pad 1 without the padding
 *   (count_include_pad=False; taps summed in row-major order, then divided by their count), 2 max-pool 3x3 / 1 pad 1
 *   (padding never wins) of in [N][H][W][C] (C % 4 == 0) into out rows of pitch ldo (ldo % 4 == 0, ldo >= C); in and
 *   out 16-byte aligned.
 * asyrp_fid_mean: out[n][c] = the mean of in [N][HW][C] over the HW pixels, summed in pixel order.
 * asyrp_fid_moments: mu [d] and sigma [d][d] (fp64) of the n rows of x fp32 [n][d]: column means and the centred
 *   covariance with the n - 1 denominator; 2 <= n <= 2^31 - 16, d % 64 == 0, d <= 65535 * 64, n d < 2^40.
 * asyrp_fid_kernel_sum: out[0] = sum over i < n, j < m of (x[i] . y[j] / d + 1)^3 in fp64, pairs i == j skipped with
 *   exclude_diag; x fp32 [n][d], y fp32 [m][d], d % 16 == 0, n <= 65535 * 64; partial:
 *   asyrp_fid_kernel_sum_partials(n, m) doubles of workspace, one per 64 x 64 tile (-1: n or m not positive, or more
 *   than 2^31 - 256 tiles, which the call refuses).
 * asyrp_fid_pack_u8: x u8 NHWC [B][H][W][3] (a decoded image file) -> out as asyrp_fid_pack: q = x, q / 255,
 *   bilinear resize to S x S, 2 v - 1 (pytorch-fid's ToTensor path); bit-identical to asyrp_fid_pack of
 *   x / 127.5 - 1 as fp32 NCHW (whose quantiser gives back q); out 16-byte aligned.
 * asyrp_fid_kernel_sum_subsets: out[z] (z < subsets, fp64) = sum over i, j < s of
 *   (x[idx_x[z][i]] . y[idx_y[z][j]] / d + 1)^3, pairs i == j skipped with exclude_diag: bit-identical to
 *   asyrp_fid_kernel_sum of the gathered rows x[idx_x[z]], y[idx_y[z]].  x fp32 [n][d], y fp32 [m][d], idx_x / idx_y
 *   int32 [subsets][s] on the device; d % 16 == 0, subsets <= 65535, s >= 2 with exclude_diag.  The indices are not
 *   checked on the device: a row outside [0, n) / [0, m) is read out of bounds (ops.fid_kernel_sum_subsets checks
 *   them).  partial: asyrp_fid_kernel_sum_subsets_partials(s, subsets) doubles of workspace (-1: too large).
 * Fixed-order reductions, no atomics, no kernel mixes samples. */
int asyrp_fid_pack(const float* x, float* out, int B, int H, int W, int S, void* stream);
int asyrp_fid_pack_u8(const unsigned char* x, float* out, int B, int H, int W, int S, void* stream);
int asyrp_fid_conv(const float* in, const float* weight, const float* bias, float* out, int N, int H, int W, int Cin,
                   int Cout, int kh, int kw, int stride, int padh, int padw, int ldo, int cstore, void* stream);
int asyrp_fid_pool(const float* in, float* out, int N, int H, int W, int C, int mode, int ldo, void* stream);
int asyrp_fid_mean(const float* in, float* out, int N, int HW, int C, void* stream);
int asyrp_fid_moments(const float* x, double* mu, double* sigma, int n, int d, void* stream);
int asyrp_fid_kernel_sum_partials(int n, int m); /* host only */
int asyrp_fid_kernel_sum(const float* x, const float* y, double* partial, double* out, int n, int m, int d,
                         int exclude_diag, void* stream);
int asyrp_fid_kernel_sum_subsets_partials(int s, int subsets); /* host only */
int asyrp_fid_kernel_sum_subsets(const float* x, const float* y, const int* idx_x, const int* idx_y, double* partial,
                                 double* out, int n, int m, int s, int subsets, int d, int exclude_diag, void* stream);

/* k-nearest-neighbour balls for precision / recall / density / coverage (csrc/prdc.cu).
 * D(u, v) = sum_c (u_c - v_c)^2, each difference and the sum in fp64, summed in feature order: identical rows give 0,
 * and a pair's D is the same bits in every launch.  The distance matrix is never written to memory.
 * asyrp_fid_knn_radii: radii[i] (fp64) = the (k + 1)-th smallest D(x[i], x[j]) over every j < n, j = i included (the
 *   squared distance to the k-th nearest other row, duplicates counted), x fp32 [n][d] row-major; 1 <= k <= 32,
 *   n >= k + 1, d >= 1.  work: asyrp_fid_knn_radii_workspace(n, k) doubles (-1: bad n or k), the per-row lists of the
 *   CTAs a row's columns are split over; the split depends on the device, the radii do not.
 * asyrp_fid_knn_counts: one pass over the n x m pairs of a fp32 [n][d] and b fp32 [m][d] with radii ra [n], rb [m]
 *   (fp64): b_in_a[j] = #{i : D(a_i, b_j) < ra[i]}, a_in_b[i] = #{j : D < rb[j]}, a_covered[i] = #{j : D < ra[i]}.
 *   The three outputs are distinct buffers and are overwritten; integer atomics keep them exact.  n, m, d >= 1,
 *   n <= 65535 * 64. */
long long asyrp_fid_knn_radii_workspace(int n, int k); /* host only */
int asyrp_fid_knn_radii(const float* x, double* radii, double* work, int n, int d, int k, void* stream);
int asyrp_fid_knn_counts(const float* a, const double* ra, int n, const float* b, const double* rb, int m, int d,
                         unsigned* b_in_a, unsigned* a_in_b, unsigned* a_covered, void* stream);

/* ---- Content preservation: PSNR, SSIM and MS-SSIM of the u8 images save_image writes (csrc/preservation.cu;
 * asyrp_official_b200/preservation.py combines the statistics).  Edited row j is compared with source row j % B.
 * asyrp_png_quantize: x fp32 NCHW [B][3][H][W] -> q u8 [B][3][H][W], the value save_image writes (as asyrp_fid_pack);
 *   lvl0 fp64 q / 255 and xq fp32 (2 q - 255) / 255 (LPIPS's input for a loaded PNG) in the same layout, each
 *   skipped when null.  x, xq 4-byte and lvl0 8-byte aligned.
 * asyrp_preserve_sse: sse[j] (int64) = sum over the plane = 3 H W elements of (edited[j] - src[j % B])^2, exact;
 *   src u8 [B][plane], edited u8 [n][plane], plane <= 2^47.
 * asyrp_ssim_level: stats[j][c] = (mean SSIM map, mean cs map) over the (H - 10) x (W - 10) valid pixels of channel c,
 *   fp64, from an 11-tap Gaussian window (sigma 1.5, normalised) applied separably without padding, C1 = 0.01^2,
 *   C2 = 0.03^2 (pytorch_msssim's _ssim with data_range 1); src fp64 [B][3][H][W], edited fp64 [n][3][H][W],
 *   stats fp64 [n][3][2]; H, W >= 11, 3 n <= 2^31 - 1.  A row's statistics are the same bits for any n and B.
 * asyrp_ssim_pool2: out = avg_pool2d(in, 2, stride 2, padding (H mod 2, W mod 2)), padding counted in the divisor,
 *   in fp64 [rows][3][H][W] -> out fp64 [rows][3][ceil(H / 2)][ceil(W / 2)]; out must not alias in.
 * No allocation, no synchronisation, no atomics. */
int asyrp_png_quantize(const float* x, unsigned char* q, double* lvl0, float* xq, int B, int H, int W, void* stream);
int asyrp_preserve_sse(const unsigned char* src, const unsigned char* edited, long long* sse, int n, int B,
                       long long plane, void* stream);
int asyrp_ssim_level(const double* src, const double* edited, double* stats, int n, int B, int H, int W, void* stream);
int asyrp_ssim_pool2(const double* in, double* out, int rows, int H, int W, void* stream);

/* Bottleneck statistics for h-space directions (csrc/hspace.cu), fp64, every sum in index order from 0:
 * asyrp_h_gram: G fp64 [n][n], G[i][j] = sum_k (x[i][k] - mu[k]) (x[j][k] - mu[k]) over the d features, the centred
 *   sample Gram (exactly symmetric); x fp32 [n][d], mu fp64 [d].  n >= 2, d > 0, n d < 2^31.
 * asyrp_h_combine: out fp64 [K][d], out[k][j] = sum_r w[k][r] (x[r][j] - mu[j]) over the n rows; w fp64 [K][n]; mu
 *   fp64 [d] or NULL (then 0).  n, d, K > 0; n d, K n and K d < 2^31.  Set means (w = 1/n), mean differences and
 *   principal directions from Gram eigenvectors (w = u_k / sqrt(lambda_k)).
 * No allocation, no synchronisation, no atomics. */
int asyrp_h_gram(const float* x, const double* mu, double* G, int n, int d, void* stream);
int asyrp_h_combine(const float* x, const double* w, const double* mu, double* out, int n, int d, int K, void* stream);

/* Region-restricted edits (csrc/region.cu): a soft mask per image from face-parsing labels, and the blend of an edit
 * pass back into the unedited trajectory outside it.
 * asyrp_blend_rows: in place, x[n][c][p] = fmaf(m, x, (1 - m) * r) in fp32 with m = mask[n % B][p] and
 *   r = ref[n % B][c][p]; x fp32 [N][C][HW], ref fp32 [B][C][HW], mask fp32 [B][HW].  m = 1 gives x and m = 0 gives r
 *   exactly.  N % B == 0; 64-bit indexing.  With HW % 4 == 0 the three pointers must be 16-byte aligned (float4
 *   loads), else 4-byte aligned.
 * asyrp_region_mask: mask fp32 [N][S][S] = 1 where a label of the pixel's footprint in labels u8 [N][512][512] (rows
 *   [ceil(y 512 / S), ceil((y + 1) 512 / S)), columns likewise) has its bit set in class_bits (labels >= 32 never),
 *   else 0.  1 <= S <= 512, 1 <= N <= 65535.
 * asyrp_mask_dilate: out = the max of in over [i - r, i + r] along axis (0: x, 1: y), indices outside the image left
 *   out; 0 <= r <= 32.  Both axes give the (2r + 1)^2 square max filter.
 * asyrp_mask_blur: out[i] = sum_{k=-R..R} taps[k + R] in[clamp(i + k, 0, S - 1)] along axis, fp32 fmaf in tap order; a
 *   window whose inputs are all equal gives that value exactly.  taps fp32 [2R + 1] on the device, 0 <= R <= 48.
 * The mask kernels take fp32 [N][S][S] images, 4-byte aligned; out must not be in.
 * asyrp_compose_rows: in place, the K attribute rows of every image replaced by one composite against the origin
 *   pass: x fp32 [K B][C][HW] attribute-major (row k B + j), ref fp32 [B][C][HW], masks fp32 [K][B][HW].  Per pixel,
 *   in fp32: s = M_1 + .. + M_K in order; w_k = M_k, w_0 = 1 - s if s <= 1, else w_k = M_k / s, w_0 = 0; then
 *   acc = w_0 r and acc = fmaf(w_k, x[k B + j], acc) for k = 1..K, written to all K rows of image j.  With K = 1 this
 *   is asyrp_blend_rows bit for bit.  1 <= K <= 8, B, C, HW > 0; 64-bit indexing.  With HW % 4 == 0 the three
 *   pointers must be 16-byte aligned (float4 loads), else 4-byte aligned.
 * No allocation, no synchronisation, no atomics. */
int asyrp_blend_rows(float* x, const float* ref, const float* mask, int N, int B, int C, int HW, void* stream);
int asyrp_compose_rows(float* x, const float* ref, const float* masks, int K, int B, int C, int HW, void* stream);
int asyrp_region_mask(const unsigned char* labels, unsigned class_bits, float* mask, int N, int S, void* stream);
int asyrp_mask_dilate(const float* in, float* out, int N, int S, int r, int axis, void* stream);
int asyrp_mask_blur(const float* in, const float* taps, float* out, int N, int S, int R, int axis, void* stream);

/* DINO ViT and the self-similarity structure distance (csrc/dino.cu): facebookresearch/dino's VisionTransformer
 * (backbone, eval mode) and Splice's key self-similarity loss.  Activations are fp32 [B][T][D], T = 1 + grid^2 <= 1025,
 * D = 64 * heads.  The patch embedding and every linear layer run on asyrp_clip_linear (epilogue 7: the exact GELU
 * 0.5 v (1 + erf(v / sqrt 2)) of fc1), cls + pos on asyrp_clip_image_tokens, the CLS cosine on asyrp_clip_cosine.
 * asyrp_dino_pack: x fp32 [B][3][S][S] in [-1, 1] (square) -> (x+1)/2 -> F.interpolate(R x R, bilinear,
 *   align_corners=False, antialias=True), R = grid*patch, with the taps of PyTorch's _upsample_bilinear2d_aa (support
 *   max(1, S/R), triangle weights normalised per output pixel; rows of taps summed first) -> (v - mean_c) / std_c with
 *   ImageNet's mean and std -> out [B*grid^2][kpad] in conv-weight column order (c, ky, kx), columns 3*patch^2 ..
 *   kpad-1 zero; kpad = 3*patch^2 rounded up to a multiple of 32.  S == R gives (x+1)/2 exactly; S, R <= 4096.
 * asyrp_dino_layernorm: LayerNorm (eps > 0) of rows in + r*ld, r < rows, into dense out [rows][width]; out may be in
 *   only when ld == width, and must not overlap it otherwise.
 * asyrp_dino_attention: non-causal softmax attention, head size 64, scale 1/8; qkv [B*T][3D] packs q | k | v, out
 *   [B*T][D].  Flash-style: key tiles of 64 in a fixed order, QK^T and PV on TF32 mma.sync m16n8k8, online softmax in
 *   fp32.  T <= 1025, B and heads <= 65535; qkv 16-byte and out 8-byte aligned; out must not overlap qkv.
 * asyrp_dino_selfsim_distance: out fp64 [P], out[p] = (1/T^2) sum_ij (Sa_ij - Sb_ij)^2 with S_ij = k^_i . k^_j,
 *   k^ = k / max(|k|, eps), the key of token i of pair p's image a at keys + (ia[p] + i) * ld (D floats) and of b at
 *   ia -> ib.  ia, ib int64 [P] on the device; ld >= D (the qkv buffer with ld = 3D at offset D gives the keys without a
 *   copy).  64 x 64 tiles over i <= j (off-diagonal tiles twice), fp32 fmaf dot products in column order, per-tile fp64
 *   partials in partial [P][asyrp_dino_selfsim_partials(T)] summed in tile order: equal rows give exactly 0.
 *   T <= 1025, P <= 65535; keys 4-byte and ia, ib, partial, out 8-byte aligned.
 * asyrp_dino_selfsim_partials: the tile pairs of T tokens (the partial columns), -1 for T outside 1..1025.
 * Fixed-order reductions, no float atomics, no kernel mixes images. */
int asyrp_dino_pack(const float* x, float* out, int B, int S, int grid, int patch, int kpad, void* stream);
int asyrp_dino_layernorm(const float* in, long long ld, const float* gamma, const float* beta, float* out, int rows,
                         int width, float eps, void* stream);
int asyrp_dino_attention(const float* qkv, float* out, int B, int T, int heads, void* stream);
int asyrp_dino_selfsim_partials(int T);
int asyrp_dino_selfsim_distance(const float* keys, long long ld, const long long* ia, const long long* ib, int P, int T,
                                int D, float eps, double* partial, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ASYRP_B200_H */
