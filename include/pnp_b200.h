/*
 * pnp_b200.h -- C-ABI of the H100-native (sm_90a) PnP-AdaNet hot path.
 *
 * The reference (carrenD/Medical-Cross-Modality-Domain-Adaptation) is pure Python over TensorFlow-1.4
 * and has no FFI of its own; the narrowest stable seam is the layers.py / ops.py operator surface
 * (SURVEY.md 8b).  Every entry point below replaces the TF-1.4 op(s) that one of those Python
 * functions instantiates; the reference call site is cited per function as file:line relative to the
 * reference tree.  The Python host layer (medical-cross-modality-domain-adaptation_b200/layers.py,
 * ops.py, ...) binds these with ctypes; INTEGRATION.md shows the stub.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise
 *   - activations NHWC fp32, conv weights HWIO fp32 ([kh][kw][Cin][Cout]) exactly like the reference
 *   - `stream` is a cudaStream_t passed as void*; launchers are asynchronous and re-entrant
 *   - return 0 on success, otherwise a cudaError_t value or one of the PNP_ERR_* codes;
 *     pnp_error_string() renders either.  Launchers never allocate device memory.
 */
#ifndef PNP_B200_H_
#define PNP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PNP_ERR_BAD_ARG 100001
#define PNP_ERR_UNSUPPORTED 100002
#define PNP_ERR_DRIVER 100003

/* activation codes for the fused BN/activation kernels */
#define PNP_ACT_NONE 0
#define PNP_ACT_RELU 1   /* tf.nn.relu         (layers.py:14) */
#define PNP_ACT_LRELU 2  /* tf.nn.leaky_relu, alpha=0.2 (layers.py:12) */

/* Geometry of one convolution.  Zero padding only: TF 'SAME' is expressed through (pad_t, pad_l)
 * with the asymmetric remainder falling on the bottom/right implicitly (out-of-range taps read 0);
 * the reference's 'SYMMETRIC' mode is pnp_mirror_pad_fwd followed by a pad-free ('VALID') conv. */
typedef struct {
  int B, H, W, Cin;   /* input  [B,H,W,Cin]    */
  int Ho, Wo, Cout;   /* output [B,Ho,Wo,Cout] */
  int kh, kw;
  int stride, dil;
  int pad_t, pad_l;
} pnp_conv_geom;

/* Optional dropout fused into producers: multiplier = (philox(seed, stream, idx) < keep) / keep.
 * seed_ptr == NULL or keep >= 1 disables it (tf.nn.dropout, layers.py:25,74,93). */
typedef struct {
  const unsigned long long* seed_ptr; /* device scalar */
  unsigned long long stream;
  float keep;
} pnp_dropout_cfg;

const char* pnp_error_string(int code);
int pnp_version(void);
/* 1 if the loaded library carries the wgmma/TMA convolution path and the device is sm_90 (Hopper) */
int pnp_tc_available(void);
/* tile configuration chosen by the most recent pnp_conv2d_tc_fwd / _dgrad call (N tile, K block, split-K factor); lets the
   benchmark attribute each timed launch to a kernel instantiation.  Host-side bookkeeping only. */
int pnp_tc_last_config(int* block_n, int* block_k, int* ksplit);

/* ---- convolution, general SIMT fp32 path (conv_simt.cu) --------------------------------------
 * replaces tf.nn.conv2d (layers.py:18,24,67,73) and tf.nn.atrous_conv2d (layers.py:86,92) plus
 * their TF-generated gradients (Conv2DBackpropInput / Conv2DBackpropFilter). */
int pnp_conv2d_fwd(const float* x, const float* w, float* y, const pnp_conv_geom* g,
                   const pnp_dropout_cfg* drop, int accumulate, void* stream);
/* dx[B,H,W,Cin] (+)= conv^T(dy, w).  wT is w with the last two axes swapped ([kh][kw][Cout][Cin]),
 * produced by pnp_weight_transpose. */
int pnp_conv2d_dgrad(const float* dy, const float* wT, float* dx, const pnp_conv_geom* g,
                     int accumulate, void* stream);
/* dw[kh][kw][Cin][Cout] += x (*) dy  (always accumulates: gradient arenas are zeroed per step) */
int pnp_conv2d_wgrad(const float* x, const float* dy, float* dw, const pnp_conv_geom* g, void* stream);
int pnp_weight_transpose(const float* w, float* wT, int taps, int Cin, int Cout, void* stream);
/* The segmenter tail in one launch: y[B, a*r, b*r, Cout] = conv_{kh x kw, SYMMETRIC}(PS_r(X), w) with X = [B, a, b, G*r*r]
 * (ops.PS ops.py:23-27 + tf.pad SYMMETRIC + tf.nn.conv2d VALID, source_segmenter.py:200-207 / adversarial.py:312-316): the
 * phase shift and the mirror padding are index maps applied by the tile loader.  w HWIO [kh][kw][G][Cout], Cout in {5, 8},
 * odd kernels up to 5x5.  order_b1: the reference's batch_size == 1 sub-pixel order (ops.py:11-20). */
int pnp_ps_mirror_conv_fwd(const float* X, const float* w, float* y, int B, int a, int b, int G, int r, int kh, int kw,
                           int Cout, int order_b1, void* stream);
/* its gradient w.r.t. X in one launch: dX = PS_r^T(mirror_pad^T(conv^T(dy, w))) (transposed convolution, fold of the mirrored
 * border, inverse phase shift), dy = [B, a*r, b*r, Cout] */
int pnp_ps_mirror_conv_bwd(const float* dy, const float* w, float* dX, int B, int a, int b, int G, int r, int kh, int kw,
                           int Cout, int order_b1, void* stream);

/* ---- convolution, wgmma + TMA tensor-core path (conv_tc.cu) ------------------------------------
 * Same math as pnp_conv2d_fwd for convolutions whose Cin and Cout are each a multiple of 64, or exactly 32 or 16 (any stride /
 * dilation / kernel <= 5x5; K blocks of 64 / 32 / 16 channels = SWIZZLE_128B / 64B / 32B operand tiles), operands pre-split into
 * bf16 planes (pnp_split_bf16); nterms = 3 gives fp32-grade results (hi*hi + hi*lo + lo*hi), nterms = 1 is the plain bf16 path
 * of BASELINE config 5.  Unsupported shapes return PNP_ERR_UNSUPPORTED (the caller then uses pnp_conv2d_*).  Layers with very
 * few tiles and a deep reduction are split along K inside the call (atomic accumulation into a zeroed y; bn_sum/bn_sumsq are then
 * produced by an internal pnp_bn_stats pass).  bn_sum/bn_sumsq with accumulate != 0 returns PNP_ERR_BAD_ARG: the statistics
 * would be of the new contribution on one path and of old + new on the other.  The weight gradient takes Cin in {32, 64k} and
 * Cout = 64k. */
int pnp_split_bf16(const float* x, uint16_t* hi, uint16_t* lo, long long n, void* stream);
/* w HWIO fp32 -> bf16 planes: for_dgrad == 0: [tap][Cout][Cin] (K-major B operand of the forward conv);
 * for_dgrad != 0: [tap][Cin][Cout] (K-major B operand of the data gradient) */
int pnp_split_weight_bf16(const float* w, uint16_t* hi, uint16_t* lo, int kh, int kw, int Cin, int Cout,
                          int for_dgrad, int cin_pad /* forward layout only: zero-pad Cin up to this (0 = none) */, void* stream);
/* [rows, C] fp32 -> [rows, Cpad] bf16 planes with zero channels >= C: Cin = 32 layers ride the 64-channel K chunk */
int pnp_split_bf16_pad(const float* x, uint16_t* hi, uint16_t* lo, long long rows, int C, int Cpad, void* stream);
int pnp_conv2d_tc_fwd(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                      float* y, const pnp_conv_geom* g, int nterms, const pnp_dropout_cfg* drop,
                      int accumulate, double* bn_sum, double* bn_sumsq, void* stream);

/* Forward convolution with a FUSED epilogue: y = act(dropout(conv) * scale[c] + shift[c] + skip) -- inference-mode batch norm
 * (tf.contrib.layers.batch_norm(is_training=False), layers.py:95-100: scale = gamma*rsqrt(moving_var+eps), shift = beta -
 * moving_mean*scale), the residual add with channel-pad skip (layers.py:160-166) and the activation (layers.py:12-14) applied
 * to the accumulator before it leaves the SM; optionally also emits the bf16 (hi, lo) operand planes of y for the next tensor-core
 * convolution (y itself may then be NULL).  This is the whole frozen-segmenter forward of the D step and the evaluation path
 * (adversarial.py:840-862, 993-1052): one kernel per layer, no z round trip.  ep == NULL: identical to pnp_conv2d_tc_fwd.
 * Batch statistics (bn_sum/bn_sumsq) are statistics of z and cannot be combined with a fused epilogue. */
typedef struct {
  const float* scale;   /* [Cout] or NULL */
  const float* shift;   /* [Cout] or NULL (both or neither) */
  const float* skip;    /* [B,Ho,Wo,skip_C] fp32 or NULL */
  int skip_C, skip_off; /* skip is added to channels [skip_off, skip_off + skip_C) */
  int act;              /* PNP_ACT_* */
  uint16_t* y_hi;       /* optional [B,Ho,Wo,Cout] bf16 planes of y */
  uint16_t* y_lo;       /* required with y_hi when nterms == 3 */
} pnp_tc_epilogue;
int pnp_conv2d_tc_fwd_fused(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                            float* y, const pnp_conv_geom* g, int nterms, const pnp_dropout_cfg* drop, int accumulate,
                            double* bn_sum, double* bn_sumsq, const pnp_tc_epilogue* ep, void* stream);

/* dx[B,H,W,Cin] (+)= conv^T(dy, w) on the tensor cores.  g is the FORWARD geometry; stride s > 1 is decomposed into s*s
 * stride-1 phase convolutions (no multiplications by the zeros a transposed convolution would insert). */
int pnp_conv2d_tc_dgrad(const uint16_t* dy_hi, const uint16_t* dy_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                        float* dx, const pnp_conv_geom* g, int nterms, int accumulate, void* stream);
/* dw[kh][kw][Cin][Cout] += x (*) dy on the tensor cores (both operands MN-major straight from the NHWC planes; pixel range split
 * across CTAs, fp32 vector atomics into dw).  x planes are the (mirror-padded) forward input. */
int pnp_conv2d_tc_wgrad(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* dy_hi, const uint16_t* dy_lo,
                        float* dw, const pnp_conv_geom* g, int nterms, int x_channels /* channels of the x planes, 0 = Cin */,
                        void* stream);

/* ---- batch norm + activation (+ residual skip) (elementwise.cu) ----------------------------------
 * replaces tf.contrib.layers.batch_norm(decay .9, eps 1e-3) (layers.py:95-100), the activation
 * (layers.py:12-14) and the residual add with channel-pad skip (layers.py:160-166,182-189). */
int pnp_bn_stats(const float* z, long long M, int C, double* sum, double* sumsq, void* stream);
/* training != 0: batch statistics (biased var), moving stats <- 0.9*moving + 0.1*(mean, unbiased var).  The variance is one-pass,
 * var = sumsq/M - mean^2 from pnp_bn_stats' fp32 partial sums (64 rows per thread, then fp64): its error is bounded by a small
 * multiple of 2^-24 * E[z^2], not of var, so the relative error of invstd grows as (mean/std)^2 (DESIGN 4.4).  invstd is within
 * 2 fp32 ulps of the correctly rounded 1/sqrt(fl(var + eps)).
 * training == 0: moving statistics.  Writes scale=gamma*invstd, shift=beta-mean*scale, mean, invstd. */
int pnp_bn_finalize(const double* sum, const double* sumsq, long long M, int C, const float* gamma,
                    const float* beta, float* moving_mean, float* moving_var, int training,
                    float* scale, float* shift, float* mean, float* invstd, void* stream);
/* pnp_bn_finalize + pnp_bn_act_apply in ONE launch: every CTA derives scale/shift from the fp64 batch sums (training) or the
 * moving statistics into shared memory; CTA 0 performs the moving-average update and writes mean / invstd (optional, for the
 * backward pass).  y may be NULL when only the planes are wanted.  C <= 1024. */
int pnp_bn_apply_fused(const float* z, const double* sum, const double* sumsq, long long M, int C, const float* gamma,
                       const float* beta, float* moving_mean, float* moving_var, int training, const float* skip, int Cs,
                       int skip_off, int act, float* y, uint16_t* y_hi, uint16_t* y_lo, float* mean_out, float* invstd_out,
                       void* stream);
/* pnp_bn_bwd_finalize + pnp_bn_bwd_apply in ONE launch (dgamma += sum_gx, dbeta += sum_g by CTA 0; sums may be NULL for a
 * frozen inference-mode batch norm: dz = gamma * invstd * g) */
int pnp_bn_bwd_apply_fused(const float* g, const float* z, const float* mean, const float* invstd, const float* gamma,
                           const double* sum_g, const double* sum_gx, long long M, int C, int training,
                           const pnp_dropout_cfg* drop, float* dgamma, float* dbeta, float* dz, uint16_t* dz_hi,
                           uint16_t* dz_lo, void* stream);
/* The same backward pass WITHOUT the fp32 g = dy*act'(y) round trip (layers whose g nobody else needs, i.e. no residual skip
 * hanging off them): pnp_bn_bwd_reduce_sums accumulates sum(g), sum(g*xhat) only; pnp_bn_bwd_apply_direct recomputes g from dy.
 * The activation sign may come from the bf16 hi plane of y (y_hi) instead of y; dz may be NULL when only the planes are wanted.
 * The two agree for every y an activation of this library writes (pnp_bn_act_apply, pnp_bn_apply_fused, the fused wgmma
 * epilogue): those flush positive subnormal activations to +0, since rn_bf16 sends 0 < y <= 2^-134 to +0.
 * 24-28 instead of 32 bytes per element. */
int pnp_bn_bwd_reduce_sums(const float* dy, const float* y, const uint16_t* y_hi, const float* z, const float* mean,
                           const float* invstd, int act, double* sum_g, double* sum_gx, long long M, int C, void* stream);
int pnp_bn_bwd_apply_direct(const float* dy, const float* y, const uint16_t* y_hi, int act, const float* z, const float* mean,
                            const float* invstd, const float* gamma, const double* sum_g, const double* sum_gx, long long M, int C,
                            int training, const pnp_dropout_cfg* drop, float* dgamma, float* dbeta, float* dz, uint16_t* dz_hi,
                            uint16_t* dz_lo, void* stream);
/* y = act(z*scale + shift + skip);  skip (optional) has Cs channels placed at channel offset skip_off.  ReLU and leaky ReLU
 * write positive subnormal results as +0 (here, in pnp_bn_apply_fused and in the wgmma fused epilogue).
 * y_hi / y_lo (optional): also emit the bf16 (hi, lo) operand planes of y for the next tensor-core convolution */
int pnp_bn_act_apply(const float* z, const float* scale, const float* shift, const float* skip, int Cs,
                     int skip_off, int act, float* y, uint16_t* y_hi, uint16_t* y_lo, long long M, int C, void* stream);
/* g = dy * act'(y);  sum_g[c] += g;  sum_gx[c] += g * xhat   (xhat = (z-mean)*invstd) */
int pnp_bn_bwd_reduce(const float* dy, const float* y, const float* z, const float* mean, const float* invstd,
                      int act, float* g, double* sum_g, double* sum_gx, long long M, int C, void* stream);
/* dgamma += sum_gx, dbeta += sum_g (if non-NULL); coef[0..C) = sum_g/M, coef[C..2C) = sum_gx/M */
int pnp_bn_bwd_finalize(const double* sum_g, const double* sum_gx, long long M, int C, float* dgamma,
                        float* dbeta, float* coef, void* stream);
/* training: dz = gamma*invstd*(g - c1 - xhat*c2) ; else dz = gamma*invstd*g ; then * dropout mult.
 * dz_hi / dz_lo (optional): bf16 operand planes of dz for the tensor-core dgrad / wgrad */
int pnp_bn_bwd_apply(const float* g, const float* z, const float* mean, const float* invstd, const float* gamma,
                     const float* coef, int training, const pnp_dropout_cfg* drop, float* dz, uint16_t* dz_hi, uint16_t* dz_lo,
                     long long M, int C, void* stream);
/* activation-only backward (no BN): g = dy * act'(y) */
int pnp_act_bwd(const float* dy, const float* y, int act, float* g, long long n, void* stream);
/* dskip[m, c] = g[m, skip_off + c], c < Cs   (gradient of the channel-pad skip) */
int pnp_channel_slice(const float* g, int C, int off, int Cs, float* out, long long M, int accumulate, void* stream);
/* standalone dropout (conv2d without BN: layers.py:74) : y = x * mult ; same call serves backward */
int pnp_dropout_apply(const float* x, float* y, long long n, const pnp_dropout_cfg* drop, void* stream);
int pnp_seed_advance(unsigned long long* seed_ptr, void* stream);

/* ---- pooling / padding / phase shift ------------------------------------------------------------- */
/* tf.nn.max_pool 2x2/2 (layers.py:102-103) */
int pnp_maxpool2_fwd(const float* x, float* y, int B, int H, int W, int C, void* stream);
int pnp_maxpool2_bwd(const float* x, const float* dy, float* dx, int B, int H, int W, int C, void* stream);
/* tf.nn.avg_pool 2x2/2 (layers.py:105-106); backward != 0: in = dy [B,H/2,W/2,C], out = dx [B,H,W,C] */
int pnp_avgpool2(const float* in, float* out, int B, int H, int W, int C, int backward, void* stream);
/* tf.nn.max_pool / tf.nn.avg_pool with ksize = strides = [1,n,n,1], padding 'SAME', any n >= 1 (layers.py:102-106): Ho = ceil(H/n),
 * the window grid is centred as TensorFlow centres it (pad_before = (Ho*n - H) / 2), padding never wins a max and is not counted by
 * the average.  avg != 0 selects the average.  y = [B,Ho,Wo,C].  Backward: dx = [B,H,W,C]; the max routes to the first maximal
 * element of a window in row-major order (x may be NULL for the average). */
int pnp_pool_fwd(const float* x, float* y, int B, int H, int W, int C, int n, int avg, void* stream);
int pnp_pool_bwd(const float* x, const float* dy, float* dx, int B, int H, int W, int C, int n, int avg, void* stream);
/* crop_and_concat (layers.py:108-115): out[B,H2,W2,C1+C2] = [ centre crop of x1[B,H1,W1,C1] to H2 x W2 (offsets (H1-H2)/2,
 * (W1-W2)/2) | x2[B,H2,W2,C2] ]; simple_concat2d (layers.py:117-127) is the H1 == H2, W1 == W2 case.  Backward: dx1 (zero outside
 * the crop) and dx2 from dout; either output may be NULL. */
int pnp_crop_concat_fwd(const float* x1, const float* x2, float* out, int B, int H1, int W1, int C1, int H2, int W2, int C2,
                        void* stream);
int pnp_crop_concat_bwd(const float* dout, float* dx1, float* dx2, int B, int H1, int W1, int C1, int H2, int W2, int C2,
                        void* stream);
/* tf.pad(..., 'SYMMETRIC') by p on each spatial side (layers.py:19-23,68-72) and its adjoint (MirrorPadGrad: each dx element
 * sums the up to 3 x 3 padded positions that mirror onto it).  Both directions require 0 <= p <= H, W (PNP_ERR_UNSUPPORTED
 * otherwise), as TensorFlow's SYMMETRIC mode does. */
int pnp_mirror_pad_fwd(const float* x, float* y, int B, int H, int W, int C, int p, void* stream);
int pnp_mirror_pad_bwd(const float* dy, float* dx, int B, int H, int W, int C, int p, void* stream);
/* PS / _phase_shift (ops.py:3-27): X[B,a,b,G*r*r] -> out[B,a*r,b*r, Ctot] channels [coff, coff+ntile*G),
 * the G output channels repeated ntile times (tf.tile, adversarial.py:326).  order_b1 != 0 selects the
 * batch_size==1 sub-pixel order of the reference. */
int pnp_phase_shift_fwd(const float* X, float* out, int B, int a, int b, int G, int r, int Ctot, int coff,
                        int ntile, int order_b1, void* stream);
int pnp_phase_shift_bwd(const float* dout, float* dX, int B, int a, int b, int G, int r, int Ctot, int coff,
                        int ntile, int order_b1, void* stream);
/* out[..., coff:coff+C] = logits ; out[..., coff+C] = float(argmax logits)  (adversarial.py:334-335) */
/* The whole discriminator input (adversarial.py:325-335) in one gather: out[B,H,W,Ctot] = [PS_r(src_0) tiled ntile_0 times | ... |
 * logits | float(argmax logits)], src_s = [B, a_s, b_s, G_s*r*r] with a_s*r == H; up to 4 sources, Ctot % 4 == 0, Ctot <= 64. */
int pnp_disc_input_fwd(const float* const* srcs, const int* a, const int* b, const int* G, const int* ntile, int nsrc,
                       const float* logits, int NC, float* out, int B, int H, int W, int r, int order_b1, void* stream);
int pnp_logits_argmax_concat(const float* logits, float* out, long long P, int C, int Ctot, int coff, void* stream);
/* out[m, 0:C] (+)= in[m, coff:coff+C]  -- strided channel slice used by the gather's backward */
/* (pnp_channel_slice above) */

/* ---- losses and metrics ---------------------------------------------------------------------------- */
/* layers.py:134-138 */
int pnp_pixel_softmax2(const float* logits, float* out, long long P, int C, void* stream);
/* tf.summary.image(name, tf.expand_dims(tf.cast(t, tf.float32), 3)) panels of one monitoring pass in one launch
 * (source_segmenter.py:398-405, adversarial.py:676-687; TF-1.4 ImageSummaryOp, float path, normalised per image).  Source s is
 * srcs[s] = fp32 NHWC [B, H, W, C[s]] and kinds[s] says which single-channel image it shows:
 *   PNP_IMG_CHANNEL          channel channel[s] (the x[:,:,:,1] input slice);
 *   PNP_IMG_ARGMAX           float(first-max index over the C[s] <= 8 channels) (tf.argmax of a one-hot label map);
 *   PNP_IMG_SOFTMAX2_ARGMAX  float(first-max index over pnp_pixel_softmax2 of the C[s] <= 8 logits) (compact_pred).
 * Images 0..n-1 (n = min(B, max_outputs) <= B) of up to 6 sources go to out[nsrc][n][H*W] (uint8). */
#define PNP_IMG_CHANNEL 0
#define PNP_IMG_ARGMAX 1
#define PNP_IMG_SOFTMAX2_ARGMAX 2
int pnp_image_summary_u8(const float* const* srcs, const int* kinds, const int* C, const int* channel, int nsrc,
                         int B, int H, int W, int n, unsigned char* out, void* stream);
/* source_segmenter.py:241-273: per-class partial sums acc[4*C] (doubles, zeroed by caller):
 * [0,C) sum y ; [C,2C) sum p*y ; [2C,3C) sum p*p ; [3C,4C) sum -y*log(clip(p,.005,1)) */
int pnp_segloss_reduce(const float* logits, const float* y, long long P, int C, double* acc, void* stream);
/* out[0]=weighted CE, out[1]=dice loss ; coef[3*C] = per-class backward coefficients */
int pnp_segloss_finalize(const double* acc, long long P, int C, float* out, float* coef, void* stream);
/* dlogits = g_wce * d wce/dlogits + g_dice * d dice/dlogits */
int pnp_segloss_bwd(const float* logits, const float* y, const float* coef, const float* g_wce, const float* g_dice,
                    float* dlogits, long long P, int C, void* stream);
/* Mean Shannon entropy of the per-pixel softmax of logits [P, C] (fp32, NHWC with P = B*H*W), TENT's test-time objective.
 * Per pixel, in fp32: m = max_c l_c; t_c = l_c - m; e_c = expf(t_c); s = sum_c e_c (ascending c); log p_c = t_c - logf(s);
 * p_c = e_c / s; H_p = -sum_c p_c * log p_c.  For finite logits every log p_c is finite: a saturated pixel gives H = 0, not NaN,
 * and nothing is clamped.  L = (1/P) sum_p H_p; dL/dl_j = -(1/P) * p_j * (log p_j + H_p).
 *   pnp_entropy_reduce:   acc[0] += sum_p H_p; acc[1 + c] += sum_p p_c (fp64 accumulation; acc[1 + C] zeroed by the caller).
 *   pnp_entropy_finalize: out[0] = (float)(acc[0] / P) = L; out[1 + c] = (float)(acc[1 + c] / P), the mean class probability
 *                         (a diagnostic: it is not differentiated).
 *   pnp_entropy_bwd:      dlogits = g[0] * dL/dlogits computed as (-g[0] / (float)P) * (p_j * (log p_j + H_p)); g is a device
 *                         scalar, so a captured graph reads it on every replay.
 * 2 <= C <= 8 and P >= 1; NULL pointers or other sizes are PNP_ERR_BAD_ARG, and nothing is launched. */
int pnp_entropy_reduce(const float* logits, long long P, int C, double* acc, void* stream);
int pnp_entropy_finalize(const double* acc, long long P, int C, float* out, void* stream);
int pnp_entropy_bwd(const float* logits, const float* g, float* dlogits, long long P, int C, void* stream);
/* lib.py:96-110 + tf.confusion_matrix: counts[C*C] (confusion, rows = truth), from logits argmax vs one-hot y */
int pnp_confusion(const float* logits, const float* y, long long P, int C, unsigned long long* counts, void* stream);
/* lib._label_decomp (lib.py:75-92): int64 label map -> one-hot fp32 [P, C], on the device */
int pnp_one_hot(const long long* labels, float* out, long long P, int C, void* stream);
/* tf.matmul [B,F]x[F,1] (adversarial.py:397,440) */
int pnp_fc_fwd(const float* x, const float* w, float* out, int B, int F, void* stream);
int pnp_fc_bwd(const float* x, const float* w, const float* dout, float* dx, float* dw, int B, int F, void* stream);
/* out[0] = ca*mean(a) + cb*mean(b) (b may be NULL)   (adversarial.py:455-459) */
int pnp_mean_combo(const float* a, float ca, const float* b, float cb, int n, float* out, void* stream);
/* cross_entropy (layers.py:140-141): out[0] = -mean(y * log(clip(p, 1e-10, 1))) over n elements; acc = one ZEROED fp64 device
 * scalar (receives the sum).  Backward from the scalar's gradient gout[0]: dy = -g/n * log(clip p), dp = -g/n * y / p where
 * 1e-10 <= p <= 1, else 0 (tf.clip_by_value's gradient); either output may be NULL. */
int pnp_cross_entropy_fwd(const float* y, const float* p, long long n, double* acc, float* out, void* stream);
int pnp_cross_entropy_bwd(const float* y, const float* p, const float* gout, long long n, float* dy, float* dp, void* stream);
/* out[0] += 0.5 * sum(w^2)   (tf.nn.l2_loss) */
int pnp_l2_loss_acc(const float* w, long long n, double* out, void* stream);

/* ---- optimizers on flat arenas ------------------------------------------------------------------------
 * chunk_seg[i] = segment id of arena elements [1024*i, 1024*i+1024); seg_wd / seg_clip are per segment.
 * grad_scale folds the data-parallel 1/N average; wd adds wd*theta to the gradient (tf.nn.l2_loss terms). */
/* tf.train.AdamOptimizer (source_segmenter.py:378) -- epsilon-hat form.  Hyper state lives in device memory so a
 * captured CUDA graph stays valid across steps: state = [beta1^t, beta2^t, lr, lr_t] (doubles).
 * pnp_adam_advance: t += 1, lr_t = lr*sqrt(1-beta2^t)/(1-beta1^t); pnp_adam_step applies the update with lr_t. */
int pnp_adam_advance(double* state, float beta1, float beta2, void* stream);
int pnp_adam_step(float* theta, const float* grad, float* m, float* v, long long n, const int* chunk_seg,
                  const float* seg_wd, const double* state, float beta1, float beta2, float eps, float grad_scale,
                  void* stream);
/* tf.train.RMSPropOptimizer (adversarial.py:643-652) + clip_by_value (adversarial.py:653-654) */
int pnp_rmsprop_step(float* theta, const float* grad, float* ms, float* mom, long long n, const int* chunk_seg,
                     const float* seg_wd, const float* seg_clip, const float* lr_ptr /* device scalar */, float decay,
                     float momentum, float eps, float grad_scale, void* stream);
/* tf.train.MomentumOptimizer (the source segmenter's other optimizer branch, source_segmenter.py:360-372): accum = momentum*accum +
 * (grad*grad_scale + wd*theta); theta -= lr*accum; lr is a device scalar (the staircase exponential decay is host logic) */
int pnp_momentum_step(float* theta, const float* grad, float* accum, long long n, const int* chunk_seg, const float* seg_wd,
                      const float* lr_ptr, float momentum, float grad_scale, void* stream);
int pnp_fill(float* p, float v, long long n, void* stream);

/* ---- exponential moving average of the trained weights (tf.train.ExponentialMovingAverage(decay, num_updates=n)) --------------
 * Every operation is fp32 and rounded on its own (no FMA contraction):
 *   pnp_ema_advance: nf = (float)n; d = fminf(decay, (1 + nf) / (10 + nf)); *c = 1 - d; n += 1.  One thread; n (int64) and c
 *                    live in device memory, so a captured graph advances the schedule on every replay.  0 < decay < 1.
 *   pnp_ema_update:  s = s - (s - x) * c for every covered float (assign_moving_average's assign_sub form), c read from device.
 *   pnp_ema_swap:    exchanges s and x.
 * The shadow is one flat buffer of arena_n + 1024 * table_n floats.  Its first arena_n floats (a multiple of 1024) mirror the
 * live optimizer arena float for float, padding included.  Each of the table_n chunks that follow belongs to one entry of
 * `table` (device memory): `len` (1..1024) live floats from `live`, the rest of the chunk is padding nobody touches.  A tensor
 * longer than 1024 floats takes ceil(len / 1024) consecutive entries.  One CTA per 1024-float chunk. */
typedef struct {
  float* live;
  long long len;
} pnp_ema_chunk;
int pnp_ema_advance(long long* num_updates, float decay, float* c, void* stream);
int pnp_ema_update(float* shadow, const float* arena, long long arena_n, const pnp_ema_chunk* table, int table_n, const float* c,
                   void* stream);
int pnp_ema_swap(float* shadow, float* arena, long long arena_n, const pnp_ema_chunk* table, int table_n, void* stream);

/* ---- batch-norm population statistics (PreciseBN / AdaBN re-estimation) ------------------------------------------------------
 * Over N batch-statistics forward passes, layer l's fp64 per-channel sums S1_b = sum z, S2_b = sum z^2 (what pnp_bn_stats or the
 * fused convolution epilogue writes) are added up, and the moving statistics are replaced by the pooled statistics of every
 * value seen.  Every operation is fp64 and rounded on its own (no FMA contraction):
 *   pnp_bn_accumulate: acc[c] += sum[c]; acc[C + c] += sumsq[c] for every entry and channel c < C (one launch per pass, so the
 *                      passes are added in the order they ran).
 *   pnp_bn_population: m = acc[c] / n; v = acc[C + c] / n - m * m; v = 0 if v < 0 (a NaN passes); moving_mean[c] = (float)m;
 *                      moving_var[c] = (float)(n > 1 ? v * (n / (n - 1)) : v), with n = count = sum of the passes' B * Ho * Wo.
 * `table` is HOST memory of n >= 1 entries; its contents travel in the launch's parameters (64 entries per launch), so the
 * caller may reuse it once the call returns, and a captured graph keeps the pointers it was captured with.  The buffers the
 * entries point to are device memory; acc is [2C] fp64.  Null table or pointers, n < 1, C < 1 or C > 1024, count < 1:
 * PNP_ERR_BAD_ARG, and nothing is launched. */
typedef struct {
  const double* sum;
  const double* sumsq;
  double* acc;
  int C;
} pnp_bn_acc_entry;
typedef struct {
  const double* acc;
  long long count;
  float* moving_mean;
  float* moving_var;
  int C;
} pnp_bn_pop_entry;
int pnp_bn_accumulate(const pnp_bn_acc_entry* table, int n, void* stream);
int pnp_bn_population(const pnp_bn_pop_entry* table, int n, void* stream);

/* ---- evaluation: 3-D surface distances ---------------------------------------------------------------------------------------
 * Per-class surface distances between a predicted label volume P and a ground truth G (medpy.metric.binary.assd / hd as the
 * papers' evaluation calls them).  pred and gt are uint8 [n0][n1][n2] (n2 fastest) on the device; labels >= C count as
 * background.  For each class c in 1 .. C-1, with A = (P == c) and B = (G == c):
 *   dA = A and not erode(A) (6-neighbour cross, one iteration; voxels outside the volume are not in A, so A's voxels on the
 *   faces of the volume are border voxels), likewise dB;
 *   d(v, S) = min over s in S of sqrt(((s0 (v0 - s0'))^2 + (s1 (v1 - s1'))^2) + (s2 (v2 - s2'))^2), spacing = (s0, s1, s2);
 *   out[(c-1)*6 + 0..5] = sum of d(v, dB) over v in dA, |dA|, max of d(v, dB) over dA,
 *                         sum of d(v, dA) over v in dB, |dB|, max of d(v, dA) over dB   (doubles, device).
 * If dA or dB is empty the four sums / maxima of that class are NaN (the counts are exact).  ASSD = (out[0]/out[1] +
 * out[3]/out[4]) / 2, HD = max(out[2], out[5]).  Each distance is exact (an exact Euclidean feature transform, then scipy's
 * expression above in fp64); with unit spacing it is bit-identical to scipy.ndimage.distance_transform_edt.  The sums run in a
 * fixed order, so repeated calls give bit-identical results.
 *
 * spacing: host pointer to 3 positive finite doubles, or NULL for unit spacing (voxel units).  1 <= n0, n1, n2 <=
 * PNP_SD_MAX_DIM and 2 <= C <= 8 (one border bit per class in a byte), else PNP_ERR_UNSUPPORTED; non-positive sizes, bad
 * spacing, NULL pointers or a workspace smaller than pnp_surface_distance_workspace's are PNP_ERR_BAD_ARG.  On any error nothing
 * is launched and out is untouched.
 *
 * Workspace (device, ws_bytes long): with N = n0*n1*n2, L = n1*n2 and A(x) = x rounded up to a multiple of 256,
 *   bytes = A(2N) + A(4N) + A(8N) + 2 A(16L) + A(8L)      (~14 bytes per voxel: 235 MB at 256^3, for any C). */
#define PNP_SD_MAX_DIM 1024
int pnp_surface_distance_workspace(int n0, int n1, int n2, int C, long long* bytes /* host */);
int pnp_surface_distance(const uint8_t* pred, const uint8_t* gt, int n0, int n1, int n2, int C, const double* spacing /* host, 3 */,
                         void* ws, long long ws_bytes, double* out, void* stream);

/* The same with a percentile of the pooled surface distances (medpy.metric.binary.hd95 at q = 95).  For each class, with dA, dB
 * and d(., .) as above, D is the multiset {d(v, dB) : v in dA} + {d(v, dA) : v in dB} of n = |dA| + |dB| values and
 *   out[(c-1)*7 + 0..5] = the six values pnp_surface_distance writes, bit-identical to it (the same kernels compute them);
 *   out[(c-1)*7 + 6]    = HD_q = numpy.percentile(D, q) with numpy's default `linear` method, operation for operation:
 *     qf = q / 100 and v = (n - 1) * qf, each rounded in fp64; lo = floor(v), hi = lo + 1, both n - 1 when v >= n - 1;
 *     gamma = v - lo, a = D(lo), b = D(hi) (order statistics, 0-based), delta = b - a;
 *     HD_q = b - delta * (1 - gamma) if gamma >= 0.5, else a + delta * gamma, each difference, product and sum rounded alone.
 * HD_q is NaN when dA or dB is empty.  q = 100 gives HD, q = 0 the smallest distance.  This is the pooled form (medpy's); the
 * larger of the two directed percentiles (MONAI) and the surfel-area-weighted form are other metrics.  The order statistics are
 * found on the device by a radix select over the distances' bit patterns with integer counts only, so HD_q is an exact function
 * of D and repeated calls are bit-identical; the call only enqueues work (no synchronisation, no copy to the host).
 *
 * q must be finite and in [0, 100], else PNP_ERR_BAD_ARG; every other check is pnp_surface_distance's, against this workspace:
 *   bytes = pnp_surface_distance_workspace's + A(16N) + A(8L) + A(8 ceil(2L / 256)) + A(16584)
 *   (~30 bytes per voxel: 506 MB at 256^3, for any C).  On any error nothing is launched and out is untouched. */
int pnp_surface_distance_pct_workspace(int n0, int n1, int n2, int C, long long* bytes /* host */);
int pnp_surface_distance_pct(const uint8_t* pred, const uint8_t* gt, int n0, int n1, int n2, int C, const double* spacing /* host, 3 */,
                             double q, void* ws, long long ws_bytes, double* out, void* stream);

/* ---- data preparation: planes resampled out of a volume (resample.cu) ----------------------------------------------------------
 * The augmented coronal slices of the data preparation (preprocess.py; the reference only describes it, README step 1) in one launch
 * per batch.  vol is fp32 and cls uint8 class ids, both C-order [n0][n1][n2] (n2 fastest) on the device.  Output plane p = b*C + k
 * has its own 3 x 3 matrix m = mats[9p .. 9p+8] (row-major, device); pixel (r, c) of plane p samples the source coordinate
 *   u_i = (m_i0 * r + m_i1 * c) + m_i2,   i = 0, 1, 2,
 * each product and each sum rounded separately in fp32 (no FMA contraction).
 *   img[b][r][c][k] (fp32 [B,H,W,C]): trilinear interpolation of vol.  Each u_i is clamped into [0, n_i - 1]; i0 = floor(u),
 *     i1 = min(i0 + 1, n_i - 1), f = u - i0; interpolation runs along axis 2, then 1, then 0, each step a + f*(b - a) with every
 *     operation rounded.  A NaN coordinate clamps to 0.
 *   lab (int64): the nearest voxel floor(u_i + 0.5) of cls (ties round up); class 0 when any u_i < -0.5, u_i >= n_i - 0.5 or
 *     u_i is NaN.  label_planes = 1 writes plane C/2 only, as lab[b][r][c] ([B,H,W], what the trainers consume); label_planes = C
 *     writes every plane, lab[b][r][c][k] ([B,H,W,C], what the record writer stores); 0 writes no labels.
 * A prepared test volume [H, W, D] is the call with B = 1 and C = D: NHWC with B = 1 is the NIfTI C-order layout.
 *
 * img may be NULL (labels only); vol may then be NULL too, and cls / lab may be NULL with label_planes = 0.  NULL mats, a NULL
 * pointer an output needs, no output at all or a non-positive size are PNP_ERR_BAD_ARG; label_planes other than 0, 1 or C, a
 * dimension n_i, H or W above PNP_RS_MAX_DIM (fp32 coordinates must resolve every voxel and n - 0.5 must be exact) or
 * n0*n1*n2, B*H*W*C or B*C*9 >= 2^31 are PNP_ERR_UNSUPPORTED.  On any error nothing is launched and the outputs are untouched.
 * Every output element is written once by one thread, so repeated calls are bit-identical. */
#define PNP_RS_MAX_DIM (1 << 23)
int pnp_resample_planes(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H, int W, int C,
                        float* img, long long* lab, int label_planes, void* stream);

/* ---- data augmentation: elastic deformation and intensity variation of the resampled planes (resample.cu) ---------------------
 * pnp_resample_planes_aug is pnp_resample_planes with three optional per-sample fields (device fp32, each may be NULL):
 *   disp [B][2][H][W]: pixel (r, c) of sample b samples the matrix at (r + d_r, c + d_c), d_r = disp[b][0][r][c],
 *     d_c = disp[b][1][r][c], each sum rounded (the image and the labels alike, every plane k of the sample);
 *   gain [B][H][W]: the image value v becomes (1 + gain[b][r][c]) * v;
 *   ab [B][2]: then a * v + b with (a, b) = (ab[2b], ab[2b + 1]);
 * out = (a * ((1 + gain) * v)) + b, every operation rounded on its own (no FMA); a NULL field skips its operations.  Every check of
 * pnp_resample_planes applies; in addition gain or ab without img is PNP_ERR_BAD_ARG and B*2*H*W >= 2^31 with disp is
 * PNP_ERR_UNSUPPORTED.  With all three NULL the output equals pnp_resample_planes' bit for bit.
 *
 * pnp_smooth_noise_field writes out [B][K][H][W] (device fp32) = min(max(amp * s, lo), hi), where s is a uniform field smoothed by a
 * separable Gaussian:
 *   x[e] = fl32(w >> 8) * 2^-23 - 1 in [-1, 1) (exact), e = ((b K + k) H + r) W + c, w = 32-bit word e & 3 of Philox4x32-10 block
 *     e >> 2 with counter (lo(e >> 2), hi(e >> 2), lo(stream_id), hi(stream_id)) and key (lo(seed), hi(seed));
 *   pass 1 (along c) y[r][c] = sum_{t=-R..R} taps[t + R] * x[r][c + t], pass 2 (along r) s[r][c] = sum_t taps[t + R] * y[r + t][c],
 *     0 outside the plane, accumulated from +0 in increasing t, every product and every sum rounded on its own (no FMA).
 * taps (device, 2R + 1 fp32) are typically the normalised Gaussian of scipy.ndimage.gaussian_filter1d (preprocess.gaussian_taps).
 * tmp (device, B*K*H*W fp32, not out) receives pass 1.  NULL taps / out / tmp, out == tmp, a non-positive size, R < 0, NaN amp or not
 * lo <= hi are PNP_ERR_BAD_ARG; R > PNP_NF_MAX_R or B*K*H*W >= 2^31 are PNP_ERR_UNSUPPORTED.  On any error nothing is launched and the
 * outputs are untouched.  Two launches; every output element is written once by one thread, so repeated calls are bit-identical. */
#define PNP_NF_MAX_R 128
int pnp_resample_planes_aug(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H, int W, int C,
                            float* img, long long* lab, int label_planes, const float* disp, const float* gain, const float* ab,
                            void* stream);
int pnp_smooth_noise_field(unsigned long long seed, unsigned long long stream_id, int B, int K, int H, int W, const float* taps, int R,
                           float amp, float lo, float hi, float* out, float* tmp, void* stream);

/* ---- native-grid labels: a prepared-grid prediction sampled back onto the scan's own voxels (resample.cu) ------------------------
 * scores: fp32 C-order [n0][n1][n2][C] class scores on the prepared grid (slice, row, column; C fastest), device.  map: 12 fp32
 * (device) taking native voxel (i, j, k) to the prepared coordinate
 *   u_a = ((m[4a] * i + m[4a+1] * j) + m[4a+2] * k) + m[4a+3],   a = 0, 1, 2,
 * each product and each sum rounded separately in fp32 (no FMA contraction).  For every native voxel of the C-order [m0][m1][m2]
 * grid (the order nifti.load(...).get_data() returns):
 *   out (uint8): 0 when any u_a is outside [-0.5, n_a - 0.5) or NaN; otherwise the argmax over c (the lowest index wins a tie) of
 *     the trilinear score of class c, with pnp_resample_planes' clamp, taps and lerp order (axis 2, then 1, then 0).
 *   cm (int64 [C][C], device, optional with gt): cm[gt][out] counted over every voxel, gt uint8 [m0][m1][m2] on the device;
 *     ground-truth labels >= C count as background.  The call zeroes cm first; integer counts make repeated calls bit-identical.
 * gt and cm are both NULL or both given.  NULL scores / map / out, only one of gt / cm, or a non-positive size are
 * PNP_ERR_BAD_ARG; C outside [2, 8], a dimension above PNP_RS_MAX_DIM, or n0*n1*n2*C or m0*m1*m2 >= 2^31 are
 * PNP_ERR_UNSUPPORTED.  On any error nothing is launched and the outputs are untouched. */
int pnp_native_labels(const float* scores, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2, uint8_t* out,
                      const uint8_t* gt, long long* cm, void* stream);

/* ---- native-grid labels of an ensemble: K predictions averaged at every native voxel before the argmax (resample.cu) ----------
 * Checkpoint ensembles and test-time augmentation.  scores: fp32 C-order [K][n0][n1][n2][C] on the device, one prepared-grid score
 * volume per member, all of one shape (member k starts at k * n0*n1*n2*C, a 64-bit offset).  maps: fp32 [K][12] on the device,
 * member k's map in pnp_native_labels' layout.  For every native voxel, in ascending k: u^k is computed as pnp_native_labels
 * computes it; member k covers the voxel when every u^k_a is inside [-0.5, n_a - 0.5) and not NaN; its class scores v^k_c are
 * pnp_native_labels' trilinear scores.  The first covering member's scores are taken as they are, each later covering member's
 * are added to them (fp32, each sum rounded, ascending k).
 *   out (uint8): the first maximum over c (the lowest index wins a tie) of the sums; 0 where no member covers the voxel.  The sum
 *     is not divided by the number of covering members: every class shares that number, and a division could create a tie.  At
 *     K = 1 out and cm are pnp_native_labels' bit for bit.
 *   cm: as pnp_native_labels counts it.
 * K <= 0 or NULL maps, and every argument pnp_native_labels rejects as PNP_ERR_BAD_ARG, are PNP_ERR_BAD_ARG; K above
 * PNP_NATIVE_MAX_MEMBERS (the maps are staged in shared memory once per CTA), and each member outside pnp_native_labels' limits,
 * are PNP_ERR_UNSUPPORTED.  On any error nothing is launched and the outputs are untouched.  Every label is written once by one
 * thread and the counts are integers, so repeated calls are bit-identical. */
#define PNP_NATIVE_MAX_MEMBERS 16
int pnp_native_labels_ensemble(const float* scores, int K, int n0, int n1, int n2, int C, const float* maps, int m0, int m1, int m2,
                               uint8_t* out, const uint8_t* gt, long long* cm, void* stream);

/* ---- native-grid labels of any number of predictions, one launch per prediction (resample.cu) ------------------------------
 * The streaming form of pnp_native_labels_ensemble, without its member cap and without K resident score volumes (the heart
 * localisation's sliding windows, native.py / localise.py).  sums: fp32 C-order [m0][m1][m2][C] and covered: uint8 [m0][m1][m2],
 * both on the device and zeroed by the caller once before the first prediction (offsets into sums are 64-bit: m0*m1*m2*C may reach
 * 2^31 and beyond).
 * pnp_native_accumulate samples one prediction (scores [n0][n1][n2][C], map: as pnp_native_labels takes them) at every native
 *   voxel with pnp_native_labels' coordinate, coverage, taps and lerps (one shared kernel body).  Where the prediction covers the
 *   voxel: if covered is 0 its class scores are stored as they are and covered is set to 1, otherwise they are added to sums (fp32,
 *   each sum rounded).  Voxels it does not cover are not touched.
 * pnp_native_accumulated_labels: out (uint8) is the first maximum over c of sums (the lowest index wins a tie) where covered is
 *   non-zero and 0 elsewhere; cm (optional with gt) as pnp_native_labels counts it (the call zeroes cm first).
 * K accumulate launches in ascending k followed by the labels call equal pnp_native_labels_ensemble on the same K members bit for
 * bit, labels and counts; K = 1 equals pnp_native_labels.
 * pnp_native_accumulate rejects what pnp_native_labels rejects (covered in the place of out, no gt / cm) and NULL sums as
 * PNP_ERR_BAD_ARG.  pnp_native_accumulated_labels: NULL sums / covered / out, only one of gt / cm or a non-positive size are
 * PNP_ERR_BAD_ARG; C outside [2, 8], a dimension above PNP_RS_MAX_DIM or m0*m1*m2 >= 2^31 are PNP_ERR_UNSUPPORTED.  On any error
 * nothing is launched and the outputs are untouched.  Each voxel is read and written by one thread per launch, so a sequence of
 * calls is bit-identical when repeated. */
int pnp_native_accumulate(const float* scores, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2, float* sums,
                          uint8_t* covered, void* stream);
int pnp_native_accumulated_labels(const float* sums, const uint8_t* covered, int m0, int m1, int m2, int C, uint8_t* out,
                                  const uint8_t* gt, long long* cm, void* stream);

/* ---- evaluation: largest connected component per class (components3d.cu) ------------------------------------------------------
 * The usual clean-up of a segmentation (nnU-Net's post-processing): every structure is one connected body, so only the largest
 * 3-D connected component of each class is kept and the rest is set to background.  labels, out and gt are uint8 C-order
 * [n0][n1][n2] (n2 fastest) on the device; labels >= C count as background.  connectivity is 6 (face neighbours) or 26 (face,
 * edge and corner neighbours): scipy.ndimage.generate_binary_structure(3, 1) and (3, 3).  For each class c in 1 .. C-1:
 *   the components of c are the connected components of {v : labels[v] == c}; voxels outside the volume belong to nothing;
 *   the kept component is the one with the most voxels; among equal sizes, the one whose smallest C-order linear index is
 *   smallest (what np.argmax(np.bincount(ndimage.label(mask, s)[0].ravel())[1:]) selects: scipy numbers components in raster
 *   order of their first voxel).  A class with no voxels keeps nothing.
 *   out[v] = c if v lies in the kept component of class c, else 0 (labels >= C become 0).  out may equal labels (in place).
 *   stats (int64 [C][3], device): stats[c] = (number of components, voxels kept, voxels removed); row 0 is (0, 0, number of labels
 *     >= C), the voxels set to 0 for being out of range.  The call zeroes stats first.
 *   cm (int64 [C][C], device, optional with gt): cm[gt][out] counted over every voxel, ground-truth labels >= C as background
 *     (as pnp_native_labels counts them).  The call zeroes cm first.
 * Union-find over an int32 parent array: each voxel is linked to its same-class neighbours of smaller linear index (3 for
 * 6-connectivity, 13 for 26), a root is only hooked under a smaller root (atomicCAS), so every root is the smallest linear index
 * of its component, and the per-class atomicMax of (size << 32) | (0xFFFFFFFF - root) picks the kept one.  The call only enqueues
 * a fixed sequence of launches (no synchronisation, no copy to the host); every quantity is an integer, so out, stats and cm are
 * exact functions of the input and repeated calls are bit-identical.
 *
 * NULL labels / out / stats / ws, only one of gt / cm, a non-positive size, or a workspace smaller than
 * pnp_largest_components_workspace's are PNP_ERR_BAD_ARG; C outside [2, 8], connectivity other than 6 or 26, or n0*n1*n2 >= 2^31
 * are PNP_ERR_UNSUPPORTED.  On any error nothing is launched and the outputs are untouched.
 *
 * Workspace (device, ws_bytes long): with N = n0*n1*n2 and A(x) = x rounded up to a multiple of 256,
 *   bytes = 2 A(4N) + 256      (parent and size, int32 per voxel, then the per-class keys: ~8 bytes per voxel, 629 MB at
 *                               512 x 512 x 300, for any C and either connectivity). */
int pnp_largest_components_workspace(int n0, int n1, int n2, int C, int connectivity, long long* bytes /* host */);
int pnp_largest_components(const uint8_t* labels, int n0, int n1, int n2, int C, int connectivity, uint8_t* out, const uint8_t* gt,
                           long long* cm, long long* stats, void* ws, long long ws_bytes, void* stream);

/* ---- per-class voxel count and bounding box (components3d.cu) -------------------------------------------------------------
 * labels: uint8 C-order [n0][n1][n2] on the device; labels >= C count as class 0.  out: int64 [C][7] on the device,
 *   out[c] = (count, lo0, hi0, lo1, hi1, lo2, hi2): the number of voxels of class c and the inclusive index bounds of them along
 *   each axis; an empty class gives (0, n0, -1, n1, -1, n2, -1).  The call initialises out itself.
 * Two launches: the empty boxes, then per-thread counts and bounds reduced per warp and folded in by integer atomics, so out is an
 * exact function of the input and repeated calls are bit-identical.
 * NULL labels / out or a non-positive size are PNP_ERR_BAD_ARG; C outside [2, 8] or n0*n1*n2 >= 2^31 are PNP_ERR_UNSUPPORTED.  On
 * any error nothing is launched and out is untouched. */
int pnp_label_boxes(const uint8_t* labels, int n0, int n1, int n2, int C, long long* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PNP_B200_H_ */
