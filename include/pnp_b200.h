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

#ifdef __cplusplus
}
#endif
#endif /* PNP_B200_H_ */
