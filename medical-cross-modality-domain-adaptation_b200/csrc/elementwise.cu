// HBM-bound kernels of the PnP-AdaNet hot path for sm_90a: batch-norm statistics / apply / backward,
// activation + residual skip, dropout, 2x2 max-pool, mirror pad, phase shift (pixel shuffle) and the
// discriminator-input gather, per-pixel softmax losses, FC + WGAN means, L2 sums, fused Adam / RMSProp+clip.
// All are coalesced 128-bit streaming kernels with warp-shuffle / shared-memory reductions and double
// precision global accumulators; grids are sized in multiples of the 132 SMs.
#include "common.cuh"
#include "../../include/pnp_b200.h"

#include <cuda_bf16.h>

namespace {

constexpr int kSMs = PNP_NUM_SMS;

// fp32 -> (hi, lo) bf16 pair with hi + lo ~ x to 2^-17 (operand planes of the wgmma convolution, conv_tc.cu)
__device__ __forceinline__ void split_pair(float x, unsigned short& hi, unsigned short& lo) {
  __nv_bfloat16 h = __float2bfloat16_rn(x);
  __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
  hi = __bfloat16_as_ushort(h);
  lo = __bfloat16_as_ushort(l);
}
__device__ __forceinline__ void store_planes(unsigned short* hi, unsigned short* lo, long long i4, float4 v) {
  ushort4 h, l;
  split_pair(v.x, h.x, l.x); split_pair(v.y, h.y, l.y); split_pair(v.z, h.z, l.z); split_pair(v.w, h.w, l.w);
  reinterpret_cast<ushort4*>(hi)[i4] = h;
  if (lo) reinterpret_cast<ushort4*>(lo)[i4] = l;
}
constexpr float kLeak = 0.2f;       // tf.nn.leaky_relu default alpha (layers.py:12)
constexpr float kBnDecay = 0.90f;   // layers.py:100
constexpr float kBnEps = 1e-3f;     // tf.contrib.layers.batch_norm default epsilon

__device__ __forceinline__ float act_fwd(float v, int act) {
  if (act == PNP_ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == PNP_ACT_LRELU) return v > 0.f ? v : kLeak * v;
  return v;
}
__device__ __forceinline__ float4 hi4_as_float4(ushort4 h) {
  return make_float4(__uint_as_float((unsigned)h.x << 16), __uint_as_float((unsigned)h.y << 16), __uint_as_float((unsigned)h.z << 16),
                     __uint_as_float((unsigned)h.w << 16));
}
__device__ __forceinline__ float act_slope(float y, int act) {
  if (act == PNP_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (act == PNP_ACT_LRELU) return y > 0.f ? 1.f : kLeak;
  return 1.f;
}

inline int grid_for(long long work_items, int per_block) {
  long long b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > PNP_NUM_SMS * 64LL) b = PNP_NUM_SMS * 64LL;
  return (int)b;
}

PnpDropout make_drop(const pnp_dropout_cfg* d) { return pnp_make_drop(d); }

// ------------------------------------------------------------------------------------------------
// BN statistics: per-channel sum and sum of squares of z[M, C] (C % 4 == 0, C <= 1024)
// ------------------------------------------------------------------------------------------------
template <bool WITH_G>
__global__ void __launch_bounds__(256)
bn_reduce_kernel(const float* __restrict__ z, const float* __restrict__ dy, const float* __restrict__ yact,
                 const unsigned short* __restrict__ yact_hi, const float* __restrict__ mean, const float* __restrict__ invstd, int act,
                 float* __restrict__ gout,
                 long long M, int C, int tpr, long long rows_per_block, double* __restrict__ out_a, double* __restrict__ out_b) {
  pnp_pdl_enter();
  // WITH_G == false: out_a += sum z, out_b += sum z^2
  // WITH_G == true : g = dy*act'(y) (written to gout); out_a += sum g ; out_b += sum g*xhat
  // thread (q, rlane) owns channel quad q and every rstep-th row; block partials are combined through shared memory
  // (no shared-memory fp64 atomics: those are CAS loops) and one fp64 global atomic per channel per block.
  __shared__ double s_part[256][8];
  const int C4 = C >> 2;
  const int q = threadIdx.x % tpr;
  const int rlane = threadIdx.x / tpr;
  const int rstep = 256 / tpr;
  long long r0 = (long long)blockIdx.x * rows_per_block;
  long long r1 = r0 + rows_per_block;
  if (r1 > M) r1 = M;
  double da[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) da[i] = 0.0;
  if (q < C4) {
    float4 mu = make_float4(0.f, 0.f, 0.f, 0.f), is = make_float4(1.f, 1.f, 1.f, 1.f);
    if (WITH_G) {
      mu = __ldg(reinterpret_cast<const float4*>(mean) + q);
      is = __ldg(reinterpret_cast<const float4*>(invstd) + q);
    }
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    int cnt = 0;
    // two rows per iteration: all loads of both rows are issued before either is consumed (memory-level parallelism)
    for (long long r = r0 + rlane; r < r1; r += 2 * rstep) {
      const long long offA = r * C4 + q;
      const bool hasB = (r + rstep) < r1;
      const long long offB = hasB ? (r + rstep) * C4 + q : offA;
      float4 zA = __ldg(reinterpret_cast<const float4*>(z) + offA);
      float4 zB = __ldg(reinterpret_cast<const float4*>(z) + offB);
      if (WITH_G) {
        float4 gA = __ldg(reinterpret_cast<const float4*>(dy) + offA);
        float4 gB = __ldg(reinterpret_cast<const float4*>(dy) + offB);
        if (act != PNP_ACT_NONE) {
          float4 yA, yB;
          if (yact_hi) {       // the sign of y from its bf16 hi plane (round-to-nearest keeps the sign; y == 0 <=> hi == 0)
            yA = hi4_as_float4(__ldg(reinterpret_cast<const ushort4*>(yact_hi) + offA));
            yB = hi4_as_float4(__ldg(reinterpret_cast<const ushort4*>(yact_hi) + offB));
          } else {
            yA = __ldg(reinterpret_cast<const float4*>(yact) + offA);
            yB = __ldg(reinterpret_cast<const float4*>(yact) + offB);
          }
          gA.x *= act_slope(yA.x, act); gA.y *= act_slope(yA.y, act); gA.z *= act_slope(yA.z, act); gA.w *= act_slope(yA.w, act);
          gB.x *= act_slope(yB.x, act); gB.y *= act_slope(yB.y, act); gB.z *= act_slope(yB.z, act); gB.w *= act_slope(yB.w, act);
        }
        if (gout) reinterpret_cast<float4*>(gout)[offA] = gA;
        a0 += gA.x; a1 += gA.y; a2 += gA.z; a3 += gA.w;
        b0 += gA.x * (zA.x - mu.x) * is.x; b1 += gA.y * (zA.y - mu.y) * is.y;
        b2 += gA.z * (zA.z - mu.z) * is.z; b3 += gA.w * (zA.w - mu.w) * is.w;
        if (hasB) {
          if (gout) reinterpret_cast<float4*>(gout)[offB] = gB;
          a0 += gB.x; a1 += gB.y; a2 += gB.z; a3 += gB.w;
          b0 += gB.x * (zB.x - mu.x) * is.x; b1 += gB.y * (zB.y - mu.y) * is.y;
          b2 += gB.z * (zB.z - mu.z) * is.z; b3 += gB.w * (zB.w - mu.w) * is.w;
        }
      } else {
        a0 += zA.x; a1 += zA.y; a2 += zA.z; a3 += zA.w;
        b0 += zA.x * zA.x; b1 += zA.y * zA.y; b2 += zA.z * zA.z; b3 += zA.w * zA.w;
        if (hasB) {
          a0 += zB.x; a1 += zB.y; a2 += zB.z; a3 += zB.w;
          b0 += zB.x * zB.x; b1 += zB.y * zB.y; b2 += zB.z * zB.z; b3 += zB.w * zB.w;
        }
      }
      if (++cnt == 32) {   // keep fp32 partial sums short (64 rows), promote to fp64
        da[0] += a0; da[1] += a1; da[2] += a2; da[3] += a3; da[4] += b0; da[5] += b1; da[6] += b2; da[7] += b3;
        a0 = a1 = a2 = a3 = b0 = b1 = b2 = b3 = 0.f;
        cnt = 0;
      }
    }
    da[0] += a0; da[1] += a1; da[2] += a2; da[3] += a3; da[4] += b0; da[5] += b1; da[6] += b2; da[7] += b3;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) s_part[threadIdx.x][i] = da[i];
  __syncthreads();
  // 2*C outputs, each the sum over the rstep row-lanes
  for (int o = threadIdx.x; o < 2 * C; o += 256) {
    const int which = o / C;            // 0: out_a, 1: out_b
    const int c = o - which * C;
    const int qq = c >> 2, j = (c & 3) + 4 * which;
    double t = 0.0;
    for (int r = 0; r < rstep; ++r) t += s_part[r * tpr + qq][j];
    atomicAdd((which ? out_b : out_a) + c, t);
  }
}

int reduce_launch_cfg(long long M, int C, int* tpr, long long* rpb, int* grid) {
  if (C % 4 != 0 || C > 1024 || C <= 0 || M <= 0) return PNP_ERR_UNSUPPORTED;
  int C4 = C / 4, t = 1;
  while (t < C4) t <<= 1;
  if (t > 256) return PNP_ERR_UNSUPPORTED;
  *tpr = t;
  int rstep = 256 / t;
  long long rows = (long long)rstep * 8;      // 8 rows per thread = 4 dependent DRAM round trips (was 32: ~17 us latency floor per launch)
  long long g = (M + rows - 1) / rows;
  long long cap = (long long)kSMs * 8;     // 8 resident CTAs of 256 threads per SM, one wave
  if (g > cap) { g = cap; rows = (M + g - 1) / g; }
  *rpb = rows;
  *grid = (int)((M + rows - 1) / rows);
  return PNP_OK;
}

__global__ void bn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, long long M, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float* moving_mean,
                                   float* moving_var, int training, float* scale, float* shift, float* mean, float* invstd) {
  pnp_pdl_enter();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mu, var;
  if (training) {
    double m = sum[c] / (double)M;
    double v = sumsq[c] / (double)M - m * m;
    if (v < 0.0) v = 0.0;
    mu = (float)m;
    var = (float)v;
    double unb = (M > 1) ? v * ((double)M / (double)(M - 1)) : v;
    moving_mean[c] = kBnDecay * moving_mean[c] + (1.f - kBnDecay) * mu;
    moving_var[c] = kBnDecay * moving_var[c] + (1.f - kBnDecay) * (float)unb;
  } else {
    mu = moving_mean[c];
    var = moving_var[c];
  }
  float is = rsqrtf(var + kBnEps);
  // one Newton step: rsqrtf is ~2 ulp, the oracle's rsqrt is correctly rounded
  is = is * (1.5f - 0.5f * (var + kBnEps) * is * is);
  float sc = gamma[c] * is;
  scale[c] = sc;
  shift[c] = beta[c] - mu * sc;
  mean[c] = mu;
  invstd[c] = is;
}

__global__ void __launch_bounds__(256)
bn_act_apply_kernel(const float* __restrict__ z, const float* __restrict__ scale, const float* __restrict__ shift,
                    const float* __restrict__ skip, int Cs, int skip_off, int act, float* __restrict__ y,
                    unsigned short* __restrict__ p_hi, unsigned short* __restrict__ p_lo, long long n4, int C4) {
  pnp_pdl_enter();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    int q = (int)(i % C4);
    float4 v = __ldg(reinterpret_cast<const float4*>(z) + i);
    if (scale) {
      float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + q);
      float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + q);
      v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y);
      v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
    }
    if (skip) {
      int c = q * 4 - skip_off;
      if (c >= 0 && c < Cs) {
        long long m = i / C4;
        float4 s = __ldg(reinterpret_cast<const float4*>(skip + m * Cs + c));
        v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w;
      }
    }
    v.x = act_fwd(v.x, act); v.y = act_fwd(v.y, act); v.z = act_fwd(v.z, act); v.w = act_fwd(v.w, act);
    reinterpret_cast<float4*>(y)[i] = v;
    if (p_hi) store_planes(p_hi, p_lo, i, v);
  }
}

// ------------------------------------------------------------------------------------------------
// batch norm with the per-channel "finalize" step folded into the streaming kernels: every CTA derives the channel
// coefficients it needs from the fp64 batch sums (or the moving statistics) into shared memory -- C <= 1024 values, a few
// hundred flops -- instead of a separate one-CTA kernel per layer (r1: 500 launches of ~5 us per two steps); CTA 0 alone
// performs the side effects (moving-average update, mean / invstd for the backward pass, dgamma / dbeta).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bn_apply_fused_kernel(const float* __restrict__ z, const double* __restrict__ sum, const double* __restrict__ sumsq, long long M,
                      int C, const float* __restrict__ gamma, const float* __restrict__ beta, float* moving_mean, float* moving_var,
                      int training, const float* __restrict__ skip, int Cs, int skip_off, int act, float* __restrict__ y,
                      unsigned short* __restrict__ p_hi, unsigned short* __restrict__ p_lo, float* mean_out, float* invstd_out,
                      long long n4) {
  pnp_pdl_enter();
  extern __shared__ float s_coef[];        // scale[C], shift[C]
  for (int c = threadIdx.x; c < C; c += 256) {
    float mu, var;
    double unb = 0.0;
    if (training) {
      double m = sum[c] / (double)M;
      double v = sumsq[c] / (double)M - m * m;
      if (v < 0.0) v = 0.0;
      mu = (float)m;
      var = (float)v;
      unb = (M > 1) ? v * ((double)M / (double)(M - 1)) : v;
    } else {
      mu = moving_mean[c];
      var = moving_var[c];
    }
    float is = rsqrtf(var + kBnEps);
    is = is * (1.5f - 0.5f * (var + kBnEps) * is * is);      // one Newton step: rsqrtf is ~2 ulp, the oracle's rsqrt is correctly rounded
    const float sc = gamma[c] * is;
    s_coef[c] = sc;
    s_coef[C + c] = beta[c] - mu * sc;
    if (blockIdx.x == 0) {
      if (training) {
        moving_mean[c] = kBnDecay * moving_mean[c] + (1.f - kBnDecay) * mu;
        moving_var[c] = kBnDecay * moving_var[c] + (1.f - kBnDecay) * (float)unb;
      }
      if (mean_out) { mean_out[c] = mu; invstd_out[c] = is; }
    }
  }
  __syncthreads();
  const int C4 = C >> 2;
  const float4* sc4 = reinterpret_cast<const float4*>(s_coef);
  const float4* sh4 = reinterpret_cast<const float4*>(s_coef + C);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const int q = (int)(i % C4);
    float4 v = __ldg(reinterpret_cast<const float4*>(z) + i);
    const float4 sc = sc4[q], sh = sh4[q];
    v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y);
    v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
    if (skip) {
      const int c = q * 4 - skip_off;
      if (c >= 0 && c < Cs) {
        const long long m = i / C4;
        const float4 s = __ldg(reinterpret_cast<const float4*>(skip + m * Cs + c));
        v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w;
      }
    }
    v.x = act_fwd(v.x, act); v.y = act_fwd(v.y, act); v.z = act_fwd(v.z, act); v.w = act_fwd(v.w, act);
    if (y) reinterpret_cast<float4*>(y)[i] = v;
    if (p_hi) store_planes(p_hi, p_lo, i, v);
  }
}

__global__ void __launch_bounds__(256)
bn_bwd_apply_fused_kernel(const float* __restrict__ g, const float* __restrict__ yact, const unsigned short* __restrict__ yact_hi,
                          int act, const float* __restrict__ z, const float* __restrict__ mean,
                          const float* __restrict__ invstd, const float* __restrict__ gamma, const double* __restrict__ sum_g,
                          const double* __restrict__ sum_gx, long long M, int C, int training, PnpDropout drop, float* dgamma,
                          float* dbeta, float* __restrict__ dz, unsigned short* __restrict__ p_hi, unsigned short* __restrict__ p_lo,
                          long long n4) {
  pnp_pdl_enter();
  extern __shared__ float s_coef[];        // k[C] = gamma*invstd, c1[C] = sum_g/M, d[C] = invstd * sum_gx/M, mu[C]
  for (int c = threadIdx.x; c < C; c += 256) {
    const float is = invstd[c];
    s_coef[c] = gamma[c] * is;
    float c1 = 0.f, c2 = 0.f, mu = 0.f;
    if (sum_g) {
      const double sg = sum_g[c], sgx = sum_gx[c];
      if (blockIdx.x == 0) {
        if (dgamma) dgamma[c] += (float)sgx;
        if (dbeta) dbeta[c] += (float)sg;
      }
      c1 = (float)(sg / (double)M);
      c2 = (float)(sgx / (double)M);
    }
    if (training) mu = mean[c];
    s_coef[C + c] = c1;
    s_coef[2 * C + c] = c2;
    s_coef[3 * C + c] = mu;
    s_coef[4 * C + c] = is;
  }
  __syncthreads();
  const int C4 = C >> 2;
  unsigned long long seed = 0ull;
  const bool drop_on = drop.seed_ptr != nullptr;
  if (drop_on) seed = *drop.seed_ptr;
  const float4* k4 = reinterpret_cast<const float4*>(s_coef);
  const float4* c14 = reinterpret_cast<const float4*>(s_coef + C);
  const float4* c24 = reinterpret_cast<const float4*>(s_coef + 2 * C);
  const float4* mu4 = reinterpret_cast<const float4*>(s_coef + 3 * C);
  const float4* is4 = reinterpret_cast<const float4*>(s_coef + 4 * C);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const int q = (int)(i % C4);
    float4 gv = __ldg(reinterpret_cast<const float4*>(g) + i);      // g, or dy when the activation derivative is applied here
    if (act != PNP_ACT_NONE) {
      const float4 yv = yact_hi ? hi4_as_float4(__ldg(reinterpret_cast<const ushort4*>(yact_hi) + i))
                                : __ldg(reinterpret_cast<const float4*>(yact) + i);
      gv.x *= act_slope(yv.x, act); gv.y *= act_slope(yv.y, act); gv.z *= act_slope(yv.z, act); gv.w *= act_slope(yv.w, act);
    }
    const float4 k = k4[q];
    float4 o;
    if (training) {
      const float4 zv = __ldg(reinterpret_cast<const float4*>(z) + i);
      const float4 mu = mu4[q], c1 = c14[q], c2 = c24[q], is = is4[q];
      o.x = k.x * (gv.x - c1.x - (zv.x - mu.x) * is.x * c2.x);
      o.y = k.y * (gv.y - c1.y - (zv.y - mu.y) * is.y * c2.y);
      o.z = k.z * (gv.z - c1.z - (zv.z - mu.z) * is.z * c2.z);
      o.w = k.w * (gv.w - c1.w - (zv.w - mu.w) * is.w * c2.w);
    } else {
      o.x = k.x * gv.x; o.y = k.y * gv.y; o.z = k.z * gv.z; o.w = k.w * gv.w;
    }
    if (drop_on) {
      const float4 mk = pnp_dropout_mult4(drop, seed, (unsigned long long)i);
      o.x *= mk.x; o.y *= mk.y; o.z *= mk.z; o.w *= mk.w;
    }
    if (dz) reinterpret_cast<float4*>(dz)[i] = o;
    if (p_hi) store_planes(p_hi, p_lo, i, o);
  }
}

__global__ void bn_bwd_finalize_kernel(const double* __restrict__ sum_g, const double* __restrict__ sum_gx, long long M,
                                       int C, float* dgamma, float* dbeta, float* coef) {
  pnp_pdl_enter();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double sg = sum_g[c], sgx = sum_gx[c];
  if (dgamma) dgamma[c] += (float)sgx;
  if (dbeta) dbeta[c] += (float)sg;
  coef[c] = (float)(sg / (double)M);
  coef[C + c] = (float)(sgx / (double)M);
}

__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ g, const float* __restrict__ z, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ coef,
                    int training, PnpDropout drop, float* __restrict__ dz, unsigned short* __restrict__ p_hi,
                    unsigned short* __restrict__ p_lo, long long n4, int C4) {
  pnp_pdl_enter();
  unsigned long long seed = 0ull;
  const bool drop_on = drop.seed_ptr != nullptr;
  if (drop_on) seed = *drop.seed_ptr;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    int q = (int)(i % C4);
    float4 gv = __ldg(reinterpret_cast<const float4*>(g) + i);
    float4 is = __ldg(reinterpret_cast<const float4*>(invstd) + q);
    float4 ga = __ldg(reinterpret_cast<const float4*>(gamma) + q);
    float4 o;
    if (training) {
      float4 zv = __ldg(reinterpret_cast<const float4*>(z) + i);
      float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + q);
      float4 c1 = __ldg(reinterpret_cast<const float4*>(coef) + q);
      float4 c2 = __ldg(reinterpret_cast<const float4*>(coef) + C4 + q);
      o.x = ga.x * is.x * (gv.x - c1.x - (zv.x - mu.x) * is.x * c2.x);
      o.y = ga.y * is.y * (gv.y - c1.y - (zv.y - mu.y) * is.y * c2.y);
      o.z = ga.z * is.z * (gv.z - c1.z - (zv.z - mu.z) * is.z * c2.z);
      o.w = ga.w * is.w * (gv.w - c1.w - (zv.w - mu.w) * is.w * c2.w);
    } else {
      o.x = ga.x * is.x * gv.x; o.y = ga.y * is.y * gv.y; o.z = ga.z * is.z * gv.z; o.w = ga.w * is.w * gv.w;
    }
    if (drop_on) {
      float4 mu = pnp_dropout_mult4(drop, seed, (unsigned long long)i);
      o.x *= mu.x; o.y *= mu.y; o.z *= mu.z; o.w *= mu.w;
    }
    reinterpret_cast<float4*>(dz)[i] = o;
    if (p_hi) store_planes(p_hi, p_lo, i, o);
  }
}

__global__ void __launch_bounds__(256)
act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, int act, float* __restrict__ g, long long n) {
  pnp_pdl_enter();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    g[i] = dy[i] * act_slope(y[i], act);
}

__global__ void __launch_bounds__(256)
channel_slice_kernel(const float* __restrict__ g, int C, int off, int Cs, float* __restrict__ out, long long total, int accumulate) {
  pnp_pdl_enter();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long m = i / Cs;
    int c = (int)(i - m * Cs);
    float v = g[m * C + off + c];
    out[i] = accumulate ? out[i] + v : v;
  }
}

__global__ void __launch_bounds__(256)
dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, PnpDropout drop) {
  pnp_pdl_enter();
  unsigned long long seed = *drop.seed_ptr;
  long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    float4 mu = pnp_dropout_mult4(drop, seed, (unsigned long long)i);
    v.x *= mu.x; v.y *= mu.y; v.z *= mu.z; v.w *= mu.w;
    reinterpret_cast<float4*>(y)[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    long long i = (n4 << 2) + threadIdx.x;
    y[i] = x[i] * pnp_dropout_mult1(drop, seed, (unsigned long long)i);
  }
}

__global__ void seed_advance_kernel(unsigned long long* s) {
  pnp_pdl_enter(); *s = *s * 6364136223846793005ull + 1442695040888963407ull; }

// ------------------------------------------------------------------------------------------------
// pooling / padding / phase shift
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void __launch_bounds__(256)
maxpool2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  pnp_pdl_enter();
  const int Ho = H / 2, Wo = W / 2, CV = C / V;
  long long total = (long long)B * Ho * Wo * CV;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int cv = (int)(i % CV);
    long long p = i / CV;
    int ox = (int)(p % Wo);
    long long t = p / Wo;
    int oy = (int)(t % Ho);
    int b = (int)(t / Ho);
    const float* base = x + (((long long)b * H + 2 * oy) * W + 2 * ox) * C + cv * V;
    float m[V];
#pragma unroll
    for (int e = 0; e < V; ++e) m[e] = base[e];
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const float* s = base + ((long long)(k >> 1) * W + (k & 1)) * C;
#pragma unroll
      for (int e = 0; e < V; ++e) m[e] = fmaxf(m[e], s[e]);
    }
#pragma unroll
    for (int e = 0; e < V; ++e) y[p * C + cv * V + e] = m[e];
  }
}

template <int V>
__global__ void __launch_bounds__(256)
maxpool2_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int B, int H, int W, int C) {
  pnp_pdl_enter();
  const int Ho = H / 2, Wo = W / 2, CV = C / V;
  long long total = (long long)B * Ho * Wo * CV;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int cv = (int)(i % CV);
    long long p = i / CV;
    int ox = (int)(p % Wo);
    long long t = p / Wo;
    int oy = (int)(t % Ho);
    int b = (int)(t / Ho);
    long long base = (((long long)b * H + 2 * oy) * W + 2 * ox) * C + cv * V;
#pragma unroll
    for (int e = 0; e < V; ++e) {
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = x[base + ((long long)(k >> 1) * W + (k & 1)) * C + e];
      int arg = 0;
      float best = v[0];
#pragma unroll
      for (int k = 1; k < 4; ++k)
        if (v[k] > best) { best = v[k]; arg = k; }   // first max in row-major window order
      float g = dy[p * C + cv * V + e];
#pragma unroll
      for (int k = 0; k < 4; ++k) dx[base + ((long long)(k >> 1) * W + (k & 1)) * C + e] = (k == arg) ? g : 0.f;
    }
  }
}

// tf.nn.avg_pool 2x2/2 (layers.py:105-106); with_grad: dx = dy/4 broadcast to the window
__global__ void __launch_bounds__(256)
avgpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C, int backward) {
  pnp_pdl_enter();
  const int Ho = H / 2, Wo = W / 2;
  long long total = (long long)B * Ho * Wo * C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int c = (int)(i % C);
    long long p = i / C;
    int ox = (int)(p % Wo);
    long long t = p / Wo;
    int oy = (int)(t % Ho);
    int b = (int)(t / Ho);
    long long base = (((long long)b * H + 2 * oy) * W + 2 * ox) * C + c;
    if (backward) {
      float g = 0.25f * in[i];
      out[base] = g; out[base + C] = g; out[base + (long long)W * C] = g; out[base + (long long)W * C + C] = g;
    } else {
      out[i] = 0.25f * (in[base] + in[base + C] + in[base + (long long)W * C] + in[base + (long long)W * C + C]);
    }
  }
}

__device__ __forceinline__ int mirror_idx(int i, int n) { return i < 0 ? (-i - 1) : (i >= n ? 2 * n - 1 - i : i); }

__global__ void __launch_bounds__(256)
mirror_pad_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C, int p) {
  pnp_pdl_enter();
  const int Hp = H + 2 * p, Wp = W + 2 * p;
  long long total = (long long)B * Hp * Wp * C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int c = (int)(i % C);
    long long t = i / C;
    int px = (int)(t % Wp);
    t /= Wp;
    int py = (int)(t % Hp);
    int b = (int)(t / Hp);
    int sy = mirror_idx(py - p, H), sx = mirror_idx(px - p, W);
    y[i] = x[(((long long)b * H + sy) * W + sx) * C + c];
  }
}

__global__ void __launch_bounds__(256)
mirror_pad_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H, int W, int C, int p) {
  pnp_pdl_enter();
  const int Hp = H + 2 * p, Wp = W + 2 * p;
  long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int c = (int)(i % C);
    long long t = i / C;
    int ix = (int)(t % W);
    t /= W;
    int iy = (int)(t % H);
    int b = (int)(t / H);
    int ys[3], xs[3], ny = 0, nx = 0;
    ys[ny++] = iy + p;
    if (iy < p) ys[ny++] = p - 1 - iy;
    if (iy >= H - p) ys[ny++] = 2 * H - 1 - iy + p;
    xs[nx++] = ix + p;
    if (ix < p) xs[nx++] = p - 1 - ix;
    if (ix >= W - p) xs[nx++] = 2 * W - 1 - ix + p;
    float acc = 0.f;
    for (int a = 0; a < ny; ++a)
      for (int e = 0; e < nx; ++e) acc += dy[(((long long)b * Hp + ys[a]) * Wp + xs[e]) * C + c];
    dx[i] = acc;
  }
}

__global__ void __launch_bounds__(256)
phase_shift_fwd_kernel(const float* __restrict__ X, float* __restrict__ out, int B, int a, int b, int G, int r, int Ctot,
                       int coff, int ntile, int order_b1) {
  pnp_pdl_enter();
  const int OH = a * r, OW = b * r;
  long long total = (long long)B * OH * OW * G;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int g = (int)(i % G);
    long long t = i / G;
    int x = (int)(t % OW);
    t /= OW;
    int y = (int)(t % OH);
    int n = (int)(t / OH);
    int iy = y / r, ry = y - iy * r, ix = x / r, rx = x - ix * r;
    int sub = order_b1 ? (ry * r + rx) : (rx * r + ry);
    float v = X[(((long long)n * a + iy) * b + ix) * ((long long)G * r * r) + (long long)g * r * r + sub];
    float* dst = out + (((long long)n * OH + y) * OW + x) * Ctot + coff + g;
    for (int tl = 0; tl < ntile; ++tl) dst[tl * G] = v;
  }
}

__global__ void __launch_bounds__(256)
phase_shift_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dX, int B, int a, int b, int G, int r, int Ctot,
                       int coff, int ntile, int order_b1) {
  pnp_pdl_enter();
  const int OH = a * r, OW = b * r, rr = r * r;
  const long long Cx = (long long)G * rr;
  long long total = (long long)B * a * b * Cx;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    int ch = (int)(i % Cx);
    long long t = i / Cx;
    int ix = (int)(t % b);
    t /= b;
    int iy = (int)(t % a);
    int n = (int)(t / a);
    int g = ch / rr, sub = ch - g * rr;
    int ry, rx;
    if (order_b1) { ry = sub / r; rx = sub - ry * r; }
    else { rx = sub / r; ry = sub - rx * r; }
    const float* src = dout + (((long long)n * OH + iy * r + ry) * OW + ix * r + rx) * Ctot + coff + g;
    float acc = 0.f;
    for (int tl = 0; tl < ntile; ++tl) acc += src[tl * G];
    dX[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// The discriminator input (adversarial.py:325-335) in ONE gather: [PS(c4) x3 | PS(c6) | PS(b7) | PS(c9) | logits | argmax]
// -> [B, H, W, Ctot].  One thread per (pixel, 4 output channels): the 128-byte pixel rows are written once, fully coalesced
// (r1: five partial-row scatter launches + one concat per call).
// ------------------------------------------------------------------------------------------------
struct DiscPlan {
  const float* src[4];
  int a[4], b[4], G[4];
  signed char ch_src[64];     // per output channel: source id 0..3, -1 = logits, -2 = argmax(logits)
  signed char ch_g[64];       // group (or logits channel)
};

__global__ void __launch_bounds__(256)
disc_input_kernel(DiscPlan plan, const float* __restrict__ logits, int NC, float* __restrict__ out, int B, int H, int W, int Ctot,
                  int r, int order_b1) {
  pnp_pdl_enter();
  const int Q = Ctot >> 2;
  const unsigned total = (unsigned)B * H * W * Q;          // < 2^31 (checked by the launcher): 32-bit index arithmetic throughout
  const int rr = r * r;
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total; i += gridDim.x * 256u) {
    const int q = (int)(i % (unsigned)Q);
    const unsigned pix = i / (unsigned)Q;
    const int x = (int)(pix % (unsigned)W);
    const unsigned t = pix / (unsigned)W;
    const int y = (int)(t % (unsigned)H);
    const int n = (int)(t / (unsigned)H);
    const int iy = y / r, ry = y - iy * r, ix = x / r, rx = x - ix * r;
    const int sub = order_b1 ? (ry * r + rx) : (rx * r + ry);
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ch = q * 4 + e;
      const int sid = plan.ch_src[ch], g = plan.ch_g[ch];
      if (sid >= 0) {
        v[e] = __ldg(plan.src[sid] + (size_t)((n * plan.a[sid] + iy) * plan.b[sid] + ix) * (size_t)(plan.G[sid] * rr) + g * rr + sub);
      } else if (sid == -1) {
        v[e] = __ldg(logits + (size_t)pix * NC + g);
      } else {
        const float* l = logits + (size_t)pix * NC;
        float best = __ldg(l);
        int arg = 0;
        for (int c = 1; c < NC; ++c) {
          const float lv = __ldg(l + c);
          if (lv > best) { best = lv; arg = c; }     // tf.argmax: lowest index on ties
        }
        v[e] = (float)arg;
      }
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// r = 8, batch >= 2 sub-pixel order: every (source pixel, group) is one contiguous 256-byte line = the 8x8 output block of one channel.
// A CTA takes 4 horizontally adjacent source pixels (8 rows x 32 output pixels): phase 1 reads their lines fully coalesced into
// shared memory, phase 2 writes the 128-byte output pixel rows fully coalesced (r2: the per-element gather above ran at the L1
// sector rate, 127 us per call for 67 MB).
struct DiscLines {
  signed char line_of[64];    // per output channel: index of its (source, group) line in the shared tile, -1 logits, -2 argmax
  signed char line_src[32];   // per line: source id
  signed char line_g[32];     // per line: group
  int nlines;
};

__global__ void __launch_bounds__(256)
disc_input_r8_kernel(DiscPlan plan, DiscLines ln, const float* __restrict__ logits, int NC, float* __restrict__ out, int B, int a, int b,
                     int Ctot) {
  pnp_pdl_enter();
  extern __shared__ float s_tile[];      // [4 source pixels][nlines][65]
  const int nl = ln.nlines;
  const int bx4 = (b + 3) >> 2;
  int t = blockIdx.x;
  const int jx = t % bx4; t /= bx4;
  const int iy = t % a;
  const int n = t / a;
  const int ix0 = jx * 4;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int it = wid; it < 4 * nl; it += 8) {
    const int j = it / nl, l = it - j * nl;
    const int ix = ix0 + j;
    float2 v = make_float2(0.f, 0.f);
    if (ix < b) {
      const int sid = ln.line_src[l];
      v = __ldg(reinterpret_cast<const float2*>(plan.src[sid] + ((size_t)(n * plan.a[sid] + iy) * plan.b[sid] + ix) * (size_t)(plan.G[sid] * 64) +
                                                ln.line_g[l] * 64 + lane * 2));
    }
    float* dst = s_tile + (size_t)(j * nl + l) * 65 + lane * 2;
    dst[0] = v.x; dst[1] = v.y;
  }
  __syncthreads();
  const int Q = Ctot >> 2;
  const int H = a * 8, W = b * 8;
  for (int idx = threadIdx.x; idx < 256 * Q; idx += 256) {
    const int q = idx % Q, p = idx / Q;               // p: pixel inside the 8 x 32 block
    const int row = p >> 5, col = p & 31;
    const int j = col >> 3, rx = col & 7;
    const int ox = ix0 * 8 + col, oy = iy * 8 + row;
    if (ox >= W) continue;
    const size_t pix = ((size_t)n * H + oy) * W + ox;
    const int sub = rx * 8 + row;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ch = q * 4 + e;
      const int l = ln.line_of[ch];
      if (l >= 0) {
        v[e] = s_tile[(size_t)(j * nl + l) * 65 + sub];
      } else if (l == -1) {
        v[e] = __ldg(logits + pix * NC + plan.ch_g[ch]);
      } else {
        const float* lg = logits + pix * NC;
        float best = __ldg(lg);
        int arg = 0;
        for (int c = 1; c < NC; ++c) {
          const float lv = __ldg(lg + c);
          if (lv > best) { best = lv; arg = c; }
        }
        v[e] = (float)arg;
      }
    }
    reinterpret_cast<float4*>(out)[pix * Q + q] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

__global__ void __launch_bounds__(256)
logits_argmax_concat_kernel(const float* __restrict__ logits, float* __restrict__ out, long long P, int C, int Ctot, int coff) {
  pnp_pdl_enter();
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256) {
    const float* l = logits + p * C;
    float* o = out + p * Ctot + coff;
    float best = l[0];
    int arg = 0;
    o[0] = best;
    for (int c = 1; c < C; ++c) {
      float v = l[c];
      o[c] = v;
      if (v > best) { best = v; arg = c; }   // tf.argmax: lowest index on ties
    }
    o[C] = (float)arg;
  }
}

// ------------------------------------------------------------------------------------------------
// losses / metrics (C <= 8 classes)
// ------------------------------------------------------------------------------------------------
constexpr int kMaxC = 8;

// pixel_wise_softmax_2 (layers.py:134-138) of one pixel's C <= kMaxC logits l[] into o[]; shared by pixel_softmax2_kernel and the
// image summaries' compact prediction, so both see the same values bit for bit
__device__ __forceinline__ void pixel_softmax2_px(const float* __restrict__ l, float* __restrict__ o, int C) {
  float e[kMaxC], s = 0.f;
  for (int c = 0; c < C; ++c) { e[c] = expf(l[c]); s += e[c]; }   // no max subtraction (layers.py:135)
  for (int c = 0; c < C; ++c) o[c] = fminf(fmaxf(e[c] / s, -1e15f), 1e15f);
}

__global__ void __launch_bounds__(256)
pixel_softmax2_kernel(const float* __restrict__ logits, float* __restrict__ out, long long P, int C) {
  pnp_pdl_enter();
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256)
    pixel_softmax2_px(logits + p * C, out + p * C, C);
}

// ---- tf.summary.image panels (TF-1.4 ImageSummaryOp, float path) --------------------------------------------------------------
constexpr int kImgMaxSrc = 6;
constexpr int kImgThreads = 512;

struct ImgPlan {
  const float* src[kImgMaxSrc];
  int kind[kImgMaxSrc];     // PNP_IMG_CHANNEL / PNP_IMG_ARGMAX / PNP_IMG_SOFTMAX2_ARGMAX
  int C[kImgMaxSrc];
  int ch[kImgMaxSrc];
};

// the single-channel value pixel p of a panel shows: channel `ch`, or the first-max class index (tf.argmax) of the C channels or
// of their pixel_wise_softmax_2 values
__device__ __forceinline__ float img_value(const float* __restrict__ x, long long p, int kind, int C, int ch) {
  const float* px = x + p * C;
  if (kind == PNP_IMG_CHANNEL) return px[ch];
  float v[kMaxC];
  if (kind == PNP_IMG_SOFTMAX2_ARGMAX) pixel_softmax2_px(px, v, C);
  else
    for (int c = 0; c < C; ++c) v[c] = px[c];
  int arg = 0;
  float best = v[0];
  for (int c = 1; c < C; ++c)
    if (v[c] > best) { best = v[c]; arg = c; }
  return (float)arg;
}

// One CTA per (source, image) panel.  NormalizeFloatImage of summary_image_op.cc: min / max over the finite pixels (a block-wide
// fmin / fmax, order-independent, so exact), then scale = 127 / max|.| with offset 128 if the min is negative, else 255 / max with
// offset 0 (scale 0 below 1e-6), pixel = uint8(trunc(v * scale + offset)), a non-finite pixel = bad_color[0] = 255.  The product and
// the sum are rounded separately (nvcc would contract them into an FMA); whether TensorFlow's own CPU build contracted them
// depends on its compiler flags and cannot be recovered, so the uncontracted form as written in the source is what is computed.
__global__ void __launch_bounds__(kImgThreads)
image_summary_u8_kernel(ImgPlan plan, int n, long long HW, unsigned char* __restrict__ out) {
  pnp_pdl_enter();
  __shared__ float s_mn[kImgThreads / 32], s_mx[kImgThreads / 32];
  __shared__ float s_scale, s_offset;
  const int s = blockIdx.x / n, i = blockIdx.x % n;
  const int kind = plan.kind[s], C = plan.C[s], ch = plan.ch[s];
  const float* x = plan.src[s] + (long long)i * HW * C;
  float mn = INFINITY, mx = -INFINITY;
  for (long long p = threadIdx.x; p < HW; p += kImgThreads) {
    const float v = img_value(x, p, kind, C, ch);
    if (isfinite(v)) { mn = fminf(mn, v); mx = fmaxf(mx, v); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kImgThreads / 32; ++w) { mn = fminf(mn, s_mn[w]); mx = fmaxf(mx, s_mx[w]); }
    const float kZeroThreshold = 1e-6f;
    float scale, offset;
    if (mn < 0.f) {
      const float max_val = fmaxf(fabsf(mn), fabsf(mx));
      scale = max_val < kZeroThreshold ? 0.f : __fdiv_rn(127.f, max_val);
      offset = 128.f;
    } else {
      scale = mx < kZeroThreshold ? 0.f : __fdiv_rn(255.f, mx);
      offset = 0.f;
    }
    s_scale = scale;
    s_offset = offset;
  }
  __syncthreads();
  const float scale = s_scale, offset = s_offset;
  unsigned char* o = out + (long long)blockIdx.x * HW;
  for (long long p = threadIdx.x; p < HW; p += kImgThreads) {
    const float v = img_value(x, p, kind, C, ch);
    o[p] = isfinite(v) ? (unsigned char)__float2uint_rz(__fadd_rn(__fmul_rn(v, scale), offset)) : (unsigned char)255;
  }
}

__device__ __forceinline__ void stable_softmax(const float* l, int C, float* p) {
  float mx = l[0];
  for (int c = 1; c < C; ++c) mx = fmaxf(mx, l[c]);
  float s = 0.f;
  for (int c = 0; c < C; ++c) { p[c] = expf(l[c] - mx); s += p[c]; }
  float inv = 1.f / s;
  for (int c = 0; c < C; ++c) p[c] *= inv;
}

__global__ void __launch_bounds__(256)
segloss_reduce_kernel(const float* __restrict__ logits, const float* __restrict__ y, long long P, int C, double* __restrict__ acc) {
  pnp_pdl_enter();
  __shared__ double s_acc[4 * kMaxC];
  if (threadIdx.x < 4 * kMaxC) s_acc[threadIdx.x] = 0.0;
  __syncthreads();
  float a[4 * kMaxC];
#pragma unroll
  for (int i = 0; i < 4 * kMaxC; ++i) a[i] = 0.f;
  int iter = 0;
  double d[4 * kMaxC];
#pragma unroll
  for (int i = 0; i < 4 * kMaxC; ++i) d[i] = 0.0;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256) {
    float l[kMaxC], pr[kMaxC];
    for (int c = 0; c < C; ++c) l[c] = logits[p * C + c];
    stable_softmax(l, C, pr);
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) {
      if (c < C) {
        float yy = y[p * C + c];
        a[c] += yy;
        a[kMaxC + c] += pr[c] * yy;
        a[2 * kMaxC + c] += pr[c] * pr[c];
        a[3 * kMaxC + c] += -yy * logf(fminf(fmaxf(pr[c], 0.005f), 1.0f));
      }
    }
    if (++iter == 32) {   // promote to double before fp32 partials grow long
#pragma unroll
      for (int i = 0; i < 4 * kMaxC; ++i) { d[i] += (double)a[i]; a[i] = 0.f; }
      iter = 0;
    }
  }
#pragma unroll
  for (int i = 0; i < 4 * kMaxC; ++i) {
    double v = pnp_warp_sum_d(d[i] + (double)a[i]);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_acc[i], v);
  }
  __syncthreads();
  if (threadIdx.x < 4 * kMaxC) {
    int q = threadIdx.x / kMaxC, c = threadIdx.x % kMaxC;
    if (c < C) atomicAdd(acc + q * C + c, s_acc[threadIdx.x]);
  }
}

__global__ void segloss_finalize_kernel(const double* __restrict__ acc, long long P, int C, float* out, float* coef) {
  pnp_pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double tot = 0.0;
  for (int c = 0; c < C; ++c) tot += acc[c];
  double wce = 0.0, dice = 0.0;
  for (int c = 0; c < C; ++c) {
    double sy = acc[c], inse = acc[C + c], l = acc[2 * C + c], ce = acc[3 * C + c];
    double w = 1.0 - sy / tot;
    wce += w * ce;
    double D = l + sy + 1e-7;
    dice += 2.0 * inse / D;
    coef[c] = (float)(w / (double)P);
    coef[C + c] = (float)(-(2.0 / C) / D);
    coef[2 * C + c] = (float)((4.0 / C) * inse / (D * D));
  }
  out[0] = (float)(wce / (double)P);
  out[1] = (float)(-dice / C);
}

__global__ void __launch_bounds__(256)
segloss_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ y, const float* __restrict__ coef,
                   const float* __restrict__ g_wce, const float* __restrict__ g_dice, float* __restrict__ dlogits,
                   long long P, int C) {
  pnp_pdl_enter();
  const float gw = g_wce ? *g_wce : 0.f;
  const float gd = g_dice ? *g_dice : 0.f;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256) {
    float l[kMaxC], pr[kMaxC], dp[kMaxC];
    for (int c = 0; c < C; ++c) l[c] = logits[p * C + c];
    stable_softmax(l, C, pr);
    float dot = 0.f;
    for (int c = 0; c < C; ++c) {
      float yy = y[p * C + c];
      float d = gd * (coef[C + c] * yy + coef[2 * C + c] * pr[c]);
      if (pr[c] >= 0.005f) d += gw * (-coef[c] * yy / pr[c]);
      dp[c] = d;
      dot += d * pr[c];
    }
    for (int c = 0; c < C; ++c) dlogits[p * C + c] = pr[c] * (dp[c] - dot);
  }
}

__global__ void __launch_bounds__(256)
confusion_kernel(const float* __restrict__ logits, const float* __restrict__ y, long long P, int C, unsigned long long* counts) {
  pnp_pdl_enter();
  __shared__ unsigned int s_cnt[kMaxC * kMaxC];
  if (threadIdx.x < kMaxC * kMaxC) s_cnt[threadIdx.x] = 0u;
  __syncthreads();
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256) {
    int pa = 0, ya = 0;
    float pb = logits[p * C], yb = y[p * C];
    for (int c = 1; c < C; ++c) {
      float v = logits[p * C + c], w = y[p * C + c];
      if (v > pb) { pb = v; pa = c; }
      if (w > yb) { yb = w; ya = c; }
    }
    atomicAdd(&s_cnt[ya * C + pa], 1u);
  }
  __syncthreads();
  if (threadIdx.x < C * C && s_cnt[threadIdx.x]) atomicAdd(counts + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

__global__ void __launch_bounds__(256)
one_hot_kernel(const long long* __restrict__ labels, float* __restrict__ out, long long P, int C) {
  pnp_pdl_enter();
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < P; p += (long long)gridDim.x * 256) {
    long long l = labels[p];
    for (int c = 0; c < C; ++c) out[p * C + c] = (l == c) ? 1.f : 0.f;
  }
}

__global__ void __launch_bounds__(256)
fc_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out, int F) {
  pnp_pdl_enter();
  __shared__ float s[8];
  const float* row = x + (long long)blockIdx.x * F;
  float acc = 0.f;
  for (int f = threadIdx.x; f < F; f += 256) acc = fmaf(row[f], w[f], acc);
  acc = pnp_warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s[i];
    out[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256)
fc_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ dout, float* __restrict__ dx,
              float* __restrict__ dw, int B, int F) {
  pnp_pdl_enter();
  int f = blockIdx.x * 256 + threadIdx.x;
  if (f >= F) return;
  float wf = w[f], acc = 0.f;
  for (int b = 0; b < B; ++b) {
    float d = dout[b];
    if (dx) dx[(long long)b * F + f] = d * wf;
    acc = fmaf(d, x[(long long)b * F + f], acc);
  }
  if (dw) dw[f] += acc;
}

__global__ void __launch_bounds__(256)
mean_combo_kernel(const float* __restrict__ a, float ca, const float* __restrict__ b, float cb, int n, float* out) {
  pnp_pdl_enter();
  __shared__ float s[8];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) acc += ca * a[i] + (b ? cb * b[i] : 0.f);
  acc = pnp_warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s[i];
    out[0] = t / (float)n;
  }
}

__global__ void __launch_bounds__(256)
l2_loss_kernel(const float* __restrict__ w, long long n, double* out) {
  pnp_pdl_enter();
  __shared__ double s[8];
  double acc = 0.0;
  float part = 0.f;
  int it = 0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float v = w[i];
    part = fmaf(v, v, part);
    if (++it == 64) { acc += (double)part; part = 0.f; it = 0; }
  }
  acc += (double)part;
  acc = pnp_warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += s[i];
    atomicAdd(out, 0.5 * t);
  }
}

// ------------------------------------------------------------------------------------------------
// optimizers over flat arenas: one CTA per 1024-element chunk, 256 threads x float4
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ theta, const float* __restrict__ grad, float* __restrict__ m, float* __restrict__ v,
            const int* __restrict__ chunk_seg, const float* __restrict__ seg_wd, const double* __restrict__ state, float b1,
            float b2, float eps, float gscale) {
  pnp_pdl_enter();
  const float wd = seg_wd[chunk_seg[blockIdx.x]];
  const float lr_t = (float)state[3];
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  float4 t = reinterpret_cast<float4*>(theta)[i];
  float4 g = __ldg(reinterpret_cast<const float4*>(grad) + i);
  float4 mm = reinterpret_cast<float4*>(m)[i];
  float4 vv = reinterpret_cast<float4*>(v)[i];
#define PNP_ADAM1(F)                                   \
  {                                                    \
    float gg = fmaf(wd, t.F, g.F * gscale);            \
    mm.F = b1 * mm.F + (1.f - b1) * gg;                \
    vv.F = b2 * vv.F + (1.f - b2) * gg * gg;           \
    t.F -= lr_t * mm.F / (sqrtf(vv.F) + eps);          \
  }
  PNP_ADAM1(x) PNP_ADAM1(y) PNP_ADAM1(z) PNP_ADAM1(w)
#undef PNP_ADAM1
  reinterpret_cast<float4*>(theta)[i] = t;
  reinterpret_cast<float4*>(m)[i] = mm;
  reinterpret_cast<float4*>(v)[i] = vv;
}

__global__ void __launch_bounds__(256)
rmsprop_kernel(float* __restrict__ theta, const float* __restrict__ grad, float* __restrict__ ms, float* __restrict__ mom,
               const int* __restrict__ chunk_seg, const float* __restrict__ seg_wd, const float* __restrict__ seg_clip,
               const float* __restrict__ lr_ptr, float decay, float momentum, float eps, float gscale) {
  pnp_pdl_enter();
  const int seg = chunk_seg[blockIdx.x];
  const float lr = *lr_ptr;
  const float wd = seg_wd[seg];
  const float clip = seg_clip ? seg_clip[seg] : 0.f;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  float4 t = reinterpret_cast<float4*>(theta)[i];
  float4 g = __ldg(reinterpret_cast<const float4*>(grad) + i);
  float4 s = reinterpret_cast<float4*>(ms)[i];
  float4 mo = reinterpret_cast<float4*>(mom)[i];
#define PNP_RMS1(F)                                              \
  {                                                              \
    float gg = fmaf(wd, t.F, g.F * gscale);                      \
    s.F = decay * s.F + (1.f - decay) * gg * gg;                 \
    mo.F = momentum * mo.F + lr * gg / sqrtf(s.F + eps);         \
    t.F -= mo.F;                                                 \
    if (clip > 0.f) t.F = fminf(fmaxf(t.F, -clip), clip);        \
  }
  PNP_RMS1(x) PNP_RMS1(y) PNP_RMS1(z) PNP_RMS1(w)
#undef PNP_RMS1
  reinterpret_cast<float4*>(theta)[i] = t;
  reinterpret_cast<float4*>(ms)[i] = s;
  reinterpret_cast<float4*>(mom)[i] = mo;
}

// tf.train.MomentumOptimizer (source_segmenter.py:371): accum = momentum*accum + g ; theta -= lr*accum   (g includes wd*theta)
__global__ void __launch_bounds__(256)
momentum_kernel(float* __restrict__ theta, const float* __restrict__ grad, float* __restrict__ accum, const int* __restrict__ chunk_seg,
                const float* __restrict__ seg_wd, const float* __restrict__ lr_ptr, float momentum, float gscale) {
  pnp_pdl_enter();
  const int seg = chunk_seg[blockIdx.x];
  const float lr = *lr_ptr;
  const float wd = seg_wd[seg];
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  float4 t = reinterpret_cast<float4*>(theta)[i];
  const float4 g = __ldg(reinterpret_cast<const float4*>(grad) + i);
  float4 ac = reinterpret_cast<float4*>(accum)[i];
  ac.x = momentum * ac.x + fmaf(wd, t.x, g.x * gscale); t.x -= lr * ac.x;
  ac.y = momentum * ac.y + fmaf(wd, t.y, g.y * gscale); t.y -= lr * ac.y;
  ac.z = momentum * ac.z + fmaf(wd, t.z, g.z * gscale); t.z -= lr * ac.z;
  ac.w = momentum * ac.w + fmaf(wd, t.w, g.w * gscale); t.w -= lr * ac.w;
  reinterpret_cast<float4*>(theta)[i] = t;
  reinterpret_cast<float4*>(accum)[i] = ac;
}

// state = [beta1^t, beta2^t, lr, lr_t]: advance t and refresh lr_t = lr*sqrt(1-beta2^t)/(1-beta1^t) (TF Adam)
__global__ void adam_advance_kernel(double* state, double b1, double b2) {
  pnp_pdl_enter();
  double p1 = state[0] * b1, p2 = state[1] * b2;
  state[0] = p1;
  state[1] = p2;
  state[3] = state[2] * sqrt(1.0 - p2) / (1.0 - p1);
}

__global__ void __launch_bounds__(256) fill_kernel(float* __restrict__ p, float v, long long n) {
  pnp_pdl_enter();
  long long n4 = n >> 2;
  float4 vv = make_float4(v, v, v, v);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256)
    reinterpret_cast<float4*>(p)[i] = vv;
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) p[(n4 << 2) + threadIdx.x] = v;
}

}  // namespace

#define S_ ((cudaStream_t)stream)

extern "C" int pnp_bn_stats(const float* z, long long M, int C, double* sum, double* sumsq, void* stream) {
  if (!z || !sum || !sumsq) return PNP_ERR_BAD_ARG;
  int tpr, grid; long long rpb;
  int rc = reduce_launch_cfg(M, C, &tpr, &rpb, &grid);
  if (rc) return rc;
  pnp_launch(bn_reduce_kernel<false>, grid, 256, 0, S_, z, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, M, C, tpr, rpb, sum, sumsq);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_finalize(const double* sum, const double* sumsq, long long M, int C, const float* gamma,
                               const float* beta, float* moving_mean, float* moving_var, int training, float* scale,
                               float* shift, float* mean, float* invstd, void* stream) {
  if (!gamma || !beta || !moving_mean || !moving_var || !scale || !shift || !mean || !invstd || C <= 0) return PNP_ERR_BAD_ARG;
  if (training && (!sum || !sumsq || M <= 0)) return PNP_ERR_BAD_ARG;
  pnp_launch(bn_finalize_kernel, pnp_cdiv(C, 128), 128, 0, S_, sum, sumsq, M, C, gamma, beta, moving_mean, moving_var, training, scale,
                                                       shift, mean, invstd);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_act_apply(const float* z, const float* scale, const float* shift, const float* skip, int Cs,
                                int skip_off, int act, float* y, uint16_t* y_hi, uint16_t* y_lo, long long M, int C, void* stream) {
  if (!z || !y || M <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (C % 4 != 0) return PNP_ERR_UNSUPPORTED;
  if (skip && (Cs % 4 != 0 || skip_off % 4 != 0 || skip_off < 0 || skip_off + Cs > C)) return PNP_ERR_UNSUPPORTED;
  if ((scale == nullptr) != (shift == nullptr)) return PNP_ERR_BAD_ARG;
  long long n4 = M * (C / 4);
  pnp_launch(bn_act_apply_kernel, grid_for(n4, 256), 256, 0, S_, z, scale, shift, skip, Cs, skip_off, act, y, y_hi, y_lo, n4, C / 4);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_bwd_reduce(const float* dy, const float* y, const float* z, const float* mean, const float* invstd,
                                 int act, float* g, double* sum_g, double* sum_gx, long long M, int C, void* stream) {
  if (!dy || !z || !mean || !invstd || !g || !sum_g || !sum_gx) return PNP_ERR_BAD_ARG;
  if (act != PNP_ACT_NONE && !y) return PNP_ERR_BAD_ARG;
  int tpr, grid; long long rpb;
  int rc = reduce_launch_cfg(M, C, &tpr, &rpb, &grid);
  if (rc) return rc;
  pnp_launch(bn_reduce_kernel<true>, grid, 256, 0, S_, z, dy, y, nullptr, mean, invstd, act, g, M, C, tpr, rpb, sum_g, sum_gx);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

/* sums only: g = dy * act'(y) is NOT written (pnp_bn_bwd_apply_direct recomputes it); the activation sign comes from y or from
 * the bf16 hi plane of y */
extern "C" int pnp_bn_bwd_reduce_sums(const float* dy, const float* y, const uint16_t* y_hi, const float* z, const float* mean,
                                      const float* invstd, int act, double* sum_g, double* sum_gx, long long M, int C, void* stream) {
  if (!dy || !z || !mean || !invstd || !sum_g || !sum_gx) return PNP_ERR_BAD_ARG;
  if (act != PNP_ACT_NONE && !y && !y_hi) return PNP_ERR_BAD_ARG;
  int tpr, grid; long long rpb;
  int rc = reduce_launch_cfg(M, C, &tpr, &rpb, &grid);
  if (rc) return rc;
  pnp_launch(bn_reduce_kernel<true>, grid, 256, 0, S_, z, dy, y, y_hi, mean, invstd, act, nullptr, M, C, tpr, rpb, sum_g, sum_gx);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_bwd_finalize(const double* sum_g, const double* sum_gx, long long M, int C, float* dgamma,
                                   float* dbeta, float* coef, void* stream) {
  if (!sum_g || !sum_gx || !coef || C <= 0 || M <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(bn_bwd_finalize_kernel, pnp_cdiv(C, 128), 128, 0, S_, sum_g, sum_gx, M, C, dgamma, dbeta, coef);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_bwd_apply(const float* g, const float* z, const float* mean, const float* invstd, const float* gamma,
                                const float* coef, int training, const pnp_dropout_cfg* drop, float* dz, uint16_t* dz_hi,
                                uint16_t* dz_lo, long long M, int C, void* stream) {
  if (!g || !invstd || !gamma || !dz || M <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (training && (!z || !mean || !coef)) return PNP_ERR_BAD_ARG;
  if (C % 4 != 0) return PNP_ERR_UNSUPPORTED;
  long long n4 = M * (C / 4);
  pnp_launch(bn_bwd_apply_kernel, grid_for(n4, 256), 256, 0, S_, g, z, mean, invstd, gamma, coef, training, make_drop(drop), dz, dz_hi, dz_lo,
                                                            n4, C / 4);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_apply_fused(const float* z, const double* sum, const double* sumsq, long long M, int C, const float* gamma,
                                  const float* beta, float* moving_mean, float* moving_var, int training, const float* skip, int Cs,
                                  int skip_off, int act, float* y, uint16_t* y_hi, uint16_t* y_lo, float* mean_out,
                                  float* invstd_out, void* stream) {
  if (!z || (!y && !y_hi) || !gamma || !beta || !moving_mean || !moving_var || M <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (training && (!sum || !sumsq)) return PNP_ERR_BAD_ARG;
  if ((mean_out == nullptr) != (invstd_out == nullptr)) return PNP_ERR_BAD_ARG;
  if (C % 4 != 0 || C > 1024) return PNP_ERR_UNSUPPORTED;
  if (skip && (Cs % 4 != 0 || skip_off % 4 != 0 || skip_off < 0 || skip_off + Cs > C)) return PNP_ERR_UNSUPPORTED;
  long long n4 = M * (C / 4);
  pnp_launch(bn_apply_fused_kernel, grid_for(n4, 256), 256, 2 * C * sizeof(float), S_, z, sum, sumsq, M, C, gamma, beta, moving_mean, moving_var,
                                                                             training, skip, Cs, skip_off, act, y, y_hi, y_lo,
                                                                             mean_out, invstd_out, n4);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_bn_bwd_apply_fused(const float* g, const float* z, const float* mean, const float* invstd, const float* gamma,
                                      const double* sum_g, const double* sum_gx, long long M, int C, int training,
                                      const pnp_dropout_cfg* drop, float* dgamma, float* dbeta, float* dz, uint16_t* dz_hi,
                                      uint16_t* dz_lo, void* stream) {
  if (!g || !invstd || !gamma || !dz || M <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (training && (!z || !mean || !sum_g || !sum_gx)) return PNP_ERR_BAD_ARG;
  if ((sum_g == nullptr) != (sum_gx == nullptr)) return PNP_ERR_BAD_ARG;
  if ((dgamma || dbeta) && !sum_g) return PNP_ERR_BAD_ARG;
  if (C % 4 != 0 || C > 1024) return PNP_ERR_UNSUPPORTED;
  long long n4 = M * (C / 4);
  pnp_launch(bn_bwd_apply_fused_kernel, grid_for(n4, 256), 256, 5 * C * sizeof(float), S_, g, nullptr, nullptr, PNP_ACT_NONE, z, mean, invstd, gamma,
                                                                                 sum_g, sum_gx, M, C, training, make_drop(drop), dgamma,
                                                                                 dbeta, dz, dz_hi, dz_lo, n4);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

/* as pnp_bn_bwd_apply_fused, but from dy: g = dy * act'(y) is recomputed on the fly (activation sign from y or from its bf16 hi
 * plane), so the fp32 g tensor never exists; dz may be NULL when only the bf16 planes are consumed (wgmma wgrad / dgrad) */
extern "C" int pnp_bn_bwd_apply_direct(const float* dy, const float* y, const uint16_t* y_hi, int act, const float* z,
                                       const float* mean, const float* invstd, const float* gamma, const double* sum_g,
                                       const double* sum_gx, long long M, int C, int training, const pnp_dropout_cfg* drop,
                                       float* dgamma, float* dbeta, float* dz, uint16_t* dz_hi, uint16_t* dz_lo, void* stream) {
  if (!dy || !invstd || !gamma || (!dz && !dz_hi) || M <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (act != PNP_ACT_NONE && !y && !y_hi) return PNP_ERR_BAD_ARG;
  if (training && (!z || !mean || !sum_g || !sum_gx)) return PNP_ERR_BAD_ARG;
  if ((sum_g == nullptr) != (sum_gx == nullptr)) return PNP_ERR_BAD_ARG;
  if ((dgamma || dbeta) && !sum_g) return PNP_ERR_BAD_ARG;
  if (C % 4 != 0 || C > 1024) return PNP_ERR_UNSUPPORTED;
  long long n4 = M * (C / 4);
  pnp_launch(bn_bwd_apply_fused_kernel, grid_for(n4, 256), 256, 5 * C * sizeof(float), S_, dy, y, y_hi, act, z, mean, invstd, gamma, sum_g, sum_gx, M,
                                                                                 C, training, make_drop(drop), dgamma, dbeta, dz, dz_hi,
                                                                                 dz_lo, n4);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_act_bwd(const float* dy, const float* y, int act, float* g, long long n, void* stream) {
  if (!dy || !y || !g || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(act_bwd_kernel, grid_for(n, 256 * 8), 256, 0, S_, dy, y, act, g, n);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_channel_slice(const float* g, int C, int off, int Cs, float* out, long long M, int accumulate, void* stream) {
  if (!g || !out || M <= 0 || Cs <= 0 || off < 0 || off + Cs > C) return PNP_ERR_BAD_ARG;
  long long total = M * Cs;
  pnp_launch(channel_slice_kernel, grid_for(total, 256 * 8), 256, 0, S_, g, C, off, Cs, out, total, accumulate);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_dropout_apply(const float* x, float* y, long long n, const pnp_dropout_cfg* drop, void* stream) {
  if (!x || !y || n <= 0) return PNP_ERR_BAD_ARG;
  PnpDropout d = make_drop(drop);
  if (!d.seed_ptr) {
    if (x != y) PNP_CUDA(cudaMemcpyAsync(y, x, n * sizeof(float), cudaMemcpyDeviceToDevice, S_));
    return PNP_OK;
  }
  pnp_launch(dropout_kernel, grid_for(n / 4 + 1, 256 * 4), 256, 0, S_, x, y, n, d);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_seed_advance(unsigned long long* seed_ptr, void* stream) {
  if (!seed_ptr) return PNP_ERR_BAD_ARG;
  pnp_launch(seed_advance_kernel, 1, 1, 0, S_, seed_ptr);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_maxpool2_fwd(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  if (!x || !y || B <= 0 || H <= 0 || W <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if ((H | W) & 1) return PNP_ERR_UNSUPPORTED;
  long long total = (long long)B * (H / 2) * (W / 2) * C;
  if (C % 4 == 0) pnp_launch(maxpool2_fwd_kernel<4>, grid_for(total / 4, 256 * 2), 256, 0, S_, x, y, B, H, W, C);
  else pnp_launch(maxpool2_fwd_kernel<1>, grid_for(total, 256 * 4), 256, 0, S_, x, y, B, H, W, C);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_maxpool2_bwd(const float* x, const float* dy, float* dx, int B, int H, int W, int C, void* stream) {
  if (!x || !dy || !dx || B <= 0 || H <= 0 || W <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if ((H | W) & 1) return PNP_ERR_UNSUPPORTED;
  long long total = (long long)B * (H / 2) * (W / 2) * C;
  if (C % 4 == 0) pnp_launch(maxpool2_bwd_kernel<4>, grid_for(total / 4, 256 * 2), 256, 0, S_, x, dy, dx, B, H, W, C);
  else pnp_launch(maxpool2_bwd_kernel<1>, grid_for(total, 256 * 4), 256, 0, S_, x, dy, dx, B, H, W, C);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_avgpool2(const float* in, float* out, int B, int H, int W, int C, int backward, void* stream) {
  if (!in || !out || B <= 0 || H <= 0 || W <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if ((H | W) & 1) return PNP_ERR_UNSUPPORTED;
  long long total = (long long)B * (H / 2) * (W / 2) * C;
  pnp_launch(avgpool2_kernel, grid_for(total, 256 * 4), 256, 0, S_, in, out, B, H, W, C, backward);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_mirror_pad_fwd(const float* x, float* y, int B, int H, int W, int C, int p, void* stream) {
  if (!x || !y || B <= 0 || H <= 0 || W <= 0 || C <= 0 || p < 0) return PNP_ERR_BAD_ARG;
  if (p > H || p > W) return PNP_ERR_UNSUPPORTED;
  long long total = (long long)B * (H + 2 * p) * (W + 2 * p) * C;
  pnp_launch(mirror_pad_fwd_kernel, grid_for(total, 256 * 8), 256, 0, S_, x, y, B, H, W, C, p);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_mirror_pad_bwd(const float* dy, float* dx, int B, int H, int W, int C, int p, void* stream) {
  if (!dy || !dx || B <= 0 || H <= 0 || W <= 0 || C <= 0 || p < 0) return PNP_ERR_BAD_ARG;
  if (2 * p > H || 2 * p > W) return PNP_ERR_UNSUPPORTED;
  long long total = (long long)B * H * W * C;
  pnp_launch(mirror_pad_bwd_kernel, grid_for(total, 256 * 8), 256, 0, S_, dy, dx, B, H, W, C, p);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_phase_shift_fwd(const float* X, float* out, int B, int a, int b, int G, int r, int Ctot, int coff,
                                   int ntile, int order_b1, void* stream) {
  if (!X || !out || B <= 0 || a <= 0 || b <= 0 || G <= 0 || r <= 0 || ntile <= 0 || coff < 0 || coff + ntile * G > Ctot)
    return PNP_ERR_BAD_ARG;
  long long total = (long long)B * a * r * b * r * G;
  pnp_launch(phase_shift_fwd_kernel, grid_for(total, 256 * 8), 256, 0, S_, X, out, B, a, b, G, r, Ctot, coff, ntile, order_b1);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_phase_shift_bwd(const float* dout, float* dX, int B, int a, int b, int G, int r, int Ctot, int coff,
                                   int ntile, int order_b1, void* stream) {
  if (!dout || !dX || B <= 0 || a <= 0 || b <= 0 || G <= 0 || r <= 0 || ntile <= 0 || coff < 0 || coff + ntile * G > Ctot)
    return PNP_ERR_BAD_ARG;
  long long total = (long long)B * a * b * G * r * r;
  pnp_launch(phase_shift_bwd_kernel, grid_for(total, 256 * 8), 256, 0, S_, dout, dX, B, a, b, G, r, Ctot, coff, ntile, order_b1);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_disc_input_fwd(const float* const* srcs, const int* a, const int* b, const int* G, const int* ntile, int nsrc,
                                  const float* logits, int NC, float* out, int B, int H, int W, int r, int order_b1, void* stream) {
  if (!srcs || !a || !b || !G || !ntile || nsrc < 1 || nsrc > 4 || !logits || !out || B <= 0 || r <= 0 || NC <= 0 || NC > kMaxC)
    return PNP_ERR_BAD_ARG;
  DiscPlan plan;
  int ch = 0;
  for (int s = 0; s < nsrc; ++s) {
    if (!srcs[s] || a[s] * r != H || b[s] * r != W || G[s] <= 0 || ntile[s] < 1) return PNP_ERR_BAD_ARG;
    plan.src[s] = srcs[s]; plan.a[s] = a[s]; plan.b[s] = b[s]; plan.G[s] = G[s];
    for (int t = 0; t < ntile[s]; ++t)
      for (int g = 0; g < G[s]; ++g) {
        if (ch >= 64) return PNP_ERR_UNSUPPORTED;
        plan.ch_src[ch] = (signed char)s; plan.ch_g[ch] = (signed char)g; ++ch;
      }
  }
  for (int s = nsrc; s < 4; ++s) { plan.src[s] = nullptr; plan.a[s] = plan.b[s] = plan.G[s] = 0; }
  for (int c = 0; c < NC; ++c) {
    if (ch >= 64) return PNP_ERR_UNSUPPORTED;
    plan.ch_src[ch] = -1; plan.ch_g[ch] = (signed char)c; ++ch;
  }
  if (ch >= 64) return PNP_ERR_UNSUPPORTED;
  plan.ch_src[ch] = -2; plan.ch_g[ch] = 0; ++ch;
  const int Ctot = ch;
  if (Ctot % 4 != 0) return PNP_ERR_UNSUPPORTED;
  for (int c = Ctot; c < 64; ++c) { plan.ch_src[c] = -1; plan.ch_g[c] = 0; }
  const long long total = (long long)B * H * W * (Ctot / 4);
  if (total >= (1LL << 31) || (long long)B * H * W * 64 >= (1LL << 31)) return PNP_ERR_UNSUPPORTED;
  bool same_grid = true;
  for (int s = 1; s < nsrc; ++s) same_grid = same_grid && a[s] == a[0] && b[s] == b[0];
  if (r == 8 && !order_b1 && same_grid) {
    // distinct (source, group) lines; tiled channels share a line
    DiscLines ln;
    ln.nlines = 0;
    bool fits = true;
    for (int c = 0; c < 64; ++c) ln.line_of[c] = -1;
    for (int c = 0; c < Ctot && fits; ++c) {
      if (plan.ch_src[c] < 0) { ln.line_of[c] = plan.ch_src[c]; continue; }
      int found = -1;
      for (int l = 0; l < ln.nlines; ++l)
        if (ln.line_src[l] == plan.ch_src[c] && ln.line_g[l] == plan.ch_g[c]) found = l;
      if (found < 0) {
        if (ln.nlines >= 32) { fits = false; break; }
        ln.line_src[ln.nlines] = plan.ch_src[c]; ln.line_g[ln.nlines] = plan.ch_g[c];
        found = ln.nlines++;
      }
      ln.line_of[c] = (signed char)found;
    }
    const size_t smem = (size_t)4 * ln.nlines * 65 * sizeof(float);
    if (fits && ln.nlines > 0 && smem <= 48 * 1024) {
      const long long blocks = (long long)B * a[0] * ((b[0] + 3) / 4);
      pnp_launch(disc_input_r8_kernel, (unsigned)blocks, 256, smem, S_, plan, ln, logits, NC, out, B, a[0], b[0], Ctot);
      PNP_LAUNCH_CHECK();
      return PNP_OK;
    }
  }
  pnp_launch(disc_input_kernel, grid_for(total, 256), 256, 0, S_, plan, logits, NC, out, B, H, W, Ctot, r, order_b1);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_logits_argmax_concat(const float* logits, float* out, long long P, int C, int Ctot, int coff, void* stream) {
  if (!logits || !out || P <= 0 || C <= 0 || coff < 0 || coff + C + 1 > Ctot) return PNP_ERR_BAD_ARG;
  pnp_launch(logits_argmax_concat_kernel, grid_for(P, 256 * 2), 256, 0, S_, logits, out, P, C, Ctot, coff);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_pixel_softmax2(const float* logits, float* out, long long P, int C, void* stream) {
  if (!logits || !out || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (C > kMaxC) return PNP_ERR_UNSUPPORTED;
  pnp_launch(pixel_softmax2_kernel, grid_for(P, 256 * 2), 256, 0, S_, logits, out, P, C);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_image_summary_u8(const float* const* srcs, const int* kinds, const int* C, const int* channel, int nsrc,
                                    int B, int H, int W, int n, unsigned char* out, void* stream) {
  if (!srcs || !kinds || !C || !channel || !out || nsrc < 1 || B <= 0 || H <= 0 || W <= 0 || n < 1 || n > B) return PNP_ERR_BAD_ARG;
  if (nsrc > kImgMaxSrc) return PNP_ERR_UNSUPPORTED;
  ImgPlan plan;
  for (int s = 0; s < kImgMaxSrc; ++s) { plan.src[s] = nullptr; plan.kind[s] = plan.C[s] = plan.ch[s] = 0; }
  for (int s = 0; s < nsrc; ++s) {
    if (!srcs[s] || C[s] <= 0) return PNP_ERR_BAD_ARG;
    if (kinds[s] == PNP_IMG_CHANNEL) {
      if (channel[s] < 0 || channel[s] >= C[s]) return PNP_ERR_BAD_ARG;
    } else if (kinds[s] == PNP_IMG_ARGMAX || kinds[s] == PNP_IMG_SOFTMAX2_ARGMAX) {
      if (C[s] > kMaxC) return PNP_ERR_UNSUPPORTED;
    } else {
      return PNP_ERR_BAD_ARG;
    }
    plan.src[s] = srcs[s]; plan.kind[s] = kinds[s]; plan.C[s] = C[s]; plan.ch[s] = channel[s];
  }
  pnp_launch(image_summary_u8_kernel, (unsigned)(nsrc * n), kImgThreads, 0, S_, plan, n, (long long)H * W, out);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_segloss_reduce(const float* logits, const float* y, long long P, int C, double* acc, void* stream) {
  if (!logits || !y || !acc || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (C > kMaxC) return PNP_ERR_UNSUPPORTED;
  pnp_launch(segloss_reduce_kernel, grid_for(P, 256 * 8), 256, 0, S_, logits, y, P, C, acc);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_segloss_finalize(const double* acc, long long P, int C, float* out, float* coef, void* stream) {
  if (!acc || !out || !coef || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(segloss_finalize_kernel, 1, 32, 0, S_, acc, P, C, out, coef);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_segloss_bwd(const float* logits, const float* y, const float* coef, const float* g_wce, const float* g_dice,
                               float* dlogits, long long P, int C, void* stream) {
  if (!logits || !y || !coef || !dlogits || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (C > kMaxC) return PNP_ERR_UNSUPPORTED;
  pnp_launch(segloss_bwd_kernel, grid_for(P, 256 * 2), 256, 0, S_, logits, y, coef, g_wce, g_dice, dlogits, P, C);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_confusion(const float* logits, const float* y, long long P, int C, unsigned long long* counts, void* stream) {
  if (!logits || !y || !counts || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (C > kMaxC) return PNP_ERR_UNSUPPORTED;
  pnp_launch(confusion_kernel, grid_for(P, 256 * 16), 256, 0, S_, logits, y, P, C, counts);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_one_hot(const long long* labels, float* out, long long P, int C, void* stream) {
  if (!labels || !out || P <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(one_hot_kernel, grid_for(P, 256 * 2), 256, 0, S_, labels, out, P, C);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_fc_fwd(const float* x, const float* w, float* out, int B, int F, void* stream) {
  if (!x || !w || !out || B <= 0 || F <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(fc_fwd_kernel, B, 256, 0, S_, x, w, out, F);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_fc_bwd(const float* x, const float* w, const float* dout, float* dx, float* dw, int B, int F, void* stream) {
  if (!x || !w || !dout || B <= 0 || F <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(fc_bwd_kernel, pnp_cdiv(F, 256), 256, 0, S_, x, w, dout, dx, dw, B, F);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_mean_combo(const float* a, float ca, const float* b, float cb, int n, float* out, void* stream) {
  if (!a || !out || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(mean_combo_kernel, 1, 256, 0, S_, a, ca, b, cb, n, out);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_l2_loss_acc(const float* w, long long n, double* out, void* stream) {
  if (!w || !out || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(l2_loss_kernel, grid_for(n, 256 * 16), 256, 0, S_, w, n, out);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_adam_advance(double* state, float beta1, float beta2, void* stream) {
  if (!state) return PNP_ERR_BAD_ARG;
  pnp_launch(adam_advance_kernel, 1, 1, 0, S_, state, (double)beta1, (double)beta2);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_adam_step(float* theta, const float* grad, float* m, float* v, long long n, const int* chunk_seg,
                             const float* seg_wd, const double* state, float beta1, float beta2, float eps, float grad_scale,
                             void* stream) {
  if (!theta || !grad || !m || !v || !chunk_seg || !seg_wd || !state || n <= 0 || (n % 1024) != 0) return PNP_ERR_BAD_ARG;
  pnp_launch(adam_kernel, (unsigned)(n / 1024), 256, 0, S_, theta, grad, m, v, chunk_seg, seg_wd, state, beta1, beta2, eps, grad_scale);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_rmsprop_step(float* theta, const float* grad, float* ms, float* mom, long long n, const int* chunk_seg,
                                const float* seg_wd, const float* seg_clip, const float* lr_ptr, float decay, float momentum,
                                float eps, float grad_scale, void* stream) {
  if (!theta || !grad || !ms || !mom || !chunk_seg || !seg_wd || !lr_ptr || n <= 0 || (n % 1024) != 0) return PNP_ERR_BAD_ARG;
  pnp_launch(rmsprop_kernel, (unsigned)(n / 1024), 256, 0, S_, theta, grad, ms, mom, chunk_seg, seg_wd, seg_clip, lr_ptr, decay, momentum, eps,
                                                      grad_scale);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_momentum_step(float* theta, const float* grad, float* accum, long long n, const int* chunk_seg, const float* seg_wd,
                                 const float* lr_ptr, float momentum, float grad_scale, void* stream) {
  if (!theta || !grad || !accum || !chunk_seg || !seg_wd || !lr_ptr || n <= 0 || (n % 1024) != 0) return PNP_ERR_BAD_ARG;
  pnp_launch(momentum_kernel, (unsigned)(n / 1024), 256, 0, S_, theta, grad, accum, chunk_seg, seg_wd, lr_ptr, momentum, grad_scale);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_fill(float* p, float v, long long n, void* stream) {
  if (!p || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(fill_kernel, grid_for(n / 4 + 1, 256 * 4), 256, 0, S_, p, v, n);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" const char* pnp_error_string(int code) {
  switch (code) {
    case 0: return "ok";
    case PNP_ERR_BAD_ARG: return "pnp: bad argument";
    case PNP_ERR_UNSUPPORTED: return "pnp: unsupported shape/configuration";
    case PNP_ERR_DRIVER: return "pnp: CUDA driver entry point unavailable";
    default: return cudaGetErrorString((cudaError_t)code);
  }
}

extern "C" int pnp_version(void) { return 100; }
