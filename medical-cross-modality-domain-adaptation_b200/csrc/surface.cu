// The members of the layers.py operator surface that the reference's graphs do not call but that a user of the module can:
// n x n pooling with TF 'SAME' geometry for any n (layers.py:102-106; the graphs use n = 2 -> elementwise.cu's maxpool2 / avgpool2),
// crop_and_concat / simple_concat2d (layers.py:108-127) and cross_entropy (layers.py:140-141).  All are streaming kernels over NHWC
// fp32 tensors: HBM-bound, one read and one write per element, 4-byte accesses coalesced along the channel axis.
#include "common.cuh"
#include "../../include/pnp_b200.h"

namespace {

inline int grid_for(long long work_items, int per_block) {
  long long b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > PNP_NUM_SMS * 64LL) b = PNP_NUM_SMS * 64LL;
  return (int)b;
}

// TF 'SAME' pooling geometry with ksize = stride = n: Ho = ceil(H / n), pad_total = Ho * n - H (< n), pad_before = pad_total / 2;
// window `o` covers input rows [o * n - pad_before, o * n - pad_before + n) clipped to the image (padding never wins a max and is not
// counted by the average).  Every input row belongs to exactly one window: o = (i + pad_before) / n.
struct PoolGeom {
  int B, H, W, C, n, Ho, Wo, pt, pl;
};

__global__ void __launch_bounds__(256)
pool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, PoolGeom g, int avg) {
  pnp_pdl_enter();
  const long long total = (long long)g.B * g.Ho * g.Wo * g.C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % g.C);
    long long p = i / g.C;
    const int ox = (int)(p % g.Wo);
    p /= g.Wo;
    const int oy = (int)(p % g.Ho);
    const int b = (int)(p / g.Ho);
    const int y0 = max(oy * g.n - g.pt, 0), y1 = min(oy * g.n - g.pt + g.n, g.H);
    const int x0 = max(ox * g.n - g.pl, 0), x1 = min(ox * g.n - g.pl + g.n, g.W);
    float m = -INFINITY, s = 0.f;
    for (int iy = y0; iy < y1; ++iy)
      for (int ix = x0; ix < x1; ++ix) {
        const float v = x[(((long long)b * g.H + iy) * g.W + ix) * g.C + c];
        m = fmaxf(m, v);
        s += v;
      }
    y[i] = avg ? s / (float)((y1 - y0) * (x1 - x0)) : m;
  }
}

// one thread per INPUT element: max pooling routes the window's gradient to the FIRST maximal element in row-major window order
// (what TF's MaxPoolGrad does, and elementwise.cu's 2x2 kernel); average pooling spreads it over the window's valid elements.
__global__ void __launch_bounds__(256)
pool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, PoolGeom g, int avg) {
  pnp_pdl_enter();
  const long long total = (long long)g.B * g.H * g.W * g.C;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % g.C);
    long long p = i / g.C;
    const int ix = (int)(p % g.W);
    p /= g.W;
    const int iy = (int)(p % g.H);
    const int b = (int)(p / g.H);
    const int oy = (iy + g.pt) / g.n, ox = (ix + g.pl) / g.n;
    const int y0 = max(oy * g.n - g.pt, 0), y1 = min(oy * g.n - g.pt + g.n, g.H);
    const int x0 = max(ox * g.n - g.pl, 0), x1 = min(ox * g.n - g.pl + g.n, g.W);
    const float gout = dy[(((long long)b * g.Ho + oy) * g.Wo + ox) * g.C + c];
    if (avg) {
      dx[i] = gout / (float)((y1 - y0) * (x1 - x0));
      continue;
    }
    float best = -INFINITY;
    int by = y0, bx = x0;
    for (int yy = y0; yy < y1; ++yy)
      for (int xx = x0; xx < x1; ++xx) {
        const float v = x[(((long long)b * g.H + yy) * g.W + xx) * g.C + c];
        if (v > best) { best = v; by = yy; bx = xx; }
      }
    dx[i] = (by == iy && bx == ix) ? gout : 0.f;
  }
}

// out[b, y, x, :] = [ x1[b, y + oy, x + ox, :] | x2[b, y, x, :] ]       (crop_and_concat; simple_concat2d is oy = ox = 0, H1 = H2, W1 = W2)
struct CatGeom {
  int B, H1, W1, C1, H2, W2, C2, oy, ox;
};

__global__ void __launch_bounds__(256)
crop_concat_fwd_kernel(const float* __restrict__ x1, const float* __restrict__ x2, float* __restrict__ out, CatGeom g) {
  pnp_pdl_enter();
  const int Ct = g.C1 + g.C2;
  const long long total = (long long)g.B * g.H2 * g.W2 * Ct;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % Ct);
    long long p = i / Ct;
    const int x = (int)(p % g.W2);
    long long t = p / g.W2;
    const int y = (int)(t % g.H2);
    const int b = (int)(t / g.H2);
    out[i] = c < g.C1 ? x1[(((long long)b * g.H1 + y + g.oy) * g.W1 + x + g.ox) * g.C1 + c] : x2[p * g.C2 + (c - g.C1)];
  }
}

// dx1 (zero outside the crop window) and dx2 from dout; either may be NULL
__global__ void __launch_bounds__(256)
crop_concat_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dx1, float* __restrict__ dx2, CatGeom g) {
  pnp_pdl_enter();
  const int Ct = g.C1 + g.C2;
  const long long n1 = dx1 ? (long long)g.B * g.H1 * g.W1 * g.C1 : 0;
  const long long n2 = dx2 ? (long long)g.B * g.H2 * g.W2 * g.C2 : 0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n1 + n2; i += (long long)gridDim.x * 256) {
    if (i < n1) {
      const int c = (int)(i % g.C1);
      long long p = i / g.C1;
      const int x = (int)(p % g.W1) - g.ox;
      long long t = p / g.W1;
      const int y = (int)(t % g.H1) - g.oy;
      const int b = (int)(t / g.H1);
      const bool in = y >= 0 && y < g.H2 && x >= 0 && x < g.W2;
      dx1[i] = in ? dout[(((long long)b * g.H2 + y) * g.W2 + x) * Ct + c] : 0.f;
    } else {
      const long long j = i - n1;
      const int c = (int)(j % g.C2);
      const long long p = j / g.C2;
      dx2[j] = dout[p * Ct + g.C1 + c];
    }
  }
}

// cross_entropy (layers.py:140-141): -mean(y * log(clip(p, 1e-10, 1))).  Forward accumulates sum(y * log(clip p)) in a zeroed fp64
// scalar (short fp32 partials per thread, fp64 across threads); the finalize kernel turns it into the fp32 result.
__global__ void __launch_bounds__(256)
cross_entropy_acc_kernel(const float* __restrict__ y, const float* __restrict__ p, long long n, double* __restrict__ acc) {
  pnp_pdl_enter();
  __shared__ double s[8];
  double a = 0.0;
  float part = 0.f;
  int it = 0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    part = fmaf(y[i], logf(fminf(fmaxf(p[i], 1e-10f), 1.0f)), part);
    if (++it == 32) { a += (double)part; part = 0.f; it = 0; }
  }
  a += (double)part;
  a = pnp_warp_sum_d(a);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += s[i];
    atomicAdd(acc, t);
  }
}

__global__ void cross_entropy_finalize_kernel(const double* __restrict__ acc, long long n, float* __restrict__ out) {
  pnp_pdl_enter();
  out[0] = (float)(-acc[0] / (double)n);
}

// d/dy = -g/n * log(clip p);  d/dp = -g/n * y / p inside [1e-10, 1] (tf.clip_by_value passes the gradient inside the range, bounds
// included, and blocks it outside)
__global__ void __launch_bounds__(256)
cross_entropy_bwd_kernel(const float* __restrict__ y, const float* __restrict__ p, const float* __restrict__ gout, long long n,
                         float* __restrict__ dy, float* __restrict__ dp) {
  pnp_pdl_enter();
  const float k = -gout[0] / (float)n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float pv = p[i];
    if (dy) dy[i] = k * logf(fminf(fmaxf(pv, 1e-10f), 1.0f));
    if (dp) dp[i] = (pv >= 1e-10f && pv <= 1.0f) ? k * y[i] / pv : 0.f;
  }
}

bool pool_geom(PoolGeom* g, int B, int H, int W, int C, int n) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || n <= 0) return false;
  g->B = B; g->H = H; g->W = W; g->C = C; g->n = n;
  g->Ho = (H + n - 1) / n;
  g->Wo = (W + n - 1) / n;
  g->pt = (g->Ho * n - H) / 2;
  g->pl = (g->Wo * n - W) / 2;
  return true;
}

bool cat_geom(CatGeom* g, int B, int H1, int W1, int C1, int H2, int W2, int C2) {
  if (B <= 0 || H1 <= 0 || W1 <= 0 || C1 <= 0 || H2 <= 0 || W2 <= 0 || C2 <= 0 || H2 > H1 || W2 > W1) return false;
  g->B = B; g->H1 = H1; g->W1 = W1; g->C1 = C1; g->H2 = H2; g->W2 = W2; g->C2 = C2;
  g->oy = (H1 - H2) / 2;
  g->ox = (W1 - W2) / 2;
  return true;
}

}  // namespace

#define S_ ((cudaStream_t)stream)

extern "C" int pnp_pool_fwd(const float* x, float* y, int B, int H, int W, int C, int n, int avg, void* stream) {
  PoolGeom g;
  if (!x || !y || !pool_geom(&g, B, H, W, C, n)) return PNP_ERR_BAD_ARG;
  pnp_launch(pool_fwd_kernel, grid_for((long long)B * g.Ho * g.Wo * C, 256 * 4), 256, 0, S_, x, y, g, avg);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_pool_bwd(const float* x, const float* dy, float* dx, int B, int H, int W, int C, int n, int avg, void* stream) {
  PoolGeom g;
  if (!dy || !dx || (!avg && !x) || !pool_geom(&g, B, H, W, C, n)) return PNP_ERR_BAD_ARG;
  pnp_launch(pool_bwd_kernel, grid_for((long long)B * H * W * C, 256 * 4), 256, 0, S_, x, dy, dx, g, avg);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_crop_concat_fwd(const float* x1, const float* x2, float* out, int B, int H1, int W1, int C1, int H2, int W2, int C2,
                                   void* stream) {
  CatGeom g;
  if (!x1 || !x2 || !out || !cat_geom(&g, B, H1, W1, C1, H2, W2, C2)) return PNP_ERR_BAD_ARG;
  pnp_launch(crop_concat_fwd_kernel, grid_for((long long)B * H2 * W2 * (C1 + C2), 256 * 4), 256, 0, S_, x1, x2, out, g);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_crop_concat_bwd(const float* dout, float* dx1, float* dx2, int B, int H1, int W1, int C1, int H2, int W2, int C2,
                                   void* stream) {
  CatGeom g;
  if (!dout || (!dx1 && !dx2) || !cat_geom(&g, B, H1, W1, C1, H2, W2, C2)) return PNP_ERR_BAD_ARG;
  const long long n = (dx1 ? (long long)B * H1 * W1 * C1 : 0) + (dx2 ? (long long)B * H2 * W2 * C2 : 0);
  pnp_launch(crop_concat_bwd_kernel, grid_for(n, 256 * 4), 256, 0, S_, dout, dx1, dx2, g);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_cross_entropy_fwd(const float* y, const float* p, long long n, double* acc, float* out, void* stream) {
  if (!y || !p || !acc || !out || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(cross_entropy_acc_kernel, grid_for(n, 256 * 16), 256, 0, S_, y, p, n, acc);
  PNP_LAUNCH_CHECK();
  pnp_launch(cross_entropy_finalize_kernel, 1, 1, 0, S_, (const double*)acc, n, out);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_cross_entropy_bwd(const float* y, const float* p, const float* gout, long long n, float* dy, float* dp, void* stream) {
  if (!y || !p || !gout || (!dy && !dp) || n <= 0) return PNP_ERR_BAD_ARG;
  pnp_launch(cross_entropy_bwd_kernel, grid_for(n, 256 * 4), 256, 0, S_, y, p, gout, n, dy, dp);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}
