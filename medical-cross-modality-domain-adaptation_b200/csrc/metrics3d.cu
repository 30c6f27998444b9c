// Evaluation: per-class average symmetric surface distance (ASSD), Hausdorff distance (HD) and, on request, a percentile of the
// pooled surface distances (HD95 at q = 95) between a predicted and a ground-truth label volume [n0][n1][n2] (uint8, n2 fastest)
// -- the second metric of the papers' per-structure tables (medpy.metric.binary.assd / hd / hd95, 6-neighbour borders).
//
//   1. sd_border_kernel: one pass over both volumes writes a border bitmask byte per voxel (bit c: class c voxel with a
//      6-neighbour of another class or on a face of the volume; labels >= C count as background).
//   2. Per class, two exact Euclidean feature transforms run side by side (t = 0: features = border of G, queries = border of
//      P; t = 1: the roles swapped), one axis at a time (Felzenszwalb & Huttenlocher, "Distance transforms of sampled
//      functions", 2012):
//        sd_pass2_kernel  axis 2 (contiguous): nearest feature in the line, f2 (int16, -1 = none).  32 lines per block are
//                         staged through shared memory so that global reads and writes stay coalesced;
//        sd_pass1_kernel  axis 1: lower envelope of g(j) + (s1 (i1 - j))^2 with g(j) = (s2 (i2 - f2))^2 -> (f1, f2);
//        sd_pass0_kernel  axis 0, fused with the query: at each query voxel the nearest feature (f0, f1, f2) gives
//                         d = sqrt(((s0 D0)^2 + (s1 D1)^2) + (s2 D2)^2) -- scipy.ndimage.distance_transform_edt's own form and
//                         order -- and every line writes (sum d, count, max d).
//      Threads own lines and neighbouring threads own neighbouring lines, so the envelope passes read and write coalesced;
//      the envelope is a stack of int16 positions in shared memory and its values are re-derived from the feature coordinates.
//   3. sd_reduce_kernel sums the per-line partials in a fixed order: no floating-point atomics, repeated calls are bit-identical.
//
// The percentile (pnp_surface_distance_pct) adds, per class:
//   a. sd_count_kernel counts the queries of every axis-0 line of both transforms and scans them within its block;
//      sd_scan_kernel scans the block totals, so that line g = t L + l owns list[off(g) .. off(g) + count(g)) -- the pooled
//      list is the distances of dA followed by those of dB -- and derives the ranks lo, hi and the weight of numpy's
//      `linear` interpolation from the pooled count n;
//   b. sd_pass0_kernel<true> also writes each query's distance (the value it adds to the line's sum) to its slot;
//   c. a radix select on the fp64 bit patterns (distances are >= +0, so their bits order like the values): sd_hist_kernel
//      histograms one 8-bit digit of the keys that match the digits picked so far (8 passes, most significant first; each
//      pass picks the previous pass's bucket itself), sd_above_kernel picks the last digit -- D(lo) exactly -- and finds
//      min{x > D(lo)} when D(hi) is not D(lo), sd_pct_kernel interpolates.  Every count is an integer and every minimum an
//      integer minimum, so the result does not depend on the order of atomics: repeated calls are bit-identical.
//
// Exactness: with unit spacing every g and every envelope test (a cross-multiplied comparison of two parabola intersections)
// is an integer below 2^53, so the transform is exact and each distance is the correctly rounded square root of the exact
// squared distance -- bit-identical to scipy's.  With other spacings the tests round, and ties may resolve to another feature
// at the same distance up to rounding.
#include <math.h>

#include "common.cuh"
#include "../../include/pnp_b200.h"

namespace {

constexpr int ROWS = 32;    // lines per block of the contiguous-axis pass
constexpr int LINES = 32;   // lines (one per thread) per block of the envelope passes

struct Dims {
  int n0, n1, n2;
  long long N;   // n0 * n1 * n2
  long long L;   // n1 * n2: lines of the axis-0 pass
};

__device__ __forceinline__ int label_of(const uint8_t* v, long long i, int C) {
  const int l = v[i];
  return l < C ? l : 0;
}

__global__ void __launch_bounds__(256)
sd_border_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt, uint8_t* __restrict__ mask, Dims d, int C) {
  pnp_pdl_enter();
  const uint8_t* v = blockIdx.y ? gt : pred;
  uint8_t* m = mask + blockIdx.y * d.N;
  const long long s1 = d.n2, s0 = d.L;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < d.N; i += (long long)gridDim.x * 256) {
    const int l = label_of(v, i, C);
    uint8_t out = 0;
    if (l) {
      const int i2 = (int)(i % d.n2);
      const long long r = i / d.n2;
      const int i1 = (int)(r % d.n1), i0 = (int)(r / d.n1);
      const bool face = i0 == 0 || i0 == d.n0 - 1 || i1 == 0 || i1 == d.n1 - 1 || i2 == 0 || i2 == d.n2 - 1;
      if (face || label_of(v, i - 1, C) != l || label_of(v, i + 1, C) != l || label_of(v, i - s1, C) != l ||
          label_of(v, i + s1, C) != l || label_of(v, i - s0, C) != l || label_of(v, i + s0, C) != l)
        out = (uint8_t)(1u << l);
    }
    m[i] = out;
  }
}

// axis 2: f2 = position of the nearest feature in the line (-1: none).  Shared memory holds ROWS lines at `stride` int16 each
// (stride = 2 mod 4, so the 32 threads scanning their own lines hit 32 different banks).
__global__ void __launch_bounds__(ROWS)
sd_pass2_kernel(const uint8_t* __restrict__ mask, int16_t* __restrict__ fa, Dims d, int cls, int stride) {
  extern __shared__ int16_t rows[];
  pnp_pdl_enter();
  const int t = blockIdx.y;
  const uint8_t* m = mask + (long long)(1 - t) * d.N;
  int16_t* f = fa + (long long)t * d.N;
  const long long r0 = (long long)blockIdx.x * ROWS;
  const int nr = (int)min((long long)ROWS, (long long)d.n0 * d.n1 - r0);
  const uint8_t bit = (uint8_t)(1u << cls);
  for (int r = 0; r < nr; ++r)
    for (int i = threadIdx.x; i < d.n2; i += ROWS) rows[r * stride + i] = (m[(r0 + r) * d.n2 + i] & bit) ? 1 : 0;
  __syncthreads();
  if ((int)threadIdx.x < nr) {
    int16_t* row = rows + threadIdx.x * stride;
    int last = -1;
    for (int i = 0; i < d.n2; ++i) {
      if (row[i]) last = i;
      row[i] = (int16_t)last;               // a feature at i reads back as row[i] == i
    }
    int next = -1;
    for (int i = d.n2 - 1; i >= 0; --i) {
      const int l = row[i];
      if (l == i) next = i;
      row[i] = (int16_t)((next >= 0 && (l < 0 || next - i < i - l)) ? next : l);
    }
  }
  __syncthreads();
  for (int r = 0; r < nr; ++r)
    for (int i = threadIdx.x; i < d.n2; i += ROWS) f[(r0 + r) * d.n2 + i] = rows[r * stride + i];
}

__device__ __forceinline__ double sq(double x) { return __dmul_rn(x, x); }

// Lower envelope of the parabolas P_j(x) = g(j) + w (x - j)^2 over the positions j < n of one line that carry a feature.
// stk[k * LINES] holds the envelope's positions left to right.  Top entry b (left neighbour a) is dropped when the new parabola
// q overtakes it no later than b overtakes a: x(a, b) >= x(b, q) with x(a, b) = ((g_b - g_a) + w (b^2 - a^2)) / (2 w (b - a)),
// compared cross-multiplied.  Returns the top index (-1: no feature on the line).
template <class Line>
__device__ __forceinline__ int envelope(const Line& line, int n, double w, int16_t* stk) {
  int k = -1;
  double gb = 0.0, ga = 0.0;   // g of the top entry and of the one below it
  for (int q = 0; q < n; ++q) {
    if (!line.has(q)) continue;
    const double gq = line.g(q);
    while (k >= 1) {
      const int a = stk[(k - 1) * LINES], b = stk[k * LINES];
      const double nab = (gb - ga) + w * (double)((b - a) * (b + a));
      const double nbq = (gq - gb) + w * (double)((q - b) * (q + b));
      if (nab * (double)(q - b) < nbq * (double)(b - a)) break;
      --k;
      gb = ga;
      ga = k >= 1 ? line.g(stk[(k - 1) * LINES]) : 0.0;
    }
    ++k;
    stk[k * LINES] = (int16_t)q;
    ga = gb;
    gb = gq;
  }
  return k;
}

// Walks the envelope left to right: `at(x)` returns the position of the parabola lowest at x (x non-decreasing between calls).
template <class Line>
struct EnvelopeWalk {
  const Line& line;
  const int16_t* stk;
  int top, e, je, jn = 0;
  double w, ge, gn = 0.0;
  __device__ EnvelopeWalk(const Line& l, const int16_t* s, int k, double w_) : line(l), stk(s), top(k), e(0), w(w_) {
    je = stk[0];
    ge = line.g(je);
    if (top > 0) {
      jn = stk[LINES];
      gn = line.g(jn);
    }
  }
  __device__ __forceinline__ int at(int x) {
    while (e < top && gn + w * sq((double)(x - jn)) <= ge + w * sq((double)(x - je))) {
      ++e;
      je = jn;
      ge = gn;
      if (e < top) {
        jn = stk[(e + 1) * LINES];
        gn = line.g(jn);
      }
    }
    return je;
  }
};

// axis-1 line (i0, *, i2) of the axis-2 result: g(j) = (s2 (i2 - f2(j)))^2
struct Line1 {
  const int16_t* f;   // f[j * n2]
  int n2, i2;
  double s2;
  __device__ __forceinline__ bool has(int j) const { return f[(long long)j * n2] >= 0; }
  __device__ __forceinline__ double g(int j) const { return sq((double)(i2 - f[(long long)j * n2]) * s2); }
};

__global__ void __launch_bounds__(LINES)
sd_pass1_kernel(const int16_t* __restrict__ fa, short2* __restrict__ fb, Dims d, double s1, double s2) {
  extern __shared__ int16_t stk1[];
  pnp_pdl_enter();
  const int t = blockIdx.z, i0 = blockIdx.y, i2 = blockIdx.x * LINES + threadIdx.x;
  if (i2 >= d.n2) return;
  const long long base = (long long)t * d.N + (long long)i0 * d.L + i2;
  const Line1 line{fa + base, d.n2, i2, s2};
  int16_t* stk = stk1 + threadIdx.x;
  short2* out = fb + base;
  const double w = sq(s1);
  const int k = envelope(line, d.n1, w, stk);
  if (k < 0) {
    for (int x = 0; x < d.n1; ++x) out[(long long)x * d.n2] = make_short2(-1, -1);
    return;
  }
  EnvelopeWalk<Line1> walk(line, stk, k, w);
  for (int x = 0; x < d.n1; ++x) {
    const int j = walk.at(x);
    out[(long long)x * d.n2] = make_short2((short)j, line.f[(long long)j * d.n2]);
  }
}

// axis-0 line (*, i1, i2) of the axis-1 result: g(j) = (s1 (i1 - f1(j)))^2 + (s2 (i2 - f2(j)))^2
struct Line0 {
  const short2* f;    // f[j * L]
  long long L;
  int i1, i2;
  double s1, s2;
  __device__ __forceinline__ bool has(int j) const { return f[j * L].x >= 0; }
  __device__ __forceinline__ double g(int j) const {
    const short2 v = f[j * L];
    return __dadd_rn(sq((double)(i1 - v.x) * s1), sq((double)(i2 - v.y) * s2));
  }
};

// EMIT: also write each query's distance to list[off(g) + i] (line g = t L + l, its i-th query; off(g) = boff[g / SCAN] + loff[g]).
// Emission does not touch sum, count or max, so the partials are those of the EMIT = false instantiation.
constexpr int SCAN = 256;   // lines per block of sd_count_kernel, and per entry of boff

template <bool EMIT>
__global__ void __launch_bounds__(LINES)
sd_pass0_kernel(const short2* __restrict__ fb, const uint8_t* __restrict__ mask, Dims d, int cls, double s0, double s1, double s2,
                double* __restrict__ psum, double* __restrict__ pmax, unsigned* __restrict__ pcnt, double* __restrict__ list,
                const unsigned* __restrict__ loff, const unsigned long long* __restrict__ boff) {
  extern __shared__ int16_t stk0[];
  pnp_pdl_enter();
  const int t = blockIdx.z, i1 = blockIdx.y, i2 = blockIdx.x * LINES + threadIdx.x;
  if (i2 >= d.n2) return;
  const long long l = (long long)i1 * d.n2 + i2;
  const Line0 line{fb + (long long)t * d.N + l, d.L, i1, i2, s1, s2};
  const uint8_t* q = mask + (long long)t * d.N + l;   // queries: the border of the other volume
  const uint8_t bit = (uint8_t)(1u << cls);
  int16_t* stk = stk0 + threadIdx.x;
  const int k = envelope(line, d.n0, sq(s0), stk);
  double sum = 0.0, mx = 0.0;
  unsigned cnt = 0;
  if (k < 0) {                       // no feature in this column means none in the volume: only count the queries
    for (int x = 0; x < d.n0; ++x) cnt += (q[x * d.L] & bit) ? 1u : 0u;
  } else {
    double* slot = nullptr;
    if (EMIT) {
      const long long g = t * d.L + l;
      slot = list + boff[g / SCAN] + loff[g];
    }
    EnvelopeWalk<Line0> walk(line, stk, k, sq(s0));
    for (int x = 0; x < d.n0; ++x) {
      if (!(q[x * d.L] & bit)) continue;
      const int j = walk.at(x);
      const short2 v = line.f[j * d.L];
      const double d0 = (double)(x - j) * s0, d1 = (double)(i1 - v.x) * s1, d2 = (double)(i2 - v.y) * s2;
      const double dist = sqrt(__dadd_rn(__dadd_rn(sq(d0), sq(d1)), sq(d2)));
      if (EMIT) slot[cnt] = dist;
      sum += dist;
      mx = fmax(mx, dist);
      ++cnt;
    }
  }
  psum[t * d.L + l] = sum;
  pmax[t * d.L + l] = mx;
  pcnt[t * d.L + l] = cnt;
}

// one block: the per-line partials of both transforms in a fixed order -> out[6] of the class
__global__ void __launch_bounds__(256)
sd_reduce_kernel(const double* __restrict__ psum, const double* __restrict__ pmax, const unsigned* __restrict__ pcnt, long long L,
                 double* __restrict__ out) {
  __shared__ double ss[256], sm[256];
  __shared__ unsigned long long sc[256];
  pnp_pdl_enter();
  const int tid = threadIdx.x;
  double res[6];
  for (int t = 0; t < 2; ++t) {
    double s = 0.0, m = 0.0;
    unsigned long long c = 0;
    for (long long i = tid; i < L; i += 256) {
      s += psum[t * L + i];
      m = fmax(m, pmax[t * L + i]);
      c += pcnt[t * L + i];
    }
    ss[tid] = s;
    sm[tid] = m;
    sc[tid] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (tid < o) {
        ss[tid] += ss[tid + o];
        sm[tid] = fmax(sm[tid], sm[tid + o]);
        sc[tid] += sc[tid + o];
      }
      __syncthreads();
    }
    res[3 * t] = ss[0];
    res[3 * t + 1] = (double)sc[0];
    res[3 * t + 2] = sm[0];
    __syncthreads();
  }
  if (tid == 0) {
    const bool empty = res[1] == 0.0 || res[4] == 0.0;   // a distance to an empty border is undefined
    for (int i = 0; i < 6; ++i) out[i] = (empty && i % 3 != 1) ? (double)NAN : res[i];
  }
}

// ---- the percentile: slots of the pooled list, radix select ------------------------------------------------------------------
typedef unsigned long long u64;

// exclusive prefix sum across the block (blockDim.x a multiple of 32, at most 1024); `total` gets the block's sum.  sh: 33 slots.
__device__ __forceinline__ u64 block_exclusive_scan(u64 x, u64* sh, u64& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  u64 inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) sh[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const u64 w = lane < nw ? sh[lane] : 0;
    u64 wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u64 y = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += y;
    }
    sh[lane] = wi - w;
    if (lane == 31) sh[32] = wi;
  }
  __syncthreads();
  total = sh[32];
  const u64 r = inc - x + sh[warp];
  __syncthreads();
  return r;
}

// line g = t L + l of the axis-0 pass: its query count, scanned within the block -> loff[g]; the block's total -> boff[block]
__global__ void __launch_bounds__(SCAN)
sd_count_kernel(const uint8_t* __restrict__ mask, Dims d, int cls, unsigned* __restrict__ loff, u64* __restrict__ boff) {
  __shared__ u64 sh[33];
  pnp_pdl_enter();
  const long long g = (long long)blockIdx.x * SCAN + threadIdx.x;
  const uint8_t bit = (uint8_t)(1u << cls);
  unsigned cnt = 0;
  if (g < 2 * d.L) {
    const long long t = g / d.L;
    const uint8_t* q = mask + t * d.N + (g - t * d.L);
    for (int x = 0; x < d.n0; ++x) cnt += (q[x * d.L] & bit) ? 1u : 0u;
  }
  u64 total;
  const u64 ex = block_exclusive_scan(cnt, sh, total);
  if (g < 2 * d.L) loff[g] = (unsigned)ex;
  if (threadIdx.x == 0) boff[blockIdx.x] = total;
}

constexpr int SEL = 256;   // threads per block of the select kernels: one per bucket of an 8-bit digit

struct Select {
  u64 n, lo, hi;           // pooled count (0 when either border is empty), the ranks of the two order statistics
  double gamma;            // interpolation weight v - lo
  u64 key, cnt_le;         // bits of D(lo), #(x <= D(lo))
  u64 above;               // min of the bits above D(lo) (an integer atomicMin)
  u64 prefix[9], rank[9];  // before pass p: the digits picked so far, and the rank sought among the keys that carry them
  u64 hist[8][SEL];        // per pass: keys that carry prefix[p], by digit p
};
static_assert(sizeof(Select) == 16584, "the workspace formula of include/pnp_b200.h counts A(16584) bytes for the select state");

// one block: the exclusive prefix sums of sd_count_kernel's block totals, in place, so that off(g) = boff[g / SCAN] + loff[g]; the pooled
// count n, |dA| = off(L) and the ranks and weight of numpy.percentile's `linear` method: v = (n - 1) qf, lo = floor(v) and
// hi = lo + 1 (both n - 1 when v >= n - 1), gamma = v - lo.  Clears the histograms.
__global__ void __launch_bounds__(1024)
sd_scan_kernel(const unsigned* __restrict__ loff, u64* __restrict__ boff, long long L, double qf, Select* __restrict__ s) {
  __shared__ u64 sh[33];
  pnp_pdl_enter();
  const long long nb = (2 * L + SCAN - 1) / SCAN;
  u64 run = 0;
  for (long long b0 = 0; b0 < nb; b0 += 1024) {
    const long long i = b0 + threadIdx.x;
    u64 total;
    const u64 ex = block_exclusive_scan(i < nb ? boff[i] : 0, sh, total);
    if (i < nb) boff[i] = run + ex;
    run += total;
  }
  for (int i = threadIdx.x; i < 8 * SEL; i += 1024) s->hist[i / SEL][i % SEL] = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    const u64 na = boff[L / SCAN] + loff[L], n = (na > 0 && run > na) ? run : 0;
    u64 lo = 0, hi = 0;
    double gamma = 0.0;
    if (n) {
      const double last = (double)(n - 1);
      const double v = __dmul_rn(last, qf);
      if (v >= last) {
        lo = hi = n - 1;
      } else {
        lo = (u64)floor(v);
        hi = lo + 1;
      }
      gamma = __dsub_rn(v, (double)lo);
    }
    s->n = n;
    s->lo = lo;
    s->hi = hi;
    s->gamma = gamma;
    s->above = ~0ull;
    s->prefix[0] = 0;
    s->rank[0] = lo;
  }
}

// the bucket of pass p that holds rank s->rank[p] -> (digits picked so far including it, rank within it, its size), in every
// thread of a SEL-thread block.  sh: 36 slots.
__device__ __forceinline__ void pick(const Select* s, int p, u64* sh, u64& prefix, u64& rank, u64& size) {
  const u64 c = s->hist[p][threadIdx.x], r = s->rank[p];
  u64 total;
  const u64 ex = block_exclusive_scan(c, sh, total);
  if (ex <= r && r < ex + c) {
    sh[33] = s->prefix[p] | ((u64)threadIdx.x << (56 - 8 * p));
    sh[34] = r - ex;
    sh[35] = c;
  }
  __syncthreads();
  prefix = sh[33];
  rank = sh[34];
  size = sh[35];
}

__device__ __forceinline__ u64 key_of(double x) { return (u64)__double_as_longlong(x); }

// pass p: picks the digit of pass p - 1 (every block alike; block 0 records it), then histograms digit p (bits 56 - 8p ..
// 63 - 8p) of the keys that carry the digits picked so far
__global__ void __launch_bounds__(SEL)
sd_hist_kernel(const double* __restrict__ list, Select* __restrict__ s, int p) {
  __shared__ unsigned h[SEL];
  __shared__ u64 sh[36];
  pnp_pdl_enter();
  const u64 n = s->n;
  if (n == 0) return;
  u64 prefix = 0;
  if (p > 0) {
    u64 rank, size;
    pick(s, p - 1, sh, prefix, rank, size);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      s->prefix[p] = prefix;
      s->rank[p] = rank;
    }
  }
  h[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 56 - 8 * p;
  const u64 high = p ? ~0ull << (shift + 8) : 0ull;
  for (u64 i = (u64)blockIdx.x * SEL + threadIdx.x; i < n; i += (u64)gridDim.x * SEL) {
    const u64 k = key_of(list[i]);
    if (((k ^ prefix) & high) == 0) atomicAdd(&h[(k >> shift) & 255], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&s->hist[p][threadIdx.x], (u64)h[threadIdx.x]);
}

// picks the last digit: D(lo) exactly and #(x <= D(lo)).  D(hi) = D(lo) when hi = lo or #(x <= D(lo)) >= hi + 1, else the
// smallest key above D(lo), which this kernel finds.
__global__ void __launch_bounds__(SEL)
sd_above_kernel(const double* __restrict__ list, Select* __restrict__ s) {
  __shared__ u64 sh[36];
  pnp_pdl_enter();
  const u64 n = s->n;
  if (n == 0) return;
  u64 key, rank, size;
  pick(s, 7, sh, key, rank, size);
  const u64 lo = s->lo, hi = s->hi, cnt_le = lo - rank + size;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    s->key = key;
    s->cnt_le = cnt_le;
  }
  if (hi == lo || cnt_le >= hi + 1) return;
  u64 m = ~0ull;
  for (u64 i = (u64)blockIdx.x * SEL + threadIdx.x; i < n; i += (u64)gridDim.x * SEL) {
    const u64 k = key_of(list[i]);
    if (k > key && k < m) m = k;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = min(m, (u64)__shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m != ~0ull) atomicMin(&s->above, m);
}

// one thread: numpy's _lerp of the two order statistics, each product and sum rounded on its own -> out[0] (NaN: empty border)
__global__ void __launch_bounds__(32)
sd_pct_kernel(const Select* __restrict__ s, double* __restrict__ out) {
  pnp_pdl_enter();
  if (threadIdx.x) return;
  if (s->n == 0) {
    out[0] = (double)NAN;
    return;
  }
  const double a = __longlong_as_double((long long)s->key);
  const double b = (s->hi == s->lo || s->cnt_le >= s->hi + 1) ? a : __longlong_as_double((long long)s->above);
  const double delta = __dsub_rn(b, a), g = s->gamma;
  out[0] = g >= 0.5 ? __dsub_rn(b, __dmul_rn(delta, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(delta, g));
}

inline long long align256(long long b) { return (b + 255) & ~255LL; }

struct Workspace {
  uint8_t* mask;
  int16_t* fa;
  short2* fb;
  double *psum, *pmax;
  unsigned* pcnt;
  double* list;     // the percentile's: pooled distances of one class
  unsigned* loff;   //   per-line slot offsets within their SCAN block
  u64* boff;        //   per SCAN block of lines: the first slot
  Select* sel;
};

// layout of the workspace; returns its size in bytes (ws == nullptr: size only).  The percentile's buffers follow the others.
long long carve(void* ws, long long N, long long L, bool pct, Workspace* w) {
  long long off = 0;
  char* base = (char*)ws;
  auto take = [&](long long bytes) -> char* {
    char* p = base ? base + off : nullptr;
    off += align256(bytes);
    return p;
  };
  w->mask = (uint8_t*)take(2 * N);
  w->fa = (int16_t*)take(2 * N * (long long)sizeof(int16_t));
  w->fb = (short2*)take(2 * N * (long long)sizeof(short2));
  w->psum = (double*)take(2 * L * (long long)sizeof(double));
  w->pmax = (double*)take(2 * L * (long long)sizeof(double));
  w->pcnt = (unsigned*)take(2 * L * (long long)sizeof(unsigned));
  w->list = nullptr;
  w->loff = nullptr;
  w->boff = nullptr;
  w->sel = nullptr;
  if (pct) {
    w->list = (double*)take(2 * N * (long long)sizeof(double));
    w->loff = (unsigned*)take(2 * L * (long long)sizeof(unsigned));
    w->boff = (u64*)take((2 * L + SCAN - 1) / SCAN * (long long)sizeof(u64));
    w->sel = (Select*)take((long long)sizeof(Select));
  }
  return off;
}

int check_shape(int n0, int n1, int n2, int C) {
  if (n0 <= 0 || n1 <= 0 || n2 <= 0) return PNP_ERR_BAD_ARG;
  if (C < 2 || C > 8 || n0 > PNP_SD_MAX_DIM || n1 > PNP_SD_MAX_DIM || n2 > PNP_SD_MAX_DIM) return PNP_ERR_UNSUPPORTED;
  return PNP_OK;
}

template <typename K>
cudaError_t allow_smem(K kernel, size_t bytes) {
  return bytes > 48 * 1024 ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) : cudaSuccess;
}

int workspace_bytes(int n0, int n1, int n2, int C, bool pct, long long* bytes) {
  if (!bytes) return PNP_ERR_BAD_ARG;
  const int rc = check_shape(n0, n1, n2, C);
  if (rc) return rc;
  Workspace w;
  *bytes = carve(nullptr, (long long)n0 * n1 * n2, (long long)n1 * n2, pct, &w);
  return PNP_OK;
}

// both entry points: q == nullptr gives out[C-1][6]; a percentile q gives out[C-1][7], column 6 = HD_q
int surface_distance(const uint8_t* pred, const uint8_t* gt, int n0, int n1, int n2, int C, const double* spacing, const double* q,
                     void* ws, long long ws_bytes, double* out, void* stream) {
  if (!pred || !gt || !ws || !out) return PNP_ERR_BAD_ARG;
  const int rc = check_shape(n0, n1, n2, C);
  if (rc) return rc;
  double s[3] = {1.0, 1.0, 1.0};
  if (spacing)
    for (int a = 0; a < 3; ++a) {
      if (!(spacing[a] > 0.0) || !isfinite(spacing[a])) return PNP_ERR_BAD_ARG;
      s[a] = spacing[a];
    }
  if (q && !(*q >= 0.0 && *q <= 100.0)) return PNP_ERR_BAD_ARG;   // NaN and infinities fail too
  const bool pct = q != nullptr;
  const int cols = pct ? 7 : 6;
  Dims d{n0, n1, n2, (long long)n0 * n1 * n2, (long long)n1 * n2};
  Workspace w;
  if (ws_bytes < carve(nullptr, d.N, d.L, pct, &w)) return PNP_ERR_BAD_ARG;
  carve(ws, d.N, d.L, pct, &w);
  cudaStream_t st = (cudaStream_t)stream;

  const long long nb = (d.N + 255) / 256;
  PNP_CUDA(pnp_launch(sd_border_kernel, dim3((unsigned)(nb < PNP_NUM_SMS * 16LL ? nb : PNP_NUM_SMS * 16LL), 2), dim3(256), 0, st,
                      pred, gt, w.mask, d, C));
  const int stride = ((n2 + 3) & ~3) + 2;
  const size_t smem2 = (size_t)ROWS * stride * sizeof(int16_t);
  const size_t smem1 = (size_t)n1 * LINES * sizeof(int16_t), smem0 = (size_t)n0 * LINES * sizeof(int16_t);
  PNP_CUDA(allow_smem(sd_pass2_kernel, smem2));
  PNP_CUDA(allow_smem(sd_pass1_kernel, smem1));
  PNP_CUDA(allow_smem(pct ? sd_pass0_kernel<true> : sd_pass0_kernel<false>, smem0));
  const unsigned gl = (unsigned)pnp_cdiv(n2, LINES);
  const unsigned gcount = (unsigned)pnp_cdiv(2 * d.L, SCAN);
  const long long sel_blocks = pnp_cdiv(2 * d.N, SEL);
  const unsigned gsel = (unsigned)(sel_blocks < PNP_NUM_SMS * 2LL ? sel_blocks : PNP_NUM_SMS * 2LL);
  for (int c = 1; c < C; ++c) {
    double* oc = out + (long long)(c - 1) * cols;
    if (pct) {
      PNP_CUDA(pnp_launch(sd_count_kernel, dim3(gcount), dim3(SCAN), 0, st, (const uint8_t*)w.mask, d, c, w.loff, w.boff));
      PNP_CUDA(pnp_launch(sd_scan_kernel, dim3(1), dim3(1024), 0, st, (const unsigned*)w.loff, w.boff, d.L, *q / 100.0, w.sel));
    }
    PNP_CUDA(pnp_launch(sd_pass2_kernel, dim3((unsigned)pnp_cdiv((long long)n0 * n1, ROWS), 2), dim3(ROWS), smem2, st,
                        (const uint8_t*)w.mask, w.fa, d, c, stride));
    PNP_CUDA(pnp_launch(sd_pass1_kernel, dim3(gl, n0, 2), dim3(LINES), smem1, st, (const int16_t*)w.fa, w.fb, d, s[1], s[2]));
    PNP_CUDA(pnp_launch(pct ? sd_pass0_kernel<true> : sd_pass0_kernel<false>, dim3(gl, n1, 2), dim3(LINES), smem0, st,
                        (const short2*)w.fb, (const uint8_t*)w.mask, d, c, s[0], s[1], s[2], w.psum, w.pmax, w.pcnt, w.list,
                        (const unsigned*)w.loff, (const u64*)w.boff));
    PNP_CUDA(pnp_launch(sd_reduce_kernel, dim3(1), dim3(256), 0, st, (const double*)w.psum, (const double*)w.pmax,
                        (const unsigned*)w.pcnt, d.L, oc));
    if (pct) {
      for (int p = 0; p < 8; ++p)
        PNP_CUDA(pnp_launch(sd_hist_kernel, dim3(gsel), dim3(SEL), 0, st, (const double*)w.list, w.sel, p));
      PNP_CUDA(pnp_launch(sd_above_kernel, dim3(gsel), dim3(SEL), 0, st, (const double*)w.list, w.sel));
      PNP_CUDA(pnp_launch(sd_pct_kernel, dim3(1), dim3(32), 0, st, (const Select*)w.sel, oc + 6));
    }
  }
  return PNP_OK;
}

}  // namespace

extern "C" int pnp_surface_distance_workspace(int n0, int n1, int n2, int C, long long* bytes) {
  return workspace_bytes(n0, n1, n2, C, false, bytes);
}

extern "C" int pnp_surface_distance(const uint8_t* pred, const uint8_t* gt, int n0, int n1, int n2, int C, const double* spacing,
                                    void* ws, long long ws_bytes, double* out, void* stream) {
  return surface_distance(pred, gt, n0, n1, n2, C, spacing, nullptr, ws, ws_bytes, out, stream);
}

extern "C" int pnp_surface_distance_pct_workspace(int n0, int n1, int n2, int C, long long* bytes) {
  return workspace_bytes(n0, n1, n2, C, true, bytes);
}

extern "C" int pnp_surface_distance_pct(const uint8_t* pred, const uint8_t* gt, int n0, int n1, int n2, int C, const double* spacing,
                                        double q, void* ws, long long ws_bytes, double* out, void* stream) {
  return surface_distance(pred, gt, n0, n1, n2, C, spacing, &q, ws, ws_bytes, out, stream);
}
