// General fp32 SIMT implicit-GEMM convolution family for sm_90a.
//
// Replaces tf.nn.conv2d / tf.nn.atrous_conv2d and their gradients as instantiated by the reference's
// layers.py:18,24,67,73,86,92.  This is the *general* path: any kernel size, stride, dilation,
// zero-pad offsets and channel counts (Cin = 3, 5, 40 ..., Cout = 5 ...).  The dense stride-1
// Cin%64==0 layers that carry ~85% of the FLOPs go through the wgmma path in conv_tc.cu; the
// layers that stay here are the HBM-leaning small-channel ones plus (for now) every wgrad.
//
//   fwd   : y[m, n]  = sum_k A(m,k) * Wmat[k, n]         m=(b,oy,ox)  k=(ky,kx,ci)  n=co
//   dgrad : dx[m, n] = sum_k A'(m,k) * WTmat[k, n]       m=(b,iy,ix)  k=(ky,kx,co)  n=ci
//           (A' gathers dy with the transposed coordinate rule, predicated on stride divisibility)
//   wgrad : dW[kk, n] += sum_m A(m,kk) * dy[m, n]        split over m across CTAs, fp32 atomics
#include "common.cuh"
#include "../../include/pnp_b200.h"

namespace {

struct GatherArgs {
  int B, IH, IW, IC;   // tensor being gathered from
  int OH, OW, OC;      // tensor being produced
  int kh, kw, stride, dil, pad_t, pad_l;
  int M;               // B*OH*OW
  int K;               // kh*kw*IC
  int accumulate;
  int phase_rows;      // TRANSPOSED, stride s > 1: rows are ordered phase-major ((oy % s, ox % s) outermost, phase_rows rows each,
                       // a multiple of BM) so that every CTA owns ONE phase and skips the k-blocks of taps that cannot reach it
  PnpDropout drop;
};

__device__ __forceinline__ int row_index(int i, int t, int T, int BT) {
  // thread t's i-th row (or column) inside a block tile of extent BT with per-thread extent T.
  // T == 8 is split in two groups of 4 that sit BT/2 apart so 128-bit shared loads are conflict free.
  if (T == 8) return (i < 4) ? (t * 4 + i) : (BT / 2 + t * 4 + (i - 4));
  return t * T + i;
}

template <int BM, int BN, int BK, int TM, int TN, int VEC, bool TRANSPOSED>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_gather_kernel(const float* __restrict__ in, const float* __restrict__ wmat, float* __restrict__ out, GatherArgs a) {
  pnp_pdl_enter();
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int KCH = BK / VEC;                                   // k-chunks per row
  constexpr int ROWS_PT = (BM >= NT) ? (BM / NT) : 1;             // rows per thread (A loader)
  constexpr int THR_PR = (BM >= NT) ? 1 : (NT / BM);              // threads per row
  constexpr int CH_PT = KCH / THR_PR;                             // k-chunks per thread per row
  static_assert(KCH % THR_PR == 0, "bad A loader split");
  constexpr int B_VEC_TOTAL = BK * BN / 4;
  constexpr int B_ITERS = (B_VEC_TOTAL + NT - 1) / NT;

  __shared__ __align__(16) float As[BK][BM];
  __shared__ __align__(16) float Bs[BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN);
  const int ty = tid / (BN / TN);
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- per-thread A-loader row bookkeeping ----
  int r_row[ROWS_PT];
  int r_y[ROWS_PT], r_x[ROWS_PT];
  long long r_base[ROWS_PT];
  bool r_ok[ROWS_PT];
  const int kc0 = (BM >= NT) ? 0 : (tid / BM);
#pragma unroll
  for (int j = 0; j < ROWS_PT; ++j) {
    int row = (BM >= NT) ? (tid + j * NT) : (tid % BM);
    r_row[j] = row;
    int m = m0 + row;
    r_ok[j] = m < a.M;
    int mm = r_ok[j] ? m : 0;
    int b, oy, ox;
    if (TRANSPOSED && a.phase_rows > 0) {
      const int p = mm / a.phase_rows, r = mm - p * a.phase_rows;
      const int PH = a.OH / a.stride, PW = a.OW / a.stride;
      b = r / (PH * PW);
      const int rem = r - b * (PH * PW);
      const int yy = rem / PW;
      oy = yy * a.stride + p / a.stride;
      ox = (rem - yy * PW) * a.stride + p % a.stride;
    } else {
      b = mm / (a.OH * a.OW);
      const int rem = mm - b * (a.OH * a.OW);
      oy = rem / a.OW;
      ox = rem - oy * a.OW;
    }
    if (TRANSPOSED) {
      r_y[j] = oy + a.pad_t;
      r_x[j] = ox + a.pad_l;
    } else {
      r_y[j] = oy * a.stride - a.pad_t;
      r_x[j] = ox * a.stride - a.pad_l;
    }
    r_base[j] = (long long)b * a.IH * a.IW * a.IC;
  }

  float a_reg[ROWS_PT][CH_PT][VEC];
  float4 b_reg[B_ITERS];

  const bool b_vec_ok = (a.OC % 4) == 0;

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int j = 0; j < ROWS_PT; ++j) {
#pragma unroll
      for (int c = 0; c < CH_PT; ++c) {
        int kc = kc0 + c * THR_PR;
        int k = k0 + kc * VEC;
        bool ok = r_ok[j] && (k < a.K);
        int tap = k / a.IC;
        int ci = k - tap * a.IC;
        int ky = tap / a.kw;
        int kx = tap - ky * a.kw;
        int iy, ix;
        if (TRANSPOSED) {
          int ty_ = r_y[j] - ky * a.dil;
          int tx_ = r_x[j] - kx * a.dil;
          iy = ty_ / a.stride;
          ix = tx_ / a.stride;
          ok = ok && ty_ >= 0 && tx_ >= 0 && (iy * a.stride == ty_) && (ix * a.stride == tx_);
        } else {
          iy = r_y[j] + ky * a.dil;
          ix = r_x[j] + kx * a.dil;
          ok = ok && iy >= 0 && ix >= 0;
        }
        ok = ok && iy < a.IH && ix < a.IW;
        if (VEC == 4) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok) v = __ldg(reinterpret_cast<const float4*>(in + r_base[j] + ((long long)iy * a.IW + ix) * a.IC + ci));
          a_reg[j][c][0] = v.x;
          a_reg[j][c][VEC > 1 ? 1 : 0] = v.y;
          a_reg[j][c][VEC > 2 ? 2 : 0] = v.z;
          a_reg[j][c][VEC > 3 ? 3 : 0] = v.w;
        } else {
          a_reg[j][c][0] = ok ? __ldg(in + r_base[j] + ((long long)iy * a.IW + ix) * a.IC + ci) : 0.f;
        }
      }
    }
#pragma unroll
    for (int it = 0; it < B_ITERS; ++it) {
      int p = tid + it * NT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p < B_VEC_TOTAL) {
        int kr = p / (BN / 4);
        int nc = (p - kr * (BN / 4)) * 4;
        int k = k0 + kr;
        int n = n0 + nc;
        if (k < a.K) {
          const float* src = wmat + (long long)k * a.OC + n;
          if (b_vec_ok && n + 3 < a.OC) {
            v = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            if (n + 0 < a.OC) v.x = __ldg(src + 0);
            if (n + 1 < a.OC) v.y = __ldg(src + 1);
            if (n + 2 < a.OC) v.z = __ldg(src + 2);
            if (n + 3 < a.OC) v.w = __ldg(src + 3);
          }
        }
      }
      b_reg[it] = v;
    }
  };

  auto store_tiles = [&]() {
#pragma unroll
    for (int j = 0; j < ROWS_PT; ++j)
#pragma unroll
      for (int c = 0; c < CH_PT; ++c) {
        int kc = kc0 + c * THR_PR;
#pragma unroll
        for (int e = 0; e < VEC; ++e) As[kc * VEC + e][r_row[j]] = a_reg[j][c][e];
      }
#pragma unroll
    for (int it = 0; it < B_ITERS; ++it) {
      int p = tid + it * NT;
      if (p < B_VEC_TOTAL) {
        int kr = p / (BN / 4);
        int nc = (p - kr * (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[kr][nc]) = b_reg[it];
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nkb = (a.K + BK - 1) / BK;
  // phase-major strided data gradient: a k-block (BK channels of one tap, IC % BK == 0) contributes to this CTA's phase only
  // if the tap offset is congruent to the phase modulo the stride -- 1 block in s*s for a dense tap grid
  const bool phased = TRANSPOSED && a.phase_rows > 0;
  const int cta_p = phased ? (m0 / a.phase_rows) : 0;
  const int cta_py = phased ? cta_p / a.stride : 0, cta_px = phased ? cta_p % a.stride : 0;
  auto next_kb = [&](int kb) {
    if (!phased) return kb;
    for (; kb < nkb; ++kb) {
      const int tap = (kb * BK) / a.IC;
      const int ky = tap / a.kw, kx = tap - ky * a.kw;
      if ((cta_py + a.pad_t - ky * a.dil) % a.stride == 0 && (cta_px + a.pad_l - kx * a.dil) % a.stride == 0) break;
    }
    return kb;
  };
  int kb_cur = next_kb(0);
  if (kb_cur < nkb) {
    load_tiles(kb_cur * BK);
    store_tiles();
  }
  __syncthreads();
  while (kb_cur < nkb) {
    const int kb_nxt = next_kb(kb_cur + 1);
    const bool more = kb_nxt < nkb;
    kb_cur = kb_nxt;
    if (more) load_tiles(kb_nxt * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float av[TM], bv[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 t4 = *reinterpret_cast<const float4*>(&As[k][row_index(i, ty, TM, BM)]);
        av[i] = t4.x; av[i + 1] = t4.y; av[i + 2] = t4.z; av[i + 3] = t4.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 t4 = *reinterpret_cast<const float4*>(&Bs[k][row_index(j, tx, TN, BN)]);
        bv[j] = t4.x; bv[j + 1] = t4.y; bv[j + 2] = t4.z; bv[j + 3] = t4.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (more) {
      store_tiles();
      __syncthreads();
    }
  }

  // ---- epilogue ----
  const bool drop_on = a.drop.seed_ptr != nullptr;
  unsigned long long seed = 0ull;
  if (drop_on) seed = *a.drop.seed_ptr;
  const bool vec_store = (a.OC % 4) == 0;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + row_index(i, ty, TM, BM);
    if (m >= a.M) continue;
    long long mlin = m;
    if (TRANSPOSED && a.phase_rows > 0) {
      const int p = m / a.phase_rows, r = m - p * a.phase_rows;
      const int PH = a.OH / a.stride, PW = a.OW / a.stride;
      const int b = r / (PH * PW);
      const int rem = r - b * (PH * PW);
      const int yy = rem / PW;
      mlin = ((long long)b * a.OH + yy * a.stride + p / a.stride) * a.OW + (rem - yy * PW) * a.stride + p % a.stride;
    }
#pragma unroll
    for (int j = 0; j < TN; j += 4) {
      int n = n0 + row_index(j, tx, TN, BN);
      if (n >= a.OC) continue;
      long long idx = mlin * a.OC + n;
      float4 v = make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
      if (vec_store && n + 3 < a.OC) {
        if (drop_on) {
          float4 mu = pnp_dropout_mult4(a.drop, seed, (unsigned long long)idx >> 2);
          v.x *= mu.x; v.y *= mu.y; v.z *= mu.z; v.w *= mu.w;
        }
        float4* dst = reinterpret_cast<float4*>(out + idx);
        if (a.accumulate) {
          float4 o = *dst;
          v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
        }
        *dst = v;
      } else {
        float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (n + e < a.OC) {
            float val = vv[e];
            if (drop_on) val *= pnp_dropout_mult1(a.drop, seed, (unsigned long long)(idx + e));
            if (a.accumulate) val += out[idx + e];
            out[idx + e] = val;
          }
        }
      }
    }
  }
}

template <int BM, int BN, int BK, int TM, int TN, int VEC, bool TR>
int launch_gather(const float* in, const float* wmat, float* out, const GatherArgs& a0, cudaStream_t s) {
  GatherArgs a = a0;
  a.phase_rows = 0;
  if (TR && a.stride > 1 && a.OH % a.stride == 0 && a.OW % a.stride == 0 && a.IC % BK == 0) {
    const long long pr = (long long)(a.M / (a.OH * a.OW)) * (a.OH / a.stride) * (a.OW / a.stride);
    if (pr % BM == 0 && pr <= 0x7fffffffLL) a.phase_rows = (int)pr;
  }
  dim3 grid(pnp_cdiv(a.M, BM), pnp_cdiv(a.OC, BN));
  dim3 block((BM / TM) * (BN / TN));
  pnp_launch(conv_gather_kernel<BM, BN, BK, TM, TN, VEC, TR>, grid, block, 0, s, in, wmat, out, a);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

template <bool TR>
int dispatch_gather(const float* in, const float* wmat, float* out, const GatherArgs& a, cudaStream_t s) {
  const bool vec = (a.IC % 4) == 0;
  if (!vec) {  // Cin in {3,5}: tiny-K scalar gather
    if (a.OC <= 8) return launch_gather<1024, 8, 8, 4, 8, 1, TR>(in, wmat, out, a, s);
    if (a.OC <= 16) return launch_gather<256, 16, 16, 4, 4, 1, TR>(in, wmat, out, a, s);
    return launch_gather<128, 64, 16, 8, 4, 1, TR>(in, wmat, out, a, s);
  }
  const bool k16 = (a.IC % 16) == 0;
  if (a.OC <= 8) return launch_gather<1024, 8, 8, 4, 8, 4, TR>(in, wmat, out, a, s);
  if (a.OC <= 16) {
    if (k16) return launch_gather<256, 16, 16, 4, 4, 4, TR>(in, wmat, out, a, s);
    return launch_gather<256, 16, 8, 4, 4, 4, TR>(in, wmat, out, a, s);
  }
  if (a.OC <= 32) {
    if (k16) return launch_gather<256, 32, 16, 8, 4, 4, TR>(in, wmat, out, a, s);
    return launch_gather<256, 32, 8, 8, 4, 4, TR>(in, wmat, out, a, s);
  }
  // grid fill heuristic: prefer the 128x128 tile only when it still yields >= 2 waves
  long long tiles128 = (long long)pnp_cdiv(a.M, 128) * pnp_cdiv(a.OC, 128);
  if (a.OC <= 64 || tiles128 < 2 * PNP_NUM_SMS) {
    if (k16) return launch_gather<128, 64, 16, 8, 4, 4, TR>(in, wmat, out, a, s);
    return launch_gather<128, 64, 8, 8, 4, 4, TR>(in, wmat, out, a, s);
  }
  if (k16) return launch_gather<128, 128, 16, 8, 8, 4, TR>(in, wmat, out, a, s);
  return launch_gather<128, 128, 8, 8, 8, 4, TR>(in, wmat, out, a, s);
}

// ------------------------------------------------------------------------------------------------
// direct convolution for very few output channels (the 5x5 40 -> 5 "output" conv on the 256x256 map,
// source_segmenter.py:206 / adversarial.py:315): an implicit GEMM would waste most of an N tile.  One CTA = 32x32 output
// pixels, 256 threads = 32 (x) x 8 (y), 4 rows per thread; 8-channel slabs of the haloed input tile and of the weights are
// staged in shared memory ([c][y][x], x fastest => conflict-free reads, weights broadcast).
// ------------------------------------------------------------------------------------------------
template <int NO>
__global__ void __launch_bounds__(256)
conv_few_out_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ y, int B, int H, int W, int Cin,
                    int Ho, int Wo, int kh, int kw, int pad_t, int pad_l) {
  pnp_pdl_enter();
  constexpr int T = 32, CC = 8, HALO = T + 4;            // kernels up to 5x5
  __shared__ float s_x[CC][HALO][HALO + 1];
  __shared__ float s_w[25][CC][NO];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * T, y0 = blockIdx.y * T, b = blockIdx.z;
  const int hh = T + kh - 1, hw = T + kw - 1;
  float acc[4][NO];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int o = 0; o < NO; ++o) acc[j][o] = 0.f;
  const float* xb = x + (long long)b * H * W * Cin;
  for (int c0 = 0; c0 < Cin; c0 += CC) {
    __syncthreads();
    for (int p = threadIdx.x; p < hh * hw * 2; p += 256) {
      const int half = p & 1, pix = p >> 1;
      const int py = pix / hw, px = pix - py * hw;
      const int iy = y0 + py - pad_t, ix = x0 + px - pad_l;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(reinterpret_cast<const float4*>(xb + ((long long)iy * W + ix) * Cin + c0 + half * 4));
      s_x[half * 4 + 0][py][px] = v.x; s_x[half * 4 + 1][py][px] = v.y;
      s_x[half * 4 + 2][py][px] = v.z; s_x[half * 4 + 3][py][px] = v.w;
    }
    for (int p = threadIdx.x; p < kh * kw * CC * NO; p += 256) {
      const int o = p % NO, c = (p / NO) % CC, t = p / (NO * CC);
      s_w[t][c][o] = __ldg(w + ((long long)t * Cin + c0 + c) * NO + o);
    }
    __syncthreads();
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx) {
        const int t = ky * kw + kx;
#pragma unroll
        for (int c = 0; c < CC; ++c) {
          float wv[NO];
#pragma unroll
          for (int o = 0; o < NO; ++o) wv[o] = s_w[t][c][o];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float a = s_x[c][ty + 8 * j + ky][tx + kx];
#pragma unroll
            for (int o = 0; o < NO; ++o) acc[j][o] = fmaf(a, wv[o], acc[j][o]);
          }
        }
      }
  }
  const int ox = x0 + tx;
  if (ox < Wo) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int oy = y0 + ty + 8 * j;
      if (oy < Ho) {
        float* dst = y + (((long long)b * Ho + oy) * Wo + ox) * NO;
#pragma unroll
        for (int o = 0; o < NO; ++o) dst[o] = acc[j][o];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// wgrad
// ------------------------------------------------------------------------------------------------
struct WgradArgs {
  int B, H, W, Cin, Ho, Wo, Cout;
  int kh, kw, stride, dil, pad_t, pad_l;
  int M;    // B*Ho*Wo
  int KK;   // kh*kw*Cin
  int m_per_split;
};

template <int BKK, int BN, int BR, int TK, int TN, int VEC>
__global__ void __launch_bounds__((BKK / TK) * (BN / TN))
conv_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dw, WgradArgs a) {
  pnp_pdl_enter();
  constexpr int NT = (BKK / TK) * (BN / TN);
  constexpr int KCH = BKK / VEC;                 // kk chunks per pixel row
  constexpr int A_TOTAL = BR * KCH;
  constexpr int A_ITERS = (A_TOTAL + NT - 1) / NT;
  constexpr int B_TOTAL = BR * BN / 4;
  constexpr int B_ITERS = (B_TOTAL + NT - 1) / NT;

  __shared__ __align__(16) float As[BR][BKK];
  __shared__ __align__(16) float Bs[BR][BN];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN);
  const int ty = tid / (BN / TN);
  const int kk0 = blockIdx.x * BKK;
  const int n0 = blockIdx.y * BN;
  const int m_begin = blockIdx.z * a.m_per_split;
  const int m_end = min(a.M, m_begin + a.m_per_split);

  // A loader: element p -> (r = p / KCH, chunk = p % KCH): kk fixed per (thread, iter) => decode once
  int a_r[A_ITERS], a_kc[A_ITERS], a_dy[A_ITERS], a_dx[A_ITERS], a_ci[A_ITERS];
  bool a_ok[A_ITERS];
#pragma unroll
  for (int it = 0; it < A_ITERS; ++it) {
    int p = tid + it * NT;
    int r = p / KCH;
    int kc = p - r * KCH;
    int kk = kk0 + kc * VEC;
    a_r[it] = r;
    a_kc[it] = kc;
    a_ok[it] = (p < A_TOTAL) && (kk < a.KK);
    int kks = a_ok[it] ? kk : 0;
    int tap = kks / a.Cin;
    a_ci[it] = kks - tap * a.Cin;
    int ky = tap / a.kw;
    int kx = tap - ky * a.kw;
    a_dy[it] = ky * a.dil - a.pad_t;
    a_dx[it] = kx * a.dil - a.pad_l;
  }
  const bool b_vec_ok = (a.Cout % 4) == 0;

  float a_reg[A_ITERS][VEC];
  float4 b_reg[B_ITERS];

  auto load_tiles = [&](int mb) {
#pragma unroll
    for (int it = 0; it < A_ITERS; ++it) {
      int m = mb + a_r[it];
      bool ok = a_ok[it] && m < m_end;
      int mm = ok ? m : 0;
      int b = mm / (a.Ho * a.Wo);
      int rem = mm - b * (a.Ho * a.Wo);
      int oy = rem / a.Wo;
      int ox = rem - oy * a.Wo;
      int iy = oy * a.stride + a_dy[it];
      int ix = ox * a.stride + a_dx[it];
      ok = ok && iy >= 0 && ix >= 0 && iy < a.H && ix < a.W;
      const float* src = x + (((long long)b * a.H + iy) * a.W + ix) * a.Cin + a_ci[it];
      if (VEC == 4) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok) v = __ldg(reinterpret_cast<const float4*>(src));
        a_reg[it][0] = v.x;
        a_reg[it][VEC > 1 ? 1 : 0] = v.y;
        a_reg[it][VEC > 2 ? 2 : 0] = v.z;
        a_reg[it][VEC > 3 ? 3 : 0] = v.w;
      } else {
        a_reg[it][0] = ok ? __ldg(src) : 0.f;
      }
    }
#pragma unroll
    for (int it = 0; it < B_ITERS; ++it) {
      int p = tid + it * NT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p < B_TOTAL) {
        int r = p / (BN / 4);
        int nc = (p - r * (BN / 4)) * 4;
        int m = mb + r;
        int n = n0 + nc;
        if (m < m_end) {
          const float* src = dy + (long long)m * a.Cout + n;
          if (b_vec_ok && n + 3 < a.Cout) {
            v = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            if (n + 0 < a.Cout) v.x = __ldg(src + 0);
            if (n + 1 < a.Cout) v.y = __ldg(src + 1);
            if (n + 2 < a.Cout) v.z = __ldg(src + 2);
            if (n + 3 < a.Cout) v.w = __ldg(src + 3);
          }
        }
      }
      b_reg[it] = v;
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int it = 0; it < A_ITERS; ++it) {
      int p = tid + it * NT;
      if (p < A_TOTAL) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) As[a_r[it]][a_kc[it] * VEC + e] = a_reg[it][e];
      }
    }
#pragma unroll
    for (int it = 0; it < B_ITERS; ++it) {
      int p = tid + it * NT;
      if (p < B_TOTAL) {
        int r = p / (BN / 4);
        int nc = (p - r * (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[r][nc]) = b_reg[it];
      }
    }
  };

  float acc[TK][TN];
#pragma unroll
  for (int i = 0; i < TK; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  if (m_begin < m_end) {
    load_tiles(m_begin);
    store_tiles();
    __syncthreads();
    for (int mb = m_begin; mb < m_end; mb += BR) {
      bool more = mb + BR < m_end;
      if (more) load_tiles(mb + BR);
#pragma unroll
      for (int r = 0; r < BR; ++r) {
        float av[TK], bv[TN];
#pragma unroll
        for (int i = 0; i < TK; ++i) av[i] = As[r][ty * TK + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) bv[j] = Bs[r][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TK; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
      if (more) {
        store_tiles();
        __syncthreads();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < TK; ++i) {
    int kk = kk0 + ty * TK + i;
    if (kk >= a.KK) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n < a.Cout) atomicAdd(dw + (long long)kk * a.Cout + n, acc[i][j]);
    }
  }
}

template <int BKK, int BN, int BR, int TK, int TN, int VEC>
int launch_wgrad(const float* x, const float* dy, float* dw, WgradArgs a, cudaStream_t s) {
  int tiles = pnp_cdiv(a.KK, BKK) * pnp_cdiv(a.Cout, BN);
  int want = (PNP_NUM_SMS * 6 + tiles - 1) / tiles;             // aim at ~6 CTAs per SM in total
  int max_splits = pnp_cdiv(a.M, BR * 4);               // at least 4 reduction blocks per CTA
  int splits = want < 1 ? 1 : want;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  int mps = pnp_cdiv(a.M, splits);
  mps = pnp_cdiv(mps, BR) * BR;
  splits = pnp_cdiv(a.M, mps);
  a.m_per_split = mps;
  dim3 grid(pnp_cdiv(a.KK, BKK), pnp_cdiv(a.Cout, BN), splits);
  pnp_launch(conv_wgrad_kernel<BKK, BN, BR, TK, TN, VEC>, grid, (BKK / TK) * (BN / TN), 0, s, x, dy, dw, a);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

__global__ void weight_transpose_kernel(const float* __restrict__ w, float* __restrict__ wT, int Cin, int Cout) {
  pnp_pdl_enter();
  // per tap: [Cin][Cout] -> [Cout][Cin]
  __shared__ float tile[32][33];
  const float* src = w + (long long)blockIdx.z * Cin * Cout;
  float* dst = wT + (long long)blockIdx.z * Cin * Cout;
  int ci0 = blockIdx.y * 32, co0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int ci = ci0 + r, co = co0 + threadIdx.x;
    tile[r][threadIdx.x] = (ci < Cin && co < Cout) ? src[(long long)ci * Cout + co] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    int co = co0 + r, ci = ci0 + threadIdx.x;
    if (co < Cout && ci < Cin) dst[(long long)co * Cin + ci] = tile[threadIdx.x][r];
  }
}

// ------------------------------------------------------------------------------------------------
// Segmenter tail in ONE kernel:  logits = conv5x5_SYMMETRIC( PS_r( X ) )     (source_segmenter.py:200-207, ops.py:23-27)
// X = conv10 output [B, a, b, G*r*r]; the phase shift (depth-to-space) and the mirror padding are pure index maps, so the
// tile loader gathers straight from X:
//     flat[n, Y, X_, g] = X[n, Y/r, X_/r, g*r*r + (X_%r)*r + (Y%r)]      (batch >= 2; the B == 1 order swaps the two residues)
//     padded[py, px]    = flat[mirror(py - p), mirror(px - p)]            (tf.pad SYMMETRIC: edge included)
// which removes the [B, 256, 256, 40] round trip through HBM twice over (r1: phase_shift 166 us + mirror_pad 108 us + conv 190 us
// per call, three calls per adversarial step).  Lanes run along Y%r first, then X_%r: for r = 8 a warp reads 128 contiguous bytes.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int mirror_i(int i, int n) { return i < 0 ? (-i - 1) : (i >= n ? 2 * n - 1 - i : i); }

template <int NO>
__global__ void __launch_bounds__(256)
ps_mirror_conv_kernel(const float* __restrict__ X, const float* __restrict__ w, float* __restrict__ y, int B, int a, int b, int G,
                      int r, int kh, int kw, int order_b1) {
  pnp_pdl_enter();
  constexpr int T = 32, CC = 8, HALO = T + 4;            // kernels up to 5x5
  __shared__ float s_x[CC][HALO][HALO + 1];
  __shared__ float s_w[25][CC][NO];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * T, y0 = blockIdx.y * T, n = blockIdx.z;
  const int H = a * r, W = b * r, rr = r * r;
  const int ph = kh / 2, pw = kw / 2;
  const int hh = T + kh - 1, hw = T + kw - 1;
  const int nby = (hh + 7) >> 3, nbx = (hw + 3) >> 2;      // loader patches of 8 (y) x 4 (x) halo pixels = one warp
  const long long Ctot = (long long)G * rr;
  float acc[4][NO];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int o = 0; o < NO; ++o) acc[j][o] = 0.f;
  const float* Xn = X + (long long)n * a * b * Ctot;
  for (int c0 = 0; c0 < G; c0 += CC) {
    __syncthreads();
    if (r == 8 && !order_b1) {
      // fast loader (r = 8, batch >= 2 sub-pixel order): one (source pixel, group) = 64 contiguous floats = the 8x8 block
      // flat[8*iy + q][8*ix + p] = X[.., g*64 + p*8 + q].  A warp reads the 256-byte line with one float2 per lane (fully
      // coalesced) and scatters it into the tile; blocks outside the image are the mirror images of the border blocks.
      const int wid = threadIdx.x >> 5, ln = threadIdx.x & 31;
      const int bY0 = (y0 - ph) >> 3, bX0 = (x0 - pw) >> 3;            // first source block touched (floor: may be -1)
      const int nbY = ((y0 - ph + hh - 1) >> 3) - bY0 + 1, nbX = ((x0 - pw + hw - 1) >> 3) - bX0 + 1;
      const int items = nbY * nbX * CC;
      const int p_ = ln >> 2, q_ = (ln & 3) * 2;                          // this lane's elements: (p_, q_) and (p_, q_ + 1)
      for (int it = wid; it < items; it += 8) {
        const int c = it % CC;
        const int rest = it / CC;
        const int sx = rest % nbX, sy = rest / nbX;
        const int bY = bY0 + sy, bX = bX0 + sx;
        const int sbY = bY < 0 ? 0 : (bY >= a ? a - 1 : bY), sbX = bX < 0 ? 0 : (bX >= b ? b - 1 : bX);
        float2 v = make_float2(0.f, 0.f);
        if (c0 + c < G)
          v = __ldg(reinterpret_cast<const float2*>(Xn + ((long long)sbY * b + sbX) * Ctot + (long long)(c0 + c) * 64 + ln * 2));
        // padded coordinate of image row Yi: itself inside the image; mirrored (edge included) for the blocks beyond the border
        const int Xi = sbX * 8 + p_;
        const int Xp = bX < 0 ? (-1 - Xi) : (bX >= b ? 2 * W - 1 - Xi : Xi);
        const int px = Xp - (x0 - pw);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int Yi = sbY * 8 + q_ + e;
          const int Yp = bY < 0 ? (-1 - Yi) : (bY >= a ? 2 * H - 1 - Yi : Yi);
          const int py = Yp - (y0 - ph);
          if (py >= 0 && py < hh && px >= 0 && px < hw) s_x[c][py][px] = e ? v.y : v.x;
        }
      }
    } else {
    const int total = nby * nbx * 32 * CC;
    for (int e = threadIdx.x; e < total; e += 256) {
      const int ly = e & 7, lx = (e >> 3) & 3;
      int rest = e >> 5;
      const int c = rest % CC;
      rest /= CC;
      const int bx = rest % nbx, by = rest / nbx;
      const int py = by * 8 + ly, px = bx * 4 + lx;
      if (py < hh && px < hw) {
        float v = 0.f;
        if (c0 + c < G) {
          const int Y = mirror_i(y0 + py - ph, H), Xc = mirror_i(x0 + px - pw, W);
          const int iy = Y / r, qy = Y - iy * r, ix = Xc / r, qx = Xc - ix * r;
          const int sub = order_b1 ? (qy * r + qx) : (qx * r + qy);
          v = __ldg(Xn + ((long long)iy * b + ix) * Ctot + (long long)(c0 + c) * rr + sub);
        }
        s_x[c][py][px] = v;
      }
    }
    }
    for (int p = threadIdx.x; p < kh * kw * CC * NO; p += 256) {
      const int o = p % NO, c = (p / NO) % CC, t = p / (NO * CC);
      s_w[t][c][o] = (c0 + c < G) ? __ldg(w + ((long long)t * G + c0 + c) * NO + o) : 0.f;
    }
    __syncthreads();
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx) {
        const int t = ky * kw + kx;
#pragma unroll
        for (int c = 0; c < CC; ++c) {
          float wv[NO];
#pragma unroll
          for (int o = 0; o < NO; ++o) wv[o] = s_w[t][c][o];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float av = s_x[c][ty + 8 * j + ky][tx + kx];
#pragma unroll
            for (int o = 0; o < NO; ++o) acc[j][o] = fmaf(av, wv[o], acc[j][o]);
          }
        }
      }
  }
  const int ox = x0 + tx;
  if (ox < W) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int oy = y0 + ty + 8 * j;
      if (oy < H) {
        float* dst = y + (((long long)n * H + oy) * W + ox) * NO;
#pragma unroll
        for (int o = 0; o < NO; ++o) dst[o] = acc[j][o];
      }
    }
  }
}

// 5x5 specialisation (the only size the graphs use), register-tiled: a thread owns a COLUMN of 8 output rows (lanes run along x, so
// every shared-memory read is conflict-free) and slides the 5 vertical taps over 12 activations held in registers: per (channel,
// kx) 12 activation loads + 7 broadcast 128-bit weight loads feed 200 FMAs, where the generic kernel above spends 9 loads per 20
// FMAs and is shared-memory-issue bound (r2: 262 us per B = 8 call at 20 TFLOP/s).  128 threads per 32x32 tile.  Measured (r2y, B = 16):
// 266 us against the generic kernel's 436 us.
template <int NO>
__global__ void __launch_bounds__(128)
ps_mirror_conv5_kernel(const float* __restrict__ X, const float* __restrict__ w, float* __restrict__ y, int B, int a, int b, int G,
                       int r, int order_b1) {
  pnp_pdl_enter();
  constexpr int T = 32, CC = 8, HALO = T + 4, RY = 8, KS = 5, NT = 128;
  constexpr int WPAD = ((KS * NO + 3) / 4) * 4;          // the KS x NO weights of one (channel, kx), padded to whole float4s
  __shared__ float s_x[CC][HALO][HALO + 1];
  __shared__ __align__(16) float s_w[CC][KS][WPAD];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * T, y0 = blockIdx.y * T, n = blockIdx.z;
  const int H = a * r, W = b * r, rr = r * r;
  constexpr int ph = 2, pw = 2, hh = HALO, hw = HALO;
  const int nby = (hh + 7) >> 3, nbx = (hw + 3) >> 2;
  const long long Ctot = (long long)G * rr;
  float acc[RY][NO];
#pragma unroll
  for (int j = 0; j < RY; ++j)
#pragma unroll
    for (int o = 0; o < NO; ++o) acc[j][o] = 0.f;
  const float* Xn = X + (long long)n * a * b * Ctot;
  for (int c0 = 0; c0 < G; c0 += CC) {
    __syncthreads();
    if (r == 8 && !order_b1) {
      // one (source pixel, group) = 64 contiguous floats = the 8x8 block flat[8*iy + q][8*ix + p] = X[.., g*64 + p*8 + q]: a warp
      // reads the 256-byte line with one float2 per lane and scatters it into the tile; blocks outside the image are the mirror
      // images of the border blocks.  Warp w owns channels w and w + 4 of the chunk and walks the (<= 6 x 6) source blocks of the
      // halo with nested loops -- no division by run-time values (ncu r2x: the first version of this kernel executed MORE
      // instructions than the generic one, 387 M vs 347 M at B = 16 against 164 M FMAs, nearly all of the surplus in a loader that
      // decoded a linear item index) -- and issues the 12 loads of one block row before scattering any of them.
      static_assert(CC == 8 && NT == 128, "loader assumes 4 warps x 2 channels");
      const int wid = threadIdx.x >> 5, ln = threadIdx.x & 31;
      const int bY0 = (y0 - ph) >> 3, bX0 = (x0 - pw) >> 3;            // first source block touched (floor: may be -1)
      const int nbY = ((y0 - ph + hh - 1) >> 3) - bY0 + 1, nbX = ((x0 - pw + hw - 1) >> 3) - bX0 + 1;      // <= 6 each
      const int p_ = ln >> 2, q_ = (ln & 3) * 2;                          // this lane's elements: (p_, q_) and (p_, q_ + 1)
      const bool on0 = c0 + wid < G, on1 = c0 + wid + 4 < G;
      const float* Xc = Xn + (long long)(c0 + wid) * 64 + ln * 2;
      for (int sy = 0; sy < nbY; ++sy) {
        const int bY = bY0 + sy;
        const int sbY = bY < 0 ? 0 : (bY >= a ? a - 1 : bY);
        const int Yi = sbY * 8 + q_;
        const bool my = bY < 0 || bY >= a;                               // mirrored block: its rows run backwards
        const int Yp = bY < 0 ? (-1 - Yi) : (bY >= a ? 2 * H - 1 - Yi : Yi);
        const int py0 = Yp - (y0 - ph), py1 = py0 + (my ? -1 : 1);
        const bool ok0 = py0 >= 0 && py0 < hh, ok1 = py1 >= 0 && py1 < hh;
        const float* Xrow = Xc + (long long)sbY * b * Ctot;
        float2 v0[6], v1[6];
#pragma unroll
        for (int sx = 0; sx < 6; ++sx) {
          const int bX = bX0 + sx;
          const int sbX = bX < 0 ? 0 : (bX >= b ? b - 1 : bX);
          const float* src = Xrow + (long long)sbX * Ctot;
          v0[sx] = (sx < nbX && on0) ? __ldg(reinterpret_cast<const float2*>(src)) : make_float2(0.f, 0.f);
          v1[sx] = (sx < nbX && on1) ? __ldg(reinterpret_cast<const float2*>(src + 4 * 64)) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int sx = 0; sx < 6; ++sx) {
          if (sx < nbX) {
            const int bX = bX0 + sx;
            const int sbX = bX < 0 ? 0 : (bX >= b ? b - 1 : bX);
            const int Xi = sbX * 8 + p_;
            const int Xp = bX < 0 ? (-1 - Xi) : (bX >= b ? 2 * W - 1 - Xi : Xi);
            const int px = Xp - (x0 - pw);
            if (px >= 0 && px < hw) {
              if (ok0) { s_x[wid][py0][px] = v0[sx].x; s_x[wid + 4][py0][px] = v1[sx].x; }
              if (ok1) { s_x[wid][py1][px] = v0[sx].y; s_x[wid + 4][py1][px] = v1[sx].y; }
            }
          }
        }
      }
    } else {
      const int total = nby * nbx * 32 * CC;
      for (int e = threadIdx.x; e < total; e += NT) {
        const int ly = e & 7, lx = (e >> 3) & 3;
        int rest = e >> 5;
        const int c = rest % CC;
        rest /= CC;
        const int bx = rest % nbx, by = rest / nbx;
        const int py = by * 8 + ly, px = bx * 4 + lx;
        if (py < hh && px < hw) {
          float v = 0.f;
          if (c0 + c < G) {
            const int Y = mirror_i(y0 + py - ph, H), Xc = mirror_i(x0 + px - pw, W);
            const int iy = Y / r, qy = Y - iy * r, ix = Xc / r, qx = Xc - ix * r;
            const int sub = order_b1 ? (qy * r + qx) : (qx * r + qy);
            v = __ldg(Xn + ((long long)iy * b + ix) * Ctot + (long long)(c0 + c) * rr + sub);
          }
          s_x[c][py][px] = v;
        }
      }
    }
    for (int p = threadIdx.x; p < KS * KS * CC * NO; p += NT) {
      const int o = p % NO, c = (p / NO) % CC, t = p / (NO * CC);
      const int ky = t / KS, kx = t - ky * KS;
      s_w[c][kx][ky * NO + o] = (c0 + c < G) ? __ldg(w + ((long long)t * G + c0 + c) * NO + o) : 0.f;
    }
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < CC; ++c) {
#pragma unroll
      for (int kx = 0; kx < KS; ++kx) {
        float av[RY + KS - 1];
#pragma unroll
        for (int i = 0; i < RY + KS - 1; ++i) av[i] = s_x[c][ty * RY + i][tx + kx];
        float wv[WPAD];
#pragma unroll
        for (int q = 0; q < WPAD / 4; ++q) {
          const float4 t4 = *reinterpret_cast<const float4*>(&s_w[c][kx][4 * q]);
          wv[4 * q] = t4.x; wv[4 * q + 1] = t4.y; wv[4 * q + 2] = t4.z; wv[4 * q + 3] = t4.w;
        }
#pragma unroll
        for (int ky = 0; ky < KS; ++ky)
#pragma unroll
          for (int j = 0; j < RY; ++j)
#pragma unroll
            for (int o = 0; o < NO; ++o) acc[j][o] = fmaf(av[j + ky], wv[ky * NO + o], acc[j][o]);
      }
    }
  }
  const int ox = x0 + tx;
  if (ox < W) {
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      const int oy = y0 + ty * RY + j;
      if (oy < H) {
        float* dst = y + (((long long)n * H + oy) * W + ox) * NO;
#pragma unroll
        for (int o = 0; o < NO; ++o) dst[o] = acc[j][o];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward of the fused tail w.r.t. its feature-map input, in ONE kernel:
//     dX = PS_r^T( mirror_pad^T( conv^T(dy, w) ) )        (the G step's path from d logits to d conv10)
// Output-stationary over the unpadded 256x256 map: dflat[Y, X, g] = sum over the padded positions (py, px) that mirror onto
// (Y, X) -- (Y+p, X+p) itself, plus the reflected rows / columns for the p border pixels -- of
//     dpadded[py, px, g] = sum_{ky,kx,o} dy[py-ky, px-kx, o] * w[ky, kx, g, o]      (dy outside the image = 0)
// and dX[n, Y/r, X/r, g*r*r + (X%r)*r + (Y%r)] = dflat[Y, X, g] (batch >= 2 order; transposed for B == 1).
// r1/r2a: transposed conv 477 us + mirror fold 108 us + inverse phase shift ~100 us per G step.
// ------------------------------------------------------------------------------------------------
template <int NO>
__global__ void __launch_bounds__(256)
ps_mirror_conv_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dX, int B, int a, int b, int G,
                          int r, int kh, int kw, int order_b1) {
  pnp_pdl_enter();
  constexpr int T = 32, CC = 8, HALO = T + 4;
  __shared__ float s_d[NO][HALO][HALO + 1];       // dy tile with halo, channel-major
  __shared__ __align__(16) float s_w[25][NO][CC];  // [tap][out channel of the forward conv][group]: 8 groups = two 128-bit broadcasts
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * T, y0 = blockIdx.y * T, n = blockIdx.z;
  const int H = a * r, W = b * r, rr = r * r;
  const int ph = kh / 2, pw = kw / 2;
  const int hh = T + kh - 1, hw = T + kw - 1;
  const long long Ctot = (long long)G * rr;
  // dy halo tile: rows y0-ph .. y0+T-1+ph of the image (zero outside): dpadded[py] with py = Y+ph reads dy rows Y+ph-ky
  const float* dyn = dy + (long long)n * H * W * NO;
  for (int p = threadIdx.x; p < hh * hw; p += 256) {
    const int py = p / hw, px = p - py * hw;
    const int iy = y0 + py - ph, ix = x0 + px - pw;
    const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
    for (int o = 0; o < NO; ++o) s_d[o][py][px] = in ? __ldg(dyn + ((long long)iy * W + ix) * NO + o) : 0.f;
  }
  // this thread's 4 output pixels (column tx, rows ty + 8j) and their mirror images: padded positions that fold onto (Y, X)
  const int X = x0 + tx;
  int xs[3], nx = 0;                           // padded columns, relative to the dy halo tile: px_rel = Xp - x0 (Xp = padded col)
  if (X < W) {
    xs[nx++] = X + pw;
    if (X < pw) xs[nx++] = pw - 1 - X;
    if (X >= W - pw) xs[nx++] = 2 * W - 1 - X + pw;
  }
  float* dXn = dX + (long long)n * a * b * Ctot;
  for (int c0 = 0; c0 < G; c0 += CC) {
    __syncthreads();
    for (int p = threadIdx.x; p < kh * kw * CC * NO; p += 256) {
      const int o = p % NO, c = (p / NO) % CC, t = p / (NO * CC);
      s_w[t][o][c] = (c0 + c < G) ? __ldg(w + ((long long)t * G + c0 + c) * NO + o) : 0.f;
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      const int Y = y0 + ty + 8 * j;
      if (Y >= H || X >= W) continue;
      int ys[3], ny = 0;
      ys[ny++] = Y + ph;
      if (Y < ph) ys[ny++] = ph - 1 - Y;
      if (Y >= H - ph) ys[ny++] = 2 * H - 1 - Y + ph;
      float acc[CC];
#pragma unroll
      for (int c = 0; c < CC; ++c) acc[c] = 0.f;
      for (int iyp = 0; iyp < ny; ++iyp)
        for (int ixp = 0; ixp < nx; ++ixp) {
          // dpadded[Yp, Xp] = sum_taps dy[Yp-ky, Xp-kx] * w[ky,kx]; tile-relative dy row of image row q is q - (y0 - ph)
          const int Yp = ys[iyp], Xp = xs[ixp];
          for (int ky = 0; ky < kh; ++ky) {
            const int ry = Yp - ky - (y0 - ph);          // image row Yp-ky, in halo coordinates
            if (ry < 0 || ry >= hh) continue;            // outside the halo == outside the image (see below)
            for (int kx = 0; kx < kw; ++kx) {
              const int rx = Xp - kx - (x0 - pw);
              if (rx < 0 || rx >= hw) continue;
              const int t = ky * kw + kx;
              float d[NO];
#pragma unroll
              for (int o = 0; o < NO; ++o) d[o] = s_d[o][ry][rx];
#pragma unroll
              for (int o = 0; o < NO; ++o) {
                const float4 w0 = *reinterpret_cast<const float4*>(&s_w[t][o][0]);
                const float4 w1 = *reinterpret_cast<const float4*>(&s_w[t][o][4]);
                acc[0] = fmaf(d[o], w0.x, acc[0]); acc[1] = fmaf(d[o], w0.y, acc[1]);
                acc[2] = fmaf(d[o], w0.z, acc[2]); acc[3] = fmaf(d[o], w0.w, acc[3]);
                acc[4] = fmaf(d[o], w1.x, acc[4]); acc[5] = fmaf(d[o], w1.y, acc[5]);
                acc[6] = fmaf(d[o], w1.z, acc[6]); acc[7] = fmaf(d[o], w1.w, acc[7]);
              }
            }
          }
        }
      const int iy = Y / r, qy = Y - iy * r, ix = X / r, qx = X - ix * r;
      const int sub = order_b1 ? (qy * r + qx) : (qx * r + qy);
      float* dst = dXn + ((long long)iy * b + ix) * Ctot + sub;
#pragma unroll
      for (int c = 0; c < CC; ++c)
        if (c0 + c < G) dst[(long long)(c0 + c) * rr] = acc[c];
    }
  }
}

// 5x5 specialisation of the backward tail, register-tiled like the forward one: a thread owns the 8 rows Y = 8*iy .. 8*iy + 7 of one
// column X -- for r = 8 exactly the 8 sub-pixel rows of ONE source pixel, i.e. 8 CONTIGUOUS floats of dX per group (the kernel above
// writes them as 8 scattered 4-byte stores per thread and runs at 85 GB/s of DRAM traffic) -- and 8 groups at a time: per (kx, o)
// 12 dy loads + 10 broadcast 128-bit weight loads feed 320 FMAs.  The mirror fold (border rows / columns receive the reflected
// padded positions as well) runs as a second, generic pass that only threads of edge pixels enter.
template <int NO>
__global__ void __launch_bounds__(128)
ps_mirror_conv5_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dX, int B, int a, int b,
                           int G, int r, int order_b1) {
  pnp_pdl_enter();
  constexpr int T = 32, CC = 8, HALO = T + 4, RY = 8, KS = 5, NT = 128;
  constexpr int ph = 2, pw = 2, hh = HALO, hw = HALO;
  __shared__ float s_d[NO][HALO][HALO + 1];                 // dy tile with halo (zero outside the image), channel-major
  __shared__ __align__(16) float s_w[KS][NO][KS][CC];       // [kx][o][ky][group]: the 40 weights of one (kx, o) are contiguous
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = blockIdx.x * T, y0 = blockIdx.y * T, n = blockIdx.z;
  const int H = a * r, W = b * r, rr = r * r;
  const long long Ctot = (long long)G * rr;
  const float* dyn = dy + (long long)n * H * W * NO;
  for (int p = threadIdx.x; p < hh * hw; p += NT) {
    const int py = p / hw, px = p - py * hw;
    const int iy = y0 + py - ph, ix = x0 + px - pw;
    const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
    for (int o = 0; o < NO; ++o) s_d[o][py][px] = in ? __ldg(dyn + ((long long)iy * W + ix) * NO + o) : 0.f;
  }
  const int X = x0 + tx;
  const int Yb = y0 + ty * RY;                               // first of this thread's 8 rows
  const bool live = X < W && Yb < H;
  // mirror images of column X in the padded frame (beyond the padded position X + pw itself)
  int xs[2], nx = 0;
  if (X < pw) xs[nx++] = pw - 1 - X;
  if (X >= W - pw && X < W) xs[nx++] = 2 * W - 1 - X + pw;
  const bool edge_rows = (Yb < ph) || (Yb + RY > H - ph);
  float* dXn = dX + (long long)n * a * b * Ctot;
  for (int c0 = 0; c0 < G; c0 += CC) {
    __syncthreads();
    for (int p = threadIdx.x; p < KS * KS * CC * NO; p += NT) {
      const int o = p % NO, c = (p / NO) % CC, t = p / (NO * CC);
      const int ky = t / KS, kx = t - ky * KS;
      s_w[kx][o][ky][c] = (c0 + c < G) ? __ldg(w + ((long long)t * G + c0 + c) * NO + o) : 0.f;
    }
    __syncthreads();
    float acc[RY][CC];
#pragma unroll
    for (int j = 0; j < RY; ++j)
#pragma unroll
      for (int c = 0; c < CC; ++c) acc[j][c] = 0.f;
    // padded position (Y + ph, X + pw) itself: dflat[Y, X] += sum_{ky,kx,o} dy[Y + ph - ky, X + pw - kx, o] * w[ky, kx, g, o];
    // in halo coordinates (origin y0 - ph, x0 - pw) that is row (Y - y0) + 2*ph - ky, column tx + 2*pw - kx
#pragma unroll 1
    for (int kx = 0; kx < KS; ++kx) {
#pragma unroll 1
      for (int o = 0; o < NO; ++o) {
        float dv[RY + KS - 1];
#pragma unroll
        for (int i = 0; i < RY + KS - 1; ++i) dv[i] = s_d[o][ty * RY + i][tx + 2 * pw - kx];
        float wv[KS * CC];
#pragma unroll
        for (int q = 0; q < KS * CC / 4; ++q) {
          const float4 t4 = *reinterpret_cast<const float4*>(&s_w[kx][o][0][0] + 4 * q);
          wv[4 * q] = t4.x; wv[4 * q + 1] = t4.y; wv[4 * q + 2] = t4.z; wv[4 * q + 3] = t4.w;
        }
#pragma unroll
        for (int ky = 0; ky < KS; ++ky)
#pragma unroll
          for (int j = 0; j < RY; ++j)
#pragma unroll
            for (int c = 0; c < CC; ++c) acc[j][c] = fmaf(dv[j + 2 * ph - ky], wv[ky * CC + c], acc[j][c]);
      }
    }
    // mirror fold: reflected padded rows / columns of edge pixels (at most 2 rows x 2 columns of the image border)
    if (live && (nx > 0 || edge_rows)) {
#pragma unroll
      for (int j = 0; j < RY; ++j) {
        const int Y = Yb + j;
        int ys[2], ny = 0;
        if (Y < ph) ys[ny++] = ph - 1 - Y;
        if (Y >= H - ph && Y < H) ys[ny++] = 2 * H - 1 - Y + ph;
        // all (row, column) combinations except (self, self): index 0 = the padded position itself
        for (int iyp = 0; iyp <= ny; ++iyp)
          for (int ixp = 0; ixp <= nx; ++ixp) {
            if (iyp == 0 && ixp == 0) continue;
            const int Yp = iyp == 0 ? Y + ph : ys[iyp - 1];
            const int Xp = ixp == 0 ? X + pw : xs[ixp - 1];
            // kept rolled: unrolled for every row j, this cold path grew to ~38k instructions at NO = 5 and ptxas spilled
            // 22 KB, the main loop's accumulators included (2.9 ms per B = 8 call instead of ~0.3)
#pragma unroll 1
            for (int ky = 0; ky < KS; ++ky) {
              const int ry = Yp - ky - (y0 - ph);
              if (ry < 0 || ry >= hh) continue;            // outside the halo == outside the image for these positions
#pragma unroll 1
              for (int kx = 0; kx < KS; ++kx) {
                const int rx = Xp - kx - (x0 - pw);
                if (rx < 0 || rx >= hw) continue;
#pragma unroll
                for (int o = 0; o < NO; ++o) {
                  const float d = s_d[o][ry][rx];
                  const float4 w0 = *reinterpret_cast<const float4*>(&s_w[kx][o][ky][0]);
                  const float4 w1 = *reinterpret_cast<const float4*>(&s_w[kx][o][ky][4]);
                  acc[j][0] = fmaf(d, w0.x, acc[j][0]); acc[j][1] = fmaf(d, w0.y, acc[j][1]);
                  acc[j][2] = fmaf(d, w0.z, acc[j][2]); acc[j][3] = fmaf(d, w0.w, acc[j][3]);
                  acc[j][4] = fmaf(d, w1.x, acc[j][4]); acc[j][5] = fmaf(d, w1.y, acc[j][5]);
                  acc[j][6] = fmaf(d, w1.z, acc[j][6]); acc[j][7] = fmaf(d, w1.w, acc[j][7]);
                }
              }
            }
          }
      }
    }
    if (live) {
      if (r == 8 && !order_b1) {
        // rows Yb .. Yb+7 are the 8 sub-pixel rows q of source pixel (Yb/8, X/8): dX[.., g*64 + (X%8)*8 + q], 32 contiguous bytes
        float* dst = dXn + ((long long)(Yb >> 3) * b + (X >> 3)) * Ctot + (X & 7) * 8;
#pragma unroll
        for (int c = 0; c < CC; ++c)
          if (c0 + c < G) {
            float4* d4 = reinterpret_cast<float4*>(dst + (long long)(c0 + c) * 64);
            d4[0] = make_float4(acc[0][c], acc[1][c], acc[2][c], acc[3][c]);
            d4[1] = make_float4(acc[4][c], acc[5][c], acc[6][c], acc[7][c]);
          }
      } else {
#pragma unroll
        for (int j = 0; j < RY; ++j) {
          const int Y = Yb + j;
          if (Y < H) {
            const int iy = Y / r, qy = Y - iy * r, ix = X / r, qx = X - ix * r;
            const int sub = order_b1 ? (qy * r + qx) : (qx * r + qy);
            float* dst = dXn + ((long long)iy * b + ix) * Ctot + sub;
#pragma unroll
            for (int c = 0; c < CC; ++c)
              if (c0 + c < G) dst[(long long)(c0 + c) * rr] = acc[j][c];
          }
        }
      }
    }
  }
}

// PNP_TAIL5: bit 0 = register-tiled 5x5 forward tail, bit 1 = register-tiled 5x5 backward tail; 0 = the generic (any odd k <= 5)
// kernels also for 5x5.  Default 3, as measured: forward 436 -> 266 us per B = 16 call (r2y; config 1: 4.44 -> 4.25 ms per step);
// backward 419 -> 298 us per B = 8 call (r2z; config 4, whose G update is the step that runs it: 28.41 -> 28.29 ms).
int tail5_mode() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("PNP_TAIL5"); v = e ? atoi(e) : 3; }
  return v;
}

bool geom_ok(const pnp_conv_geom* g) {
  return g && g->B > 0 && g->H > 0 && g->W > 0 && g->Cin > 0 && g->Ho > 0 && g->Wo > 0 && g->Cout > 0 && g->kh > 0 &&
         g->kw > 0 && g->stride > 0 && g->dil > 0 && g->pad_t >= 0 && g->pad_l >= 0;
}

PnpDropout make_drop(const pnp_dropout_cfg* d) { return pnp_make_drop(d); }

}  // namespace

extern "C" int pnp_conv2d_fwd(const float* x, const float* w, float* y, const pnp_conv_geom* g,
                              const pnp_dropout_cfg* drop, int accumulate, void* stream) {
  if (!geom_ok(g) || !x || !w || !y) return PNP_ERR_BAD_ARG;
  long long M = (long long)g->B * g->Ho * g->Wo;
  if (M > 0x7fffffffLL || (long long)g->kh * g->kw * g->Cin > 0x7fffffffLL) return PNP_ERR_UNSUPPORTED;
  GatherArgs a;
  a.B = g->B; a.IH = g->H; a.IW = g->W; a.IC = g->Cin;
  a.OH = g->Ho; a.OW = g->Wo; a.OC = g->Cout;
  a.kh = g->kh; a.kw = g->kw; a.stride = g->stride; a.dil = g->dil; a.pad_t = g->pad_t; a.pad_l = g->pad_l;
  a.M = (int)M; a.K = g->kh * g->kw * g->Cin; a.accumulate = accumulate;
  a.drop = make_drop(drop);
  if ((g->Cout == 5 || g->Cout == 8) && g->Cin % 8 == 0 && g->stride == 1 && g->dil == 1 && g->kh <= 5 && g->kw <= 5 && !accumulate &&
      a.drop.seed_ptr == nullptr && g->B <= 65535) {
    dim3 grid(pnp_cdiv(g->Wo, 32), pnp_cdiv(g->Ho, 32), g->B);
    if (g->Cout == 5)
      pnp_launch(conv_few_out_kernel<5>, grid, 256, 0, (cudaStream_t)stream, x, w, y, g->B, g->H, g->W, g->Cin, g->Ho, g->Wo, g->kh, g->kw,
                                                                     g->pad_t, g->pad_l);
    else
      pnp_launch(conv_few_out_kernel<8>, grid, 256, 0, (cudaStream_t)stream, x, w, y, g->B, g->H, g->W, g->Cin, g->Ho, g->Wo, g->kh, g->kw,
                                                                     g->pad_t, g->pad_l);
    PNP_LAUNCH_CHECK();
    return PNP_OK;
  }
  return dispatch_gather<false>(x, w, y, a, (cudaStream_t)stream);
}

extern "C" int pnp_ps_mirror_conv_fwd(const float* X, const float* w, float* y, int B, int a, int b, int G, int r, int kh, int kw,
                                      int Cout, int order_b1, void* stream) {
  if (!X || !w || !y || B <= 0 || a <= 0 || b <= 0 || G <= 0 || r <= 0) return PNP_ERR_BAD_ARG;
  if (kh > 5 || kw > 5 || kh < 1 || kw < 1 || (kh & 1) == 0 || (kw & 1) == 0 || B > 65535) return PNP_ERR_UNSUPPORTED;
  if (kh / 2 > a * r || kw / 2 > b * r) return PNP_ERR_UNSUPPORTED;
  dim3 grid(pnp_cdiv(b * r, 32), pnp_cdiv(a * r, 32), B);
  if (kh == 5 && kw == 5 && (Cout == 5 || Cout == 8) && (tail5_mode() & 1)) {      // the graphs' 5x5 output convolution: register-tiled kernel
    if (Cout == 5) pnp_launch(ps_mirror_conv5_kernel<5>, grid, 128, 0, (cudaStream_t)stream, X, w, y, B, a, b, G, r, order_b1);
    else pnp_launch(ps_mirror_conv5_kernel<8>, grid, 128, 0, (cudaStream_t)stream, X, w, y, B, a, b, G, r, order_b1);
    PNP_LAUNCH_CHECK();
    return PNP_OK;
  }
  if (Cout == 5) pnp_launch(ps_mirror_conv_kernel<5>, grid, 256, 0, (cudaStream_t)stream, X, w, y, B, a, b, G, r, kh, kw, order_b1);
  else if (Cout == 8) pnp_launch(ps_mirror_conv_kernel<8>, grid, 256, 0, (cudaStream_t)stream, X, w, y, B, a, b, G, r, kh, kw, order_b1);
  else return PNP_ERR_UNSUPPORTED;
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_ps_mirror_conv_bwd(const float* dy, const float* w, float* dX, int B, int a, int b, int G, int r, int kh, int kw,
                                      int Cout, int order_b1, void* stream) {
  if (!dy || !w || !dX || B <= 0 || a <= 0 || b <= 0 || G <= 0 || r <= 0) return PNP_ERR_BAD_ARG;
  if (kh > 5 || kw > 5 || kh < 1 || kw < 1 || (kh & 1) == 0 || (kw & 1) == 0 || B > 65535) return PNP_ERR_UNSUPPORTED;
  if (kh / 2 > a * r || kw / 2 > b * r) return PNP_ERR_UNSUPPORTED;
  dim3 grid(pnp_cdiv(b * r, 32), pnp_cdiv(a * r, 32), B);
  if (kh == 5 && kw == 5 && (Cout == 5 || Cout == 8) && (tail5_mode() & 2)) {
    if (Cout == 5) pnp_launch(ps_mirror_conv5_bwd_kernel<5>, grid, 128, 0, (cudaStream_t)stream, dy, w, dX, B, a, b, G, r, order_b1);
    else pnp_launch(ps_mirror_conv5_bwd_kernel<8>, grid, 128, 0, (cudaStream_t)stream, dy, w, dX, B, a, b, G, r, order_b1);
    PNP_LAUNCH_CHECK();
    return PNP_OK;
  }
  if (Cout == 5) pnp_launch(ps_mirror_conv_bwd_kernel<5>, grid, 256, 0, (cudaStream_t)stream, dy, w, dX, B, a, b, G, r, kh, kw, order_b1);
  else if (Cout == 8) pnp_launch(ps_mirror_conv_bwd_kernel<8>, grid, 256, 0, (cudaStream_t)stream, dy, w, dX, B, a, b, G, r, kh, kw, order_b1);
  else return PNP_ERR_UNSUPPORTED;
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_conv2d_dgrad(const float* dy, const float* wT, float* dx, const pnp_conv_geom* g,
                                int accumulate, void* stream) {
  if (!geom_ok(g) || !dy || !wT || !dx) return PNP_ERR_BAD_ARG;
  long long M = (long long)g->B * g->H * g->W;
  if (M > 0x7fffffffLL) return PNP_ERR_UNSUPPORTED;
  GatherArgs a;
  a.B = g->B; a.IH = g->Ho; a.IW = g->Wo; a.IC = g->Cout;   // gather from dy
  a.OH = g->H; a.OW = g->W; a.OC = g->Cin;                  // produce dx
  a.kh = g->kh; a.kw = g->kw; a.stride = g->stride; a.dil = g->dil; a.pad_t = g->pad_t; a.pad_l = g->pad_l;
  a.M = (int)M; a.K = g->kh * g->kw * g->Cout; a.accumulate = accumulate;
  a.drop = make_drop(nullptr);
  return dispatch_gather<true>(dy, wT, dx, a, (cudaStream_t)stream);
}

extern "C" int pnp_conv2d_wgrad(const float* x, const float* dy, float* dw, const pnp_conv_geom* g, void* stream) {
  if (!geom_ok(g) || !x || !dy || !dw) return PNP_ERR_BAD_ARG;
  long long M = (long long)g->B * g->Ho * g->Wo;
  if (M > 0x7fffffffLL) return PNP_ERR_UNSUPPORTED;
  WgradArgs a;
  a.B = g->B; a.H = g->H; a.W = g->W; a.Cin = g->Cin; a.Ho = g->Ho; a.Wo = g->Wo; a.Cout = g->Cout;
  a.kh = g->kh; a.kw = g->kw; a.stride = g->stride; a.dil = g->dil; a.pad_t = g->pad_t; a.pad_l = g->pad_l;
  a.M = (int)M; a.KK = g->kh * g->kw * g->Cin; a.m_per_split = (int)M;
  cudaStream_t s = (cudaStream_t)stream;
  const bool vec = (g->Cin % 4) == 0;
  if (!vec) {
    if (g->Cout <= 16) return launch_wgrad<64, 16, 16, 4, 1, 1>(x, dy, dw, a, s);
    return launch_wgrad<64, 64, 16, 4, 4, 1>(x, dy, dw, a, s);
  }
  if (g->Cout <= 8) return launch_wgrad<128, 8, 16, 4, 1, 4>(x, dy, dw, a, s);
  if (g->Cout <= 16) return launch_wgrad<64, 16, 16, 4, 1, 4>(x, dy, dw, a, s);
  if (g->Cout <= 32) return launch_wgrad<64, 32, 16, 4, 2, 4>(x, dy, dw, a, s);
  if (g->Cout <= 64 || a.KK < 128) return launch_wgrad<64, 64, 16, 4, 4, 4>(x, dy, dw, a, s);
  return launch_wgrad<128, 128, 16, 8, 8, 4>(x, dy, dw, a, s);
}

extern "C" int pnp_weight_transpose(const float* w, float* wT, int taps, int Cin, int Cout, void* stream) {
  if (!w || !wT || taps <= 0 || Cin <= 0 || Cout <= 0) return PNP_ERR_BAD_ARG;
  dim3 grid(pnp_cdiv(Cout, 32), pnp_cdiv(Cin, 32), taps);
  pnp_launch(weight_transpose_kernel, grid, dim3(32, 8), 0, (cudaStream_t)stream, w, wT, Cin, Cout);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}
