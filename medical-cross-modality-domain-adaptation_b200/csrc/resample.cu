// Planes resampled out of a device-resident volume: the data-preparation hot path (preprocess.py).  One launch draws every
// augmented coronal slice of a batch -- images by trilinear interpolation of the z-scored intensities, labels by the nearest voxel
// of the class-id volume -- straight into the trainers' NHWC layout, so a trainer can draw fresh augmentations every step
// without record files or a host-to-device image copy.  A grid-stride gather: the writes are coalesced along the NHWC index,
// the reads follow the sampled coordinates.  The way back (native.py): pnp_native_labels samples the class scores of the prepared
// grid at every voxel of the subject's native grid with the same taps and lerps, and labels it by their argmax;
// pnp_native_labels_ensemble sums the scores of several members (checkpoints, test-time transforms) first, and
// pnp_native_accumulate / pnp_native_accumulated_labels do the same for any number of members, one launch per member into a
// native-grid sum volume, then one argmax launch.  The opt-in
// augmentations: pnp_smooth_noise_field draws smoothed Philox noise fields (elastic displacement, bias gain) and
// pnp_resample_planes_aug resamples at the displaced pixels and applies gain, contrast and offset.
#include "common.cuh"
#include "../../include/pnp_b200.h"

#include <initializer_list>

namespace {

// a + f (b - a) with each operation rounded (no FMA contraction): the host restatement (oracle/resample_exact.py) computes
// the same three roundings
__device__ __forceinline__ float lerp_rn(float a, float b, float f) { return __fadd_rn(a, __fmul_rn(f, __fsub_rn(b, a))); }

// trilinear taps along one axis: clamp into [0, n - 1], i0 = floor, i1 = min(i0 + 1, n - 1), f = x - i0 (exact for x >= 0).
// fmaxf sends a NaN coordinate to 0.
__device__ __forceinline__ void axis_taps(float u, int n, int& i0, int& i1, float& f) {
  const float x = fminf(fmaxf(u, 0.f), (float)(n - 1));
  const float fl = floorf(x);
  i0 = (int)fl;
  i1 = min(i0 + 1, n - 1);
  f = __fsub_rn(x, fl);
}

// u inside [-0.5, n - 0.5), false for a NaN coordinate.  n <= 2^23 keeps n - 0.5 exact.
__device__ __forceinline__ bool axis_inside(float u, int n) { return u >= -0.5f && u < __fsub_rn((float)n, 0.5f); }

// nearest voxel floor(u + 0.5) (ties round up), -1 outside [-0.5, n - 0.5) or for a NaN coordinate; the min() only guards the
// index.
__device__ __forceinline__ int axis_nearest(float u, int n) {
  if (!axis_inside(u, n)) return -1;
  return min((int)floorf(__fadd_rn(u, 0.5f)), n - 1);
}

// Per-sample augmentation fields of pnp_resample_planes_aug; every pointer may be NULL.  disp [B][2][H][W]: (d_r, d_c) added to
// the output pixel before its matrix; gain [B][H][W]: g - 1 of the multiplicative bias field; ab [B][2]: contrast a, offset b.
struct AugFields {
  const float* disp;
  const float* gain;
  const float* ab;
};

// Item q of the NHWC output: k = q % Cw (or C / 2 when only the middle label plane is written, Cw == 1), pixel = q / Cw.
// AUG = false is pnp_resample_planes (aug unused); AUG = true is pnp_resample_planes_aug.
template <bool AUG>
__global__ void __launch_bounds__(256)
resample_planes_kernel(const float* __restrict__ vol, const uint8_t* __restrict__ cls, int n0, int n1, int n2,
                       const float* __restrict__ mats, int H, int W, int C, int Cw, long long total, float* __restrict__ img,
                       long long* __restrict__ lab, int label_planes, AugFields aug) {
  pnp_pdl_enter();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const unsigned q = (unsigned)i;
    const int k = Cw == C ? (int)(q % (unsigned)C) : C / 2;
    const unsigned pix = q / (unsigned)Cw;                  // (b H + r) W + c
    const unsigned row = pix / (unsigned)W;
    const int c = (int)(pix - row * (unsigned)W), r = (int)(row % (unsigned)H), b = (int)(row / (unsigned)H);
    const float* m = mats + (long long)(b * C + k) * 9;
    float fr = (float)r, fc = (float)c;
    if (AUG && aug.disp) {                                  // d_r at b 2HW + r W + c = pix + b HW, d_c one plane later
      const float* d = aug.disp + (long long)pix + (long long)b * H * W;
      fr = __fadd_rn(fr, __ldg(d));
      fc = __fadd_rn(fc, __ldg(d + (long long)H * W));
    }
    float u[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) u[a] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 3 * a), fr), __fmul_rn(__ldg(m + 3 * a + 1), fc)),
                                                 __ldg(m + 3 * a + 2));
    const long long o = (long long)pix * C + k;
    if (img) {
      int a0, b0, a1, b1, a2, b2;
      float f0, f1, f2;
      axis_taps(u[0], n0, a0, b0, f0);
      axis_taps(u[1], n1, a1, b1, f1);
      axis_taps(u[2], n2, a2, b2, f2);
      const float* p00 = vol + (a0 * n1 + a1) * n2;
      const float* p01 = vol + (a0 * n1 + b1) * n2;
      const float* p10 = vol + (b0 * n1 + a1) * n2;
      const float* p11 = vol + (b0 * n1 + b1) * n2;
      const float v00 = lerp_rn(__ldg(p00 + a2), __ldg(p00 + b2), f2);
      const float v01 = lerp_rn(__ldg(p01 + a2), __ldg(p01 + b2), f2);
      const float v10 = lerp_rn(__ldg(p10 + a2), __ldg(p10 + b2), f2);
      const float v11 = lerp_rn(__ldg(p11 + a2), __ldg(p11 + b2), f2);
      float v = lerp_rn(lerp_rn(v00, v01, f1), lerp_rn(v10, v11, f1), f0);
      if (AUG && aug.gain) v = __fmul_rn(__fadd_rn(1.f, __ldg(aug.gain + pix)), v);
      if (AUG && aug.ab) v = __fadd_rn(__fmul_rn(__ldg(aug.ab + 2 * b), v), __ldg(aug.ab + 2 * b + 1));
      img[o] = v;
    }
    if (label_planes) {
      const int j0 = axis_nearest(u[0], n0), j1 = axis_nearest(u[1], n1), j2 = axis_nearest(u[2], n2);
      const long long v = (j0 < 0 || j1 < 0 || j2 < 0) ? 0LL : (long long)__ldg(cls + (j0 * n1 + j1) * n2 + j2);
      if (label_planes == C) lab[o] = v;
      else if (k == C / 2) lab[pix] = v;
    }
  }
}

// Native voxel q = (i m1 + j) m2 + k: trilinear class scores at its prepared-grid coordinate, first-max argmax, and with gt the
// (truth, prediction) pair in a per-CTA histogram flushed by one global atomic per non-zero bin.  One body serves three kernels:
// ENS = false, ACC = false is pnp_native_labels: one member, its map held in registers (K and stride unused).
// ENS = true is pnp_native_labels_ensemble: member k's scores start at scores + k stride and its map at map + 12 k; the maps are
// staged in shared memory once per CTA, and the class scores of the members covering the voxel are summed in ascending k (the
// first one taken as it is) before the argmax.
// ACC = true is pnp_native_accumulate: one member as pnp_native_labels samples it, its class scores stored into sums[q][.] where
// out[q] (the coverage flags) is 0 -- out[q] is then set to 1 -- and added to them elsewhere (gt, cm, K and stride unused).
template <bool ENS, bool ACC>
__device__ __forceinline__ void native_labels_body(const float* __restrict__ scores, int n0, int n1, int n2, int C,
                                                   const float* __restrict__ map, int m1, int m2, long long total,
                                                   uint8_t* __restrict__ out, const uint8_t* __restrict__ gt, long long* __restrict__ cm,
                                                   int K, long long stride, float* __restrict__ sums) {
  __shared__ unsigned int hist[64];
  __shared__ float maps[ENS ? 12 * PNP_NATIVE_MAX_MEMBERS : 1];
  pnp_pdl_enter();
  if (cm) {
    if (threadIdx.x < 64) hist[threadIdx.x] = 0u;
    __syncthreads();
  }
  float m[12];
  if (ENS) {
    if (threadIdx.x < 12 * K) maps[threadIdx.x] = __ldg(map + threadIdx.x);
    __syncthreads();
  } else {
#pragma unroll
    for (int t = 0; t < 12; ++t) m[t] = __ldg(map + t);
  }
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const unsigned q = (unsigned)i;
    const unsigned row = q / (unsigned)m2;
    const float fk = (float)(q - row * (unsigned)m2), fj = (float)(row % (unsigned)m1), fi = (float)(row / (unsigned)m1);
    int best = 0;
    float sum[8];                        // ENS: the summed class scores (C <= 8, fully unrolled: they stay in registers)
    bool covered = false;                // ENS: some member covers the voxel
    for (int e = 0; e < (ENS ? K : 1); ++e) {
      const float* mk = ENS ? maps + 12 * e : m;
      const float* member = ENS ? scores + (long long)e * stride : scores;
      float u[3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
        u[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(mk[4 * a], fi), __fmul_rn(mk[4 * a + 1], fj)), __fmul_rn(mk[4 * a + 2], fk)),
                         mk[4 * a + 3]);
      if (axis_inside(u[0], n0) && axis_inside(u[1], n1) && axis_inside(u[2], n2)) {
        int a0, b0, a1, b1, a2, b2;
        float f0, f1, f2;
        axis_taps(u[0], n0, a0, b0, f0);
        axis_taps(u[1], n1, a1, b1, f1);
        axis_taps(u[2], n2, a2, b2, f2);
        const float* p00 = member + (long long)((a0 * n1 + a1) * n2) * C;
        const float* p01 = member + (long long)((a0 * n1 + b1) * n2) * C;
        const float* p10 = member + (long long)((b0 * n1 + a1) * n2) * C;
        const float* p11 = member + (long long)((b0 * n1 + b1) * n2) * C;
        const int o0 = a2 * C, o1 = b2 * C;
        float top = 0.f;
        float* s = ACC ? sums + (long long)q * C : nullptr;      // 64-bit: m0 m1 m2 C may reach 2^31
        const bool first = ACC && out[q] == 0;
#pragma unroll
        for (int c = 0; c < (ENS ? 8 : C); ++c) {     // ENS unrolls to 8 classes and stops at C
          if (ENS && c >= C) break;
          const float v00 = lerp_rn(__ldg(p00 + o0 + c), __ldg(p00 + o1 + c), f2);
          const float v01 = lerp_rn(__ldg(p01 + o0 + c), __ldg(p01 + o1 + c), f2);
          const float v10 = lerp_rn(__ldg(p10 + o0 + c), __ldg(p10 + o1 + c), f2);
          const float v11 = lerp_rn(__ldg(p11 + o0 + c), __ldg(p11 + o1 + c), f2);
          const float v = lerp_rn(lerp_rn(v00, v01, f1), lerp_rn(v10, v11, f1), f0);
          if (ACC) {
            s[c] = first ? v : __fadd_rn(s[c], v);             // the first covering member is taken as it is
          } else if (ENS) {
            sum[c] = covered ? __fadd_rn(sum[c], v) : v;     // the first covering member is taken as it is
          } else if (c == 0 || v > top) {       // strictly greater: the lowest index wins a tie
            top = v;
            best = c;
          }
        }
        if (ACC && first) out[q] = 1;
        covered = true;
      }
    }
    if (ENS && covered) {
      float top = sum[0];
#pragma unroll
      for (int c = 1; c < 8; ++c) {
        if (c < C && sum[c] > top) {     // strictly greater: the lowest index wins a tie
          top = sum[c];
          best = c;
        }
      }
    }
    if (ACC) continue;
    out[q] = (uint8_t)best;
    if (cm) {
      int g = __ldg(gt + q);
      if (g >= C) g = 0;
      atomicAdd(&hist[g * C + best], 1u);
    }
  }
  if (cm) {
    __syncthreads();
    if (threadIdx.x < C * C && hist[threadIdx.x])
      atomicAdd((unsigned long long*)cm + threadIdx.x, (unsigned long long)hist[threadIdx.x]);
  }
}

template <bool ENS>
__global__ void __launch_bounds__(256)
native_labels_kernel(const float* __restrict__ scores, int n0, int n1, int n2, int C, const float* __restrict__ map, int m1, int m2,
                     long long total, uint8_t* __restrict__ out, const uint8_t* __restrict__ gt, long long* __restrict__ cm, int K,
                     long long stride) {
  native_labels_body<ENS, false>(scores, n0, n1, n2, C, map, m1, m2, total, out, gt, cm, K, stride, nullptr);
}

// pnp_native_accumulate: covered[q] is read and written by the one thread that samples voxel q
__global__ void __launch_bounds__(256)
native_accumulate_kernel(const float* __restrict__ scores, int n0, int n1, int n2, int C, const float* __restrict__ map, int m1, int m2,
                         long long total, float* __restrict__ sums, uint8_t* __restrict__ covered) {
  native_labels_body<false, true>(scores, n0, n1, n2, C, map, m1, m2, total, covered, nullptr, nullptr, 1, 0, sums);
}

// pnp_native_accumulated_labels: the first maximum of each covered voxel's sums, 0 where nothing covers it, with
// pnp_native_labels' (truth, prediction) counts
__global__ void __launch_bounds__(256)
native_accumulated_labels_kernel(const float* __restrict__ sums, const uint8_t* __restrict__ covered, int C, long long total,
                                 uint8_t* __restrict__ out, const uint8_t* __restrict__ gt, long long* __restrict__ cm) {
  __shared__ unsigned int hist[64];
  pnp_pdl_enter();
  if (cm) {
    if (threadIdx.x < 64) hist[threadIdx.x] = 0u;
    __syncthreads();
  }
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const unsigned q = (unsigned)i;
    int best = 0;
    if (__ldg(covered + q)) {
      const float* sum = sums + (long long)q * C;       // 64-bit: m0 m1 m2 C may reach 2^31
      float top = __ldg(sum);
#pragma unroll
      for (int c = 1; c < 8; ++c) {
        if (c >= C) break;
        const float v = __ldg(sum + c);
        if (v > top) {                   // strictly greater: the lowest index wins a tie (pnp_native_labels_ensemble's rule)
          top = v;
          best = c;
        }
      }
    }
    out[q] = (uint8_t)best;
    if (cm) {
      int g = __ldg(gt + q);
      if (g >= C) g = 0;
      atomicAdd(&hist[g * C + best], 1u);
    }
  }
  if (cm) {
    __syncthreads();
    if (threadIdx.x < C * C && hist[threadIdx.x])
      atomicAdd((unsigned long long*)cm + threadIdx.x, (unsigned long long)hist[threadIdx.x]);
  }
}

// ---- smooth noise field (pnp_smooth_noise_field): uniforms on [-1, 1) from Philox, a separable Gaussian along c, then along r
constexpr int NF_LINE = 256;          // pass 1: outputs per tile, one segment of one row
constexpr int NF_TC = 32, NF_TR = 64;  // pass 2: a tile of NF_TR rows x NF_TC columns, 256 threads as 8 row groups of 32 columns

// element e of the field: word e & 3 of Philox block e >> 2 of (seed, stream) -> fl32(x >> 8) 2^-23 - 1, exact in fp32
__device__ __forceinline__ float nf_uniform(unsigned long long seed, unsigned long long stream, unsigned long long e) {
  const uint4 x = pnp_philox4x32_10(make_uint4((uint32_t)(e >> 2), (uint32_t)(e >> 34), (uint32_t)stream, (uint32_t)(stream >> 32)),
                                    make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t w = (e & 2) ? ((e & 1) ? x.w : x.z) : ((e & 1) ? x.y : x.x);
  return __fsub_rn(__fmul_rn((float)(w >> 8), 0x1p-23f), 1.f);
}

// s = sum over t = 0 .. n-1 of w[t] x[t * stride], from +0 in increasing t, every product and sum rounded on its own
__device__ __forceinline__ float nf_taps(const float* ws, const float* x, int n, int stride) {
  float s = 0.f;
  for (int t = 0; t < n; ++t) s = __fadd_rn(s, __fmul_rn(ws[t], x[t * stride]));
  return s;
}

// pass 1: tile = NF_LINE outputs of one row (line = (b K + k) H + r); the uniforms of the tile and its +-R halo (0 outside the
// row) are generated into shared memory, so no noise buffer exists.
__global__ void __launch_bounds__(256)
noise_field_cols_kernel(unsigned long long seed, unsigned long long stream, int W, const float* __restrict__ taps, int R,
                        int tiles_per_line, long long tiles, float* __restrict__ tmp) {
  __shared__ float ws[2 * PNP_NF_MAX_R + 1];
  __shared__ float xs[NF_LINE + 2 * PNP_NF_MAX_R];
  pnp_pdl_enter();
  const int n = 2 * R + 1;
  for (int t = threadIdx.x; t < n; t += 256) ws[t] = __ldg(taps + t);
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long line = tile / tiles_per_line;
    const int c0 = (int)(tile - line * tiles_per_line) * NF_LINE;
    __syncthreads();                                       // the previous tile's reads (and the taps) are done
    for (int i = threadIdx.x; i < NF_LINE + 2 * R; i += 256) {
      const int c = c0 - R + i;
      xs[i] = (c >= 0 && c < W) ? nf_uniform(seed, stream, (unsigned long long)(line * W + c)) : 0.f;
    }
    __syncthreads();
    const int c = c0 + (int)threadIdx.x;
    if (c < W) tmp[line * W + c] = nf_taps(ws, xs + threadIdx.x, n, 1);
  }
}

// pass 2: tile = NF_TR rows x NF_TC columns of one plane (b K + k), its rows +-R halo (0 outside the plane) staged in shared
// memory; out = min(max(amp s, lo), hi)
__global__ void __launch_bounds__(256)
noise_field_rows_kernel(const float* __restrict__ tmp, int H, int W, const float* __restrict__ taps, int R, int tiles_r,
                        int tiles_c, long long tiles, float amp, float lo, float hi, float* __restrict__ out) {
  __shared__ float ws[2 * PNP_NF_MAX_R + 1];
  __shared__ float ys[(NF_TR + 2 * PNP_NF_MAX_R) * NF_TC];
  pnp_pdl_enter();
  const int n = 2 * R + 1;
  for (int t = threadIdx.x; t < n; t += 256) ws[t] = __ldg(taps + t);
  const int tx = threadIdx.x % NF_TC, ty = threadIdx.x / NF_TC;
  const long long plane_px = (long long)H * W;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long plane = tile / ((long long)tiles_r * tiles_c);
    const int rest = (int)(tile - plane * tiles_r * tiles_c);
    const int r0 = (rest / tiles_c) * NF_TR, c0 = (rest % tiles_c) * NF_TC;
    const float* src = tmp + plane * plane_px;
    __syncthreads();
    for (int i = threadIdx.x; i < (NF_TR + 2 * R) * NF_TC; i += 256) {
      const int r = r0 - R + i / NF_TC, c = c0 + i % NF_TC;
      ys[i] = (r >= 0 && r < H && c < W) ? src[(long long)r * W + c] : 0.f;
    }
    __syncthreads();
    const int c = c0 + tx;
    for (int rl = ty; rl < NF_TR; rl += 256 / NF_TC) {
      const int r = r0 + rl;
      if (r < H && c < W)
        out[plane * plane_px + (long long)r * W + c] = fminf(fmaxf(__fmul_rn(amp, nf_taps(ws, ys + rl * NF_TC + tx, n, NF_TC)), lo), hi);
    }
  }
}

// a product of positive ints below 2^31 (each factor is, so no partial product overflows)
bool count_below_2_31(std::initializer_list<int> dims) {
  long long n = 1;
  for (int d : dims) {
    n *= d;
    if (n >= (1LL << 31)) return false;
  }
  return true;
}

// the checks of pnp_resample_planes, shared by pnp_resample_planes_aug
int check_resample(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H, int W, int C,
                   const float* img, const long long* lab, int label_planes) {
  if (!mats || n0 <= 0 || n1 <= 0 || n2 <= 0 || B <= 0 || H <= 0 || W <= 0 || C <= 0) return PNP_ERR_BAD_ARG;
  if (label_planes != 0 && label_planes != 1 && label_planes != C) return PNP_ERR_UNSUPPORTED;
  if (!img && !label_planes) return PNP_ERR_BAD_ARG;
  if ((img && !vol) || (label_planes && (!cls || !lab))) return PNP_ERR_BAD_ARG;
  if (n0 > PNP_RS_MAX_DIM || n1 > PNP_RS_MAX_DIM || n2 > PNP_RS_MAX_DIM || H > PNP_RS_MAX_DIM || W > PNP_RS_MAX_DIM)
    return PNP_ERR_UNSUPPORTED;
  if (!count_below_2_31({n0, n1, n2}) || !count_below_2_31({B, H, W, C}) || !count_below_2_31({B, C, 9})) return PNP_ERR_UNSUPPORTED;
  return PNP_OK;
}

template <bool AUG>
int launch_resample(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H, int W, int C,
                    float* img, long long* lab, int label_planes, AugFields aug, void* stream) {
  const int Cw = (img || label_planes != 1) ? C : 1;
  const long long total = (long long)B * H * W * Cw;
  PNP_CUDA(pnp_launch(resample_planes_kernel<AUG>, grid_for(total, 256 * 4), 256, 0, (cudaStream_t)stream, vol, cls, n0, n1, n2, mats,
                      H, W, C, Cw, total, img, lab, label_planes, aug));
  return PNP_OK;
}

// the checks of pnp_native_labels, shared by pnp_native_labels_ensemble (whose every member has the shape n0 x n1 x n2 x C)
int check_native(const float* scores, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2, const uint8_t* out,
                 const uint8_t* gt, const long long* cm) {
  if (!scores || !map || !out || (!gt) != (!cm) || n0 <= 0 || n1 <= 0 || n2 <= 0 || m0 <= 0 || m1 <= 0 || m2 <= 0)
    return PNP_ERR_BAD_ARG;
  if (C < 2 || C > 8) return PNP_ERR_UNSUPPORTED;
  if (n0 > PNP_RS_MAX_DIM || n1 > PNP_RS_MAX_DIM || n2 > PNP_RS_MAX_DIM || m0 > PNP_RS_MAX_DIM || m1 > PNP_RS_MAX_DIM ||
      m2 > PNP_RS_MAX_DIM)
    return PNP_ERR_UNSUPPORTED;
  if (!count_below_2_31({n0, n1, n2, C}) || !count_below_2_31({m0, m1, m2})) return PNP_ERR_UNSUPPORTED;
  return PNP_OK;
}

template <bool ENS>
int launch_native(const float* scores, int K, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2, uint8_t* out,
                  const uint8_t* gt, long long* cm, void* stream) {
  const long long total = (long long)m0 * m1 * m2;
  const long long stride = (long long)n0 * n1 * n2 * C;
  if (cm) PNP_CUDA(cudaMemsetAsync(cm, 0, sizeof(long long) * C * C, (cudaStream_t)stream));
  PNP_CUDA(pnp_launch(native_labels_kernel<ENS>, grid_for(total, 256 * 4), 256, 0, (cudaStream_t)stream, scores, n0, n1, n2, C, map,
                      m1, m2, total, out, gt, cm, K, stride));
  return PNP_OK;
}

// the checks of the accumulator pair: sums [m0][m1][m2][C] may hold 2^31 floats or more (64-bit offsets), the voxel count may not
int check_accumulated(const float* sums, const uint8_t* covered, int m0, int m1, int m2, int C) {
  if (!sums || !covered || m0 <= 0 || m1 <= 0 || m2 <= 0) return PNP_ERR_BAD_ARG;
  if (C < 2 || C > 8) return PNP_ERR_UNSUPPORTED;
  if (m0 > PNP_RS_MAX_DIM || m1 > PNP_RS_MAX_DIM || m2 > PNP_RS_MAX_DIM || !count_below_2_31({m0, m1, m2})) return PNP_ERR_UNSUPPORTED;
  return PNP_OK;
}

}  // namespace

extern "C" int pnp_resample_planes(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H, int W,
                                   int C, float* img, long long* lab, int label_planes, void* stream) {
  const int rc = check_resample(vol, cls, n0, n1, n2, mats, B, H, W, C, img, lab, label_planes);
  if (rc != PNP_OK) return rc;
  return launch_resample<false>(vol, cls, n0, n1, n2, mats, B, H, W, C, img, lab, label_planes, AugFields{nullptr, nullptr, nullptr},
                                stream);
}

extern "C" int pnp_resample_planes_aug(const float* vol, const uint8_t* cls, int n0, int n1, int n2, const float* mats, int B, int H,
                                       int W, int C, float* img, long long* lab, int label_planes, const float* disp,
                                       const float* gain, const float* ab, void* stream) {
  const int rc = check_resample(vol, cls, n0, n1, n2, mats, B, H, W, C, img, lab, label_planes);
  if (rc != PNP_OK) return rc;
  if (!img && (gain || ab)) return PNP_ERR_BAD_ARG;
  if (disp && !count_below_2_31({B, 2, H, W})) return PNP_ERR_UNSUPPORTED;
  return launch_resample<true>(vol, cls, n0, n1, n2, mats, B, H, W, C, img, lab, label_planes, AugFields{disp, gain, ab}, stream);
}

extern "C" int pnp_smooth_noise_field(unsigned long long seed, unsigned long long stream_id, int B, int K, int H, int W,
                                      const float* taps, int R, float amp, float lo, float hi, float* out, float* tmp, void* stream) {
  if (!taps || !out || !tmp || out == tmp || B <= 0 || K <= 0 || H <= 0 || W <= 0 || R < 0) return PNP_ERR_BAD_ARG;
  if (!(lo <= hi) || !(amp == amp)) return PNP_ERR_BAD_ARG;
  if (R > PNP_NF_MAX_R || !count_below_2_31({B, K, H, W})) return PNP_ERR_UNSUPPORTED;
  const int tiles_per_line = pnp_cdiv(W, NF_LINE), tiles_r = pnp_cdiv(H, NF_TR), tiles_c = pnp_cdiv(W, NF_TC);
  const long long t1 = (long long)B * K * H * tiles_per_line, t2 = (long long)B * K * tiles_r * tiles_c;
  PNP_CUDA(pnp_launch(noise_field_cols_kernel, grid_for(t1, 1), 256, 0, (cudaStream_t)stream, seed, stream_id, W, taps, R,
                      tiles_per_line, t1, tmp));
  PNP_CUDA(pnp_launch(noise_field_rows_kernel, grid_for(t2, 1), 256, 0, (cudaStream_t)stream, (const float*)tmp, H, W, taps, R,
                      tiles_r, tiles_c, t2, amp, lo, hi, out));
  return PNP_OK;
}

extern "C" int pnp_native_labels(const float* scores, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2,
                                 uint8_t* out, const uint8_t* gt, long long* cm, void* stream) {
  const int rc = check_native(scores, n0, n1, n2, C, map, m0, m1, m2, out, gt, cm);
  if (rc != PNP_OK) return rc;
  return launch_native<false>(scores, 1, n0, n1, n2, C, map, m0, m1, m2, out, gt, cm, stream);
}

extern "C" int pnp_native_labels_ensemble(const float* scores, int K, int n0, int n1, int n2, int C, const float* maps, int m0, int m1,
                                          int m2, uint8_t* out, const uint8_t* gt, long long* cm, void* stream) {
  if (K <= 0 || !maps) return PNP_ERR_BAD_ARG;
  const int rc = check_native(scores, n0, n1, n2, C, maps, m0, m1, m2, out, gt, cm);
  if (rc != PNP_OK) return rc;
  if (K > PNP_NATIVE_MAX_MEMBERS) return PNP_ERR_UNSUPPORTED;
  return launch_native<true>(scores, K, n0, n1, n2, C, maps, m0, m1, m2, out, gt, cm, stream);
}

extern "C" int pnp_native_accumulate(const float* scores, int n0, int n1, int n2, int C, const float* map, int m0, int m1, int m2,
                                     float* sums, uint8_t* covered, void* stream) {
  if (!sums) return PNP_ERR_BAD_ARG;
  const int rc = check_native(scores, n0, n1, n2, C, map, m0, m1, m2, covered, nullptr, nullptr);
  if (rc != PNP_OK) return rc;
  const long long total = (long long)m0 * m1 * m2;
  PNP_CUDA(pnp_launch(native_accumulate_kernel, grid_for(total, 256 * 4), 256, 0, (cudaStream_t)stream, scores, n0, n1, n2, C, map, m1,
                      m2, total, sums, covered));
  return PNP_OK;
}

extern "C" int pnp_native_accumulated_labels(const float* sums, const uint8_t* covered, int m0, int m1, int m2, int C, uint8_t* out,
                                             const uint8_t* gt, long long* cm, void* stream) {
  if (!out || (!gt) != (!cm)) return PNP_ERR_BAD_ARG;
  const int rc = check_accumulated(sums, covered, m0, m1, m2, C);
  if (rc != PNP_OK) return rc;
  const long long total = (long long)m0 * m1 * m2;
  if (cm) PNP_CUDA(cudaMemsetAsync(cm, 0, sizeof(long long) * C * C, (cudaStream_t)stream));
  PNP_CUDA(pnp_launch(native_accumulated_labels_kernel, grid_for(total, 256 * 4), 256, 0, (cudaStream_t)stream, sums, covered, C, total,
                      out, gt, cm));
  return PNP_OK;
}
