// wgmma + TMA implicit-GEMM convolution for sm_90a (Hopper H100).
//
// Replaces tf.nn.conv2d / tf.nn.atrous_conv2d (layers.py:18,67,86) for the dense layers that carry the
// FLOPs of the PnP-AdaNet hot path: kxk convolutions (dilated or strided) with Cin and Cout each a multiple of 64, or exactly
// 32 or 16 -- groups 3..10 of the segmenter and most of the feature discriminator -- and their data gradients (a stride-1
// dgrad is the same convolution with flipped taps and swapped channels) and weight gradients.
//
// Formulation: D[m, n] = sum_{tap, c} A_tap[m, c] * W_tap[n, c]
//   m = output pixel inside a tile of (tn images) x (th rows) x (tw cols), tn*th*tw <= 128
//   A_tap tile = one 4-D TMA box {BK ch, tw, th, tn} of the NHWC bf16 activation plane at the
//                tap-shifted coordinate; TMA zero-fills out-of-range pixels, which *is* the zero padding
//   W_tap tile = one 2-D TMA box {BK ch, BLOCK_N} of the [tap][Cout][Cin] bf16 weight plane
//   both land in shared memory K-major with the 128/64/32-byte swizzle and are consumed straight from shared memory by
//   wgmma.mma_async (bf16 x bf16 -> fp32); the accumulator lives in the registers of the two consumer warpgroups, whose
//   epilogue streams it to HBM (dropout / accumulate / BN partial statistics / inference BN + skip + activation fused).
//
// Precision: fp32 operands are pre-split into bf16 (hi, lo) planes (pnp_split_bf16).  NTERMS == 3 issues
// hi*hi + hi*lo + lo*hi (error ~2^-16 per product: meets the 1e-3 parity bar through 36 layers);
// NTERMS == 1 is the plain bf16 path of BASELINE config 5.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (accumulator rows 0..63 and 64..127: one m64nNk16 wgmma
// each per K step), warp 8 = TMA producer (one lane).  Tiles of at most 64 columns run two CTAs per SM (96 registers per
// thread, half the shared-memory ring each), the 128-column tiles one.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <cuda_bf16.h>
#include "common.cuh"
#include "../../include/pnp_b200.h"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // bf16 elements = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int CONSUMER_THREADS = 256;
constexpr int CONSUMER_WARPS = CONSUMER_THREADS / 32;
constexpr int TC_THREADS = CONSUMER_THREADS + 32;

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a broken TMA descriptor / barrier protocol must trap, never hang the GPU.  No printf here: a function call
// between wgmma issue and wgmma.wait_group makes ptxas serialize every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > 4000000000ull) __trap();   // 4 s
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// the consumer warpgroups only (the producer warp never joins): named barrier 1
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory"); }

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers while an asynchronous wgmma may still write them
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma.mma_async m64nNk16, bf16 x bf16 -> fp32 in registers; both operands from shared memory descriptors.
// TA / TB: 0 = K-major, 1 = MN-major (transposed) operand.  scale_d == 0 overwrites the accumulator.

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7"
      "}, %8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (N == 16) wgmma_m64n16k16<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 32) wgmma_m64n32k16<TA, TB>(d, da, db, scale_d);
  else if constexpr (N == 64) wgmma_m64n64k16<TA, TB>(d, da, db, scale_d);
  else wgmma_m64n128k16<TA, TB>(d, da, db, scale_d);
}

// Shared-memory matrix descriptor of wgmma: [0,14) start address >> 4, [16,30) leading byte offset >> 4, [32,46) stride byte
// offset >> 4, [62,64) swizzle (1 = 128B, 2 = 64B, 3 = 32B).  All tiles are 1024-byte aligned (base offset 0).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, int swizzle) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)swizzle << 62;
  return d;
}
// K-major operand tile whose rows are BK bf16 wide: BK = 64 -> 128-byte rows, SWIZZLE_128B (8-row group = 1024 B);
// BK = 32 -> 64-byte rows, SWIZZLE_64B (512 B); BK = 16 -> 32-byte rows, SWIZZLE_32B (256 B).  The narrow tiles serve the
// Cin = 32 / 16 layers natively (no zero-padded K).  The leading byte offset is unused for swizzled K-major tiles.
template <int BK>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
  return make_smem_desc(smem_addr, 16, 8 * BK * 2, BK == 64 ? 1 : (BK == 32 ? 2 : 3));
}

__device__ __forceinline__ void split1(float x, uint16_t& hi, uint16_t& lo) {
  __nv_bfloat16 h = __float2bfloat16_rn(x);
  __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
  hi = __bfloat16_as_ushort(h);
  lo = __bfloat16_as_ushort(l);
}

constexpr int MAX_TAPS = 25;
struct TcArgs {
  int B, OH, OW, Cout;        // full output tensor [B, OH, OW, Cout]
  int U, V;                   // extent of the tiled grid: output pixel (u, v) -> (u*out_mul + out_py, v*out_mul + out_px)
  int out_mul, out_py, out_px;
  int in_mul;                 // TMA coordinate of tile origin = origin * in_mul + tap offset (stride of a strided forward conv)
  int Cin;                    // GEMM K per tap
  int kchunks;                // Cin / BK
  int ntaps;
  short tap_oy[MAX_TAPS], tap_ox[MAX_TAPS];
  int tap_wrow[MAX_TAPS];     // first row of the tap's [N][K] slab in the weight plane
  int tw, th, tn;             // pixel tile
  int tiles_x, tiles_y, tiles_n;
  int accumulate;
  PnpDropout drop;
  double* bn_sum;
  double* bn_sumsq;
  // fused epilogue (forward only): y = act(z * ep_scale[c] + ep_shift[c] + skip) -- inference-mode batch norm, the residual
  // add with channel-pad skip and the activation folded into the convolution; optional bf16 (hi, lo) planes of y for the next
  // tensor-core convolution; out may be null when only the planes are wanted
  const float* ep_scale;
  const float* ep_shift;
  const float* ep_skip;
  int ep_skip_c, ep_skip_off, ep_act;
  uint16_t* out_hi;
  uint16_t* out_lo;
  // phases: a strided data gradient is s*s independent stride-1 convolutions ("phases"), each over its own subset of the
  // taps (every tap belongs to exactly one phase) and its own output sub-grid; all of them run in ONE persistent launch.
  int total_tiles;            // all phases, all (m, n) tiles, times ksplit
  int rot_mul;                // k-loop rotation per m-tile (see the producer)
  int taps_inner;             // k-block order: 1 = channel chunk outer / taps inner (the shifted windows of one chunk hit L2)
  int ksplit;                 // > 1: each (m, n) tile's k-blocks are divided among ksplit CTAs that atomically add their partial
                              // sums into a zeroed output (few-tile, deep-K layers: 4x4 / 16x16 maps with 512 channels)
  int nphases;                // 0: single phase described by the fields above
  struct Phase {
    short tap_begin, tap_count, py, px;
    int U, V, tiles_x, tiles_y, tile_base;    // tile_base: first global tile id of this phase
  } ph[16];
};

struct TileCoord {
  int x0, y0, img0, n0, tap_begin, tap_count, U, V, py, px, kb_begin, kb_count, mt;
};

template <int BLOCK_N>
__device__ __forceinline__ TileCoord decode_tile(const TcArgs& a, int t, int n_tiles) {
  TileCoord c;
  int tiles_x = a.tiles_x, tiles_y = a.tiles_y;
  int ks = 0;
  if (a.ksplit > 1) { ks = t % a.ksplit; t /= a.ksplit; }
  c.tap_begin = 0; c.tap_count = a.ntaps; c.U = a.U; c.V = a.V; c.py = a.out_py; c.px = a.out_px;
  if (a.nphases > 0) {
    int p = 0;
    while (p + 1 < a.nphases && t >= a.ph[p + 1].tile_base) ++p;
    t -= a.ph[p].tile_base;
    tiles_x = a.ph[p].tiles_x; tiles_y = a.ph[p].tiles_y;
    c.tap_begin = a.ph[p].tap_begin; c.tap_count = a.ph[p].tap_count;
    c.U = a.ph[p].U; c.V = a.ph[p].V; c.py = a.ph[p].py; c.px = a.ph[p].px;
  }
  int mt = t / n_tiles;
  c.mt = mt;
  c.n0 = (t - mt * n_tiles) * BLOCK_N;
  const int txi = mt % tiles_x;
  mt /= tiles_x;
  const int tyi = mt % tiles_y;
  const int tni = mt / tiles_y;
  c.x0 = txi * a.tw; c.y0 = tyi * a.th; c.img0 = tni * a.tn;
  const int nkb = c.tap_count * a.kchunks;
  if (a.ksplit > 1) {
    c.kb_begin = (int)((long long)nkb * ks / a.ksplit);
    c.kb_count = (int)((long long)nkb * (ks + 1) / a.ksplit) - c.kb_begin;
  } else {
    c.kb_begin = 0; c.kb_count = nkb;
  }
  return c;
}

// k-block i of a tile -> (absolute tap, channel chunk)
__device__ __forceinline__ void kblock_of(const TcArgs& a, const TileCoord& tc, int i, int kchunks, int& tap, int& kc) {
  const int rot = (tc.kb_count >= 16) ? (int)(((long long)tc.mt * a.rot_mul) % tc.kb_count) : 0;
  int kr = i + rot;
  if (kr >= tc.kb_count) kr -= tc.kb_count;
  const int kb = tc.kb_begin + kr;
  int tl;
  if (a.taps_inner) { kc = kb / tc.tap_count; tl = kb - kc * tc.tap_count; }
  else { tl = kb / kchunks; kc = kb - tl * kchunks; }
  tap = tc.tap_begin + tl;
}

// CTAs resident per SM: two for the accumulators of at most 64 columns (32 fp32 registers per thread), so that one CTA's
// epilogue runs while the other issues MMAs; the 128-column tiles need more than the 96 registers per thread two CTAs of
// 288 threads can have (registers are allocated per 16K-register SM sub-partition, and 18 warps put five on one), and stay
// at one
constexpr int tc_ctas_per_sm(int block_n) { return block_n <= 64 ? 2 : 1; }

template <int BLOCK_N, int NTERMS, int BK, int CTAS_PER_SM>
struct TcCfg {
  static constexpr int A_TILE_BYTES = BLOCK_M * BK * 2;
  static constexpr int B_TILE_BYTES = BLOCK_N * BK * 2;
  static constexpr int NPLANES = (NTERMS == 1) ? 1 : 2;
  static constexpr int STAGE_BYTES = NPLANES * (A_TILE_BYTES + B_TILE_BYTES);
  // the ~200 KB ring budget of an SM is shared by its resident CTAs
  static constexpr int STAGES_RAW = (200 * 1024 / CTAS_PER_SM) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  // fp64 BN partial sums of the current n-tile, one [sum | sumsq][BLOCK_N] row per consumer warp (16 KB at BLOCK_N = 128)
  static constexpr int STAT_BYTES = CONSUMER_WARPS * 2 * BLOCK_N * 8;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAT_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(STAGES >= 2, "pipeline needs two stages");
  // the ring is sized before the statistics rows: they must fit beside it, never cost it a stage
  static_assert(SMEM_BYTES <= 227 * 1024, "H100 allows 227 KB of shared memory per block");
  // every resident CTA also takes 1 KB of shared memory the system reserves, out of the SM's 228 KB
  static_assert(CTAS_PER_SM * (SMEM_BYTES + 1024) <= 228 * 1024, "the resident CTAs must fit in one SM's shared memory");
};

// 32-bit word k (0..3, may differ per lane) of a Philox block
__device__ __forceinline__ uint32_t word_of(const uint4& r, int k) { return k == 0 ? r.x : k == 1 ? r.y : k == 2 ? r.z : r.w; }

template <int BLOCK_N, int NTERMS, int BK, int CTAS_PER_SM>
__global__ void __launch_bounds__(TC_THREADS, CTAS_PER_SM)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
               float* __restrict__ out, TcArgs a) {
  pnp_pdl_trigger();      // the wait comes after the prologue (barriers, tensor-map prefetch touch no predecessor data)
  // PERSISTENT: CTAS_PER_SM CTAs per SM walk tiles t = blockIdx.x, blockIdx.x + gridDim.x, ...; the smem ring and its phases
  // run across tile boundaries, so the producer prefetches the next tile's operands while the consumers run the epilogue, and
  // with two CTAs on an SM the other CTA's MMAs run during it too.
  using Cfg = TcCfg<BLOCK_N, NTERMS, BK, CTAS_PER_SM>;
  constexpr int A_TILE_BYTES = Cfg::A_TILE_BYTES;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int ACC = BLOCK_N / 2;                   // fp32 accumulator registers per thread (m64 x BLOCK_N per warpgroup)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  double* stat = reinterpret_cast<double*>(smem + STAGES * Cfg::STAGE_BYTES);    // [consumer warp][sum | sumsq][BLOCK_N]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stat + CONSUMER_WARPS * 2 * BLOCK_N);   // [0..S) full, [S..2S) empty

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tiles = a.Cout / BLOCK_N;
  const int kchunks = a.kchunks;
  const bool bn_on = a.bn_sum != nullptr;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_b_hi);
    if (NTERMS > 1) { tma_prefetch_desc(&map_a_lo); tma_prefetch_desc(&map_b_lo); }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);
      mbar_init(smem_u32(&bars[STAGES + s]), CONSUMER_WARPS);     // one arrival per consumer warp frees a slot
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < CONSUMER_WARPS * 2 * BLOCK_N; i += TC_THREADS) stat[i] = 0.0;
  __syncthreads();
  pnp_pdl_wait();                             // from here on the predecessor kernel's results are read / its buffers written

  if (warp == CONSUMER_WARPS) {
    // ================= TMA producer =================
    if (lane == 0) {
      const uint32_t box_a_bytes = (uint32_t)(a.tw * a.th * a.tn) * BK * 2;
      const uint32_t tx_bytes = Cfg::NPLANES * (box_a_bytes + (uint32_t)Cfg::B_TILE_BYTES);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        const TileCoord tc = decode_tile<BLOCK_N>(a, t, n_tiles);
        // CTAs that share a weight tile (same n0, different m-tile) would otherwise request the same L2 lines in lockstep;
        // rotating each m-tile's starting k-block spreads those requests over the whole weight slab (sum order is free)
        for (int i = 0; i < tc.kb_count; ++i) {
          int tap, kc;
          kblock_of(a, tc, i, kchunks, tap, kc);
          mbar_wait(smem_u32(&bars[STAGES + stage]), phase ^ 1);
          const uint32_t full = smem_u32(&bars[stage]);
          mbar_expect_tx(full, tx_bytes);
          uint8_t* st = smem + stage * Cfg::STAGE_BYTES;
          const int cx = tc.x0 * a.in_mul + a.tap_ox[tap];
          const int cy = tc.y0 * a.in_mul + a.tap_oy[tap];
          const int wrow = a.tap_wrow[tap] + tc.n0;
          tma_load_4d(smem_u32(st), &map_a_hi, full, kc * BK, cx, cy, tc.img0);
          tma_load_2d(smem_u32(st + Cfg::NPLANES * A_TILE_BYTES), &map_b_hi, full, kc * BK, wrow);
          if (NTERMS > 1) {
            tma_load_4d(smem_u32(st + A_TILE_BYTES), &map_a_lo, full, kc * BK, cx, cy, tc.img0);
            tma_load_2d(smem_u32(st + 2 * A_TILE_BYTES + Cfg::B_TILE_BYTES), &map_b_lo, full, kc * BK, wrow);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ================= consumer warpgroups: MMA + epilogue =================
  // wgmma accumulator layout (m64nN, fp32): thread (warp w of the warpgroup, lane l) holds rows 16w + l/4 and 16w + l/4 + 8,
  // and of every 8-column group j the columns 8j + 2(l%4) + {0, 1}: d[4j + {0,1}] in the first row, d[4j + {2,3}] in the second
  const int wg = warp >> 2;
  const int q = lane & 3;
  const int cq = q * 2;
  const int per_img = a.th * a.tw;
  const bool drop_on = a.drop.seed_ptr != nullptr;
  unsigned long long seed = 0ull;
  if (drop_on) seed = *a.drop.seed_ptr;
  // At two CTAs per SM a thread has 96 registers, a third of them the accumulator.  The empty asm statements guarded by
  // SHORT_LIVES below keep the compiler from holding values over the K loop or the epilogue's loops that it can form again
  // cheaply; the one-CTA instantiations have the registers to spare and are compiled as before.
  constexpr bool SHORT_LIVES = CTAS_PER_SM > 1;
  // BN partial statistics: warp-reduced in fp32, then summed in fp64 over every tile of this CTA that shares an n-tile, in the
  // warp's own shared-memory row (one writer per slot: plain adds, no shared-memory atomics, which sm_90 runs as CAS loops on
  // fp64).  When the n-tile changes (and at the end) the eight rows are summed in a fixed order and each column takes one fp64
  // global atomic, not one per tile.
  double* wstat = stat + warp * 2 * BLOCK_N;
  int stat_n0 = -1;
  auto flush_stats = [&]() {
    consumer_sync();
    for (int i = threadIdx.x; i < 2 * BLOCK_N; i += CONSUMER_THREADS) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < CONSUMER_WARPS; ++w) {
        t += stat[w * 2 * BLOCK_N + i];
        stat[w * 2 * BLOCK_N + i] = 0.0;
      }
      atomicAdd((i < BLOCK_N ? a.bn_sum : a.bn_sumsq) + stat_n0 + (i % BLOCK_N), t);
    }
    consumer_sync();
  };

  float acc[ACC];
  int stage = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
    const TileCoord tk = decode_tile<BLOCK_N>(a, t, n_tiles);
    if (bn_on && tk.n0 != stat_n0) {
      if (stat_n0 >= 0) flush_stats();
      stat_n0 = tk.n0;
    }
    const int kb_count = tk.kb_count;
    if (kb_count == 0) {
#pragma unroll
      for (int i = 0; i < ACC; ++i) acc[i] = 0.f;
    }
    int prev = -1;
    for (int kb = 0; kb < kb_count; ++kb) {
      mbar_wait(smem_u32(&bars[stage]), phase);
      wgmma_fence();
      const uint32_t st = smem_u32(smem + stage * Cfg::STAGE_BYTES);
      const uint32_t a_hi = st + wg * 64 * BK * 2;      // this warpgroup's 64 activation rows
      const uint32_t a_lo = a_hi + A_TILE_BYTES;
      const uint32_t b_hi = st + Cfg::NPLANES * A_TILE_BYTES;
      const uint32_t b_lo = b_hi + Cfg::B_TILE_BYTES;
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k) {
        const uint32_t koff = k * WGMMA_K * 2;   // bytes inside the swizzled row
        const uint64_t da_hi = make_kmajor_desc<BK>(a_hi + koff);
        const uint64_t db_hi = make_kmajor_desc<BK>(b_hi + koff);
        if (NTERMS > 1) {
          const uint64_t da_lo = make_kmajor_desc<BK>(a_lo + koff);
          const uint64_t db_lo = make_kmajor_desc<BK>(b_lo + koff);
          // small cross terms first, then the dominant hi*hi term
          wgmma_bf16<BLOCK_N, 0, 0>(acc, da_lo, db_hi, (kb | k) != 0);
          wgmma_bf16<BLOCK_N, 0, 0>(acc, da_hi, db_lo, 1);
          wgmma_bf16<BLOCK_N, 0, 0>(acc, da_hi, db_hi, 1);
        } else {
          wgmma_bf16<BLOCK_N, 0, 0>(acc, da_hi, db_hi, (kb | k) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                 // the previous stage's MMAs have retired: hand its slot back to the producer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars[STAGES + prev]));
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars[STAGES + prev]));
    }

    // the tile's coordinates: with SHORT_LIVES decoded again rather than held over the K loop (the asm hides that t_ep is
    // the t decoded above); otherwise the compiler merges this with the decode above
    int t_ep = t;
    if constexpr (SHORT_LIVES) asm volatile("" : "+r"(t_ep));
    const TileCoord tc = decode_tile<BLOCK_N>(a, t_ep, n_tiles);
    const int n0 = tc.n0;
    // the rows' coordinates are derived per tile rather than kept live across the K loop
    long long pix[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;     // accumulator row = pixel index inside the tile
      const int rni = m / per_img;
      const int rem = m - rni * per_img;
      const int ryy = rem / a.tw;
      const int img = tc.img0 + rni, u = tc.y0 + ryy, v_ = tc.x0 + (rem - ryy * a.tw);
      valid[h] = (rni < a.tn) && (img < a.B) && (u < tc.U) && (v_ < tc.V);
      const int oy = u * a.out_mul + tc.py, ox = v_ * a.out_mul + tc.px;
      pix[h] = ((long long)img * a.OH + oy) * a.OW + ox;
    }
    if (drop_on) {
      // element e draws half (e & 1) of word (e & 7) >> 1 of the Philox block e >> 3 (pnp_dropout_mult8), so the four lanes of
      // a quad (one row; columns 2q, 2q + 1 of every 8-column group) need the same block, word q each.  Lane q draws the block
      // of group 4 jg + q, and three xor shuffles transpose the quad's 4 x 4 words: got[s] = word q of the block of group
      // 4 jg + (q ^ s).  Invalid rows (and, at 16 columns, the groups past the tile) draw too, unused, so that every lane
      // reaches every shuffle.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const unsigned long long blk0 = (unsigned long long)(pix[h] * a.Cout + n0 + q * 8) >> 3;
#pragma unroll
        for (int jg = 0; jg < (BLOCK_N / 8 + 3) / 4; ++jg) {
          const uint4 blk = pnp_dropout_bits8(a.drop, seed, blk0 + 4 * jg);
          uint32_t got[4];
          got[0] = word_of(blk, q);
#pragma unroll
          for (int s = 1; s < 4; ++s) got[s] = __shfl_xor_sync(0xffffffffu, word_of(blk, q ^ s), s);
#pragma unroll
          for (int jq = 0; jq < 4; ++jq) {
            const int j = 4 * jg + jq;
            if (j >= BLOCK_N / 8) break;
            const int sj = q ^ jq;
            const uint32_t w = sj == 0 ? got[0] : sj == 1 ? got[1] : sj == 2 ? got[2] : got[3];
            acc[4 * j + 2 * h] *= pnp_drop_sel(a.drop, w & 0xffffu);
            acc[4 * j + 2 * h + 1] *= pnp_drop_sel(a.drop, w >> 16);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int c0 = j * 8 + cq;                     // column inside the tile
      const int ch = n0 + c0;
      float v[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        v[h][0] = acc[4 * j + 2 * h];
        v[h][1] = acc[4 * j + 2 * h + 1];
      }
      if (bn_on) {
        float s0 = (valid[0] ? v[0][0] : 0.f) + (valid[1] ? v[1][0] : 0.f);
        float s1 = (valid[0] ? v[0][1] : 0.f) + (valid[1] ? v[1][1] : 0.f);
        float q0 = (valid[0] ? v[0][0] * v[0][0] : 0.f) + (valid[1] ? v[1][0] * v[1][0] : 0.f);
        float q1 = (valid[0] ? v[0][1] * v[0][1] : 0.f) + (valid[1] ? v[1][1] * v[1][1] : 0.f);
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) {      // over the 8 lanes that share these columns: the warp's 16 rows
          s0 += __shfl_xor_sync(0xffffffffu, s0, off);
          s1 += __shfl_xor_sync(0xffffffffu, s1, off);
          q0 += __shfl_xor_sync(0xffffffffu, q0, off);
          q1 += __shfl_xor_sync(0xffffffffu, q1, off);
        }
        // lanes q, q + 4, .., q + 28 now hold the same four sums of columns c0, c0 + 1; lane 4r + q adds the r-th of them
        if (lane < 16) {
          const int r = lane >> 2;
          const float x = r == 0 ? s0 : r == 1 ? s1 : r == 2 ? q0 : q1;
          wstat[(r >> 1) * BLOCK_N + c0 + (r & 1)] += (double)x;
        }
      }
      float2 sc = make_float2(1.f, 1.f), sh = make_float2(0.f, 0.f);
      if (a.ep_scale != nullptr) {
        sc = __ldg(reinterpret_cast<const float2*>(a.ep_scale + ch));
        sh = __ldg(reinterpret_cast<const float2*>(a.ep_shift + ch));
      }
      const bool skip_on = a.ep_skip != nullptr && ch >= a.ep_skip_off && ch < a.ep_skip_off + a.ep_skip_c;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!valid[h]) continue;
        // with SHORT_LIVES the row's addresses are formed per column group: hoisted out of the unrolled loop, the 64-bit row
        // pointers of y, its planes and the skip would take a dozen registers through the whole column loop
        long long p = pix[h];
        if constexpr (SHORT_LIVES) asm volatile("" : "+l"(p));
        float2 o = make_float2(v[h][0], v[h][1]);
        if (a.ep_scale != nullptr) { o.x = fmaf(o.x, sc.x, sh.x); o.y = fmaf(o.y, sc.y, sh.y); }
        if (skip_on) {
          const float2 sk = __ldg(reinterpret_cast<const float2*>(a.ep_skip + p * a.ep_skip_c - a.ep_skip_off + ch));
          o.x += sk.x; o.y += sk.y;
        }
        // positive subnormals go to +0, as in elementwise.cu act_fwd: the hi plane of y then carries the sign of y exactly
        // (rn_bf16 sends 0 < y <= 2^-134 to +0), which the backward kernels read instead of y
        constexpr float kMinNormal = 1.17549435e-38f;   // FLT_MIN
        if (a.ep_act == PNP_ACT_RELU) {
          o.x = o.x >= kMinNormal ? o.x : 0.f; o.y = o.y >= kMinNormal ? o.y : 0.f;
        } else if (a.ep_act == PNP_ACT_LRELU) {
          o.x = o.x >= kMinNormal ? o.x : (o.x > 0.f ? 0.f : 0.2f * o.x);
          o.y = o.y >= kMinNormal ? o.y : (o.y > 0.f ? 0.f : 0.2f * o.y);
        }
        const long long e0 = p * a.Cout + ch;        // flat element index of this thread's pair
        if (out != nullptr) {
          float2* dst = reinterpret_cast<float2*>(out + e0);
          if (a.ksplit > 1) {
            atomicAdd(dst, o);
          } else {
            if (a.accumulate) {
              const float2 p = *dst;
              o.x += p.x; o.y += p.y;
            }
            *dst = o;
          }
        }
        if (a.out_hi != nullptr) {
          uint16_t h0, l0, h1, l1;
          split1(o.x, h0, l0);
          split1(o.y, h1, l1);
          *reinterpret_cast<uint32_t*>(a.out_hi + e0) = (uint32_t)h0 | ((uint32_t)h1 << 16);
          if (a.out_lo) *reinterpret_cast<uint32_t*>(a.out_lo + e0) = (uint32_t)l0 | ((uint32_t)l1 << 16);
        }
      }
    }
  }
  if (bn_on && stat_n0 >= 0) flush_stats();
}


// ---------------------------------------------------------------------------------------------
// operand preparation
// ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256)
split_bf16_kernel(const float* __restrict__ x, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, long long n) {
  pnp_pdl_enter();
  long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    ushort4 h, l;
    split1(v.x, h.x, l.x); split1(v.y, h.y, l.y); split1(v.z, h.z, l.z); split1(v.w, h.w, l.w);
    reinterpret_cast<ushort4*>(hi)[i] = h;
    if (lo) reinterpret_cast<ushort4*>(lo)[i] = l;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    long long i = (n4 << 2) + threadIdx.x;
    uint16_t h, l;
    split1(x[i], h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

// [rows, C] fp32 -> [rows, Cpad] bf16 planes, channels >= C zero (lets Cin = 32 layers ride the 64-channel K chunk)
__global__ void __launch_bounds__(256)
split_bf16_pad_kernel(const float* __restrict__ x, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, long long rows, int C,
                      int Cpad) {
  pnp_pdl_enter();
  const int q4 = Cpad >> 2;
  long long total = rows * q4;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    long long r = i / q4;
    int c = (int)(i - r * q4) * 4;
    ushort4 h = make_ushort4(0, 0, 0, 0), l = make_ushort4(0, 0, 0, 0);
    if (c < C) {
      float4 v = __ldg(reinterpret_cast<const float4*>(x + r * C + c));
      split1(v.x, h.x, l.x); split1(v.y, h.y, l.y); split1(v.z, h.z, l.z); split1(v.w, h.w, l.w);
    }
    reinterpret_cast<ushort4*>(hi)[i] = h;
    if (lo) reinterpret_cast<ushort4*>(lo)[i] = l;
  }
}

// w HWIO [taps][Cin][Cout] -> fwd : out[tap][co][ci]          (B operand rows = co, K = ci)
//                             dgrad: out[tap][ci][co]          (B operand rows = ci, K = co)
__global__ void __launch_bounds__(256)
split_weight_kernel(const float* __restrict__ w, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int taps, int Cin,
                    int Cout, int for_dgrad, int CinP) {
  pnp_pdl_enter();
  __shared__ float tile[32][33];
  const int tap = blockIdx.z;
  const float* src = w + (long long)tap * Cin * Cout;
  if (for_dgrad) {
    long long obase = (long long)tap * Cin * Cout;
    int ci = blockIdx.y * 32 + threadIdx.y * 4;
    int co = blockIdx.x * 32 + threadIdx.x;
    for (int r = 0; r < 4; ++r) {
      if (ci + r < Cin && co < Cout) {
        uint16_t h, l;
        split1(src[(long long)(ci + r) * Cout + co], h, l);
        hi[obase + (long long)(ci + r) * Cout + co] = h;
        if (lo) lo[obase + (long long)(ci + r) * Cout + co] = l;
      }
    }
    return;
  }
  int ci0 = blockIdx.y * 32, co0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int ci = ci0 + r, co = co0 + threadIdx.x;
    tile[r][threadIdx.x] = (ci < Cin && co < Cout) ? src[(long long)ci * Cout + co] : 0.f;
  }
  __syncthreads();
  long long obase = (long long)tap * CinP * Cout;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int co = co0 + r, ci = ci0 + threadIdx.x;
    if (co < Cout && ci < CinP) {       // ci in [Cin, CinP): zero padding (tile[] holds 0 there)
      uint16_t h, l;
      split1(tile[threadIdx.x][r], h, l);
      hi[obase + (long long)co * CinP + ci] = h;
      if (lo) lo[obase + (long long)co * CinP + ci] = l;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host: tensor maps
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// ---------------------------------------------------------------------------------------------
// wgrad on wgmma:  dW[tap][ci][co] += sum_pixels x[pixel + tap offset][ci] * dy[pixel][co]
//   GEMM per tap: M = ci (128 per CTA, 64 per consumer warpgroup), N = co (BLOCK_N), K = pixels.  Both operands are
//   *MN-major*: the very same NHWC TMA boxes {64 ch, tw, th, tn} as the forward pass (one 128-byte row per pixel = one K index,
//   64 channels = 64 M/N indices), two boxes side by side for 128/BLOCK_N channels (leading byte offset = box size), 8-pixel
//   swizzle atoms 1024 B apart (stride byte offset).  The pixel range is split across CTAs (gridDim.y); partial tiles are added
//   to the fp32 gradient arena with vector atomics.
// ---------------------------------------------------------------------------------------------
constexpr int WG_PB = 64;                                  // pixels per pipeline stage
constexpr int WG_BOX_BYTES = WG_PB * BLOCK_K * 2;          // one {64 ch x 64 px} box = 8 KB

struct WgArgs {
  int B, Cin, Cout;
  int ntaps;
  // taps packed along the 128-row M tile: 1 = 128 consecutive channels of one tap (two 64-channel boxes); 2 = Cin 64: two taps;
  // 4 = Cin 32: four taps of 32-channel (64-byte, SWIZZLE_64B) boxes -- a narrow layer still fills the whole MMA
  int pack, ngroups;
  short tap_oy[MAX_TAPS], tap_ox[MAX_TAPS];
  int in_mul;
  int tw, th, tn, tiles_x, tiles_y, tiles_n;
  int num_pb, pb_per_split;
  int mt, nt;
  float* dw;
};

template <int BLOCK_N, int NTERMS>
struct WgCfg {
  static constexpr int NPLANES = (NTERMS == 1) ? 1 : 2;
  static constexpr int A_BYTES = 2 * WG_BOX_BYTES;                       // 128 ci
  static constexpr int B_BYTES = (BLOCK_N / 64) * WG_BOX_BYTES;
  static constexpr int STAGE_BYTES = NPLANES * (A_BYTES + B_BYTES);
  static constexpr int STAGES_RAW = (200 * 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

template <int BLOCK_N, int NTERMS>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                     const __grid_constant__ CUtensorMap map_dy_hi, const __grid_constant__ CUtensorMap map_dy_lo, WgArgs a) {
  pnp_pdl_trigger();
  using Cfg = WgCfg<BLOCK_N, NTERMS>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int ACC = BLOCK_N / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  int t = blockIdx.x;
  const int ni = t % a.nt;
  t /= a.nt;
  const int mi = t % a.mt;
  const int tap = t / a.mt;
  const int ci0 = mi * 128, co0 = ni * BLOCK_N;
  const int pb_begin = blockIdx.y * a.pb_per_split;
  const int pb_end = min(a.num_pb, pb_begin + a.pb_per_split);
  const int num_kb = pb_end - pb_begin;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_x_hi);
    tma_prefetch_desc(&map_dy_hi);
    if (NTERMS > 1) { tma_prefetch_desc(&map_x_lo); tma_prefetch_desc(&map_dy_lo); }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bars[s]), 1);
      mbar_init(smem_u32(&bars[STAGES + s]), CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pnp_pdl_wait();
  if (num_kb <= 0) return;

  if (warp == CONSUMER_WARPS) {
    // ================= TMA producer =================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int oy = a.tap_oy[tap], ox = a.tap_ox[tap];
      for (int kb = 0; kb < num_kb; ++kb) {
        int pb = pb_begin + kb;
        const int txi = pb % a.tiles_x;
        pb /= a.tiles_x;
        const int tyi = pb % a.tiles_y;
        const int tni = pb / a.tiles_y;
        const int x0 = txi * a.tw, y0 = tyi * a.th, img0 = tni * a.tn;
        mbar_wait(smem_u32(&bars[STAGES + stage]), phase ^ 1);
        const uint32_t full = smem_u32(&bars[stage]);
        mbar_expect_tx(full, Cfg::STAGE_BYTES);
        uint8_t* st = smem + stage * Cfg::STAGE_BYTES;
        const int cx = x0 * a.in_mul + ox, cy = y0 * a.in_mul + oy;
#pragma unroll
        for (int p = 0; p < Cfg::NPLANES; ++p) {
          const CUtensorMap* mx = p ? &map_x_lo : &map_x_hi;
          const CUtensorMap* md = p ? &map_dy_lo : &map_dy_hi;
          uint8_t* sa = st + p * Cfg::A_BYTES;
          uint8_t* sb = st + Cfg::NPLANES * Cfg::A_BYTES + p * Cfg::B_BYTES;
          if (a.pack == 1) {
            tma_load_4d(smem_u32(sa), mx, full, ci0, cx, cy, img0);
            tma_load_4d(smem_u32(sa + WG_BOX_BYTES), mx, full, ci0 + 64, cx, cy, img0);   // beyond Cin: zero filled
          } else {
            const int nb = a.pack;                       // 2 boxes of 8 KB or 4 boxes of 4 KB
            const int bbytes = 2 * WG_BOX_BYTES / nb;
            for (int j = 0; j < nb; ++j) {
              int tp = tap * nb + j;
              if (tp >= a.ntaps) tp = a.ntaps - 1;       // dummy rows of the last group (never written back)
              tma_load_4d(smem_u32(sa + j * bbytes), mx, full, 0, x0 * a.in_mul + a.tap_ox[tp], y0 * a.in_mul + a.tap_oy[tp], img0);
            }
          }
#pragma unroll
          for (int g = 0; g < BLOCK_N / 64; ++g) tma_load_4d(smem_u32(sb + g * WG_BOX_BYTES), md, full, co0 + g * 64, x0, y0, img0);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ================= consumer warpgroups =================
  // warpgroup wg owns M rows [64 wg, 64 wg + 64) = the second half of the A tile: one 64-channel box (pack 1, 2) or two
  // 32-channel boxes (pack 4); both start WG_BOX_BYTES * wg into the A operand
  const int wg = warp >> 2;
  float acc[ACC];
  int stage = 0;
  uint32_t phase = 0;
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(smem_u32(&bars[stage]), phase);
    wgmma_fence();
    const uint32_t st = smem_u32(smem + stage * Cfg::STAGE_BYTES);
    const uint32_t a_hi = st + wg * WG_BOX_BYTES, a_lo = a_hi + Cfg::A_BYTES;
    const uint32_t b_hi = st + Cfg::NPLANES * Cfg::A_BYTES, b_lo = b_hi + Cfg::B_BYTES;
#pragma unroll
    for (int k = 0; k < WG_PB / WGMMA_K; ++k) {
      const uint32_t koff = k * (WGMMA_K / 8) * 1024;       // 16 pixels = two 8-row swizzle atoms
      const uint32_t koff_a = (a.pack == 4) ? koff / 2 : koff;
      const uint64_t da_hi = (a.pack == 4) ? make_smem_desc(a_hi + koff_a, WG_BOX_BYTES / 2, 512, 2)
                                           : make_smem_desc(a_hi + koff_a, WG_BOX_BYTES, 1024, 1);
      const uint64_t db_hi = make_smem_desc(b_hi + koff, WG_BOX_BYTES, 1024, 1);
      if (NTERMS > 1) {
        const uint64_t da_lo = (a.pack == 4) ? make_smem_desc(a_lo + koff_a, WG_BOX_BYTES / 2, 512, 2)
                                             : make_smem_desc(a_lo + koff_a, WG_BOX_BYTES, 1024, 1);
        const uint64_t db_lo = make_smem_desc(b_lo + koff, WG_BOX_BYTES, 1024, 1);
        wgmma_bf16<BLOCK_N, 1, 1>(acc, da_lo, db_hi, (kb | k) != 0);
        wgmma_bf16<BLOCK_N, 1, 1>(acc, da_hi, db_lo, 1);
        wgmma_bf16<BLOCK_N, 1, 1>(acc, da_hi, db_hi, 1);
      } else {
        wgmma_bf16<BLOCK_N, 1, 1>(acc, da_hi, db_hi, (kb | k) != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars[STAGES + prev]));
    }
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  fence_acc(acc);

  const int cq = (lane & 3) * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    int ci = ci0 + m, tap_w = tap;
    if (a.pack == 2) { tap_w = tap * 2 + (m >> 6); ci = m & 63; }
    else if (a.pack == 4) { tap_w = tap * 4 + (m >> 5); ci = m & 31; }
    if (ci >= a.Cin || tap_w >= a.ntaps) continue;
    float* orow = a.dw + ((long long)tap_w * a.Cin + ci) * a.Cout + co0 + cq;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j)
      atomicAdd(reinterpret_cast<float2*>(orow + j * 8), make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
  }
}

// ---------------------------------------------------------------------------------------------
// host: tensor maps, tile selection, launches
// ---------------------------------------------------------------------------------------------
int make_act_map(CUtensorMap* m, const uint16_t* ptr, int B, int H, int W, int C, int tw, int th, int tn, int stride, int bk = BLOCK_K) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return PNP_ERR_DRIVER;
  if (tw * stride > 256 || th * stride > 256 || tn > 256) return PNP_ERR_UNSUPPORTED;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  // traversal stride: TMA loads ceil(box/stride) elements per dimension, i.e. every stride-th pixel (strided convolutions)
  cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(tw * stride), (cuuint32_t)(th * stride), (cuuint32_t)tn};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? PNP_OK : PNP_ERR_DRIVER;
}

int make_w_map(CUtensorMap* m, const uint16_t* ptr, long long rows, int K, int block_n, int bk = BLOCK_K) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return PNP_ERR_DRIVER;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)block_n};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? PNP_OK : PNP_ERR_DRIVER;
}

// pixel tile of `rows` (128 for conv, 64 for wgrad) over a U x V grid; exact != 0 demands tw*th*tn == rows (reduction dim)
int choose_tile(int U, int V, int B, int rows, int exact, int* tw, int* th, int* tn) {
  if (V >= rows) {
    if (V % rows != 0) return PNP_ERR_UNSUPPORTED;
    *tw = rows; *th = 1; *tn = 1;
    return PNP_OK;
  }
  *tw = V;
  *th = rows / V;
  if (*th > U) *th = U;
  *tn = (*th == U) ? (rows / (*tw * *th)) : 1;
  if (*tn < 1) *tn = 1;
  if (exact) {
    if ((*tw) * (*th) * (*tn) != rows || (U % *th) != 0) return PNP_ERR_UNSUPPORTED;
  } else if (*tn > B) {
    *tn = B;
  }
  return PNP_OK;
}

int g_last_cfg[3] = {0, 0, 0};   // {N tile, K block, split-K factor} of the most recent conv launch (profiling aid)

int sm_count() {
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      num_sms = PNP_NUM_SMS;
  }
  return num_sms;
}

// {CTAs per SM, grid size} of the most recent conv launch, and the largest residency a launch may use (profiling aids)
int g_last_residency[2] = {0, 0};
int g_residency_cap = 2;

template <int BLOCK_N, int NTERMS, int BK>
int launch_tc(const CUtensorMap& ma_hi, const CUtensorMap& ma_lo, const CUtensorMap& mb_hi, const CUtensorMap& mb_lo,
              float* y, const TcArgs& a, cudaStream_t s) {
  constexpr int CTAS = tc_ctas_per_sm(BLOCK_N);
  using Cfg = TcCfg<BLOCK_N, NTERMS, BK, CTAS>;
  auto kernel = conv_tc_kernel<BLOCK_N, NTERMS, BK, CTAS>;
  static int resident = 0;            // CTAs per SM the device actually fits, checked on the first launch
  if (resident == 0) {
    PNP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    int fit = 0;
    PNP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, kernel, TC_THREADS, Cfg::SMEM_BYTES));
    resident = fit >= CTAS ? CTAS : 1;      // a device that fits fewer runs the same kernel at one CTA per SM
  }
  const int ctas = resident < g_residency_cap ? resident : g_residency_cap;
  const long long slots = (long long)ctas * sm_count();
  const long long tiles = a.total_tiles;
  dim3 grid((unsigned)(tiles < slots ? tiles : slots));     // persistent: the resident CTAs walk the tile list
  g_last_residency[0] = ctas; g_last_residency[1] = (int)grid.x;
  pnp_launch(kernel, grid, TC_THREADS, Cfg::SMEM_BYTES, s, ma_hi, ma_lo, mb_hi, mb_lo, y, a);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

template <int BLOCK_N, int NTERMS>
int launch_wg(const CUtensorMap& mx_hi, const CUtensorMap& mx_lo, const CUtensorMap& md_hi, const CUtensorMap& md_lo,
              const WgArgs& a, int splits, cudaStream_t s) {
  using Cfg = WgCfg<BLOCK_N, NTERMS>;
  static bool attr_set = false;
  if (!attr_set) {
    PNP_CUDA(cudaFuncSetAttribute(conv_wgrad_tc_kernel<BLOCK_N, NTERMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid(a.ngroups * a.mt * a.nt, splits);
  pnp_launch(conv_wgrad_tc_kernel<BLOCK_N, NTERMS>, grid, TC_THREADS, Cfg::SMEM_BYTES, s, mx_hi, mx_lo, md_hi, md_lo, a);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

PnpDropout make_drop(const pnp_dropout_cfg* d) { return pnp_make_drop(d); }

// one launch of the generalized tap-table convolution: A planes [B, AH, AW, Cin] -> out [B, OH, OW, Cout]
int run_tc(const uint16_t* a_hi, const uint16_t* a_lo, int AH, int AW, int a_stride, const uint16_t* w_hi, const uint16_t* w_lo,
           long long w_rows, float* out, TcArgs& a, int nterms, cudaStream_t s) {
  int rc = choose_tile(a.U, a.V, a.B, BLOCK_M, 0, &a.tw, &a.th, &a.tn);     // (a.U, a.V): largest phase extent
  if (rc) return rc;
  a.tiles_x = pnp_cdiv(a.V, a.tw);
  if (a.nphases == 0 && a.V % a.tw != 0) return PNP_ERR_UNSUPPORTED;
  a.tiles_y = pnp_cdiv(a.U, a.th);
  a.tiles_n = pnp_cdiv(a.B, a.tn);
  // N tile: the widest of 128 / 64 / 32 / 16 that divides Cout.  128 columns is the widest accumulator two consumer
  // warpgroups hold in registers next to the epilogue (64 fp32 registers per thread)
  const int block_n = (a.Cout % 128 == 0) ? 128 : ((a.Cout % 64 == 0) ? 64 : ((a.Cout % 32 == 0) ? 32 : 16));
  // K-block width: 64 (SWIZZLE_128B) unless the reduction is 32 or 16 channels per tap
  int bk = (a.Cin % 64 == 0) ? 64 : ((a.Cin % 32 == 0) ? 32 : 16);
  {
    // experiment knobs: 32-wide K blocks for the 128- and 64-column tiles of 64-multiple reductions (twice the pipeline stages of
    // half the size)
    static int bk128_env = -1, bk64_env = -1;
    if (bk128_env < 0) { const char* e = getenv("PNP_TC_BK128"); bk128_env = e ? atoi(e) : 64; }
    if (bk64_env < 0) { const char* e = getenv("PNP_TC_BK64"); bk64_env = e ? atoi(e) : 64; }
    if (block_n == 128 && bk == 64 && bk128_env == 32) bk = 32;
    if (block_n == 64 && bk == 64 && bk64_env == 32) bk = 32;
  }
  a.kchunks = a.Cin / bk;
  g_last_cfg[0] = block_n; g_last_cfg[1] = bk; g_last_cfg[2] = 1;
  {
    const int n_tiles = a.Cout / block_n;
    if (a.nphases == 0) {
      a.total_tiles = a.tiles_x * a.tiles_y * a.tiles_n * n_tiles;
    } else {
      int base = 0;
      for (int p = 0; p < a.nphases; ++p) {
        a.ph[p].tiles_x = pnp_cdiv(a.ph[p].V, a.tw);
        a.ph[p].tiles_y = pnp_cdiv(a.ph[p].U, a.th);
        a.ph[p].tile_base = base;
        base += a.ph[p].tiles_x * a.ph[p].tiles_y * a.tiles_n * n_tiles;
      }
      a.total_tiles = base;
    }
  }
  // split-K: a layer with far fewer tiles than SMs and a deep reduction (cls_5's 5x5 stride-4 conv: 4 tiles x 200 k-blocks)
  // would otherwise run its whole K loop on a handful of SMs
  {
    static int rot_env = -1;
    static int order_env = -1;
    if (rot_env < 0) { const char* e = getenv("PNP_TC_ROT"); rot_env = e ? atoi(e) : 7; }
    if (order_env < 0) { const char* e = getenv("PNP_TC_ORDER"); order_env = e ? atoi(e) : 0; }
    a.rot_mul = rot_env;
    a.taps_inner = order_env;
  }
  a.ksplit = 1;
  double* bn_sum_after = nullptr;
  double* bn_sumsq_after = nullptr;
  {
    int min_taps = a.ntaps;
    for (int p = 0; p < a.nphases; ++p) min_taps = a.ph[p].tap_count < min_taps ? a.ph[p].tap_count : min_taps;
    const int min_kb = min_taps * a.kchunks;
    const int sms = sm_count();
    const bool fused_ep = a.ep_scale != nullptr || a.ep_skip != nullptr || a.ep_act != PNP_ACT_NONE || a.out_hi != nullptr;
    if (!fused_ep && a.total_tiles * 2 <= sms && min_kb >= 8) {
      int ks = sms / a.total_tiles;
      if (ks > min_kb / 4) ks = min_kb / 4;
      if (ks > 32) ks = 32;
      if (ks > 1) {
        a.ksplit = ks;
        g_last_cfg[2] = ks;
        a.total_tiles *= ks;
        if (!a.accumulate) PNP_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)a.B * a.OH * a.OW * a.Cout, s));
        bn_sum_after = a.bn_sum; bn_sumsq_after = a.bn_sumsq;      // statistics of partial sums are meaningless: separate pass
        a.bn_sum = nullptr; a.bn_sumsq = nullptr;
      }
    }
  }
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  rc = make_act_map(&ma_hi, a_hi, a.B, AH, AW, a.Cin, a.tw, a.th, a.tn, a_stride, bk);
  if (rc) return rc;
  rc = make_w_map(&mb_hi, w_hi, w_rows, a.Cin, block_n, bk);
  if (rc) return rc;
  if (nterms == 3) {
    rc = make_act_map(&ma_lo, a_lo, a.B, AH, AW, a.Cin, a.tw, a.th, a.tn, a_stride, bk);
    if (rc) return rc;
    rc = make_w_map(&mb_lo, w_lo, w_rows, a.Cin, block_n, bk);
    if (rc) return rc;
  } else {
    ma_lo = ma_hi;
    mb_lo = mb_hi;
  }
#define PNP_TC_GO(N_, K_)                                                                                  \
  rc = (nterms == 3) ? launch_tc<N_, 3, K_>(ma_hi, ma_lo, mb_hi, mb_lo, out, a, s)                         \
                     : launch_tc<N_, 1, K_>(ma_hi, ma_lo, mb_hi, mb_lo, out, a, s)
  if (block_n == 128 && bk == 64) { PNP_TC_GO(128, 64); }
  else if (block_n == 128 && bk == 32) { PNP_TC_GO(128, 32); }
  else if (block_n == 64 && bk == 64) { PNP_TC_GO(64, 64); }
  else if (block_n == 64 && bk == 32) { PNP_TC_GO(64, 32); }
  else if (block_n == 32 && bk == 64) { PNP_TC_GO(32, 64); }
  else if (block_n == 32 && bk == 32) { PNP_TC_GO(32, 32); }
  else if (block_n == 32 && bk == 16) { PNP_TC_GO(32, 16); }
  else if (block_n == 16 && bk == 16) { PNP_TC_GO(16, 16); }
  else if (block_n == 16 && bk == 32) { PNP_TC_GO(16, 32); }
  else return PNP_ERR_UNSUPPORTED;      // (no layer of the graphs needs the remaining tile shapes)
#undef PNP_TC_GO
  if (rc) return rc;
  if (bn_sum_after) return pnp_bn_stats(out, (long long)a.B * a.OH * a.OW, a.Cout, bn_sum_after, bn_sumsq_after, (void*)s);
  return PNP_OK;
}

bool tc_geom_ok(const pnp_conv_geom* g) {
  return g && g->B > 0 && g->H > 0 && g->W > 0 && g->Ho > 0 && g->Wo > 0 && g->kh > 0 && g->kw > 0 && g->dil > 0 && g->stride > 0 &&
         g->kh * g->kw <= MAX_TAPS && (g->Cin % 64 == 0 || g->Cin == 32 || g->Cin == 16) &&
         (g->Cout % 64 == 0 || g->Cout == 32 || g->Cout == 16);
}

}  // namespace

extern "C" int pnp_tc_last_config(int* block_n, int* block_k, int* ksplit) {
  if (block_n) *block_n = g_last_cfg[0];
  if (block_k) *block_k = g_last_cfg[1];
  if (ksplit) *ksplit = g_last_cfg[2];
  return PNP_OK;
}

// Residency of the wgmma forward / data-gradient launches, for tests and profiling (not part of the C-ABI header):
// pnp_tc_last_residency reports the CTAs per SM and the grid of the most recent launch; pnp_tc_set_residency_cap(1) runs
// every later launch at one CTA per SM (2 restores the default) and returns the previous cap.
extern "C" int pnp_tc_last_residency(int* ctas_per_sm, int* grid) {
  if (ctas_per_sm) *ctas_per_sm = g_last_residency[0];
  if (grid) *grid = g_last_residency[1];
  return PNP_OK;
}

extern "C" int pnp_tc_set_residency_cap(int cap) {
  const int prev = g_residency_cap;
  if (cap == 1 || cap == 2) g_residency_cap = cap;
  return prev;
}

extern "C" int pnp_tc_available(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return (major == 9 && get_encode_fn() != nullptr) ? 1 : 0;
}

extern "C" int pnp_split_bf16(const float* x, uint16_t* hi, uint16_t* lo, long long n, void* stream) {
  if (!x || !hi || n <= 0) return PNP_ERR_BAD_ARG;
  long long blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > PNP_NUM_SMS * 32LL) blocks = PNP_NUM_SMS * 32LL;
  pnp_launch(split_bf16_kernel, (unsigned)blocks, 256, 0, (cudaStream_t)stream, x, hi, lo, n);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_split_bf16_pad(const float* x, uint16_t* hi, uint16_t* lo, long long rows, int C, int Cpad, void* stream) {
  if (!x || !hi || rows <= 0 || C <= 0 || Cpad < C || (C % 4) != 0 || (Cpad % 4) != 0) return PNP_ERR_BAD_ARG;
  long long blocks = (rows * (Cpad / 4) + 255) / 256;
  if (blocks > PNP_NUM_SMS * 32LL) blocks = PNP_NUM_SMS * 32LL;
  pnp_launch(split_bf16_pad_kernel, (unsigned)blocks, 256, 0, (cudaStream_t)stream, x, hi, lo, rows, C, Cpad);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_split_weight_bf16(const float* w, uint16_t* hi, uint16_t* lo, int kh, int kw, int Cin, int Cout,
                                     int for_dgrad, int cin_pad, void* stream) {
  if (!w || !hi || kh <= 0 || kw <= 0 || Cin <= 0 || Cout <= 0) return PNP_ERR_BAD_ARG;
  const int CinP = (cin_pad > Cin) ? cin_pad : Cin;
  if (for_dgrad && CinP != Cin) return PNP_ERR_UNSUPPORTED;
  dim3 grid(pnp_cdiv(Cout, 32), pnp_cdiv(CinP, 32), kh * kw);
  pnp_launch(split_weight_kernel, grid, dim3(32, 8), 0, (cudaStream_t)stream, w, hi, lo, kh * kw, Cin, Cout, for_dgrad, CinP);
  PNP_LAUNCH_CHECK();
  return PNP_OK;
}

extern "C" int pnp_conv2d_tc_fwd_fused(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                                       float* y, const pnp_conv_geom* g, int nterms, const pnp_dropout_cfg* drop, int accumulate,
                                       double* bn_sum, double* bn_sumsq, const pnp_tc_epilogue* ep, void* stream) {
  if (!g || !x_hi || !w_hi) return PNP_ERR_BAD_ARG;
  if (!y && !(ep && ep->y_hi)) return PNP_ERR_BAD_ARG;
  if (nterms != 1 && nterms != 3) return PNP_ERR_BAD_ARG;
  if (nterms == 3 && (!x_lo || !w_lo)) return PNP_ERR_BAD_ARG;
  if ((bn_sum == nullptr) != (bn_sumsq == nullptr)) return PNP_ERR_BAD_ARG;
  // the epilogue reduces the statistics of the new contribution, the split-K path those of old + new: no single meaning
  if (accumulate && bn_sum) return PNP_ERR_BAD_ARG;
  if (!tc_geom_ok(g)) return PNP_ERR_UNSUPPORTED;
  TcArgs a;
  a.B = g->B; a.OH = g->Ho; a.OW = g->Wo; a.Cout = g->Cout; a.Cin = g->Cin;
  a.U = g->Ho; a.V = g->Wo; a.out_mul = 1; a.out_py = 0; a.out_px = 0; a.in_mul = g->stride; a.nphases = 0;
  a.ntaps = g->kh * g->kw;
  for (int ky = 0; ky < g->kh; ++ky)
    for (int kx = 0; kx < g->kw; ++kx) {
      int t = ky * g->kw + kx;
      a.tap_oy[t] = (short)(ky * g->dil - g->pad_t);
      a.tap_ox[t] = (short)(kx * g->dil - g->pad_l);
      a.tap_wrow[t] = t * g->Cout;
    }
  a.accumulate = accumulate;
  a.drop = make_drop(drop);
  a.bn_sum = bn_sum;
  a.bn_sumsq = bn_sumsq;
  a.ep_scale = nullptr; a.ep_shift = nullptr; a.ep_skip = nullptr; a.ep_skip_c = 0; a.ep_skip_off = 0; a.ep_act = PNP_ACT_NONE;
  a.out_hi = nullptr; a.out_lo = nullptr;
  if (ep) {
    if ((ep->scale == nullptr) != (ep->shift == nullptr)) return PNP_ERR_BAD_ARG;
    if (accumulate) return PNP_ERR_BAD_ARG;                               // a fused epilogue produces final values
    if (bn_sum && (ep->scale || ep->skip || ep->act != PNP_ACT_NONE || ep->y_hi)) return PNP_ERR_BAD_ARG;   // batch statistics are of z
    if (ep->skip && (ep->skip_C % 4 != 0 || ep->skip_off % 4 != 0 || ep->skip_off < 0 || ep->skip_off + ep->skip_C > g->Cout))
      return PNP_ERR_BAD_ARG;
    if (ep->y_hi && nterms == 3 && !ep->y_lo) return PNP_ERR_BAD_ARG;
    a.ep_scale = ep->scale; a.ep_shift = ep->shift;
    a.ep_skip = ep->skip; a.ep_skip_c = ep->skip_C; a.ep_skip_off = ep->skip_off;
    a.ep_act = ep->act;
    a.out_hi = ep->y_hi; a.out_lo = ep->y_lo;
  }
  return run_tc(x_hi, x_lo, g->H, g->W, g->stride, w_hi, w_lo, (long long)g->kh * g->kw * g->Cout, y, a, nterms, (cudaStream_t)stream);
}

extern "C" int pnp_conv2d_tc_fwd(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                                 float* y, const pnp_conv_geom* g, int nterms, const pnp_dropout_cfg* drop, int accumulate,
                                 double* bn_sum, double* bn_sumsq, void* stream) {
  if (!y) return PNP_ERR_BAD_ARG;
  return pnp_conv2d_tc_fwd_fused(x_hi, x_lo, w_hi, w_lo, y, g, nterms, drop, accumulate, bn_sum, bn_sumsq, nullptr, stream);
}

// dx[B,H,W,Cin] (+)= conv^T(dy, w): `g` is the FORWARD geometry, dy planes [B,Ho,Wo,Cout], weight planes from
// pnp_split_weight_bf16(for_dgrad = 1) = [tap][Cin][Cout].  stride 1: one launch; stride s: s*s phase launches, each a
// stride-1 convolution over dy with the taps whose offset is divisible by s, writing every s-th pixel of dx.
extern "C" int pnp_conv2d_tc_dgrad(const uint16_t* dy_hi, const uint16_t* dy_lo, const uint16_t* w_hi, const uint16_t* w_lo,
                                   float* dx, const pnp_conv_geom* g, int nterms, int accumulate, void* stream) {
  if (!g || !dy_hi || !w_hi || !dx) return PNP_ERR_BAD_ARG;
  if (nterms != 1 && nterms != 3) return PNP_ERR_BAD_ARG;
  if (nterms == 3 && (!dy_lo || !w_lo)) return PNP_ERR_BAD_ARG;
  if (!tc_geom_ok(g)) return PNP_ERR_UNSUPPORTED;
  const int s = g->stride;
  // every phase needs at least one tap per axis, otherwise part of dx would stay unwritten
  for (int p = 0; p < s; ++p) {
    bool hy = false, hx = false;
    for (int k = 0; k < g->kh; ++k) hy = hy || ((p + g->pad_t - k * g->dil) % s == 0);
    for (int k = 0; k < g->kw; ++k) hx = hx || ((p + g->pad_l - k * g->dil) % s == 0);
    if (!hy || !hx) return PNP_ERR_UNSUPPORTED;
  }
  TcArgs a;
  a.B = g->B; a.OH = g->H; a.OW = g->W; a.Cout = g->Cin; a.Cin = g->Cout;
  a.out_mul = s; a.out_py = 0; a.out_px = 0; a.in_mul = 1;
  a.accumulate = accumulate;
  a.drop = make_drop(nullptr);
  a.bn_sum = nullptr;
  a.bn_sumsq = nullptr;
  a.ep_scale = nullptr; a.ep_shift = nullptr; a.ep_skip = nullptr; a.ep_skip_c = 0; a.ep_skip_off = 0; a.ep_act = PNP_ACT_NONE;
  a.out_hi = nullptr; a.out_lo = nullptr;
  a.U = 0; a.V = 0;
  int np = 0, nt = 0;
  for (int py = 0; py < s; ++py)
    for (int px = 0; px < s; ++px) {
      const int U = (g->H - py + s - 1) / s, V = (g->W - px + s - 1) / s;
      if (U <= 0 || V <= 0) continue;
      a.ph[np].tap_begin = (short)nt;
      for (int ky = 0; ky < g->kh; ++ky) {
        int ny = py + g->pad_t - ky * g->dil;
        if (ny % s != 0) continue;
        for (int kx = 0; kx < g->kw; ++kx) {
          int nx = px + g->pad_l - kx * g->dil;
          if (nx % s != 0) continue;
          a.tap_oy[nt] = (short)(ny / s);
          a.tap_ox[nt] = (short)(nx / s);
          a.tap_wrow[nt] = (ky * g->kw + kx) * g->Cin;
          ++nt;
        }
      }
      a.ph[np].tap_count = (short)(nt - a.ph[np].tap_begin);
      a.ph[np].py = (short)py; a.ph[np].px = (short)px;
      a.ph[np].U = U; a.ph[np].V = V;
      if (U > a.U) a.U = U;
      if (V > a.V) a.V = V;
      ++np;
    }
  a.ntaps = nt;
  a.nphases = (s == 1) ? 0 : np;
  if (s == 1) { a.out_py = 0; a.out_px = 0; }
  int rc = run_tc(dy_hi, dy_lo, g->Ho, g->Wo, 1, w_hi, w_lo, (long long)g->kh * g->kw * g->Cin, dx, a, nterms, (cudaStream_t)stream);
  if (rc) return rc;
  return PNP_OK;
}

// dw[kh][kw][Cin][Cout] += x (*) dy on the tensor cores (x planes [B,H,W,Cin] -- the mirror-padded input for SYMMETRIC convs)
extern "C" int pnp_conv2d_tc_wgrad(const uint16_t* x_hi, const uint16_t* x_lo, const uint16_t* dy_hi, const uint16_t* dy_lo,
                                   float* dw, const pnp_conv_geom* g, int nterms, int x_channels, void* stream) {
  if (!g || !x_hi || !dy_hi || !dw) return PNP_ERR_BAD_ARG;
  if (nterms != 1 && nterms != 3) return PNP_ERR_BAD_ARG;
  if (nterms == 3 && (!x_lo || !dy_lo)) return PNP_ERR_BAD_ARG;
  const int xc = x_channels > 0 ? x_channels : g->Cin;     // channel count of the x planes (>= Cin, zero padded)
  {
    pnp_conv_geom t = *g;
    t.Cin = xc;
    if (xc < g->Cin || !tc_geom_ok(&t) || (xc % 64 != 0 && !(xc == 32 && g->Cin == 32)) || g->Cout % 64 != 0) return PNP_ERR_UNSUPPORTED;
  }
  WgArgs a;
  a.B = g->B; a.Cin = g->Cin; a.Cout = g->Cout; a.in_mul = g->stride; a.dw = dw;
  a.ntaps = g->kh * g->kw;
  for (int ky = 0; ky < g->kh; ++ky)
    for (int kx = 0; kx < g->kw; ++kx) {
      a.tap_oy[ky * g->kw + kx] = (short)(ky * g->dil - g->pad_t);
      a.tap_ox[ky * g->kw + kx] = (short)(kx * g->dil - g->pad_l);
    }
  int rc = choose_tile(g->Ho, g->Wo, g->B, WG_PB, 1, &a.tw, &a.th, &a.tn);
  if (rc) return rc;
  a.tiles_x = g->Wo / a.tw;
  a.tiles_y = g->Ho / a.th;
  a.tiles_n = pnp_cdiv(g->B, a.tn);
  a.num_pb = a.tiles_x * a.tiles_y * a.tiles_n;
  const int block_n = (g->Cout % 128 == 0) ? 128 : 64;
  a.mt = pnp_cdiv(g->Cin, 128);
  a.nt = g->Cout / block_n;
  a.pack = 1;
  if (g->Cin == 64 && xc == 64) a.pack = 2;
  else if (g->Cin == 32 && xc == 32) a.pack = 4;
  a.ngroups = pnp_cdiv(a.ntaps, a.pack);
  const int x_bk = (a.pack == 4) ? 32 : 64;
  const int tiles = a.ngroups * a.mt * a.nt;
  int splits = (2 * sm_count()) / tiles;       // floor: tiles * splits CTAs must fit two full waves (one CTA per SM), never spill into a third
  int max_splits = a.num_pb / 4;
  if (max_splits < 1) max_splits = 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  a.pb_per_split = pnp_cdiv(a.num_pb, splits);
  splits = pnp_cdiv(a.num_pb, a.pb_per_split);
  CUtensorMap mx_hi, mx_lo, md_hi, md_lo;
  rc = make_act_map(&mx_hi, x_hi, g->B, g->H, g->W, xc, a.tw, a.th, a.tn, g->stride, x_bk);
  if (rc) return rc;
  rc = make_act_map(&md_hi, dy_hi, g->B, g->Ho, g->Wo, g->Cout, a.tw, a.th, a.tn, 1);
  if (rc) return rc;
  if (nterms == 3) {
    rc = make_act_map(&mx_lo, x_lo, g->B, g->H, g->W, xc, a.tw, a.th, a.tn, g->stride, x_bk);
    if (rc) return rc;
    rc = make_act_map(&md_lo, dy_lo, g->B, g->Ho, g->Wo, g->Cout, a.tw, a.th, a.tn, 1);
    if (rc) return rc;
  } else {
    mx_lo = mx_hi;
    md_lo = md_hi;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (block_n == 128) {
    if (nterms == 3) return launch_wg<128, 3>(mx_hi, mx_lo, md_hi, md_lo, a, splits, s);
    return launch_wg<128, 1>(mx_hi, mx_lo, md_hi, md_lo, a, splits, s);
  }
  if (nterms == 3) return launch_wg<64, 3>(mx_hi, mx_lo, md_hi, md_lo, a, splits, s);
  return launch_wg<64, 1>(mx_hi, mx_lo, md_hi, md_lo, a, splits, s);
}
