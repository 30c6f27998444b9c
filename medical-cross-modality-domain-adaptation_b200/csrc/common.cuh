// Shared device/host helpers for the PnP-AdaNet H100 hot path (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// streaming multiprocessors of an H100 SXM: grid-stride kernels size their grids in multiples of it
#define PNP_NUM_SMS 132

#define PNP_OK 0
#define PNP_ERR_BAD_ARG 100001
#define PNP_ERR_UNSUPPORTED 100002
#define PNP_ERR_DRIVER 100003

#define PNP_LAUNCH_CHECK()                        \
  do {                                            \
    cudaError_t _e = cudaGetLastError();          \
    if (_e != cudaSuccess) return (int)_e;        \
  } while (0)

#define PNP_CUDA(call)                            \
  do {                                            \
    cudaError_t _e = (call);                      \
    if (_e != cudaSuccess) return (int)_e;        \
  } while (0)

static inline int pnp_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------------
// Programmatic dependent launch (opt-in: PNP_PDL=1).  A step is ~860 short kernels in stream order (inside one CUDA graph).
// Every kernel of this library starts with pnp_pdl_enter(): `griddepcontrol.launch_dependents` lets the NEXT kernel of the
// stream become resident as soon as all CTAs of this one have started (its CTAs take whatever SM resources are free),
// `griddepcontrol.wait` then blocks until the PREVIOUS kernel has completed and its writes are visible -- no kernel touches
// global memory before that, so stream-order semantics are kept and only launch latency, CTA scheduling and the per-kernel
// prologue (the tensor-core kernels wait after their barrier set-up) overlap the predecessor's tail.  With PNP_PDL=1 launches
// carry cudaLaunchAttributeProgrammaticStreamSerialization (stream capture turns it into a programmatic graph edge); without
// it both instructions are no-ops.  Inside a CUDA graph most launch latency is already hidden: default OFF.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pnp_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pnp_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pnp_pdl_enter() {
  pnp_pdl_trigger();
  pnp_pdl_wait();
}

#ifdef __CUDACC__
#include <stdlib.h>
static inline int pnp_pdl_on() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("PNP_PDL"); v = e ? atoi(e) : 0; }
  return v;
}
template <typename... KArgs, typename... Args>
static inline cudaError_t pnp_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pnp_pdl_on() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// ------------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG.  One call yields the 4 uniforms for the 4 consecutive elements
// [4*idx4, 4*idx4+3] of a tensor; `stream` separates dropout call sites, the seed lives in device
// memory so that a captured CUDA graph sees a fresh seed on every replay.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 pnp_philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

struct PnpDropout {
  const unsigned long long* seed_ptr;  // device scalar; nullptr => dropout disabled
  unsigned long long stream;           // call-site id
  float keep;                          // keep probability
  float inv_keep;                      // 1/keep
  uint32_t thresh;                     // keep * 2^16 (an element is kept when its 16-bit draw is below it)
};

// One Philox call yields 128 bits = the 16-bit draws of the EIGHT consecutive elements [8*idx8, 8*idx8+7] (element e uses the
// low / high half of word (e & 7) >> 1).  16 bits resolve keep_prob to 1.5e-5 (0.75 is exact); halving the Philox calls per
// element matters in the convolution epilogue, where the mask generation used to cost more issue slots than everything else.
__device__ __forceinline__ uint4 pnp_dropout_bits8(const PnpDropout& d, unsigned long long seed, unsigned long long idx8) {
  return pnp_philox4x32_10(make_uint4((uint32_t)idx8, (uint32_t)(idx8 >> 32), (uint32_t)d.stream, (uint32_t)(d.stream >> 32)),
                           make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}
__device__ __forceinline__ float pnp_drop_sel(const PnpDropout& d, uint32_t u16) { return (u16 < d.thresh) ? d.inv_keep : 0.f; }

// multipliers (0 or 1/keep) for elements 8*idx8 .. 8*idx8+7
__device__ __forceinline__ void pnp_dropout_mult8(const PnpDropout& d, unsigned long long seed, unsigned long long idx8, float (&m)[8]) {
  const uint4 r = pnp_dropout_bits8(d, seed, idx8);
  m[0] = pnp_drop_sel(d, r.x & 0xffffu); m[1] = pnp_drop_sel(d, r.x >> 16);
  m[2] = pnp_drop_sel(d, r.y & 0xffffu); m[3] = pnp_drop_sel(d, r.y >> 16);
  m[4] = pnp_drop_sel(d, r.z & 0xffffu); m[5] = pnp_drop_sel(d, r.z >> 16);
  m[6] = pnp_drop_sel(d, r.w & 0xffffu); m[7] = pnp_drop_sel(d, r.w >> 16);
}

// multipliers for elements 4*idx4 .. 4*idx4+3 (the lower or upper half of their group of eight)
__device__ __forceinline__ float4 pnp_dropout_mult4(const PnpDropout& d, unsigned long long seed, unsigned long long idx4) {
  const uint4 r = pnp_dropout_bits8(d, seed, idx4 >> 1);
  const uint32_t w0 = (idx4 & 1ull) ? r.z : r.x, w1 = (idx4 & 1ull) ? r.w : r.y;
  float4 m;
  m.x = pnp_drop_sel(d, w0 & 0xffffu); m.y = pnp_drop_sel(d, w0 >> 16);
  m.z = pnp_drop_sel(d, w1 & 0xffffu); m.w = pnp_drop_sel(d, w1 >> 16);
  return m;
}

__device__ __forceinline__ float pnp_dropout_mult1(const PnpDropout& d, unsigned long long seed, unsigned long long idx) {
  float4 m = pnp_dropout_mult4(d, seed, idx >> 2);
  int l = (int)(idx & 3);
  return l == 0 ? m.x : (l == 1 ? m.y : (l == 2 ? m.z : m.w));
}

// host: (seed pointer, stream id, keep) of the C-ABI -> kernel argument; keep >= 1 or a null seed disables dropout
template <class Cfg>
static inline PnpDropout pnp_make_drop(const Cfg* d) {
  PnpDropout r;
  r.seed_ptr = nullptr; r.stream = 0; r.keep = 1.f; r.inv_keep = 1.f; r.thresh = 65536u;
  if (d && d->seed_ptr && d->keep < 1.0f) {
    r.seed_ptr = d->seed_ptr; r.stream = d->stream; r.keep = d->keep; r.inv_keep = 1.0f / d->keep;
    float t = d->keep * 65536.0f + 0.5f;
    r.thresh = t <= 0.f ? 0u : (t >= 65536.f ? 65536u : (uint32_t)t);
  }
  return r;
}

__device__ __forceinline__ float pnp_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double pnp_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
