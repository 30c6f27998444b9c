// Largest connected component per class of a 3-D label volume (native.py's optional post-processing of a native-grid prediction).
// Union-find over an int32 parent array in the style of Playne & Hawick 2018 with ECL-CC's hooking and path halving
// (Jaiganesh & Burtscher 2018): every voxel links to its same-class neighbours of smaller linear index (3 for 6-connectivity, 13 for
// 26), a root is only ever hooked under a smaller root by atomicCAS, so every root ends as the smallest linear index of its
// component.  A fixed sequence of five launches, whatever the content: no convergence loop on the host, no copy back.
//   init      parent[v] = v, size[v] = 0
//   merge     union of v with each same-class backward neighbour (template on the neighbour set)
//   flatten   parent[v] = root(v) (a read-only walk), size[root] += 1 (warp-aggregated atomics)
//   select    per class: number of roots, atomicMax of (size << 32) | (0xFFFFFFFF - root)  -> the largest, first in C order
//   write     out[v] = class if v's root is its class's kept root, else 0; stats kept / removed; cm[gt][out]
// Every quantity is an integer, so out, stats and cm are exact functions of the input and repeated calls are bit-identical.
// pnp_label_boxes (native.py's heart localisation) reduces each class's voxel count and bounding box: per-thread registers, a warp
// reduction, then one integer atomic per warp, class and field.
#include "common.cuh"
#include "../../include/pnp_b200.h"

namespace {

typedef unsigned long long u64;

constexpr int THREADS = 256;

// the class of a label (0 for background and labels >= C)
__device__ __forceinline__ int class_of(int l, int C) { return l < C ? l : 0; }

// root of x with path halving.  Parents only decrease (parent[v] <= v) and only roots are ever hooked, so a store into a non-root
// replaces one of its ancestors by another and races with other finds are benign.  volatile: other CTAs hook and halve concurrently.
__device__ __forceinline__ int find_root(volatile int* parent, int x) {
  int cur = parent[x];
  if (cur == x) return x;
  int prev = x, next;
  while (cur > (next = parent[cur])) {
    parent[prev] = next;
    prev = cur;
    cur = next;
  }
  return cur;
}

// root of x without writing: the flatten pass stores each voxel's final root, and a halving store landing after that one would
// leave an intermediate ancestor behind
__device__ __forceinline__ int walk_root(volatile const int* parent, int x) {
  int next;
  while ((next = parent[x]) != x) x = next;
  return x;
}

// the larger of the two roots is hooked under the smaller one, and only while it is still a root
__device__ __forceinline__ void unite(int* parent, int a, int b) {
  volatile int* p = parent;
  while (true) {
    a = find_root(p, a);
    b = find_root(p, b);
    if (a == b) return;
    if (a < b) {
      const int t = a;
      a = b;
      b = t;
    }
    if (atomicCAS(parent + a, a, b) == a) return;
  }
}

__global__ void __launch_bounds__(THREADS) lcc_init_kernel(int* __restrict__ parent, int* __restrict__ size, long long total) {
  pnp_pdl_enter();
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    parent[i] = (int)i;
    size[i] = 0;
  }
}

// Backward neighbours (d0, d1, d2) with a smaller linear index: 6-connectivity the three face neighbours, 26-connectivity the 13
// offsets that are lexicographically negative.
template <int CONN>
struct Backward;
template <>
struct Backward<6> {
  static constexpr int count = 3;
  static __device__ __forceinline__ int3 at(int t) { return t == 0 ? make_int3(-1, 0, 0) : (t == 1 ? make_int3(0, -1, 0) : make_int3(0, 0, -1)); }
};
template <>
struct Backward<26> {
  static constexpr int count = 13;
  static __device__ __forceinline__ int3 at(int t) {
    // t < 9: d0 = -1 with (d1, d2) over {-1, 0, 1}^2; 9..11: d0 = 0, d1 = -1, d2 = -1 .. 1; 12: (0, 0, -1)
    if (t < 9) return make_int3(-1, t / 3 - 1, t % 3 - 1);
    if (t < 12) return make_int3(0, -1, t - 10);
    return make_int3(0, 0, -1);
  }
};

template <int CONN>
__global__ void __launch_bounds__(THREADS)
lcc_merge_kernel(const uint8_t* __restrict__ labels, int n1, int n2, int C, long long total, int* parent) {
  pnp_pdl_enter();
  const int plane = n1 * n2;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int v = (int)i;
    const int c = class_of(__ldg(labels + v), C);
    if (c == 0) continue;
    const int row = v / n2;
    const int k = v - row * n2, j = row % n1, i0 = row / n1;
#pragma unroll
    for (int t = 0; t < Backward<CONN>::count; ++t) {
      const int3 d = Backward<CONN>::at(t);
      if (i0 + d.x < 0 || j + d.y < 0 || j + d.y >= n1 || k + d.z < 0 || k + d.z >= n2) continue;
      const int u = v + d.x * plane + d.y * n2 + d.z;
      if (__ldg(labels + u) == c) unite(parent, v, u);
    }
  }
}

// Every warp walks whole 32-voxel groups (the stride is a multiple of 32), so the full-mask match below is always converged.
__global__ void __launch_bounds__(THREADS)
lcc_flatten_kernel(const uint8_t* __restrict__ labels, int C, long long total, int* parent, int* __restrict__ size) {
  pnp_pdl_enter();
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * THREADS + (threadIdx.x & ~31); base < total; base += (long long)gridDim.x * THREADS) {
    const long long i = base + lane;
    int r = -1;
    if (i < total && class_of(__ldg(labels + i), C) != 0) {
      r = walk_root((volatile const int*)parent, (int)i);
      parent[i] = r;
    }
    const unsigned same = __match_any_sync(0xffffffffu, r);
    if (r >= 0 && lane == __ffs(same) - 1) atomicAdd(size + r, __popc(same));
  }
}

// best[c]: (size << 32) | (0xFFFFFFFF - root), the atomicMax of which is the largest component, the smallest root among equals
__global__ void __launch_bounds__(THREADS)
lcc_select_kernel(const uint8_t* __restrict__ labels, int C, long long total, const int* __restrict__ parent,
                  const int* __restrict__ size, u64* __restrict__ best, long long* __restrict__ stats) {
  __shared__ u64 sbest[8];
  __shared__ unsigned scount[8];
  pnp_pdl_enter();
  if (threadIdx.x < 8) {
    sbest[threadIdx.x] = 0ull;
    scount[threadIdx.x] = 0u;
  }
  __syncthreads();
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int v = (int)i;
    if (__ldg(parent + v) != v) continue;
    const int c = class_of(__ldg(labels + v), C);
    if (c == 0) continue;
    atomicMax(sbest + c, ((u64)(unsigned)__ldg(size + v) << 32) | (u64)(0xFFFFFFFFu - (unsigned)v));
    atomicAdd(scount + c, 1u);
  }
  __syncthreads();
  if (threadIdx.x > 0 && threadIdx.x < C && scount[threadIdx.x]) {
    atomicMax(best + threadIdx.x, sbest[threadIdx.x]);
    atomicAdd((u64*)stats + 3 * threadIdx.x, (u64)scount[threadIdx.x]);
  }
}

// labels and out may alias: each voxel's label is read and its output written by the same thread, nothing else reads labels here
__global__ void __launch_bounds__(THREADS)
lcc_write_kernel(const uint8_t* labels, int C, long long total, const int* __restrict__ parent, const u64* __restrict__ best,
                 uint8_t* out, const uint8_t* __restrict__ gt, long long* __restrict__ stats, long long* __restrict__ cm) {
  __shared__ unsigned hist[64];
  __shared__ unsigned kept[8], removed[8];
  pnp_pdl_enter();
  if (threadIdx.x < 64) hist[threadIdx.x] = 0u;
  if (threadIdx.x < 8) {
    kept[threadIdx.x] = 0u;
    removed[threadIdx.x] = 0u;
  }
  __syncthreads();
  unsigned keep_root[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) keep_root[c] = c < C ? 0xFFFFFFFFu - (unsigned)__ldg(best + c) : 0xFFFFFFFFu;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int v = (int)i;
    const int l = labels[v];
    int o = 0;
    if (l >= C) {
      atomicAdd(removed, 1u);
    } else if (l > 0) {
      unsigned root = (unsigned)__ldg(parent + v), want = keep_root[0];
#pragma unroll
      for (int c = 1; c < 8; ++c)
        if (c == l) want = keep_root[c];
      if (root == want) {
        o = l;
        atomicAdd(kept + l, 1u);
      } else {
        atomicAdd(removed + l, 1u);
      }
    }
    out[v] = (uint8_t)o;
    if (cm) {
      int g = __ldg(gt + v);
      if (g >= C) g = 0;
      atomicAdd(&hist[g * C + o], 1u);
    }
  }
  __syncthreads();
  if (cm && threadIdx.x < C * C && hist[threadIdx.x]) atomicAdd((u64*)cm + threadIdx.x, (u64)hist[threadIdx.x]);
  if (threadIdx.x < C) {
    if (kept[threadIdx.x]) atomicAdd((u64*)stats + 3 * threadIdx.x + 1, (u64)kept[threadIdx.x]);
    if (removed[threadIdx.x]) atomicAdd((u64*)stats + 3 * threadIdx.x + 2, (u64)removed[threadIdx.x]);
  }
}

// out[c] = (count, lo0, hi0, lo1, hi1, lo2, hi2): the empty box (0, n0, -1, n1, -1, n2, -1) that the atomics shrink onto the voxels
__global__ void __launch_bounds__(THREADS) box_init_kernel(int n0, int n1, int n2, int C, long long* __restrict__ out) {
  pnp_pdl_enter();
  const int t = threadIdx.x, f = t % 7;
  if (t < 7 * C) out[t] = f == 0 ? 0 : (f % 2 == 0 ? -1 : (f == 1 ? n0 : (f == 3 ? n1 : n2)));
}

// Each thread keeps every class's count and bounds in registers (the class selects its slot through an unrolled compare, so no
// local memory); after the grid-stride loop, which every thread leaves, each warp reduces them with __reduce_*_sync and lane 0
// folds the warp's result into out with one integer atomic per non-empty class and field.
__global__ void __launch_bounds__(THREADS)
label_boxes_kernel(const uint8_t* __restrict__ labels, int n1, int n2, int C, long long total, long long* __restrict__ out) {
  pnp_pdl_enter();
  unsigned cnt[8];
  int lo0[8], hi0[8], lo1[8], hi1[8], lo2[8], hi2[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    cnt[c] = 0u;
    lo0[c] = lo1[c] = lo2[c] = 0x7FFFFFFF;
    hi0[c] = hi1[c] = hi2[c] = -1;
  }
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int v = (int)i;
    const int l = class_of(__ldg(labels + v), C);
    const int row = v / n2;
    const int k = v - row * n2, j = row % n1, i0 = row / n1;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      if (c == l) {
        cnt[c] += 1u;
        lo0[c] = min(lo0[c], i0);
        hi0[c] = max(hi0[c], i0);
        lo1[c] = min(lo1[c], j);
        hi1[c] = max(hi1[c], j);
        lo2[c] = min(lo2[c], k);
        hi2[c] = max(hi2[c], k);
      }
    }
  }
  const unsigned full = 0xffffffffu;
  const bool lead = (threadIdx.x & 31) == 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (c >= C) break;
    const unsigned n = __reduce_add_sync(full, cnt[c]);
    const int a0 = __reduce_min_sync(full, lo0[c]), b0 = __reduce_max_sync(full, hi0[c]);
    const int a1 = __reduce_min_sync(full, lo1[c]), b1 = __reduce_max_sync(full, hi1[c]);
    const int a2 = __reduce_min_sync(full, lo2[c]), b2 = __reduce_max_sync(full, hi2[c]);
    if (lead && n) {
      long long* o = out + 7 * c;
      atomicAdd((u64*)o, (u64)n);
      atomicMin(o + 1, (long long)a0);
      atomicMax(o + 2, (long long)b0);
      atomicMin(o + 3, (long long)a1);
      atomicMax(o + 4, (long long)b1);
      atomicMin(o + 5, (long long)a2);
      atomicMax(o + 6, (long long)b2);
    }
  }
}

inline long long align256(long long b) { return (b + 255) & ~255LL; }

// bytes = 2 A(4N) + 256: parent and size (int32 per voxel), then the 8 per-class keys
long long workspace_size(long long N) { return 2 * align256(4 * N) + 256; }

int check_shape(int n0, int n1, int n2, int C, int connectivity) {
  if (n0 <= 0 || n1 <= 0 || n2 <= 0) return PNP_ERR_BAD_ARG;
  if (C < 2 || C > 8 || (connectivity != 6 && connectivity != 26)) return PNP_ERR_UNSUPPORTED;
  if ((long long)n0 * n1 * n2 >= (1LL << 31)) return PNP_ERR_UNSUPPORTED;
  return PNP_OK;
}

}  // namespace

extern "C" int pnp_largest_components_workspace(int n0, int n1, int n2, int C, int connectivity, long long* bytes) {
  if (!bytes) return PNP_ERR_BAD_ARG;
  const int rc = check_shape(n0, n1, n2, C, connectivity);
  if (rc) return rc;
  *bytes = workspace_size((long long)n0 * n1 * n2);
  return PNP_OK;
}

extern "C" int pnp_largest_components(const uint8_t* labels, int n0, int n1, int n2, int C, int connectivity, uint8_t* out,
                                      const uint8_t* gt, long long* cm, long long* stats, void* ws, long long ws_bytes,
                                      void* stream) {
  if (!labels || !out || (!gt) != (!cm) || !stats || !ws) return PNP_ERR_BAD_ARG;
  const int rc = check_shape(n0, n1, n2, C, connectivity);
  if (rc) return rc;
  const long long N = (long long)n0 * n1 * n2;
  if (ws_bytes < workspace_size(N)) return PNP_ERR_BAD_ARG;
  int* parent = (int*)ws;
  int* size = (int*)((char*)ws + align256(4 * N));
  u64* best = (u64*)((char*)ws + 2 * align256(4 * N));
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(N, THREADS * 4);
  PNP_CUDA(cudaMemsetAsync(best, 0, 8 * sizeof(u64), st));
  PNP_CUDA(cudaMemsetAsync(stats, 0, sizeof(long long) * 3 * C, st));
  if (cm) PNP_CUDA(cudaMemsetAsync(cm, 0, sizeof(long long) * C * C, st));
  PNP_CUDA(pnp_launch(lcc_init_kernel, grid, THREADS, 0, st, parent, size, N));
  if (connectivity == 6)
    PNP_CUDA(pnp_launch(lcc_merge_kernel<6>, grid, THREADS, 0, st, labels, n1, n2, C, N, parent));
  else
    PNP_CUDA(pnp_launch(lcc_merge_kernel<26>, grid, THREADS, 0, st, labels, n1, n2, C, N, parent));
  PNP_CUDA(pnp_launch(lcc_flatten_kernel, grid, THREADS, 0, st, labels, C, N, parent, size));
  PNP_CUDA(pnp_launch(lcc_select_kernel, grid, THREADS, 0, st, labels, C, N, (const int*)parent, (const int*)size, best, stats));
  PNP_CUDA(pnp_launch(lcc_write_kernel, grid, THREADS, 0, st, labels, C, N, (const int*)parent, (const u64*)best, out, gt, stats,
                      cm));
  return PNP_OK;
}

extern "C" int pnp_label_boxes(const uint8_t* labels, int n0, int n1, int n2, int C, long long* out, void* stream) {
  if (!labels || !out || n0 <= 0 || n1 <= 0 || n2 <= 0) return PNP_ERR_BAD_ARG;
  if (C < 2 || C > 8 || (long long)n0 * n1 * n2 >= (1LL << 31)) return PNP_ERR_UNSUPPORTED;
  const long long N = (long long)n0 * n1 * n2;
  cudaStream_t st = (cudaStream_t)stream;
  PNP_CUDA(pnp_launch(box_init_kernel, 1, THREADS, 0, st, n0, n1, n2, C, out));
  PNP_CUDA(pnp_launch(label_boxes_kernel, grid_for(N, THREADS * 4), THREADS, 0, st, labels, n1, n2, C, N, out));
  return PNP_OK;
}
