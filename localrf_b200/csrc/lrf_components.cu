// lrf_components.cu -- connected components of an exported mesh or point cloud on the device, so that the small ones
// (the floaters an optimised radiance field leaves in free space) can be dropped.
//
// Union-find over a parent array that starts as parent[v] = v and only ever decreases: a union finds both roots with
// path halving (each shortcut an atomicMin) and hooks the higher root under the lower one with atomicCAS, retrying
// from the new parent when the CAS finds the root already hooked.  So parent[v] <= v at every moment, and the root of
// a component is its lowest index whatever order the threads run in.  Sizes are integer atomics at the root, so
// labels and sizes are bitwise deterministic.
//
// Mesh: each triangle unites its three vertices.  Cloud: each point's cell, floor((x - origin) / cell_size) keyed by
// cell_key as lrf_frame_points keys its voxels, is claimed once in an lrf_table.cuh table whose slot keeps the cell's
// lowest point (atomicMin); a point unites with the one its atomicMin replaced or lost to, so a cell's points form one
// set, and each cell unites its lowest point with those of its 13 forward neighbours among the 26 (the neighbour
// relation is symmetric, so that covers all 26).
//
// lrf_components_select ranks the components by size (descending, ties by label) and compacts the kept vertices in
// their original order, both with KeySlotSort.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"
#include "lrf_table.cuh"

namespace lrf {

namespace {

constexpr int CC_THREADS = 256;
constexpr int NO_INDEX = 0x7fffffff;       // an empty cell's lowest point
constexpr unsigned long long SIZE_MAX31 = 0x7fffffffull;

// The root of v.  Path halving: v's parent becomes its grandparent (atomicMin, so a shortcut never raises a parent
// another thread lowered), and the walk goes on from there.
__device__ __forceinline__ int find_root(int* parent, int v) {
  int p = __ldcg(parent + v);
  while (p != v) {
    const int g = __ldcg(parent + p);
    if (g == p) return p;
    atomicMin(parent + v, g);
    v = g;
    p = __ldcg(parent + v);
  }
  return v;
}

// One set of a and b: the higher root is hooked under the lower, and a CAS that finds the higher one no longer a root
// retries from the root of its new parent.
__device__ __forceinline__ void unite(int* parent, int a, int b) {
  a = find_root(parent, a);
  b = find_root(parent, b);
  while (a != b) {
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicCAS(parent + b, b, a);
    if (old == b) return;
    b = find_root(parent, old);
  }
}

// size[r] += 1 for each lane with ok, one atomic per distinct r in the warp (every lane of the warp calls it)
__device__ __forceinline__ void add_sizes(unsigned long long* size, bool ok, int r) {
  const unsigned active = __ballot_sync(0xffffffffu, ok);
  if (!ok) return;
  const unsigned peers = __match_any_sync(active, r);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(size + r, (unsigned long long)__popc(peers));
}

// adds the warp's lanes with `flag` to *counter (every lane of the warp calls it)
__device__ __forceinline__ void count_lanes(unsigned long long* counter, bool flag) {
  const unsigned m = __ballot_sync(0xffffffffu, flag);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(counter, (unsigned long long)__popc(m));
}

// parent[v] = v and size[v] = 0 for v < n; an empty table of `cap` slots (cap may be 0); stats[0, n_stats) = 0
__global__ void __launch_bounds__(CC_THREADS) init_kernel(int* parent, unsigned long long* size, long long n,
                                                          unsigned long long* keys, int* first, long long cap,
                                                          unsigned long long* stats, int n_stats) {
  const long long i = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  if (i < n) { parent[i] = (int)i; size[i] = 0; }
  if (i < cap) { keys[i] = 0; first[i] = NO_INDEX; }
  if (i < n_stats) stats[i] = 0;
}

// One thread per triangle: its vertices in one set; a triangle with an index outside [0, V) is counted in stats[0]
__global__ void __launch_bounds__(CC_THREADS) mesh_link_kernel(const int* __restrict__ faces, long long T, int V,
                                                               int* parent, unsigned long long* stats) {
  const long long t = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  bool bad = false;
  if (t < T) {
    const int a = __ldg(faces + 3 * t), b = __ldg(faces + 3 * t + 1), c = __ldg(faces + 3 * t + 2);
    bad = (unsigned)a >= (unsigned)V || (unsigned)b >= (unsigned)V || (unsigned)c >= (unsigned)V;
    if (!bad) {
      unite(parent, a, b);
      unite(parent, a, c);
    }
  }
  count_lanes(stats, bad);
}

// One thread per vertex once every union is done: parent[v] = its root (only ever lowered, so the other threads'
// shortcuts cannot undo it); with `size`, each vertex adds 1 to its root's
__global__ void __launch_bounds__(CC_THREADS) label_kernel(int* parent, long long n, unsigned long long* size) {
  const long long v = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  int r = 0;
  if (v < n) {
    r = find_root(parent, (int)v);
    atomicMin(parent + v, r);
  }
  if (size) add_sizes(size, v < n, r);
}

// One thread per triangle: 1 to the size of its component (at the label of its first vertex)
__global__ void __launch_bounds__(CC_THREADS) mesh_size_kernel(const int* __restrict__ faces, long long T, int V,
                                                               const int* __restrict__ label,
                                                               unsigned long long* size) {
  const long long t = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  bool ok = false;
  int r = 0;
  if (t < T) {
    const int a = __ldg(faces + 3 * t), b = __ldg(faces + 3 * t + 1), c = __ldg(faces + 3 * t + 2);
    ok = (unsigned)a < (unsigned)V && (unsigned)b < (unsigned)V && (unsigned)c < (unsigned)V;
    if (ok) r = __ldg(label + a);
  }
  add_sizes(size, ok, r);
}

struct CellGrid {
  float origin[3];
  float cell;
};

// One thread per point: its cell claimed in the table (claim counter stats[0]), the point's index into the slot's
// minimum, and a union with the point that minimum held before (every point of a cell but the first to arrive finds
// one).  A point that is not finite or whose cell lies outside [-2^20, 2^20) stays alone and is counted in stats[1].
__global__ void __launch_bounds__(CC_THREADS) point_cells_kernel(const float* __restrict__ xyz, long long n,
                                                                 const CellGrid g, unsigned long long* keys,
                                                                 int* first, long long cap, int* parent,
                                                                 unsigned long long* stats) {
  const long long p = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  bool in = false, out = false;
  unsigned long long key = 0;
  if (p < n && !table_full(stats, cap)) {
    in = cell_key(xyz + 3 * p, g.origin, g.cell, key, [](int, float, float) {});
    out = !in;
  }
  count_lanes(stats + 1, out);
  if (!in) return;
  int held = NO_INDEX;
  find_or_claim(keys, cap, stats, key, [&](unsigned long long slot, bool) { held = atomicMin(first + slot, (int)p); });
  if (held != NO_INDEX) unite(parent, (int)p, held);
}

// One thread per slot once every cell is claimed: the cell's lowest point united with those of the occupied cells
// among its 13 forward neighbours, offsets (dx, dy, dz) in {-1, 0, 1}^3 after (0, 0, 0) in lexicographic order.
__global__ void __launch_bounds__(CC_THREADS) cell_link_kernel(const unsigned long long* __restrict__ keys,
                                                               const int* __restrict__ first, long long cap,
                                                               const unsigned long long* stats, int* parent) {
  const long long s = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  if (s >= cap || table_full(stats, cap)) return;
  const unsigned long long tag = __ldg(keys + s);
  if (tag == 0) return;
  const int rep = __ldg(first + s);
  const int k[3] = {(int)cell_field(tag - 1, 0), (int)cell_field(tag - 1, 1), (int)cell_field(tag - 1, 2)};
  for (int o = 14; o < 27; ++o) {
    const int m[3] = {k[0] + o / 9 - 1, k[1] + (o / 3) % 3 - 1, k[2] + o % 3 - 1};
    const unsigned field = (unsigned)KEY_FIELD;
    if ((unsigned)m[0] > field || (unsigned)m[1] > field || (unsigned)m[2] > field) continue;
    const int ns = find_slot(keys, cap, cell_key_of(m));
    if (ns >= 0) unite(parent, rep, __ldg(first + ns));
  }
}

// sort input: the rank key (2^31 - 1 - size) << 31 | v at each root v (label[v] == v), size clamped to [0, 2^31 - 1],
// NO_KEY (sorted last) at the other vertices; comp_rank[v] = -1 and counts = 0 until the later launches write them
__global__ void __launch_bounds__(CC_THREADS) rank_keys_kernel(const int* __restrict__ label,
                                                               const long long* __restrict__ size, long long n,
                                                               unsigned long long* keys, unsigned int* slots,
                                                               int* comp_rank, long long* counts) {
  const long long v = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  if (v < 4) counts[v] = 0;
  if (v >= n) return;
  unsigned long long key = NO_KEY;
  if (__ldg(label + v) == (int)v) {
    const long long s = __ldg(size + v);
    const unsigned long long c = s <= 0 ? 0 : s < (long long)SIZE_MAX31 ? (unsigned long long)s : SIZE_MAX31;
    key = ((SIZE_MAX31 - c) << 31) | (unsigned long long)v;
  }
  keys[v] = key;
  slots[v] = (unsigned int)v;
  comp_rank[v] = -1;
}

// the size a rank key holds
__device__ __forceinline__ long long key_size(unsigned long long key) { return (long long)(SIZE_MAX31 - (key >> 31)); }

// component i of the ranking -> sizes_sorted[i]; a kept one (size >= min_size, and i < keep unless keep is 0) gets
// comp_rank[its label] = i.  The kept ones are a prefix of the ranking; counts[1] = kept, counts[2] = components,
// counts[3] += the kept sizes.
__global__ void __launch_bounds__(CC_THREADS) rank_write_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                long long keep, long long min_size, int* comp_rank,
                                                                long long* sizes_sorted, long long* counts) {
  const long long i = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  const unsigned long long key = i < n ? keys[i] : NO_KEY;
  const unsigned long long next = i + 1 < n ? keys[i + 1] : NO_KEY;
  const bool is = key != NO_KEY;
  const bool kept = is && key_size(key) >= min_size && (keep == 0 || i < keep);
  const bool next_kept = next != NO_KEY && key_size(next) >= min_size && (keep == 0 || i + 1 < keep);
  unsigned long long s = kept ? (unsigned long long)key_size(key) : 0;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd((unsigned long long*)counts + 3, s);
  if (!is) return;
  sizes_sorted[i] = key_size(key);
  if (kept) comp_rank[key & SIZE_MAX31] = (int)i;
  if (kept && !next_kept) counts[1] = i + 1;
  if (next == NO_KEY) counts[2] = i + 1;
}

// sort input of the compaction: v for a kept vertex, NO_KEY for a dropped one (whose new_index is -1)
__global__ void __launch_bounds__(CC_THREADS) kept_keys_kernel(const int* __restrict__ label, long long n,
                                                               const int* __restrict__ comp_rank,
                                                               unsigned long long* keys, unsigned int* slots,
                                                               int* new_index) {
  const long long v = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  if (v >= n) return;
  const int l = __ldg(label + v);
  const bool kept = l >= 0 && l < n && __ldg(comp_rank + l) >= 0;
  keys[v] = kept ? (unsigned long long)v : NO_KEY;
  slots[v] = (unsigned int)v;
  if (!kept) new_index[v] = -1;
}

// row j of the sorted kept vertices: new_index[v] = j, rank[j] = v's component rank; counts[0] = the kept rows
__global__ void __launch_bounds__(CC_THREADS) kept_write_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                const int* __restrict__ label,
                                                                const int* __restrict__ comp_rank, int* new_index,
                                                                int* rank, long long* counts) {
  const long long j = (long long)blockIdx.x * CC_THREADS + threadIdx.x;
  if (j >= n) return;
  const unsigned long long v = keys[j];
  if (v == NO_KEY) return;
  new_index[v] = (int)j;
  rank[j] = comp_rank[label[v]];
  if (j + 1 == n || keys[j + 1] == NO_KEY) counts[0] = j + 1;
}

}  // namespace

cudaError_t launch_mesh_components(const int* faces, long long T, long long V, int* label, unsigned long long* size,
                                   unsigned long long* stats, cudaStream_t stream) {
  init_kernel<<<item_ctas(V > 1 ? V : 1, CC_THREADS), CC_THREADS, 0, stream>>>(label, size, V, nullptr, nullptr, 0,
                                                                               stats, 1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || T == 0) return e;
  mesh_link_kernel<<<item_ctas(T, CC_THREADS), CC_THREADS, 0, stream>>>(faces, T, (int)V, label, stats);
  if ((e = cudaGetLastError()) != cudaSuccess || V == 0) return e;
  label_kernel<<<item_ctas(V, CC_THREADS), CC_THREADS, 0, stream>>>(label, V, nullptr);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  mesh_size_kernel<<<item_ctas(T, CC_THREADS), CC_THREADS, 0, stream>>>(faces, T, (int)V, label, size);
  return cudaGetLastError();
}

cudaError_t launch_point_components(const float* xyz, long long n, const float* origin, float cell_size,
                                    unsigned long long* keys, int* first, long long cap, int* label,
                                    unsigned long long* size, unsigned long long* stats, cudaStream_t stream) {
  init_kernel<<<item_ctas(n > cap ? n : cap, CC_THREADS), CC_THREADS, 0, stream>>>(label, size, n, keys, first, cap,
                                                                                   stats, 2);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || n == 0) return e;
  const CellGrid g = {{origin[0], origin[1], origin[2]}, cell_size};
  point_cells_kernel<<<item_ctas(n, CC_THREADS), CC_THREADS, 0, stream>>>(xyz, n, g, keys, first, cap, label, stats);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  cell_link_kernel<<<item_ctas(cap, CC_THREADS), CC_THREADS, 0, stream>>>(keys, first, cap, stats, label);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  label_kernel<<<item_ctas(n, CC_THREADS), CC_THREADS, 0, stream>>>(label, n, size);
  return cudaGetLastError();
}

// the sort's key and index buffers, the rank of each root, then the sort's temporary storage
ExtractScratch components_select_scratch(long long n) { return ExtractScratch{n, n, 0}; }

cudaError_t launch_components_select(const int* label, const long long* size, long long n, long long keep,
                                     long long min_size, int* new_index, int* rank, long long* sizes_sorted,
                                     long long* counts, void* scratch, cudaStream_t stream) {
  if (n == 0) return cudaMemsetAsync(counts, 0, 4 * sizeof(long long), stream);
  ExtractScratch x = components_select_scratch(n);
  cudaError_t e = x.carve(scratch);
  if (e != cudaSuccess) return e;
  const KeySlotSort& pairs = x.pairs[0];
  int* comp_rank = x.index;
  const unsigned blocks = item_ctas(n, CC_THREADS);
  rank_keys_kernel<<<blocks, CC_THREADS, 0, stream>>>(label, size, n, pairs.keys(), pairs.slots(), comp_rank, counts);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = x.pairs[0].sort(n, x.temp, x.temp_bytes, stream)) != cudaSuccess) return e;
  rank_write_kernel<<<blocks, CC_THREADS, 0, stream>>>(pairs.keys(), n, keep, min_size, comp_rank, sizes_sorted,
                                                       counts);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  kept_keys_kernel<<<blocks, CC_THREADS, 0, stream>>>(label, n, comp_rank, pairs.keys(), pairs.slots(), new_index);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = x.pairs[0].sort(n, x.temp, x.temp_bytes, stream)) != cudaSuccess) return e;
  kept_write_kernel<<<blocks, CC_THREADS, 0, stream>>>(pairs.keys(), n, label, comp_rank, new_index, rank, counts);
  return cudaGetLastError();
}

}  // namespace lrf
