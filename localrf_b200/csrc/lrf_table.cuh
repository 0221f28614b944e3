// lrf_table.cuh -- the open-addressing table of the geometry exports (LrfVoxelTable of lrf_export.cu, LrfMeshTable of
// lrf_mesh.cu, the cell table of lrf_components.cu), keyed by 64-bit integers below ~0.
//
// Slot i of `keys` holds tag = key + 1, 0 while empty; a slot, once claimed by CAS, never changes.  A key's probe
// starts at probe_start(key) & (capacity - 1) and steps by one slot, wrapping from the last to 0.  A claim counter
// counts the claims, and the table holds at most capacity / 2 keys: the claim that finds the counter there or above
// is an overflow, as is every probe that starts or continues once it is past.  The extracts sort the tables by key,
// with NO_KEY (sorted last) for the slots they leave out (lrf_launchers.cuh, KeySlotSort, ExtractScratch).  The
// voxel and cell tables are keyed by cell_key below.
#pragma once
#include <cuda_runtime.h>

namespace lrf {

constexpr unsigned long long NO_KEY = ~0ull;

// splitmix64's finaliser: the probe start of a key
__device__ __forceinline__ unsigned long long probe_start(unsigned long long x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// whether the table has overflowed: more than capacity / 2 claims so far (a volatile read of the claim counter, to
// which other threads add while the table fills)
__device__ __forceinline__ bool table_full(const unsigned long long* counter, long long capacity) {
  return *reinterpret_cast<const volatile unsigned long long*>(counter) > ((unsigned long long)capacity >> 1);
}

// The slot of `key` (capacity is at most 2^30), claimed when no slot holds it yet -> -1 once the table has
// overflowed.  Before it returns a slot it calls on_slot(slot, claimed), claimed when this call made the claim.  The
// caller's work at the slot sits in the probe loop that way, where the compiler keeps it on the claim and find paths
// without a join.
template <typename OnSlot>
__device__ __forceinline__ int find_or_claim(unsigned long long* keys, long long capacity, unsigned long long* counter,
                                             unsigned long long key, OnSlot on_slot) {
  const unsigned long long half = (unsigned long long)capacity >> 1, mask = (unsigned long long)capacity - 1;
  const unsigned long long tag = key + 1;
  unsigned long long slot = probe_start(key) & mask;
  for (long long probe = 0; probe < capacity; ++probe, slot = (slot + 1) & mask) {
    unsigned long long cur = __ldcg(keys + slot);
    if (cur == 0) {
      cur = atomicCAS(keys + slot, 0ull, tag);
      if (cur == 0) {
        if (atomicAdd(counter, 1ull) >= half) return -1;   // more than capacity / 2 keys: overflow
        on_slot(slot, true);
        return (int)slot;
      }
    }
    if (cur == tag) {
      on_slot(slot, false);
      return (int)slot;
    }
    if (table_full(counter, capacity)) return -1;
  }
  return -1;
}

// The cell key of the point cloud's voxels (lrf_export.cu) and of the components' cells (lrf_components.cu): cell
// k = floor(q), q = (p - origin) / size with round-to-nearest fp32 operations in that order, on each axis; a cell with
// every k in [-2^20, 2^20) is keyed by k + 2^20 in KEY_BITS bits per axis, x highest (63 bits, below NO_KEY).
constexpr int KEY_BITS = 21;
constexpr float KEY_LIM = 1048576.0f;           // 2^20
constexpr unsigned long long KEY_FIELD = (1ull << KEY_BITS) - 1;

// The cell of point p (p[0 .. 2]) -> whether it lies in the key range (false for NaN), and then its key.  On each
// axis a whose cell and those before it are in range it calls on_axis(a, q, k) as it packs k, so the caller's
// per-axis work sits in the loop.
template <typename OnAxis>
__device__ __forceinline__ bool cell_key(const float* p, const float* origin, float size, unsigned long long& key,
                                         OnAxis on_axis) {
  bool in_range = true;
  key = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float q = __fdiv_rn(__fsub_rn(p[a], origin[a]), size);
    const float k = floorf(q);
    in_range = in_range && k >= -KEY_LIM && k < KEY_LIM;
    if (in_range) {
      on_axis(a, q, k);
      key = (key << KEY_BITS) | (unsigned long long)((int)k + (1 << 20));
    }
  }
  return in_range;
}

// axis a's field k + 2^20 of a cell key (x: a = 0), in [0, 2^21)
__device__ __forceinline__ unsigned long long cell_field(unsigned long long key, int a) {
  return (key >> (KEY_BITS * (2 - a))) & KEY_FIELD;
}

// the key of the cell whose fields are f (each in [0, 2^21))
__device__ __forceinline__ unsigned long long cell_key_of(const int (&f)[3]) {
  return ((unsigned long long)f[0] << (2 * KEY_BITS)) | ((unsigned long long)f[1] << KEY_BITS) |
         (unsigned long long)f[2];
}

// The slot holding `key` in a table no thread is claiming in -> -1 when none holds it.  The table is at most half
// full, so an empty slot ends every probe for an absent key.
__device__ __forceinline__ int find_slot(const unsigned long long* keys, long long capacity, unsigned long long key) {
  const unsigned long long mask = (unsigned long long)capacity - 1, tag = key + 1;
  unsigned long long slot = probe_start(key) & mask;
  for (long long probe = 0; probe < capacity; ++probe, slot = (slot + 1) & mask) {
    const unsigned long long cur = __ldg(keys + slot);
    if (cur == tag) return (int)slot;
    if (cur == 0) return -1;
  }
  return -1;
}

}  // namespace lrf
