// lrf_select.cuh -- order statistics on the device: the order-preserving 32-bit float keys shared by every kernel
// that selects (lrf_losses.cu sorts them within a view), and an exact device-wide k-th smallest value of fp32 arrays
// of up to 2^31 - 1 elements (lrf_panels.cu).
//
// The selection is a radix select on the keys, most significant byte first: four passes, each one histogram launch
// (integer counts in shared memory, then integer atomics into the job's histogram: the counts do not depend on the
// order in which threads add them) and one tiny launch that picks the byte holding the k-th key and narrows the
// prefix.  The choice runs on the device, so a selection costs eight launches and no host round-trip.  Several jobs
// (array, rank) run in the same launches; blockIdx.y is the job.  A job may also ask for the value at rank k + 1 (the
// upper neighbour of a linear quantile): it is the k-th key itself when that key's run of equal keys reaches k + 1,
// else the smallest key above it, which one more pass finds with an integer atomicMin, only for the jobs that need it.
//
// The keys order -0 before +0.  numpy and torch select by comparison, where the two zeros are equal, so a zero order
// statistic may come back with the other sign than theirs; every other value (NaN included) is the same bits.
//
// Translation units that only need the keys define LRF_SELECT_KEYS_ONLY before including this header.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lrf_launch.cuh"

namespace lrf {

// order-preserving; every NaN becomes the canonical +NaN first, so that NaNs of either sign sort after +inf and
// share one key (0xffffffff, which no other value has)
__device__ inline unsigned int f2key(float f) {
  const unsigned int u = isnan(f) ? 0x7fffffffu : __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ inline float key32_to_f(unsigned int u) { return __uint_as_float(u ^ ((u >> 31) ? 0x80000000u : 0xffffffffu)); }
// the value of a 64-bit (key << 32 | index) sort key
__device__ inline float key2f(unsigned long long k) { return key32_to_f((unsigned int)(k >> 32)); }

#ifndef LRF_SELECT_KEYS_ONLY

constexpr unsigned int SEL_NAN_KEY = 0xffffffffu;
constexpr int SEL_THREADS = 256, SEL_BINS = 256, SEL_PASSES = 4, SEL_MAX_JOBS = 16;

struct SelectJob {
  const float* x;              // [n] device or pinned
  unsigned int n;              // 1 .. 2^31 - 1
  unsigned int k;              // rank, 0-based, < n
  int want_next;               // also find the value at rank k + 1 (k + 1 < n)
};
struct SelectJobs {            // passed by value: no upload
  SelectJob j[SEL_MAX_JOBS];
};

// per job, in device memory: zeroed before the first pass
struct SelectState {
  unsigned int prefix;         // the high bytes of the k-th key chosen so far; after the last pass, its key
  unsigned int k;              // the rank within the keys that share the prefix
  unsigned int n_nan;          // NaNs in the array (counted in pass 0)
  unsigned int need_next;      // after the last pass: rank k + 1 holds a larger key than rank k
  unsigned int next;           // that key (the smallest key above the k-th), when need_next
  unsigned int pad[3];
  unsigned int hist[SEL_PASSES][SEL_BINS];
};

// pass p counts the byte (3 - p) of every key whose higher bytes equal the prefix chosen so far
static __global__ void __launch_bounds__(SEL_THREADS) select_hist_kernel(const SelectJobs jobs,
                                                                          SelectState* __restrict__ st, int pass) {
  __shared__ unsigned int h[SEL_BINS];
  __shared__ unsigned int nan_block;
  const SelectJob& J = jobs.j[blockIdx.y];
  SelectState& S = st[blockIdx.y];
  for (int b = threadIdx.x; b < SEL_BINS; b += blockDim.x) h[b] = 0;
  if (threadIdx.x == 0) nan_block = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const unsigned int mask = pass == 0 ? 0u : 0xffffffffu << (32 - 8 * pass);
  const unsigned int prefix = pass == 0 ? 0u : S.prefix;
  const int lane = threadIdx.x & 31;
  unsigned int nan_count = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  // the loop bound is rounded up to whole warps so that every lane of a warp takes part in the match below
  const long long n_round = ((long long)J.n + 31) & ~31ll;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i - lane < n_round; i += stride) {
    unsigned int digit = SEL_BINS;                   // no bin: outside the array or outside the prefix
    if (i < J.n) {
      const unsigned int key = f2key(J.x[i]);
      if ((key & mask) == prefix) digit = (key >> shift) & 0xffu;
      nan_count += key == SEL_NAN_KEY;
    }
    // warp-aggregated: one shared atomic per distinct digit of the warp (a frame of equal values stays cheap)
    const unsigned int peers = __match_any_sync(0xffffffffu, digit);
    if (digit < SEL_BINS && lane == __ffs(peers) - 1) atomicAdd(&h[digit], (unsigned int)__popc(peers));
  }
  if (pass == 0 && nan_count) atomicAdd(&nan_block, nan_count);
  __syncthreads();
  for (int b = threadIdx.x; b < SEL_BINS; b += blockDim.x)
    if (h[b]) atomicAdd(&S.hist[pass][b], h[b]);
  if (pass == 0 && threadIdx.x == 0 && nan_block) atomicAdd(&S.n_nan, nan_block);
}

// one thread per job: the byte whose bin holds the k-th remaining key.  After the last pass every key of the chosen
// bin equals the k-th key, so rank k + 1 holds the same key unless the bin's count is exhausted.
static __global__ void select_choose_kernel(SelectState* __restrict__ st, const SelectJobs jobs, int n_jobs, int pass) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  SelectState& S = st[j];
  unsigned int k = pass == 0 ? jobs.j[j].k : S.k, prefix = pass == 0 ? 0u : S.prefix;
  unsigned int b = 0;
  for (; b < SEL_BINS - 1; ++b) {
    const unsigned int c = S.hist[pass][b];
    if (k < c) break;
    k -= c;
  }
  S.prefix = prefix | (b << (24 - 8 * pass));
  S.k = k;
  if (pass == SEL_PASSES - 1) {
    S.need_next = jobs.j[j].want_next && k + 1 >= S.hist[pass][b];
    S.next = 0xffffffffu;
  }
}

// the smallest key above the k-th, for the jobs whose rank k + 1 lies beyond the k-th key's run
static __global__ void __launch_bounds__(SEL_THREADS) select_next_kernel(const SelectJobs jobs,
                                                                          SelectState* __restrict__ st) {
  const SelectJob& J = jobs.j[blockIdx.y];
  SelectState& S = st[blockIdx.y];
  if (!S.need_next) return;
  const unsigned int K = S.prefix;
  unsigned int m = 0xffffffffu;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < J.n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned int key = f2key(J.x[i]);
    if (key > K && key < m) m = key;
  }
  m = __reduce_min_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m != 0xffffffffu) atomicMin(&S.next, m);
}

// the k-th smallest value of a finished job, and the value at rank k + 1 of a job that asked for it
__device__ inline float select_value(const SelectState& S) { return key32_to_f(S.prefix); }
__device__ inline float select_next_value(const SelectState& S) { return key32_to_f(S.need_next ? S.next : S.prefix); }

// Enqueues the four passes over n_jobs <= SEL_MAX_JOBS jobs (states zeroed by the caller), and the successor pass
// when a job asks for rank k + 1.
inline cudaError_t launch_select(const SelectJobs& jobs, SelectState* st, int n_jobs, unsigned int n_max, int n_sms,
                                 cudaStream_t stream) {
  const dim3 grid(cta_count(n_max, SEL_THREADS * 8, n_sms, 8), (unsigned)n_jobs);   // about 8 keys per thread
  for (int pass = 0; pass < SEL_PASSES; ++pass) {
    select_hist_kernel<<<grid, SEL_THREADS, 0, stream>>>(jobs, st, pass);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    select_choose_kernel<<<(n_jobs + 31) / 32, 32, 0, stream>>>(st, jobs, n_jobs, pass);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  bool any_next = false;
  for (int j = 0; j < n_jobs; ++j) any_next = any_next || jobs.j[j].want_next;
  if (any_next) {
    select_next_kernel<<<grid, SEL_THREADS, 0, stream>>>(jobs, st);
    return cudaGetLastError();
  }
  return cudaSuccess;
}

#endif  // LRF_SELECT_KEYS_ONLY

}  // namespace lrf
