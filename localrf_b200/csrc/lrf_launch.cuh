// lrf_launch.cuh -- the launch conventions the kernel files share: the fixed-order fp64 CTA sum, the CTA count of a
// capped grid-stride launch and of a one-thread-per-item launch, the carving of a caller's scratch block, and the
// one-time opt-in to large dynamic shared memory and choice of the shared-memory carveout.
//
// Not included from lrf_common.cuh or lrf_device.cuh: tests/host_emul compiles those with a host compiler.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace lrf {

// The sum of v over the CTA: warp shuffles down, then the warps' sums in warp order by thread 0.  The order depends
// on blockDim alone, so the result is bitwise repeatable.  red holds blockDim.x / 32 doubles; the result is valid in
// thread 0.
__device__ inline double block_sum_fp64(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();                                   // red may still be read by a previous call
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < nw; ++w) s += red[w];
  return s;
}

// CTAs for `work` items at `per_cta` items each, at most `per_sm` CTAs per SM and at least one.  The kernels loop over
// what a capped grid leaves, and the cap is part of each kernel's summation order where it sums.
inline unsigned int cta_count(long long work, long long per_cta, int n_sms, int per_sm) {
  const long long want = (work + per_cta - 1) / per_cta, cap = (long long)n_sms * per_sm;
  return (unsigned int)(want < 1 ? 1 : (want < cap ? want : cap));
}

// CTAs of `threads` for a kernel with one thread per item of n.  Not capped: these kernels do not loop.
inline unsigned int item_ctas(long long n, int threads) { return (unsigned int)((n + threads - 1) / threads); }

// Consecutive arrays in a caller's scratch block.  take(bytes, align) returns the next `bytes` from the first offset
// that is a multiple of `align` (a power of two).  On a null base it only counts: the *_scratch_bytes functions and
// the launchers run the same description of a layout, the former for its size.
struct ScratchCarver {
  unsigned char* base;
  size_t off = 0;

  explicit ScratchCarver(void* b) : base(static_cast<unsigned char*>(b)) {}

  template <typename T = unsigned char>
  T* take(size_t bytes, size_t align) {
    off = (off + align - 1) & ~(align - 1);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += bytes;
    return p;
  }
  // the bytes taken so far, rounded up to a multiple of `align`
  size_t size(size_t align = 1) const { return (off + align - 1) & ~(align - 1); }
};

// Lets `kernel` launch with `bytes` of dynamic shared memory on the current device: sets the attribute when bytes
// exceeds what this kernel already has there.  Safe under concurrent callers; a kernel already configured takes no
// lock.  Defined in lrf_abi.cu.
cudaError_t set_max_dynamic_smem(const void* kernel, int bytes);

// Sets `kernel`'s shared-memory carveout on the current device to the smallest step that holds a CTA of `cta_bytes`
// of shared memory, when it was last set for another CTA size.  Safe under concurrent callers, as above.  Defined in
// lrf_abi.cu.
cudaError_t set_smem_carveout(const void* kernel, int cta_bytes);

}  // namespace lrf
