// lrf_optim.cu -- one Adam step over any number of fp32 tensors in one launch: what torch.optim.Adam.step does on
// CUDA with its default options (torch 2.11's _multi_tensor_adam, the non-capturable branch), bit for bit.
//
// Work is split into (tensor, chunk) items of ADAM_CHUNK elements, one CTA each; a CTA finds its tensor by a
// binary search of the prefix table in the kernel parameters and loops over its chunk in passes of 256 threads x 4
// elements.  16-byte accesses when all four operands of the tensor are 16-byte aligned, scalar otherwise and in the
// tail.  Every element is updated by one thread with the five roundings of torch's foreach sequence:
//   exp_avg    = lerp(exp_avg, g, 1 - beta1)                  _foreach_lerp_      (ATen/native/Lerp.h)
//   exp_avg_sq = exp_avg_sq * beta2                           _foreach_mul_
//   exp_avg_sq = fma(1 - beta2, g * g, exp_avg_sq)            _foreach_addcmul_   (DeviceAddCmulCdiv.cuh)
//   d          = sqrt(exp_avg_sq) / bc2_sqrt + eps            _foreach_sqrt, _foreach_div_, _foreach_add_
//   param      = fma(step_size, exp_avg / d, param)           _foreach_addcdiv_   (DeviceAddCmulCdiv.cuh)
// The intrinsics make each rounding explicit.  Lerp.h leaves `self + weight * (end - self)` to the compiler, which
// contracts it into one fma in ATen's build; the same is written out here.  No atomics, no host synchronisation:
// results are bitwise repeatable.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launchers.cuh"

namespace lrf {

namespace {

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_CHUNK = 16384;   // elements per work item: 16 passes of 256 threads x 4
constexpr int ADAM_MAX_T = 448;     // tensors per launch: the table stays under the 32 KB parameter limit

struct AdamTable {
  int32_t n;
  int32_t chunk_start[ADAM_MAX_T + 1];   // first work item of tensor i; [n] = the launch's total
  LrfAdamTensor t[ADAM_MAX_T];
};
static_assert(sizeof(AdamTable) <= 32764, "kernel parameters are limited to 32764 bytes");

struct AdamScalars {
  float w, one_minus_w, beta2, omb2, eps, step_size, bc2;
  bool small;
};

__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, const AdamScalars& s) {
  // at::native::lerp (Lerp.h): the small-weight branch for |w| < 0.5
  const float diff = __fsub_rn(g, m);
  m = s.small ? __fmaf_rn(s.w, diff, m) : __fmaf_rn(-diff, s.one_minus_w, g);
  v = __fmul_rn(v, s.beta2);
  v = __fmaf_rn(s.omb2, __fmul_rn(g, g), v);
  const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), s.bc2), s.eps);
  p = __fmaf_rn(s.step_size, __fdiv_rn(m, d), p);
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_kernel(const __grid_constant__ AdamTable tab) {
  const int b = blockIdx.x;
  int lo = 0, hi = tab.n - 1;                 // the last tensor whose first item is <= b
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab.chunk_start[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  const LrfAdamTensor& T = tab.t[lo];
  AdamScalars s;
  s.w = T.one_minus_beta1;
  s.one_minus_w = __fsub_rn(1.0f, s.w);
  s.small = fabsf(s.w) < 0.5f;
  s.beta2 = T.beta2;
  s.omb2 = T.one_minus_beta2;
  s.eps = T.eps;
  s.step_size = T.step_size;
  s.bc2 = T.bc2_sqrt;
  const long long start = (long long)(b - tab.chunk_start[lo]) * ADAM_CHUNK;
  const int len = (int)min((long long)ADAM_CHUNK, T.numel - start);
  float* p = T.param + start;
  const float* g = T.grad + start;
  float* m = T.exp_avg + start;
  float* v = T.exp_avg_sq + start;

  int done = 0;
  if ((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0) {
    const int n4 = len >> 2;
    for (int i = threadIdx.x; i < n4; i += ADAM_THREADS) {
      float4 P = reinterpret_cast<const float4*>(p)[i];
      const float4 G = __ldcs(reinterpret_cast<const float4*>(g) + i);
      float4 M = reinterpret_cast<const float4*>(m)[i];
      float4 V = reinterpret_cast<const float4*>(v)[i];
      adam_update(P.x, G.x, M.x, V.x, s);
      adam_update(P.y, G.y, M.y, V.y, s);
      adam_update(P.z, G.z, M.z, V.z, s);
      adam_update(P.w, G.w, M.w, V.w, s);
      reinterpret_cast<float4*>(p)[i] = P;
      reinterpret_cast<float4*>(m)[i] = M;
      reinterpret_cast<float4*>(v)[i] = V;
    }
    done = n4 << 2;
  }
  for (int i = done + threadIdx.x; i < len; i += ADAM_THREADS) {
    float P = p[i], M = m[i], V = v[i];
    adam_update(P, g[i], M, V, s);
    p[i] = P;
    m[i] = M;
    v[i] = V;
  }
}

}  // namespace

// Launches the step over t[0..n) on `stream`, ADAM_MAX_T tensors per launch.  Tensors without elements are skipped.
// The table travels in the kernel parameters, which the launch copies: nothing on the host outlives the call.
cudaError_t launch_adam_step(const LrfAdamTensor* t, long long n, cudaStream_t stream) {
  AdamTable tab;
  tab.n = 0;
  long long items = 0;
  for (long long i = 0; i <= n; ++i) {
    const long long c = i < n ? (t[i].numel + ADAM_CHUNK - 1) / ADAM_CHUNK : 0;
    const bool flush = i == n || tab.n == ADAM_MAX_T || items + c > 0x7fffffffLL;
    if (flush && tab.n > 0) {
      tab.chunk_start[tab.n] = (int32_t)items;
      adam_kernel<<<(unsigned)items, ADAM_THREADS, 0, stream>>>(tab);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return e;
      tab.n = 0;
      items = 0;
    }
    if (i == n || c == 0) continue;
    tab.chunk_start[tab.n] = (int32_t)items;
    tab.t[tab.n++] = t[i];
    items += c;
  }
  return cudaSuccess;
}

}  // namespace lrf
