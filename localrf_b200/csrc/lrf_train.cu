// lrf_train.cu -- the training call of LocalTensorfs.forward (local_tensorfs.py:397-499, is_train) around the render
// kernel and its backward: gradients of the cameras, intrinsics, exposure and world2rf.
//
//   forward   lrf_render in ray-generation mode with finalize = 0 writes rgb_linear; exposure_clamp_kernel then
//             writes rgb = clamp(E_v rgb_linear, 0, 1) with the render kernel's own finalize arithmetic.
//   backward  1. ray_prologue_kernel: per ray, the generated rays (generate_ray, the render kernel's function) go to
//                scratch; g' = g [0 <= E x <= 1] (both ends pass, as torch's clamp backward does); g_lin = E^T g'.
//             2. the field backward of lrf_backward.cu (march, shade, density) on the scratch rays -> d_rays, with
//                each shaded sample's colour-branch position gradient in its own slot (dpos) rather than added
//                atomically per ray, so d_rays -- and everything stage 3 derives from it -- is repeatable.
//             3. cam_view_kernel: one CTA per view reduces d_cam2world, d_exposure and the view's partials of
//                d_world2rf / d_intrinsics; cam_final_kernel sums the partials over the views.
// The reductions use fp64 accumulators in a fixed order (per-thread strides, xor butterflies, warps in order,
// views in order) and no atomics, so the camera gradients are bitwise repeatable.
#include "../../include/localrf_b200.h"
#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

namespace {

constexpr int PART = 8;            // per-view fp64 partials: d_world2rf [3], d_intrinsics [3], 2 unused
constexpr int CAM_THREADS = 256;
constexpr int CAM_ACC = 24;        // d_cam2world [12], d_exposure [9], d_intrinsics [3]

struct TrainScratch {
  float *rays, *dirs, *g_lin, *g_clip, *d_rays, *dpos;
  double* part;
  void* field;                     // the field backward's own block
};

// in the order of the header's description, each array 16-byte aligned
TrainScratch carve(ScratchCarver& c, long long n, int S, long long V) {
  TrainScratch s;
  s.rays = c.take<float>((size_t)n * 6 * 4, 16);
  s.dirs = c.take<float>((size_t)n * 3 * 4, 16);
  s.g_lin = c.take<float>((size_t)n * 3 * 4, 16);
  s.g_clip = c.take<float>((size_t)n * 3 * 4, 16);
  s.d_rays = c.take<float>((size_t)n * 6 * 4, 16);
  s.part = c.take<double>((size_t)V * PART * 8, 16);
  s.dpos = c.take<float>((size_t)n * S * 3 * 4, 16);
  s.field = c.take(backward_scratch_bytes(n, S), 16);
  return s;
}

}  // namespace

__global__ void exposure_clamp_kernel(const float* __restrict__ x, const float* __restrict__ E, long long n,
                                      long long rpv, float* __restrict__ rgb) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    float c[3] = {x[3 * r], x[3 * r + 1], x[3 * r + 2]};
    finalize_rgb(E ? E + 9 * (r / rpv) : nullptr, c);
    rgb[3 * r] = c[0]; rgb[3 * r + 1] = c[1]; rgb[3 * r + 2] = c[2];
  }
}

__global__ void ray_prologue_kernel(const BatchDev B, const float* __restrict__ x, const float* __restrict__ g,
                                    TrainScratch s) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < B.n_rays;
       r += (long long)gridDim.x * blockDim.x) {
    const long long view = r / B.rays_per_view;
    float o[3], d[3];
    generate_ray(B, r, view, o, d, s.dirs + 3 * r, nullptr);
#pragma unroll
    for (int a = 0; a < 3; ++a) { s.rays[6 * r + a] = o[a]; s.rays[6 * r + 3 + a] = d[a]; }
    const float* E = B.exposure ? B.exposure + 9 * view : nullptr;
    float y[3] = {x[3 * r], x[3 * r + 1], x[3 * r + 2]};
    expose_rgb(E, y);                                              // the forward's pre-clamp value
    float gp[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      gp[a] = (y[a] >= 0.0f && y[a] <= 1.0f) ? g[3 * r + a] : 0.0f;
      s.g_clip[3 * r + a] = gp[a];
    }
#pragma unroll
    for (int b = 0; b < 3; ++b)                                    // g_lin = E^T g'
      s.g_lin[3 * r + b] = E ? __fmaf_rn(E[6 + b], gp[2], __fmaf_rn(E[3 + b], gp[1], __fmul_rn(E[b], gp[0]))) : gp[b];
  }
}

__global__ void __launch_bounds__(CAM_THREADS)
cam_view_kernel(const BatchDev B, const float* __restrict__ x, const float* __restrict__ d_rays,
                const float* __restrict__ g_dirs, const TrainScratch s, float* d_c2w, float* d_expo) {
  __shared__ double red[CAM_THREADS / 32][CAM_ACC];
  const long long v = blockIdx.x, R = B.rays_per_view;
  const float* c = B.c2w + 12 * v;
  double Rm[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) Rm[3 * a + b] = c[4 * a + b];
  double focal = B.focal;
  if (B.intrinsics) focal = B.intrinsics[0];
  double acc[CAM_ACC];
#pragma unroll
  for (int k = 0; k < CAM_ACC; ++k) acc[k] = 0.0;
  for (long long t = threadIdx.x; t < R; t += CAM_THREADS) {
    const long long r = v * R + t;
    double dd[3], dc[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      dd[a] = d_rays[6 * r + 3 + a];
      dc[a] = s.dirs[3 * r + a];
      acc[4 * a + 3] += d_rays[6 * r + a];                         // rays_o = t + world2rf
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)                                    // rays_d = R dc
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[4 * a + b] += dd[a] * dc[b];
#pragma unroll
    for (int a = 0; a < 3; ++a)                                    // rgb = clamp(E x): dE = g' x^T
#pragma unroll
      for (int b = 0; b < 3; ++b) acc[12 + 3 * a + b] += (double)s.g_clip[3 * r + a] * (double)x[3 * r + b];
    if (!B.fov360) {                                               // dc = ((i - cx) / f, -(j - cy) / f, -1)
      double ddc[2];
#pragma unroll
      for (int b = 0; b < 2; ++b)
        ddc[b] = Rm[b] * dd[0] + Rm[3 + b] * dd[1] + Rm[6 + b] * dd[2] + (g_dirs ? (double)g_dirs[3 * r + b] : 0.0);
      acc[21] += -(ddc[0] * dc[0] + ddc[1] * dc[1]) / focal;
      acc[22] += -ddc[0] / focal;
      acc[23] += ddc[1] / focal;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < CAM_ACC; ++k) {
    double u = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) u += __shfl_xor_sync(0xffffffffu, u, o);
    if (lane == 0) red[warp][k] = u;
  }
  __syncthreads();
  if (threadIdx.x < CAM_ACC) {
    const int k = threadIdx.x;
    double u = 0.0;
    for (int w = 0; w < CAM_THREADS / 32; ++w) u += red[w][k];
    if (k < 12) {
      if (d_c2w) d_c2w[12 * v + k] = (float)u;
      if (k % 4 == 3) s.part[PART * v + k / 4] = u;
    } else if (k < 21) {
      if (d_expo) d_expo[9 * v + k - 12] = (float)u;
    } else {
      s.part[PART * v + 3 + (k - 21)] = u;
    }
  }
}

__global__ void cam_final_kernel(const TrainScratch s, long long V, int fov360, float* d_intr, float* d_w2rf) {
  const int k = threadIdx.x;
  if (k >= 6) return;
  double u = 0.0;
  for (long long v = 0; v < V; ++v) u += s.part[PART * v + k];
  if (k < 3) {
    if (d_w2rf) d_w2rf[k] = (float)u;
  } else if (d_intr) {
    d_intr[k - 3] = fov360 ? 0.0f : (float)u;
  }
}

// ---- host-side launchers --------------------------------------------------------------------------
size_t train_backward_scratch_bytes(long long n, int S, long long V) {
  ScratchCarver c(nullptr);
  carve(c, n, S, V);
  return c.size(16);
}

cudaError_t launch_exposure_clamp(const float* x, const float* E, long long n, long long V, float* rgb, int n_sms,
                                  cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  exposure_clamp_kernel<<<cta_count(n, 256, n_sms, 8), 256, 0, stream>>>(x, E, n, n / V, rgb);
  return cudaGetLastError();
}

cudaError_t launch_render_backward_batch(const FieldDev& F, const BatchDev& B, const float* bp, const float* x,
                                         const float* g_rgb, const float* g_depth, const float* g_dirs,
                                         const LrfGradients& G, const LrfCameraGrads& CG, void* scratch,
                                         long long n_views, int n_sms, cudaStream_t stream) {
  ScratchCarver c(scratch);
  const TrainScratch s = carve(c, B.n_rays, F.S, n_views);
  cudaError_t e = cudaMemsetAsync(s.dpos, 0, (size_t)B.n_rays * F.S * 3 * 4, stream);
  if (e != cudaSuccess) return e;
  ray_prologue_kernel<<<cta_count(B.n_rays, 256, n_sms, 8), 256, 0, stream>>>(B, x, g_rgb, s);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  LrfGradients G2 = G;
  if (!G2.d_rays) G2.d_rays = s.d_rays;
  e = launch_render_backward_abi(F, s.rays, B.n_rays, B.white_bg, s.g_lin, g_depth, bp, G2, s.field, n_sms, stream,
                                 s.dpos);
  if (e != cudaSuccess) return e;
  cam_view_kernel<<<(unsigned)n_views, CAM_THREADS, 0, stream>>>(B, x, G2.d_rays, g_dirs, s, CG.d_cam2world,
                                                               CG.d_exposure);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  cam_final_kernel<<<1, 32, 0, stream>>>(s, n_views, B.fov360, CG.d_intrinsics, CG.d_world2rf);
  return cudaGetLastError();
}

}  // namespace lrf
