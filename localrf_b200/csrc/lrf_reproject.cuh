// lrf_reproject.cuh -- the optical-flow reprojection of the reference (get_cam2cams, get_pred_flow, pts2px,
// utils/utils.py:15-48) as device functions, shared by the training losses (lrf_losses.cu) and the test-frame
// panels (lrf_panels.cu).
#pragma once
#include <cuda_runtime.h>

namespace lrf {

__device__ inline float clamp_min(float x, float lo) { return x < lo ? lo : x; }   // NaN passes, as ATen's clamp

// the cam2cam transform from camera `rel` to camera `k` of cam2world [n][3][4] (R = [:, :3], t = [:, 3]):
// Rcc = Rk^T Rrel row-major in m[0..8], tcc = Rk^T trel - Rk^T tk in m[9..11]
__device__ inline void cam2cam(const float* cam2world, long long rel, long long k, float m[12]) {
  const float* K = cam2world + 12 * k;
  const float* Rl = cam2world + 12 * rel;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      m[3 * i + j] = K[0 * 4 + i] * Rl[0 * 4 + j] + K[1 * 4 + i] * Rl[1 * 4 + j] + K[2 * 4 + i] * Rl[2 * 4 + j];
    const float a = K[0 * 4 + i] * Rl[3] + K[1 * 4 + i] * Rl[7] + K[2 * 4 + i] * Rl[11];
    const float c = K[0 * 4 + i] * K[3] + K[1 * 4 + i] * K[7] + K[2 * 4 + i] * K[11];
    m[9 + i] = a + (-c);
  }
}

// the reprojection of one camera-space point through one cam2cam, minus the ray's pixel (get_pred_flow, pts2px)
struct Proj {
  float q[3], z, u, v;
  int zpass;
};
__device__ inline Proj project(const float* m, const float p[3], float f, float cx, float cy, float i, float j) {
  Proj r;
  for (int a = 0; a < 3; ++a) r.q[a] = m[3 * a] * p[0] + m[3 * a + 1] * p[1] + m[3 * a + 2] * p[2] + m[9 + a];
  const float nz = -r.q[2];
  r.zpass = nz >= 1e-6f;
  r.z = clamp_min(nz, 1e-6f);
  r.u = r.q[0] / r.z * f + cx - 0.5f - i;
  r.v = -r.q[1] / r.z * f + cy - 0.5f - j;
  return r;
}

}  // namespace lrf
