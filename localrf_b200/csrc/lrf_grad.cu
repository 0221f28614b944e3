// lrf_grad.cu -- differentiable VM lookups for the training path: the 72 plane x line appearance
// products (forward) and the backward of the density / appearance lookups (gradients to the
// channel-last planes and lines by atomic adds, and to the sample coordinates).
//
// Reference semantics: F.grid_sample(align_corners=True, padding_mode="border") forward/backward as
// used by compute_densityfeature / compute_appfeature (models/tensoRF.py:112-196); a clipped
// coordinate gets zero gradient (ATen clip_coordinates_set_grad).
#include "lrf_device.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

// forward: prod[m][i*C + c] = bilinear(plane_i[c]) * linear(line_i[c])      (tensoRF.py:174-194)
__global__ void app_products_kernel(const FieldDev F, const float* __restrict__ xyz, long long M,
                                    float* __restrict__ out) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float q[3] = {xyz[3 * m], xyz[3 * m + 1], xyz[3 * m + 2]};
  float feat[CA];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    app_plane_features_t<false>(F, i, q, feat);
#pragma unroll
    for (int c = 0; c < CA; c += 4)
      *reinterpret_cast<float4*>(out + m * NF + i * CA + c) =
          make_float4(feat[c], feat[c + 1], feat[c + 2], feat[c + 3]);
  }
}

struct GradPtrs {
  float* plane[3];
  float* line[3];
};

__global__ void density_backward_kernel(const FieldDev F, const GradPtrs G,
                                        const float* __restrict__ xyz,
                                        const float* __restrict__ gout, long long M,
                                        float* __restrict__ dxyz) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float q[3] = {xyz[3 * m], xyz[3 * m + 1], xyz[3 * m + 2]};
  const float gm = gout[m];
  float dq[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int i = 0; i < 3; ++i)
    vm_pair_backward<CD>(F.g, i, F.dplane[i], F.dline[i], G.plane[i], G.line[i], q,
                         [&](int) { return gm; }, dq);
  if (dxyz) { dxyz[3 * m] = dq[0]; dxyz[3 * m + 1] = dq[1]; dxyz[3 * m + 2] = dq[2]; }
}

__global__ void app_products_backward_kernel(const FieldDev F, const GradPtrs G,
                                             const float* __restrict__ xyz,
                                             const float* __restrict__ gout, long long M,
                                             float* __restrict__ dxyz) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float q[3] = {xyz[3 * m], xyz[3 * m + 1], xyz[3 * m + 2]};
  const float* gm = gout + m * NF;
  float dq[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int i = 0; i < 3; ++i)
    vm_pair_backward<CA>(F.g, i, F.aplane[i], F.aline[i], G.plane[i], G.line[i], q,
                         [&](int c) { return __ldg(gm + i * CA + c); }, dq);
  if (dxyz) { dxyz[3 * m] = dq[0]; dxyz[3 * m + 1] = dq[1]; dxyz[3 * m + 2] = dq[2]; }
}

// ---- host-side launchers --------------------------------------------------------------------------
cudaError_t launch_app_products(const FieldDev& F, const float* xyz, long long M, float* out,
                                cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  app_products_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(F, xyz, M, out);
  return cudaGetLastError();
}

cudaError_t launch_density_backward(const FieldDev& F, float* const* d_plane, float* const* d_line,
                                    const float* xyz, const float* gout, long long M, float* dxyz,
                                    cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  GradPtrs G;
  for (int i = 0; i < 3; ++i) { G.plane[i] = d_plane[i]; G.line[i] = d_line[i]; }
  density_backward_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(F, G, xyz, gout, M, dxyz);
  return cudaGetLastError();
}

cudaError_t launch_app_products_backward(const FieldDev& F, float* const* d_plane,
                                         float* const* d_line, const float* xyz, const float* gout,
                                         long long M, float* dxyz, cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  GradPtrs G;
  for (int i = 0; i < 3; ++i) { G.plane[i] = d_plane[i]; G.line[i] = d_line[i]; }
  app_products_backward_kernel<<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(F, G, xyz, gout, M,
                                                                                 dxyz);
  return cudaGetLastError();
}

}  // namespace lrf
