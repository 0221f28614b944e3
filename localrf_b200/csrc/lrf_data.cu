// lrf_data.cu -- the supervision gather of a training batch from device-resident frames: what
// LocalRFDataset.sample (dataLoader/localrf_dataset.py:273-315) does with numpy fancy indexing over the host arrays
// of every active frame, after the host has drawn the view and pixel ids.
//
// One thread per ray reads its view id and pixel, finds the frame's slot (frame f lives in slot f % capacity) and
// copies the ray's rgb, loss weight and, when the store has them, inverse depth, flows and flow masks.  A ray whose
// view is not the frame its slot holds, or whose pixel is outside the frame, gets NaN in every row instead: no
// other frame's data is ever read.  A batch is ~4096 rays x 11 floats, so the launch is latency-bound (one wave of
// 16 CTAs, dependent loads of the ids then the data); there is nothing to tune.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launchers.cuh"

namespace lrf {

namespace {

constexpr int GATHER_THREADS = 256;

__global__ void __launch_bounds__(GATHER_THREADS) gather_rays_kernel(const LrfFrameStore s, const LrfRayGather g) {
  const long long r = (long long)blockIdx.x * GATHER_THREADS + threadIdx.x;
  if (r >= g.n_rays) return;
  const long long view = g.ids[r / (g.n_rays / g.n_views)];
  const long long pix = g.ids[g.n_views + r];
  g.idx[r] = view * s.n_px + pix;
  const long long slot = view >= 0 ? view % s.capacity : 0;
  const bool ok = view >= 0 && pix >= 0 && pix < s.n_px && s.slot_frame[slot] == view;
  const long long p = slot * s.n_px + pix;           // only dereferenced when ok
  const float nan = __int_as_float(0x7fc00000);
  for (int c = 0; c < 3; ++c) g.rgb[3 * r + c] = ok ? s.rgb[3 * p + c] : nan;
  g.loss_weight[r] = ok ? s.loss_weight[p] : nan;
  if (s.invdepth) g.invdepth[r] = ok ? s.invdepth[p] : nan;
  if (s.fwd_flow) {
    for (int c = 0; c < 2; ++c) {
      g.fwd_flow[2 * r + c] = ok ? s.fwd_flow[2 * p + c] : nan;
      g.bwd_flow[2 * r + c] = ok ? s.bwd_flow[2 * p + c] : nan;
    }
    g.fwd_mask[r] = ok ? s.fwd_mask[p] : nan;
    g.bwd_mask[r] = ok ? s.bwd_mask[p] : nan;
  }
}

}  // namespace

cudaError_t launch_gather_rays(const LrfFrameStore& s, const LrfRayGather& g, cudaStream_t stream) {
  if (g.n_rays == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((g.n_rays + GATHER_THREADS - 1) / GATHER_THREADS);
  gather_rays_kernel<<<blocks, GATHER_THREADS, 0, stream>>>(s, g);
  return cudaGetLastError();
}

}  // namespace lrf
