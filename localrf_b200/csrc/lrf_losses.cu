// lrf_losses.cu -- the supervision losses of one training step (train.py:369-423) and their backward: the
// loss-weighted L1 rgb term, the optical-flow reprojection term (get_fwd_bwd_cam2cams, get_pred_flow, pts2px,
// utils/utils.py:15-48) with its per-view cut at the 0.9 quantile, and the scale- and shift-invariant
// monocular-depth term (compute_depth_loss, utils/utils.py:50-59) with per-view lower medians and a cut at the
// 0.8 quantile.
//
// Forward: one CTA per view sorts (value, ray index) keys in shared memory (bitonic), so the selections are
// exact: the medians are torch.median's (the lower median sorted[(R-1)/2], or NaN when the view holds one; of the
// rays holding that value, the one with the lowest index) and
// each quantile is torch.quantile's linear interpolation, fp32 rank and fused two-branch lerp included, so the
// thresholds are bit-identical to torch's over the same rows.  The per-ray e and d, both thresholds, the median
// indices and the MAD scales go to caller scratch with the per-view partial sums; a one-CTA kernel sums the
// partials in a fixed order.  Backward: one CTA per view recomputes the per-ray terms but takes every hard
// decision (cut sets, medians) from the forward's scratch; a one-CTA kernel chains the per-view cam2cam
// gradients to cam2world in view order and sums the intrinsics' partials.  No atomics, no host
// synchronisation: results are bitwise repeatable.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launch.cuh"
#include "lrf_reproject.cuh"
#define LRF_SELECT_KEYS_ONLY
#include "lrf_select.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

constexpr int LOSS_THREADS = 256, LOSS_MAX_R = 4096, LOSS_NPART = 32;
constexpr float LOSS_Q_FLOW = 0.9f, LOSS_Q_DEPTH = 0.8f;
// per-view doubles in scratch: 0 rgb sum, 1 weight sum, 2 cut flow sum, 3 cut depth sum, 4..6 d focal / cx / cy,
// 8..19 d(Rcc, tcc) of the backward direction, 20..31 of the forward direction (row-major 3x4)
constexpr int P_RGB = 0, P_W = 1, P_FLOW = 2, P_DEPTH = 3, P_INTR = 4, P_CAM = 8;

struct LossPtrs {                     // scratch, carved
  float *e, *d, *tau_f, *tau_d, *mad;
  int* med;
  double *glob, *part;
};

// The leading part is documented in the header (lrf_supervision_losses): e [N], d [N], tau [2][V], med [V][2].
static LossPtrs carve(ScratchCarver& c, long long N, long long V) {
  LossPtrs p;
  p.e = c.take<float>(4 * (size_t)N, 4);
  p.d = c.take<float>(4 * (size_t)N, 4);
  p.tau_f = c.take<float>(4 * (size_t)V, 4);
  p.tau_d = c.take<float>(4 * (size_t)V, 4);
  p.med = c.take<int>(8 * (size_t)V, 4);
  p.mad = c.take<float>(8 * (size_t)V, 4);
  p.glob = c.take<double>(16, 8);
  p.part = c.take<double>((size_t)LOSS_NPART * 8 * (size_t)V, 8);
  return p;
}

// ---- device helpers -------------------------------------------------------------------------------------
__device__ inline int key2idx(unsigned long long k) { return (int)(k & 0xffffffffu); }

// ascending bitonic sort of P (a power of two) keys; every thread of the CTA calls it
__device__ void bitonic_sort(unsigned long long* k, int P) {
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const unsigned long long a = k[i], b = k[j];
        if ((a > b) == ((i & size) == 0)) {
          k[i] = b;
          k[j] = a;
        }
      }
    }
  __syncthreads();
}

// torch.quantile(row, q, interpolation="linear") over R sorted keys: rank q*(R-1) in fp32, lerp of the two
// neighbours with ATen's two-branch formula (fused as ATen's kernels compute it); a NaN in the row gives NaN
__device__ inline float sorted_quantile(const unsigned long long* k, int R, float q) {
  const float last = key2f(k[R - 1]);
  if (isnan(last)) return last;
  const float r = __fmul_rn(q, (float)(R - 1));
  const int lo = (int)floorf(r), hi = (int)ceilf(r);
  const float w = __fsub_rn(r, (float)lo);
  const float a = key2f(k[lo]), b = key2f(k[hi]);
  const float diff = __fsub_rn(b, a);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, diff, a) : __fmaf_rn(-diff, __fsub_rn(1.0f, w), b);
}

// torch.median(row) over R sorted keys: the lower median sorted[(R-1)/2], or NaN when the row holds one.  Keys order
// equal values by ray index, so the first key of the value's run is the lowest ray holding it.
__device__ inline unsigned long long sorted_median(const unsigned long long* k, int R) {
  int hi = isnan(key2f(k[R - 1])) ? R - 1 : (R - 1) >> 1;
  const unsigned long long run = k[hi] & 0xffffffff00000000ull;
  int lo = 0;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (k[mid] < run) lo = mid + 1;
    else hi = mid;
  }
  return k[lo];
}

// block_sum_fp64, broadcast to every thread
__device__ inline double block_sum_all(double v, double* red) {
  const double s = block_sum_fp64(v, red);
  __syncthreads();
  if (threadIdx.x == 0) red[0] = s;
  __syncthreads();
  return red[0];
}

__device__ inline float sgn(float x) { return (float)((x > 0.f) - (x < 0.f)); }

// one view's two cam2cam transforms (index 0: k = rel - 1, the backward flow; 1: k = rel + 1, the forward flow)
struct ViewCams {
  float m[2][12];     // Rcc row-major 3x3 in [0..8], tcc in [9..11]
  int rel, k[2], valid, fwd_off;
};

__device__ void view_cams(const LrfLossBatch& b, int v, ViewCams& vc) {
  const long long vid = b.view_ids[v];
  const long long rel = vid - b.starting_id;
  vc.valid = rel >= 0 && rel < b.n_cams;
  vc.fwd_off = vid == b.n_cams - 1;                 // the reference compares the absolute id with len(cam2world) - 1
  vc.rel = (int)rel;
  for (int o = 0; o < 2; ++o) {
    long long k = rel + (o ? 1 : -1);
    k = k < 0 ? 0 : (k > b.n_cams - 1 ? b.n_cams - 1 : k);
    vc.k[o] = (int)k;
    if (!vc.valid) {
      for (int i = 0; i < 12; ++i) vc.m[o][i] = __int_as_float(0x7fffffff);
      continue;
    }
    cam2cam(b.cam2world, rel, k, vc.m[o]);
  }
}

// ---- forward ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LOSS_THREADS) losses_view_kernel(LrfLossBatch b, int R, int P, LossPtrs s) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);      // [P]
  float* buf = reinterpret_cast<float*>(keys + P);                             // [R]
  __shared__ double red[LOSS_THREADS / 32];
  __shared__ ViewCams vc;
  __shared__ float sel[2];
  const int v = blockIdx.x;
  const long long base = (long long)v * R;
  double* part = s.part + (size_t)LOSS_NPART * v;

  // rgb: sum_n w_n (|d0| + |d1| + |d2|) and sum_n w_n
  double srgb = 0.0, sw = 0.0;
  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    const long long n = base + i;
    const float w = b.loss_weights[n];
    const float a = fabsf(b.rgb_map[3 * n] - b.rgb_train[3 * n]) * w;
    const float c = fabsf(b.rgb_map[3 * n + 1] - b.rgb_train[3 * n + 1]) * w;
    const float d = fabsf(b.rgb_map[3 * n + 2] - b.rgb_train[3 * n + 2]) * w;
    srgb += (double)a + (double)c + (double)d;
    sw += (double)w;
  }
  srgb = block_sum_fp64(srgb, red);
  sw = block_sum_fp64(sw, red);
  if (threadIdx.x == 0) {
    part[P_RGB] = srgb;
    part[P_W] = sw;
  }

  if (b.use_flow) {
    if (threadIdx.x == 0) view_cams(b, v, vc);
    __syncthreads();
    const float f = b.focal[0], cx = b.center[0], cy = b.center[1];
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
      unsigned long long key = ~0ull;
      if (i < R) {
        const long long n = base + i;
        const float dep = b.depth_map[n];
        const float p[3] = {b.directions[3 * n] * dep, b.directions[3 * n + 1] * dep, b.directions[3 * n + 2] * dep};
        const float pi = (float)b.ij[2 * n], pj = (float)b.ij[2 * n + 1];
        const Proj pb = project(vc.m[0], p, f, cx, cy, pi, pj);
        const Proj pf = project(vc.m[1], p, f, cx, cy, pi, pj);
        float e = (fabsf(pb.u - b.bwd_flow[2 * n]) + fabsf(pb.v - b.bwd_flow[2 * n + 1])) * b.bwd_mask[n];
        e += (fabsf(pf.u - b.fwd_flow[2 * n]) + fabsf(pf.v - b.fwd_flow[2 * n + 1])) * (vc.fwd_off ? 0.f : b.fwd_mask[n]);
        if (!vc.valid) e = __int_as_float(0x7fffffff);
        s.e[n] = e;
        key = ((unsigned long long)f2key(e) << 32) | (unsigned int)i;
      }
      keys[i] = key;
    }
    bitonic_sort(keys, P);
    if (threadIdx.x == 0) sel[0] = sorted_quantile(keys, R, LOSS_Q_FLOW);
    __syncthreads();
    const float tau = sel[0];
    double sf = 0.0;
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
      const float e = key2f(keys[i]);
      if (!(e > tau)) sf += (double)e;
    }
    sf = block_sum_fp64(sf, red);
    if (threadIdx.x == 0) {
      s.tau_f[v] = tau;
      part[P_FLOW] = sf;
    }
  }

  if (b.use_depth) {
    // x = 1 / clamp(depth, 1e-6): lower median t, MAD scale s, xn = (x - t) / s into buf[ray]
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
      unsigned long long key = ~0ull;
      if (i < R) key = ((unsigned long long)f2key(1.0f / clamp_min(b.depth_map[base + i], 1e-6f)) << 32) | (unsigned int)i;
      keys[i] = key;
    }
    for (int pass = 0; pass < 2; ++pass) {           // 0: x (rendered), 1: g (invdepths)
      if (pass == 1) {
        __syncthreads();
        for (int i = threadIdx.x; i < P; i += blockDim.x)
          keys[i] = i < R ? ((unsigned long long)f2key(b.invdepths[base + i]) << 32) | (unsigned int)i : ~0ull;
      }
      bitonic_sort(keys, P);
      const unsigned long long mk = sorted_median(keys, R);
      const float t = key2f(mk);
      double mad = 0.0;
      for (int i = threadIdx.x; i < R; i += blockDim.x) mad += (double)fabsf(key2f(keys[i]) - t);
      mad = block_sum_all(mad, red);
      const float sc = (float)mad / (float)R;
      for (int i = threadIdx.x; i < R; i += blockDim.x) {
        const unsigned long long k = keys[i];
        const float xn = (key2f(k) - t) / sc;
        if (pass == 0) {
          buf[key2idx(k)] = xn;
        } else {
          const float df = buf[key2idx(k)] - xn;
          buf[key2idx(k)] = df * df;
        }
      }
      if (threadIdx.x == 0) {
        s.med[2 * v + pass] = key2idx(mk);
        s.mad[2 * v + pass] = sc;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
      unsigned long long key = ~0ull;
      if (i < R) {
        s.d[base + i] = buf[i];
        key = ((unsigned long long)f2key(buf[i]) << 32) | (unsigned int)i;
      }
      keys[i] = key;
    }
    bitonic_sort(keys, P);
    if (threadIdx.x == 0) sel[1] = sorted_quantile(keys, R, LOSS_Q_DEPTH);
    __syncthreads();
    const float tau = sel[1];
    double sd = 0.0;
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
      const float d = key2f(keys[i]);
      if (!(d > tau)) sd += (double)d;
    }
    sd = block_sum_fp64(sd, red);
    if (threadIdx.x == 0) {
      s.tau_d[v] = tau;
      part[P_DEPTH] = sd;
    }
  }
}

__global__ void __launch_bounds__(LOSS_THREADS) losses_final_kernel(LrfLossBatch b, LossPtrs s, float* losses) {
  __shared__ double red[LOSS_THREADS / 32];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long v = threadIdx.x; v < b.n_views; v += blockDim.x)
    for (int j = 0; j < 4; ++j) acc[j] += s.part[LOSS_NPART * v + j];
  for (int j = 0; j < 4; ++j) acc[j] = block_sum_fp64(acc[j], red);
  if (threadIdx.x == 0) {
    const double N = (double)b.n_rays;
    const double mean_w = acc[P_W] / N;
    s.glob[0] = mean_w;
    losses[0] = (float)(0.25 * acc[P_RGB] / mean_w / (3.0 * N));
    losses[1] = b.use_flow ? (float)(acc[P_FLOW] / N * (double)b.flow_weight) : 0.f;
    losses[2] = b.use_depth ? (float)(acc[P_DEPTH] / N * (double)b.depth_weight) : 0.f;
  }
}

// ---- backward ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LOSS_THREADS) losses_view_backward_kernel(LrfLossBatch b, int R, LossPtrs s,
                                                                            const float* gl, LrfLossGrads g) {
  __shared__ double red[LOSS_THREADS / 32];
  __shared__ double wsum[LOSS_THREADS / 32][27];
  __shared__ ViewCams vc;
  const int v = blockIdx.x;
  const long long base = (long long)v * R;
  const double N = (double)b.n_rays;
  double* part = s.part + (size_t)LOSS_NPART * v;
  const float g_rgb = (float)((double)gl[0] / (3.0 * N) / s.glob[0] * 0.25);
  const float g_flow = (float)((double)gl[1] * (double)b.flow_weight / N);
  const float g_depth = (float)((double)gl[2] * (double)b.depth_weight / N);

  // depth: the per-view sums the median and MAD scale chain through
  float t[2] = {0.f, 0.f}, sc[2] = {1.f, 1.f}, dsd = 0.f, dtx = 0.f;
  int mx = -1;
  if (b.use_depth) {
    mx = s.med[2 * v];
    const int mg = s.med[2 * v + 1];
    t[0] = 1.0f / clamp_min(b.depth_map[base + mx], 1e-6f);
    t[1] = b.invdepths[base + mg];
    sc[0] = s.mad[2 * v];
    sc[1] = s.mad[2 * v + 1];
    const float tau = s.tau_d[v];
    double A = 0.0, B = 0.0, Cs = 0.0;
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
      const long long n = base + i;
      const float x = 1.0f / clamp_min(b.depth_map[n], 1e-6f);
      const float xn = (x - t[0]) / sc[0], gn = (b.invdepths[n] - t[1]) / sc[1];
      const float a = (s.d[n] > tau) ? 0.f : g_depth * 2.f * (xn - gn);
      A += (double)a;
      B += (double)a * (double)xn;
      Cs += (double)sgn(x - t[0]);
    }
    A = block_sum_all(A, red);
    B = block_sum_all(B, red);
    Cs = block_sum_all(Cs, red);
    dsd = (float)(-B / (double)sc[0]);                                   // dL/ds
    dtx = (float)(-A / (double)sc[0] + (double)dsd * (-Cs / (double)R)); // dL/dt, directly and through s
  }

  if (b.use_flow && threadIdx.x == 0) view_cams(b, v, vc);
  __syncthreads();
  const float f = b.use_flow ? b.focal[0] : 0.f, cx = b.use_flow ? b.center[0] : 0.f,
              cy = b.use_flow ? b.center[1] : 0.f;
  const float tau_f = b.use_flow ? s.tau_f[v] : 0.f;
  float acc[27];
#pragma unroll
  for (int j = 0; j < 27; ++j) acc[j] = 0.f;

  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    const long long n = base + i;
    if (g.d_rgb) {
      const float w = b.loss_weights[n] * g_rgb;
      for (int c = 0; c < 3; ++c) g.d_rgb[3 * n + c] = w * sgn(b.rgb_map[3 * n + c] - b.rgb_train[3 * n + c]);
    }
    float dd = 0.f, ddir[3] = {0.f, 0.f, 0.f};
    if (b.use_flow && !(s.e[n] > tau_f)) {
      const float dep = b.depth_map[n];
      const float dir[3] = {b.directions[3 * n], b.directions[3 * n + 1], b.directions[3 * n + 2]};
      const float p[3] = {dir[0] * dep, dir[1] * dep, dir[2] * dep};
      const float pi = (float)b.ij[2 * n], pj = (float)b.ij[2 * n + 1];
      float dp[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        const float* m = vc.m[o];
        const Proj pr = project(m, p, f, cx, cy, pi, pj);
        const float* fl = o ? b.fwd_flow : b.bwd_flow;
        const float mk = o ? (vc.fwd_off ? 0.f : b.fwd_mask[n]) : b.bwd_mask[n];
        const float c = g_flow * mk;
        const float gu = c * sgn(pr.u - fl[2 * n]), gv = c * sgn(pr.v - fl[2 * n + 1]);
        const float iz = 1.0f / pr.z;
        const float xz = pr.q[0] * iz, yz = pr.q[1] * iz;
        float dq[3];
        dq[0] = gu * f * iz;
        dq[1] = -gv * f * iz;
        const float dz = (-gu * xz + gv * yz) * f * iz;
        dq[2] = pr.zpass ? -dz : 0.f;
        acc[0] += gu * xz - gv * yz;          // d focal
        acc[1] += gu;                         // d cx
        acc[2] += gv;                         // d cy
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
          for (int k = 0; k < 3; ++k) acc[3 + 12 * o + 3 * a + k] += dq[a] * p[k];
          acc[3 + 12 * o + 9 + a] += dq[a];
          for (int k = 0; k < 3; ++k) dp[k] += m[3 * a + k] * dq[a];
        }
      }
      for (int k = 0; k < 3; ++k) {
        ddir[k] = dp[k] * dep;
        dd += dp[k] * dir[k];
      }
    }
    if (b.use_depth) {
      const float dm = b.depth_map[n];
      const float x = 1.0f / clamp_min(dm, 1e-6f);
      const float xn = (x - t[0]) / sc[0], gn = (b.invdepths[n] - t[1]) / sc[1];
      const float a = (s.d[n] > s.tau_d[v]) ? 0.f : g_depth * 2.f * (xn - gn);
      float dx = a / sc[0] + dsd * sgn(x - t[0]) / (float)R;
      if (i == mx) dx += dtx;
      if (dm >= 1e-6f) dd += dx * (-(x * x));
    }
    if (g.d_depth) g.d_depth[n] = dd;
    if (g.d_directions)
      for (int k = 0; k < 3; ++k) g.d_directions[3 * n + k] = ddir[k];
  }

  if (b.use_flow) {        // 27 per-view sums: warp shuffles, then warps in order
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 27; ++j) {
      double x = (double)acc[j];
      for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
      if (lane == 0) wsum[warp][j] = x;
    }
    __syncthreads();
    if (threadIdx.x < 27) {
      double x = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) x += wsum[w][threadIdx.x];
      part[threadIdx.x < 3 ? P_INTR + threadIdx.x : P_CAM + threadIdx.x - 3] = x;
    }
  }
}

// without the flow term nothing depends on the cameras or the intrinsics: their gradients are zero
__global__ void __launch_bounds__(LOSS_THREADS) losses_final_backward_kernel(LrfLossBatch b, LossPtrs s,
                                                                             LrfLossGrads g) {
  const int V = b.use_flow ? (int)b.n_views : 0;
  if (threadIdx.x < 3) {
    double x = 0.0;
    for (int v = 0; v < V; ++v) x += s.part[(size_t)LOSS_NPART * v + P_INTR + threadIdx.x];
    if (threadIdx.x == 0 && g.d_focal) g.d_focal[0] = (float)x;
    if (threadIdx.x > 0 && g.d_center) g.d_center[threadIdx.x - 1] = (float)x;
  }
  if (!g.d_cam2world) return;
  const float* C = b.cam2world;
  for (long long idx = threadIdx.x; idx < 12 * b.n_cams; idx += blockDim.x) {
    const int c = (int)(idx / 12), r = (int)(idx % 12) / 4, col = (int)(idx % 4);
    double x = 0.0;
    for (int v = 0; v < V; ++v) {
      const long long rel = b.view_ids[v] - b.starting_id;
      if (rel < 0 || rel >= b.n_cams) continue;       // such a view's loss is NaN; it reaches no camera
      const float* Rl = C + 12 * rel;
      for (int o = 0; o < 2; ++o) {
        long long k = rel + (o ? 1 : -1);
        k = k < 0 ? 0 : (k > b.n_cams - 1 ? b.n_cams - 1 : k);
        if (c != rel && c != k) continue;
        const float* K = C + 12 * k;
        const double* dm = s.part + (size_t)LOSS_NPART * v + P_CAM + 12 * o;   // dRcc [0..8], dtcc [9..11]
        if (c == rel) {                                // Rcc = Rk^T Rrel, tcc = Rk^T (trel - tk)
          if (col < 3) {
            for (int m = 0; m < 3; ++m) x += (double)K[4 * r + m] * dm[3 * m + col];
          } else {
            for (int m = 0; m < 3; ++m) x += (double)K[4 * r + m] * dm[9 + m];
          }
        }
        if (c == k) {
          if (col < 3) {
            for (int j = 0; j < 3; ++j) x += (double)Rl[4 * r + j] * dm[3 * col + j];
            x += ((double)Rl[4 * r + 3] - (double)K[4 * r + 3]) * dm[9 + col];
          } else {
            for (int m = 0; m < 3; ++m) x -= (double)K[4 * r + m] * dm[9 + m];
          }
        }
      }
    }
    g.d_cam2world[idx] = (float)x;
  }
}

// ---- host side --------------------------------------------------------------------------------------------
size_t losses_scratch_bytes(long long N, long long V) {
  ScratchCarver c(nullptr);
  carve(c, N, V);
  return c.size();
}

static int pow2_at_least(int R) {
  int P = 1;
  while (P < R) P <<= 1;
  return P;
}

cudaError_t launch_supervision_losses(const LrfLossBatch& b, float* losses, void* scratch, cudaStream_t stream) {
  cudaError_t e = set_max_dynamic_smem((const void*)losses_view_kernel, LOSS_MAX_R * (8 + 4));
  if (e != cudaSuccess) return e;
  const int R = (int)(b.n_rays / b.n_views), P = pow2_at_least(R);
  ScratchCarver c(scratch);
  const LossPtrs s = carve(c, b.n_rays, b.n_views);
  losses_view_kernel<<<(unsigned)b.n_views, LOSS_THREADS, (size_t)P * 8 + (size_t)R * 4, stream>>>(b, R, P, s);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  losses_final_kernel<<<1, LOSS_THREADS, 0, stream>>>(b, s, losses);
  return cudaGetLastError();
}

cudaError_t launch_supervision_losses_backward(const LrfLossBatch& b, const float* grad_losses, const LrfLossGrads& g,
                                               void* scratch, cudaStream_t stream) {
  const int R = (int)(b.n_rays / b.n_views);
  ScratchCarver c(scratch);
  const LossPtrs s = carve(c, b.n_rays, b.n_views);
  losses_view_backward_kernel<<<(unsigned)b.n_views, LOSS_THREADS, 0, stream>>>(b, R, s, grad_losses, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (g.d_focal || g.d_center || g.d_cam2world) {
    losses_final_backward_kernel<<<1, LOSS_THREADS, 0, stream>>>(b, s, g);
    e = cudaGetLastError();
  }
  return e;
}

}  // namespace lrf
