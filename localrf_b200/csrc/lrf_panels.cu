// lrf_panels.cu -- the flow and depth comparison panels of one held-out frame (renderer.py:79-124): the forward and
// backward optical flow of the rendered depth against the dataset's flows, each channel scaled by the 0.9 quantile
// of [predicted; ground truth] (np.quantile, linear), with the masked error below; and the rendered inverse depth
// against the dataset's, each normalised by its lower median and mean absolute deviation (compute_depth_loss,
// utils/utils.py:50-59), with the squared difference below.
//
// Per frame, all on the caller's stream:
//   prep      one thread per pixel: the nearest-neighbour map of the ground truth (cv2.INTER_NEAREST), the two
//             predicted flows (the reprojection of lrf_reproject.cuh), the error rows of the flow panels, and the
//             arrays the statistics are taken over;
//   select    the exact order statistics (lrf_select.cuh): per flow array numpy's two neighbours in one job (the
//             lower rank, then its successor), per depth array the median;
//   mad       per-block fp64 sums of |v - median| (depth only);
//   stats     one CTA: numpy's lerp between the selected neighbours, the medians, and the MAD sums in a fixed order;
//   finish    one thread per pixel: the normalised, clamped rows.
// No float atomics and no host synchronisation: bitwise repeatable.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launch.cuh"
#include "lrf_reproject.cuh"
#include "lrf_select.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

constexpr int PAN_THREADS = 256, PAN_MAD_BLOCKS = 1024, PAN_NSTATS = 8;
// selection jobs: c + 2 d selects the lower neighbour of flow array (d: 0 fwd, 1 bwd; c: channel) and, when numpy's
// upper neighbour is the next rank, that one too; the medians of x and g follow (or come first without the flow
// branch).  Only above 2^24 values can numpy's float32 index put the upper neighbour two ranks up: it then gets a job
// of its own after the medians.

// what the host folds for the device: np.quantile's rank and weight for n = 2 W H values
struct QuantRule {
  unsigned int lo, hi;
  float gamma;
};

struct PanelArgs {
  LrfPanelFrame f;
  int flow, depth;
  long long n;                 // W H
  double ifx, ify;             // OpenCV's 1 / (dsize / ssize)
  QuantRule q;
  int job_x;                   // first depth job
  int hi_mode;                 // numpy's upper neighbour: 0 the lower one, 1 the next rank, 2 its own job
  int job_hi;                  // first of those jobs (hi_mode 2)
  SelectState* st;
  float* stats;                // [8] in scratch
  double* mad;                 // [2][PAN_MAD_BLOCKS]
  int mad_blocks;
  float* cmp;                  // [4][2 n]: pred_c rows, then gt_c rows
  float* xg;                   // [2][n]: x, g
};

// the scratch: the selection states, the statistics, the MAD partials, cmp, xg
static void carve(ScratchCarver& c, PanelArgs& a) {
  a.st = c.take<SelectState>((size_t)SEL_MAX_JOBS * sizeof(SelectState), 8);
  a.stats = c.take<float>(64, 8);
  a.mad = c.take<double>((size_t)2 * PAN_MAD_BLOCKS * sizeof(double), 8);
  a.cmp = c.take<float>((size_t)4 * 2 * a.n * sizeof(float), 8);
  a.xg = c.take<float>((size_t)2 * a.n * sizeof(float), 8);
}

// clamp(0, 1) as torch's and numpy's: NaN and -0 pass through (only values strictly outside are replaced)
__device__ inline float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }

// cv2.resize(..., INTER_NEAREST): source index min(floor(x * (1 / (dst / src))), src - 1), in double as OpenCV does
__device__ inline int nearest_src(int x, double inv, int src) {
  const int s = (int)floor((double)x * inv);
  return s < src - 1 ? s : src - 1;
}

__global__ void __launch_bounds__(PAN_THREADS) panels_prep_kernel(PanelArgs a) {
  __shared__ float m[2][12];
  const LrfPanelFrame& f = a.f;
  if (a.flow && threadIdx.x < 2) {                  // 0: forward (idx + 1), 1: backward (idx - 1), clamped
    long long k = f.idx + (threadIdx.x == 0 ? 1 : -1);
    k = k < 0 ? 0 : (k > f.n_cams - 1 ? f.n_cams - 1 : k);
    cam2cam(f.cam2world, f.idx, k, m[threadIdx.x]);
  }
  __syncthreads();
  const int W = f.W;
  const long long W2 = 2 * (long long)f.W, n = a.n;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / W), x = (int)(p % W);
    const long long s = (long long)nearest_src(y, a.ify, f.h0) * f.w0 + nearest_src(x, a.ifx, f.w0);
    const float dep = f.depth[p];
    if (a.flow) {
      const float fo = f.intrinsics[0], cx = f.intrinsics[1], cy = f.intrinsics[2];
      const float pt[3] = {f.directions[3 * p] * dep, f.directions[3 * p + 1] * dep, f.directions[3 * p + 2] * dep};
      for (int d = 0; d < 2; ++d) {
        const Proj pr = project(m[d], pt, fo, cx, cy, (float)x, (float)y);
        const float* gf = d ? f.bwd_flow : f.fwd_flow;
        const float mk = (d ? f.bwd_mask : f.fwd_mask)[s];
        const float g0 = gf[2 * s], g1 = gf[2 * s + 1];
        float* c0 = a.cmp + (size_t)(2 * d) * 2 * n;
        float* c1 = c0 + 2 * n;
        c0[p] = pr.u;
        c0[n + p] = g0;
        c1[p] = pr.v;
        c1[n + p] = g1;
        float* panel = d ? f.bwd_panel : f.fwd_panel;            // [3H][2W]; the error rows start at 2H
        panel[(2 * (long long)f.H + y) * W2 + x] = clamp01(fabsf(pr.u - g0) * mk / (float)W);
        panel[(2 * (long long)f.H + y) * W2 + W + x] = clamp01(fabsf(pr.v - g1) * mk / (float)W);
        float* pred = d ? f.bwd_pred : f.fwd_pred;
        if (pred) {
          pred[2 * p] = pr.u;
          pred[2 * p + 1] = pr.v;
        }
      }
    }
    if (a.depth) {
      a.xg[p] = 1.0f / clamp_min(dep, 1e-6f);
      a.xg[n + p] = f.invdepth[s];
    }
  }
}

// torch.median's NaN rule on top of the selection: a NaN anywhere gives NaN
__device__ inline float selected(const SelectState& S) {
  return S.n_nan ? __int_as_float(0x7fffffff) : select_value(S);
}

// blockIdx.y: 0 x, 1 g.  Every block sums a fixed slice of the pixels, so the order depends on n alone.
__global__ void __launch_bounds__(PAN_THREADS) panels_mad_kernel(PanelArgs a) {
  __shared__ double red[PAN_THREADS / 32];
  const int which = blockIdx.y;
  const float t = selected(a.st[a.job_x + which]);
  const float* v = a.xg + (size_t)which * a.n;
  double s = 0.0;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < a.n; p += (long long)gridDim.x * blockDim.x)
    s += (double)fabsf(__fsub_rn(v[p], t));
  s = block_sum_fp64(s, red);
  if (threadIdx.x == 0) a.mad[which * PAN_MAD_BLOCKS + blockIdx.x] = s;
}

// np.quantile(a, 0.9) with numpy's float32 arithmetic: d = b - a; a + d g, or b - d (1 - g) when g >= 0.5
__device__ inline float numpy_lerp(float lo, float hi, float g) {
  const float d = __fsub_rn(hi, lo);
  return g >= 0.5f ? __fsub_rn(hi, __fmul_rn(d, __fsub_rn(1.0f, g))) : __fadd_rn(lo, __fmul_rn(d, g));
}

__global__ void __launch_bounds__(PAN_THREADS) panels_stats_kernel(PanelArgs a) {
  __shared__ double red[PAN_THREADS / 32];
  const float nan = __int_as_float(0x7fffffff);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) {
      const SelectState& lo = a.st[i];
      const float b = a.hi_mode == 0 ? select_value(lo)
                      : a.hi_mode == 1 ? select_next_value(lo) : select_value(a.st[a.job_hi + i]);
      a.stats[i] = !a.flow ? nan : lo.n_nan ? nan : numpy_lerp(select_value(lo), b, a.q.gamma);
    }
  }
  for (int which = 0; which < 2; ++which) {
    double s = 0.0;
    if (a.depth)
      for (int b = threadIdx.x; b < a.mad_blocks; b += blockDim.x) s += a.mad[which * PAN_MAD_BLOCKS + b];
    s = block_sum_fp64(s, red);
    if (threadIdx.x == 0) {
      a.stats[4 + 2 * which] = a.depth ? selected(a.st[a.job_x + which]) : nan;
      a.stats[5 + 2 * which] = a.depth ? (float)(s / (double)a.n) : nan;
    }
  }
}

__global__ void __launch_bounds__(PAN_THREADS) panels_finish_kernel(PanelArgs a) {
  const LrfPanelFrame& f = a.f;
  __shared__ float st[PAN_NSTATS];
  if (threadIdx.x < PAN_NSTATS) st[threadIdx.x] = a.stats[threadIdx.x];
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x < PAN_NSTATS && f.stats) f.stats[threadIdx.x] = st[threadIdx.x];
  const int W = f.W;
  const long long W2 = 2 * (long long)f.W, n = a.n;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / W), x = (int)(p % W);
    if (a.flow) {
      for (int d = 0; d < 2; ++d) {
        float* panel = d ? f.bwd_panel : f.fwd_panel;
        for (int c = 0; c < 2; ++c) {
          const float q = st[2 * d + c];
          const float* cm = a.cmp + (size_t)(2 * d + c) * 2 * n;
          panel[y * W2 + c * W + x] = clamp01(cm[p] / q);
          panel[((long long)f.H + y) * W2 + c * W + x] = clamp01(cm[n + p] / q);
        }
      }
    }
    if (a.depth) {
      const float xn = (a.xg[p] - st[4]) / st[5], gn = (a.xg[n + p] - st[6]) / st[7];
      const float df = __fsub_rn(xn, gn);
      f.depth_panel[p] = clamp01(__fmul_rn(0.5f, xn));
      f.depth_panel[n + p] = clamp01(__fmul_rn(0.5f, gn));
      f.depth_panel[2 * n + p] = clamp01(__fmul_rn(df, df));
    }
  }
}

// ---- host side --------------------------------------------------------------------------------------------
size_t panels_scratch_bytes(long long n_px) {
  PanelArgs a;
  a.n = n_px;
  ScratchCarver c(nullptr);
  carve(c, a);
  return c.size();
}

// numpy 2.x, method="linear", float32 input: q is float32(0.9); the virtual index (n - 1) * q is float32 (the Python
// int n - 1 is cast to float32 first), floor() and + 1 stay float32, and gamma = index - floor(index) is float32.
static QuantRule numpy_quantile_rule(long long n, float q) {
  const volatile float vi = (float)(n - 1) * q;      // volatile: one float32 rounding, as numpy's float32 multiply
  const float prev = floorf(vi);
  const volatile float next = prev + 1.0f;
  QuantRule r;
  r.lo = (unsigned int)prev;
  r.hi = (unsigned int)next;
  if (vi >= (float)(n - 1)) r.lo = r.hi = (unsigned int)(n - 1);   // numpy takes the last value there
  if (r.hi > (unsigned int)(n - 1)) r.hi = (unsigned int)(n - 1);
  r.gamma = vi - prev;
  return r;
}

cudaError_t launch_test_panels(const LrfPanelFrame& f, void* scratch, int n_sms, cudaStream_t stream) {
  PanelArgs a;
  a.f = f;
  a.flow = f.fwd_flow != nullptr;
  a.depth = f.invdepth != nullptr;
  if (!a.flow && !a.depth) return cudaSuccess;
  a.n = (long long)f.W * f.H;
  a.ifx = 1.0 / ((double)f.W / (double)f.w0);
  a.ify = 1.0 / ((double)f.H / (double)f.h0);
  a.q = numpy_quantile_rule(2 * a.n, 0.9f);
  a.job_x = a.flow ? 4 : 0;
  a.hi_mode = a.q.hi == a.q.lo ? 0 : (a.q.hi == a.q.lo + 1 ? 1 : 2);
  a.job_hi = a.job_x + (a.depth ? 2 : 0);
  ScratchCarver c(scratch);
  carve(c, a);
  const long long mb = (a.n + 4095) / 4096;
  a.mad_blocks = (int)(mb < PAN_MAD_BLOCKS ? mb : PAN_MAD_BLOCKS);

  SelectJobs jobs = {};
  int n_jobs = 0;
  if (a.flow)
    for (int i = 0; i < 4; ++i)
      jobs.j[n_jobs++] = {a.cmp + (size_t)i * 2 * a.n, (unsigned int)(2 * a.n), a.q.lo, a.hi_mode == 1};
  if (a.depth)
    for (int i = 0; i < 2; ++i)
      jobs.j[n_jobs++] = {a.xg + (size_t)i * a.n, (unsigned int)a.n, (unsigned int)((a.n - 1) / 2), 0};
  if (a.flow && a.hi_mode == 2)
    for (int i = 0; i < 4; ++i) jobs.j[n_jobs++] = {a.cmp + (size_t)i * 2 * a.n, (unsigned int)(2 * a.n), a.q.hi, 0};

  cudaError_t e = cudaMemsetAsync(a.st, 0, (size_t)n_jobs * sizeof(SelectState), stream);
  if (e != cudaSuccess) return e;
  const unsigned int grid = cta_count(a.n, PAN_THREADS, n_sms, 16);
  panels_prep_kernel<<<grid, PAN_THREADS, 0, stream>>>(a);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  e = launch_select(jobs, a.st, n_jobs, (unsigned int)(a.flow ? 2 * a.n : a.n), n_sms, stream);
  if (e != cudaSuccess) return e;
  if (a.depth) {
    panels_mad_kernel<<<dim3((unsigned)a.mad_blocks, 2), PAN_THREADS, 0, stream>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  panels_stats_kernel<<<1, PAN_THREADS, 0, stream>>>(a);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  panels_finish_kernel<<<grid, PAN_THREADS, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace lrf
