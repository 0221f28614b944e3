// lrf_metrics.cu -- test-frame MSE and SSIM of one H x W x 3 fp32 frame against its ground truth
// (renderer.py:162-163; rgb_ssim, utils/utils.py:232-287).
//
// The reference's inputs are float32 and its filter is float64, so the squares and the cross product are fp32
// products (rounded before they are filtered) while every filter, moment and map operation is fp64.  The filter
// sums each window from its last pixel to its first, as scipy.signal.convolve2d does, and all fp64 arithmetic
// uses the _rn intrinsics so that nvcc cannot contract it into FMAs.  Identical images then give a map of exactly
// 1, and the moments differ from the reference's by about one rounding.
//
// One CTA owns a 16 x 32 tile of input pixels.  It sums the MSE terms of that tile and computes the SSIM
// outputs whose window starts in the tile, so the grid covers every input pixel once and every output once.
// The tile plus its (fs - 1) halo is staged in shared memory as fp32; the vertical pass of the separable filter
// writes five fp64 moments per channel to shared memory and the horizontal pass runs in registers.  Per-CTA
// fp64 partial sums go to scratch, and one more CTA sums them in a fixed order: results are bitwise
// deterministic, with no atomics.
#include <cuda_runtime.h>

#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

constexpr int MET_TH = 16, MET_TW = 32, MET_THREADS = 256, MET_MAX_FS = 16;

struct MetricTaps {
  double f[MET_MAX_FS];
};

__host__ __device__ inline size_t metrics_smem_bytes(int fs) {
  const int rows = MET_TH + fs - 1, cols = MET_TW + fs - 1;
  return (size_t)5 * MET_TH * cols * sizeof(double) + (size_t)2 * 3 * rows * cols * sizeof(float);
}

__global__ void __launch_bounds__(MET_THREADS) metrics_tile_kernel(
    const float* __restrict__ img, int img_stride, const float* __restrict__ gt, int gt_stride, int H, int W,
    int fs, MetricTaps taps, double c1, double c2, double* __restrict__ ssim_map, double* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int rows = MET_TH + fs - 1, cols = MET_TW + fs - 1;
  const int Ho = H - fs + 1, Wo = W - fs + 1;
  double* V = reinterpret_cast<double*>(smem);                     // [5][MET_TH][cols]
  float* A = reinterpret_cast<float*>(V + 5 * MET_TH * cols);      // [3][rows][cols]  img
  float* B = A + 3 * rows * cols;                                  // [3][rows][cols]  gt
  __shared__ double red[MET_THREADS / 32];
  __shared__ double f[MET_MAX_FS];                                 // indexed taps: shared, not a local copy
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < MET_MAX_FS; ++k) f[k] = taps.f[k];
  }

  const int r0 = blockIdx.y * MET_TH, c0 = blockIdx.x * MET_TW;
  double mse = 0.0, ssim = 0.0;

  // stage the tile + halo (channel fastest, so a warp reads consecutive floats); MSE of the owned pixels
  for (int i = threadIdx.x; i < rows * cols * 3; i += MET_THREADS) {
    const int c = i % 3, p = i / 3, x = p % cols, r = p / cols;
    const int gr = r0 + r, gc = c0 + x;
    float a = 0.f, b = 0.f;
    if (gr < H && gc < W) {
      const long long pix = (long long)gr * W + gc;
      a = img[pix * img_stride + c];
      b = gt[pix * gt_stride + c];
      if (r < MET_TH && x < MET_TW) {
        const float d = __fsub_rn(b, a);
        mse += (double)__fmul_rn(d, d);
      }
    }
    A[(c * rows + r) * cols + x] = a;
    B[(c * rows + r) * cols + x] = b;
  }
  __syncthreads();

  const int out_rows = min(MET_TH, Ho - r0), out_cols = min(MET_TW, Wo - c0);   // may be <= 0 at the edges
  for (int ch = 0; ch < 3; ++ch) {
    // vertical pass: moments of rows r .. r+fs-1 for every staged column
    if (out_rows > 0 && out_cols > 0) {
      const int need = out_cols + fs - 1;
      for (int i = threadIdx.x; i < out_rows * need; i += MET_THREADS) {
        const int r = i / need, x = i % need;
        const float* a = A + (ch * rows + r) * cols + x;
        const float* b = B + (ch * rows + r) * cols + x;
        double m0 = 0.0, m1 = 0.0, m00 = 0.0, m11 = 0.0, m01 = 0.0;
        for (int k = fs - 1; k >= 0; --k) {
          const float av = a[k * cols], bv = b[k * cols];
          const double fk = f[k];
          m0 = __dadd_rn(m0, __dmul_rn(fk, (double)av));
          m1 = __dadd_rn(m1, __dmul_rn(fk, (double)bv));
          m00 = __dadd_rn(m00, __dmul_rn(fk, (double)__fmul_rn(av, av)));
          m11 = __dadd_rn(m11, __dmul_rn(fk, (double)__fmul_rn(bv, bv)));
          m01 = __dadd_rn(m01, __dmul_rn(fk, (double)__fmul_rn(av, bv)));
        }
        const int o = r * cols + x;
        V[0 * MET_TH * cols + o] = m0;
        V[1 * MET_TH * cols + o] = m1;
        V[2 * MET_TH * cols + o] = m00;
        V[3 * MET_TH * cols + o] = m11;
        V[4 * MET_TH * cols + o] = m01;
      }
    }
    __syncthreads();
    // horizontal pass + the SSIM map
    for (int i = threadIdx.x; i < MET_TH * MET_TW; i += MET_THREADS) {
      const int r = i / MET_TW, x = i % MET_TW;
      if (r >= out_rows || x >= out_cols) continue;
      double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
      for (int k = fs - 1; k >= 0; --k) {
        const double fk = f[k];
#pragma unroll
        for (int j = 0; j < 5; ++j) m[j] = __dadd_rn(m[j], __dmul_rn(fk, V[j * MET_TH * cols + r * cols + x + k]));
      }
      const double mu00 = __dmul_rn(m[0], m[0]), mu11 = __dmul_rn(m[1], m[1]), mu01 = __dmul_rn(m[0], m[1]);
      const double s00 = fmax(0.0, __dsub_rn(m[2], mu00));
      const double s11 = fmax(0.0, __dsub_rn(m[3], mu11));
      double s01 = __dsub_rn(m[4], mu01);
      const double sgn = s01 > 0.0 ? 1.0 : (s01 < 0.0 ? -1.0 : 0.0);
      s01 = __dmul_rn(sgn, fmin(sqrt(__dmul_rn(s00, s11)), fabs(s01)));
      const double numer = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu01), c1), __dadd_rn(__dmul_rn(2.0, s01), c2));
      const double denom = __dmul_rn(__dadd_rn(__dadd_rn(mu00, mu11), c1), __dadd_rn(__dadd_rn(s00, s11), c2));
      const double v = numer / denom;
      ssim += v;
      if (ssim_map) ssim_map[((long long)(r0 + r) * Wo + (c0 + x)) * 3 + ch] = v;
    }
    __syncthreads();                                 // V is rewritten by the next channel
  }

  const double mse_cta = block_sum_fp64(mse, red);
  const double ssim_cta = block_sum_fp64(ssim, red);
  if (threadIdx.x == 0) {
    const int cta = blockIdx.y * gridDim.x + blockIdx.x;
    partial[2 * cta] = mse_cta;
    partial[2 * cta + 1] = ssim_cta;
  }
}

__global__ void __launch_bounds__(1024) metrics_final_kernel(const double* __restrict__ partial, int n,
                                                             double n_pix, double n_map, double* __restrict__ out) {
  __shared__ double red[32];
  double mse = 0.0, ssim = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    mse += partial[2 * i];
    ssim += partial[2 * i + 1];
  }
  mse = block_sum_fp64(mse, red);
  ssim = block_sum_fp64(ssim, red);
  if (threadIdx.x == 0) {
    out[0] = mse / n_pix;
    out[1] = ssim / n_map;
  }
}

size_t metrics_scratch_bytes(int H, int W) {
  const size_t ctas = (size_t)((H + MET_TH - 1) / MET_TH) * ((W + MET_TW - 1) / MET_TW);
  return 2 * ctas * sizeof(double);
}

// The reference's normalised Gaussian: hw = fs // 2, shift = (2 hw - fs + 1) / 2, f = exp(-0.5 ((k - hw + shift) /
// sigma)^2) / sum.  numpy's vectorised exp and summation order may differ from these in the last bit of a tap;
// that moves the results by about 1e-16.
static MetricTaps gaussian_taps(int fs, double sigma) {
  MetricTaps t = {};
  const int hw = fs / 2;
  const double shift = (2 * hw - fs + 1) / 2.0;
  double sum = 0.0;
  for (int k = 0; k < fs; ++k) {
    const double x = ((double)(k - hw) + shift) / sigma;
    t.f[k] = exp(-0.5 * (x * x));
    sum += t.f[k];
  }
  for (int k = 0; k < fs; ++k) t.f[k] /= sum;
  return t;
}

cudaError_t launch_image_metrics(const float* img, int img_stride, const float* gt, int gt_stride, int H, int W,
                                 int fs, double sigma, double c1, double c2, double* out, double* ssim_map,
                                 void* scratch, cudaStream_t stream) {
  cudaError_t e = set_max_dynamic_smem((const void*)metrics_tile_kernel, (int)metrics_smem_bytes(MET_MAX_FS));
  if (e != cudaSuccess) return e;
  const MetricTaps t = gaussian_taps(fs, sigma);
  const dim3 grid((W + MET_TW - 1) / MET_TW, (H + MET_TH - 1) / MET_TH);
  double* partial = static_cast<double*>(scratch);
  metrics_tile_kernel<<<grid, MET_THREADS, metrics_smem_bytes(fs), stream>>>(
      img, img_stride, gt, gt_stride, H, W, fs, t, c1, c2, ssim_map, partial);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const double n_map = 3.0 * (double)(H - fs + 1) * (double)(W - fs + 1);
  metrics_final_kernel<<<1, 1024, 0, stream>>>(partial, (int)(grid.x * grid.y), 3.0 * (double)H * (double)W, n_map,
                                               out);
  return cudaGetLastError();
}

}  // namespace lrf
