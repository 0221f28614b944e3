// lrf_sched.cu -- the schedule-time operators around the render path, as kernels on the field's
// channel-last tensors (SURVEY.md 8f ranks 2-3 and the AABB sampler north_star names):
//
//   dense alpha + occupancy mask   getDenseAlpha / updateAlphaMask     models/tensorBase.py:501-536
//   grid upsampling                up_sampling_VM                      models/tensoRF.py:198-221
//   density_L1                     (no 8*G^3 intermediate)             models/tensoRF.py:83-92
//   TV loss on planes / lines      TVLoss                              utils/utils.py:293-312
//   sample_ray                     ray-AABB intersection sampler       models/tensorBase.py:396-417
#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

// torch.linspace(0, 1, n)[i] in fp32 (ATen: symmetric evaluation around the midpoint)
__device__ __forceinline__ float linspace01(int i, int n) {
  if (n <= 1) return 0.0f;
  const float step = __fdiv_rn(1.0f, (float)(n - 1));
  return i < n / 2 ? __fmul_rn(step, (float)i) : __fsub_rn(1.0f, __fmul_rn(step, (float)(n - i - 1)));
}

// ---- getDenseAlpha (tensorBase.py:501-515) + compute_alpha (:538-558) ---------------------------------
// alpha[i][j][k] at lattice point aabb0*(1-t) + aabb1*t, t = linspace(0,1,dims) per axis; an existing
// alpha mask culls (sigma = 0) exactly as compute_alpha does.
__global__ void dense_alpha_kernel(const FieldDev F, const float3 amax, int gx, int gy, int gz,
                                   float length, float* __restrict__ alpha) {
  const long long n = (long long)gx * gy * gz;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(e % gz), j = (int)((e / gz) % gy), i = (int)(e / ((long long)gz * gy));
    const float t[3] = {linspace01(i, gx), linspace01(j, gy), linspace01(k, gz)};
    const float hi[3] = {amax.x, amax.y, amax.z};
    float p[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(__fmul_rn(F.amin[a], __fsub_rn(1.0f, t[a])), __fmul_rn(hi[a], t[a]));
    alpha[e] = dense_alpha_at(F, p, length);
  }
}

// updateAlphaMask (tensorBase.py:517-536): clamp(0,1) -> transpose(0,2) -> max_pool3d(k=3, pad=1) ->
// {>= thres: 1, < thres: 0}.  in: alpha [gx][gy][gz]; out: mask [gz][gy][gx]; kept += #ones
__global__ void alpha_pool_kernel(const float* __restrict__ alpha, int gx, int gy, int gz, float thres,
                                  float* __restrict__ mask, unsigned long long* __restrict__ kept) {
  const long long n = (long long)gx * gy * gz;
  unsigned int mine = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(e % gx), y = (int)((e / gx) % gy), z = (int)(e / ((long long)gx * gy));
    float m = -INFINITY;
    for (int dx = -1; dx <= 1; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= gx) continue;
      for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= gy) continue;
#pragma unroll
        for (int dz = -1; dz <= 1; ++dz) {
          const int zz = z + dz;
          if (zz < 0 || zz >= gz) continue;
          const float a = __ldg(alpha + ((long long)xx * gy + yy) * gz + zz);
          m = fmaxf(m, fminf(fmaxf(a, 0.0f), 1.0f));
        }
      }
    }
    const float v = m >= thres ? 1.0f : (m < thres ? 0.0f : m);
    mask[e] = v;
    mine += v == 1.0f;
  }
  mine = __reduce_add_sync(0xffffffffu, mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(kept, (unsigned long long)mine);
}

// ---- up_sampling_VM (tensoRF.py:198-221): F.interpolate(bilinear, align_corners=True) ------------------
// channel-last in and out: src [H][W][C] -> dst [H2][W2][C]; lines are H = L, W = 1.
__global__ void upsample_kernel(const float* __restrict__ src, int H, int W, float* __restrict__ dst,
                                int H2, int W2, int C4 /* C / 4 */) {
  const long long n = (long long)H2 * W2 * C4;
  const float sy = H2 > 1 ? __fdiv_rn((float)(H - 1), (float)(H2 - 1)) : 0.0f;   // area_pixel_compute_scale
  const float sx = W2 > 1 ? __fdiv_rn((float)(W - 1), (float)(W2 - 1)) : 0.0f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(e % C4), x = (int)((e / C4) % W2), y = (int)(e / ((long long)C4 * W2));
    const float fy = __fmul_rn(sy, (float)y), fx = __fmul_rn(sx, (float)x);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float hy = 1.0f - ly, hx = 1.0f - lx;
    const float4 a = ldg4(src + (((long long)y0 * W + x0) * C4 + c4) * 4);
    const float4 b = ldg4(src + (((long long)y0 * W + x1) * C4 + c4) * 4);
    const float4 c = ldg4(src + (((long long)y1 * W + x0) * C4 + c4) * 4);
    const float4 d = ldg4(src + (((long long)y1 * W + x1) * C4 + c4) * 4);
    float4 o;   // ATen: h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d)
    o.x = hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x);
    o.y = hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y);
    o.z = hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z);
    o.w = hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w);
    *reinterpret_cast<float4*>(dst + e * 4) = o;
  }
}

// ---- density_L1 (tensoRF.py:83-92) -------------------------------------------------------------------
// The reference materialises, per plane i, bmm(plane_i [C,P_i,1], line_i [C,1,L_i]) = C*G^3 floats and
// sums them at the same FLAT index n = p*L_i + l for all three i (the flat order is what it is:
// [C, P_i*L_i] views of the three products are added element by element).  Here every n is
// evaluated on the fly: f[n] = sum_i <plane_i[n / L_i], line_i[n % L_i]> (8 channels, one 32-byte
// texel each), loss = mean sqrt(clamp(feature2density(f), 1e-5)); nothing of size G^3 is stored.
__device__ __forceinline__ float dot8(const float* a, const float* b) {
  const float4 a0 = ldg4(a), a1 = ldg4(a + 4), b0 = ldg4(b), b1 = ldg4(b + 4);
  return a0.x * b0.x + a0.y * b0.y + a0.z * b0.z + a0.w * b0.w + a1.x * b1.x + a1.y * b1.y +
         a1.z * b1.z + a1.w * b1.w;
}
__device__ __forceinline__ float l1_feature(const FieldDev& F, long long n) {
  float f = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int L = F.g[vecm(i)];
    const long long p = n / L;
    const int l = (int)(n - p * L);
    f += dot8(F.dplane[i] + p * CD, F.dline[i] + (long long)l * CD);
  }
  return f;
}
__device__ __forceinline__ float block_sum(float v, float* red /*[32]*/) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.0f;
  if (warp == 0) v = warp_sum(v);
  return v;                                   // valid in thread 0
}

__global__ void density_l1_fwd_kernel(const FieldDev F, long long N, double* __restrict__ sum) {
  __shared__ float red[32];
  float acc = 0.0f;
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N;
       n += (long long)gridDim.x * blockDim.x) {
    const float s = feature2density(l1_feature(F, n), F.density_shift, F.act);
    acc += sqrtf(fmaxf(s, 1e-5f));
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) atomicAdd(sum, (double)acc);
}

// d loss / d f[n], times the upstream gradient / N
__device__ __forceinline__ float l1_dfeature(const FieldDev& F, float f, float gscale) {
  float s, ds;
  if (F.act == 0) {
    const float x = f + F.density_shift;
    s = x > 20.0f ? x : log1pf(expf(x));
    ds = x > 20.0f ? 1.0f : __fdiv_rn(1.0f, 1.0f + expf(-x));
  } else {
    s = fmaxf(f, 0.0f);
    ds = f > 0.0f ? 1.0f : 0.0f;
  }
  if (!(s >= 1e-5f)) return 0.0f;                                  // clamp(min) passes no gradient below
  return gscale * __fdiv_rn(0.5f, sqrtf(s)) * ds;
}

// gradients of plane I / line I: one block owns a slice of plane texels p (so d_plane rows are written
// without atomics) and sweeps all L line positions for each; line gradients accumulate in registers
// over the slice and are added atomically once per block.
constexpr int L1_THREADS = 256, L1_SLOTS = 4, L1_PSLICE = 64;
template <int I>
__global__ void __launch_bounds__(L1_THREADS)
density_l1_bwd_kernel(const FieldDev F, long long P, const float* __restrict__ gout, float inv_n,
                      float* __restrict__ d_plane, float* __restrict__ d_line) {
  __shared__ float red[8][L1_THREADS / 32];
  const int L = F.g[vecm(I)];
  const float gscale = __ldg(gout) * inv_n;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float ul[L1_SLOTS][CD];
#pragma unroll
  for (int k = 0; k < L1_SLOTS; ++k)
#pragma unroll
    for (int c = 0; c < CD; ++c) ul[k][c] = 0.0f;
  const long long p_lo = (long long)blockIdx.x * L1_PSLICE;
  const long long p_hi = p_lo + L1_PSLICE < P ? p_lo + L1_PSLICE : P;
  for (long long p = p_lo; p < p_hi; ++p) {
    float pl[CD];
    {
      const float4 a = ldg4(F.dplane[I] + p * CD), b = ldg4(F.dplane[I] + p * CD + 4);
      pl[0] = a.x; pl[1] = a.y; pl[2] = a.z; pl[3] = a.w; pl[4] = b.x; pl[5] = b.y; pl[6] = b.z; pl[7] = b.w;
    }
    float v[CD];
#pragma unroll
    for (int c = 0; c < CD; ++c) v[c] = 0.0f;
#pragma unroll
    for (int k = 0; k < L1_SLOTS; ++k) {
      const int l = tid + k * L1_THREADS;
      if (l < L) {
        const long long n = p * L + l;
        const float df = l1_dfeature(F, l1_feature(F, n), gscale);
        const float4 a = ldg4(F.dline[I] + (long long)l * CD), b = ldg4(F.dline[I] + (long long)l * CD + 4);
        const float ln[CD] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int c = 0; c < CD; ++c) { v[c] = fmaf(df, ln[c], v[c]); ul[k][c] = fmaf(df, pl[c], ul[k][c]); }
      }
    }
    // tail of very long lines (L > SLOTS * THREADS): per-element atomics
    for (int l = tid + L1_SLOTS * L1_THREADS; l < L; l += L1_THREADS) {
      const long long n = p * L + l;
      const float df = l1_dfeature(F, l1_feature(F, n), gscale);
#pragma unroll
      for (int c = 0; c < CD; ++c) {
        v[c] = fmaf(df, __ldg(F.dline[I] + (long long)l * CD + c), v[c]);
        atomicAdd(d_line + (long long)l * CD + c, df * pl[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < CD; ++c) v[c] = warp_sum(v[c]);
    __syncthreads();
    if (lane == 0)
#pragma unroll
      for (int c = 0; c < CD; ++c) red[c][warp] = v[c];
    __syncthreads();
    if (tid < CD) {
      float s = 0.0f;
#pragma unroll
      for (int w = 0; w < L1_THREADS / 32; ++w) s += red[tid][w];
      d_plane[p * CD + tid] += s;                                   // this block owns texel p
    }
  }
#pragma unroll
  for (int k = 0; k < L1_SLOTS; ++k) {
    const int l = tid + k * L1_THREADS;
    if (l < L)
#pragma unroll
      for (int c = 0; c < CD; ++c) atomicAdd(d_line + (long long)l * CD + c, ul[k][c]);
  }
}

// ---- TVLoss (utils/utils.py:293-312) on a channel-last [H][W][C] tensor ---------------------------------
// sums[0] += sum (x[y+1]-x[y])^2, sums[1] += sum (x[.,x+1]-x[.,x])^2
__global__ void tv_fwd_kernel(const float* __restrict__ x, int H, int W, int C, double* __restrict__ sums) {
  __shared__ float red[32];
  const long long n = (long long)H * W * C, row = (long long)W * C;
  float sh = 0.0f, sw = 0.0f;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)((e / C) % W), yy = (int)(e / row);
    const float v = __ldg(x + e);
    if (yy + 1 < H) { const float d = __ldg(x + e + row) - v; sh = fmaf(d, d, sh); }
    if (xx + 1 < W) { const float d = __ldg(x + e + C) - v; sw = fmaf(d, d, sw); }
  }
  sh = block_sum(sh, red);
  sw = block_sum(sw, red);
  if (threadIdx.x == 0) { atomicAdd(sums, (double)sh); atomicAdd(sums + 1, (double)sw); }
}
// dx += gh * d(sum_h)/dx + gw * d(sum_w)/dx   (gh, gw already hold upstream * weight * 2 / count)
__global__ void tv_bwd_kernel(const float* __restrict__ x, int H, int W, int C, const float* __restrict__ gout,
                              float kh, float kw, float* __restrict__ dx) {
  const long long n = (long long)H * W * C, row = (long long)W * C;
  const float g = __ldg(gout), gh = g * kh, gw = g * kw;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)((e / C) % W), yy = (int)(e / row);
    const float v = __ldg(x + e);
    float dh = 0.0f, dw = 0.0f;
    if (yy > 0) dh += v - __ldg(x + e - row);
    if (yy + 1 < H) dh -= __ldg(x + e + row) - v;
    if (xx > 0) dw += v - __ldg(x + e - C);
    if (xx + 1 < W) dw -= __ldg(x + e + C) - v;
    dx[e] += 2.0f * (gh * dh + gw * dw);
  }
}

// ---- sample_ray (tensorBase.py:396-417): ray-AABB entry distance + uniform steps --------------------------
// rays [N][6] (o, d as given: the reference does not normalise here); jitter [N] or NULL (train: one
// uniform draw per ray, tensorBase.py:404-406).  out: pts [N][S][3], z [N][S], inside [N][S] (uint8)
__global__ void sample_ray_kernel(const float* __restrict__ rays, const float* __restrict__ jitter,
                                  long long N, int S, float3 amin, float3 amax, float near, float far,
                                  float step, float* __restrict__ pts, float* __restrict__ z,
                                  unsigned char* __restrict__ inside) {
  const long long total = N * S;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / S;
    const int k = (int)(e - r * S);
    const float* ray = rays + 6 * r;
    const float lo[3] = {amin.x, amin.y, amin.z}, hi[3] = {amax.x, amax.y, amax.z};
    float tmin = -INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float d = ray[3 + a];
      const float vec = d == 0.0f ? 1e-6f : d;
      const float ra = __fdiv_rn(hi[a] - ray[a], vec), rb = __fdiv_rn(lo[a] - ray[a], vec);
      tmin = fmaxf(tmin, fminf(ra, rb));
    }
    tmin = fminf(fmaxf(tmin, near), far);
    float rng = (float)k;
    if (jitter) rng = __fadd_rn(rng, jitter[r]);
    const float t = __fadd_rn(tmin, __fmul_rn(step, rng));
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float p = __fadd_rn(ray[a], __fmul_rn(ray[3 + a], t));
      pts[e * 3 + a] = p;
      in = in && !(lo[a] > p) && !(p > hi[a]);
    }
    z[e] = t;
    inside[e] = in ? 1 : 0;
  }
}

// ---- frame post-processing (renderer.py:126-131,173-176; utils/utils.py:179-197) -------------------------
// rgb -> 8-bit BGR (what cv2.imwrite receives: 255 * rgb[..., ::-1], saturating round-to-nearest-even) and
// depth -> colour-mapped 8-bit BGR through a 256-entry lookup table (cv2.applyColorMap of
// (255 * clip((d - lo) / (hi - lo + 1e-8), 0, 1)).astype(uint8)); both are written where the caller points --
// pinned host memory included, so a finished frame leaves the GPU as 6 bytes per pixel.
// The depth bounds arrive as lo = (float)d_lo and den = (float)(d_hi - d_lo + 1e-8), the denominator formed in
// double on the host: numpy does exactly this with a float32 frame and Python-number bounds.
// rgb equals OpenCV's x86-64 float -> 8U conversion for |255 v| < 2^31, NaN and -inf (both 0).  At or above 2^31
// and at +inf this writes 255 where OpenCV's cvRound overflows to INT_MIN and writes 0; the renderer clamps rgb
// to [0, 1] first, so a rendered frame never reaches that range.
__global__ void frame_u8_kernel(const float* __restrict__ rgb, int rgb_stride, const float* __restrict__ depth,
                                int depth_stride, long long N, float d_lo, float d_den,
                                const unsigned char* __restrict__ lut, unsigned char* __restrict__ rgb8,
                                unsigned char* __restrict__ depth8) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < N;
       r += (long long)gridDim.x * blockDim.x) {
    if (rgb8) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __fmul_rn(255.0f, rgb[(long long)rgb_stride * r + c]);
        rgb8[3 * r + (2 - c)] = (unsigned char)min(max(__float2int_rn(v), 0), 255);   // cv::saturate_cast<uchar>
      }
    }
    if (depth8) {
      float d = depth[(long long)depth_stride * r];
      if (d != d) d = 0.0f;                                                     // np.nan_to_num
      float x = __fdiv_rn(__fsub_rn(d, d_lo), d_den);
      x = fminf(fmaxf(x, 0.0f), 1.0f);
      const int idx = (int)__fmul_rn(255.0f, x);                                // astype(uint8) truncates
      depth8[3 * r] = lut[3 * idx]; depth8[3 * r + 1] = lut[3 * idx + 1]; depth8[3 * r + 2] = lut[3 * idx + 2];
    }
  }
}

cudaError_t launch_frame_u8(const float* rgb, int rgb_stride, const float* depth, int depth_stride, long long N,
                            double d_lo, double d_hi, const unsigned char* lut, unsigned char* rgb8,
                            unsigned char* depth8, int n_sms, cudaStream_t stream) {
  if (N == 0) return cudaSuccess;
  frame_u8_kernel<<<cta_count(N, 256, n_sms, 16), 256, 0, stream>>>(rgb, rgb_stride, depth, depth_stride, N,
                                                                    (float)d_lo, (float)(d_hi - d_lo + 1e-8), lut,
                                                                    rgb8, depth8);
  return cudaGetLastError();
}

// ---- launchers -------------------------------------------------------------------------------------------
cudaError_t launch_alpha_mask_build(const FieldDev& F, const float* aabb_max, const int* dims, float length,
                                    float thres, float* alpha_scratch, float* mask,
                                    unsigned long long* kept, int n_sms, cudaStream_t stream) {
  const long long n = (long long)dims[0] * dims[1] * dims[2];
  if (n == 0) return cudaSuccess;
  dense_alpha_kernel<<<cta_count(n, 256, n_sms, 16), 256, 0, stream>>>(
      F, make_float3(aabb_max[0], aabb_max[1], aabb_max[2]), dims[0], dims[1], dims[2], length, alpha_scratch);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || !mask) return e;
  alpha_pool_kernel<<<cta_count(n, 256, n_sms, 16), 256, 0, stream>>>(alpha_scratch, dims[0], dims[1], dims[2],
                                                                   thres, mask, kept);
  return cudaGetLastError();
}

cudaError_t launch_upsample(const float* src, int H, int W, float* dst, int H2, int W2, int C, int n_sms,
                            cudaStream_t stream) {
  const long long n = (long long)H2 * W2 * (C / 4);
  if (n == 0) return cudaSuccess;
  upsample_kernel<<<cta_count(n, 256, n_sms, 16), 256, 0, stream>>>(src, H, W, dst, H2, W2, C / 4);
  return cudaGetLastError();
}

cudaError_t launch_density_l1(const FieldDev& F, double* sum, int n_sms, cudaStream_t stream) {
  const long long N = (long long)F.g[0] * F.g[1] * F.g[2];
  density_l1_fwd_kernel<<<cta_count(N, 256, n_sms, 16), 256, 0, stream>>>(F, N, sum);
  return cudaGetLastError();
}

cudaError_t launch_density_l1_backward(const FieldDev& F, const float* gout, float* const* d_plane,
                                       float* const* d_line, cudaStream_t stream) {
  const long long N = (long long)F.g[0] * F.g[1] * F.g[2];
  const float inv_n = (float)(1.0 / (double)N);
  const long long P0 = N / F.g[vecm(0)], P1 = N / F.g[vecm(1)], P2 = N / F.g[vecm(2)];
  density_l1_bwd_kernel<0><<<(unsigned)((P0 + L1_PSLICE - 1) / L1_PSLICE), L1_THREADS, 0, stream>>>(
      F, P0, gout, inv_n, d_plane[0], d_line[0]);
  density_l1_bwd_kernel<1><<<(unsigned)((P1 + L1_PSLICE - 1) / L1_PSLICE), L1_THREADS, 0, stream>>>(
      F, P1, gout, inv_n, d_plane[1], d_line[1]);
  density_l1_bwd_kernel<2><<<(unsigned)((P2 + L1_PSLICE - 1) / L1_PSLICE), L1_THREADS, 0, stream>>>(
      F, P2, gout, inv_n, d_plane[2], d_line[2]);
  return cudaGetLastError();
}

cudaError_t launch_tv(const float* x, int H, int W, int C, double* sums, int n_sms, cudaStream_t stream) {
  const long long n = (long long)H * W * C;
  if (n == 0) return cudaSuccess;
  tv_fwd_kernel<<<cta_count(n, 256, n_sms, 16), 256, 0, stream>>>(x, H, W, C, sums);
  return cudaGetLastError();
}

cudaError_t launch_tv_backward(const float* x, int H, int W, int C, const float* gout, float kh, float kw,
                               float* dx, int n_sms, cudaStream_t stream) {
  const long long n = (long long)H * W * C;
  if (n == 0) return cudaSuccess;
  tv_bwd_kernel<<<cta_count(n, 256, n_sms, 16), 256, 0, stream>>>(x, H, W, C, gout, kh, kw, dx);
  return cudaGetLastError();
}

cudaError_t launch_sample_ray(const float* rays, const float* jitter, long long N, int S, const float* aabb,
                              float near, float far, float step, float* pts, float* z,
                              unsigned char* inside, int n_sms, cudaStream_t stream) {
  if (N * S == 0) return cudaSuccess;
  sample_ray_kernel<<<cta_count(N * S, 256, n_sms, 16), 256, 0, stream>>>(
      rays, jitter, N, S, make_float3(aabb[0], aabb[1], aabb[2]), make_float3(aabb[3], aabb[4], aabb[5]),
      near, far, step, pts, z, inside);
  return cudaGetLastError();
}

}  // namespace lrf
