// lrf_backward.cu -- backward of the per-ray-batch render (TensorBase.forward with
// floater_thresh = 0; tensorBase.py:567-636): dL/d(rgb_map), dL/d(depth_map) -> dL/d(rays) and
// dL/d(every parameter of the field), in three launches that share a scratch block in HBM:
//
//   bwd_march_kernel    warp = ray, lane = sample.  Marches the ray again (feature, alpha,
//                       transmittance by a warp-shuffle scan, weight), stores the per-sample tables,
//                       seeds dL/dw with the depth / background terms and appends the shaded samples
//                       (weight > rayMarch_weight_thres) to one global list.
//   bwd_shade_kernel    persistent CTAs over 64-sample tiles of that list.  Recomputes the 72 plane x
//                       line products and the MLP (folded layer 1, layer 2, layer 3 + sigmoid) and runs
//                       its backward as register-tiled fp32 GEMMs out of shared memory; every thread
//                       owns a fixed block of dW2 / d(W1 @ basis) in registers for the whole launch
//                       (flushed once), product gradients scatter to the appearance planes / lines,
//                       the position gradient goes through the contraction Jacobian to the ray, and
//                       g . rgb is added to the sample's dL/dw.
//   bwd_density_kernel  warp = ray, lane = sample.  dL/dw -> dL/dalpha by a reverse (suffix) scan,
//                       through alpha = 1 - exp(-sigma dist scale) and softplus / relu to the density
//                       feature, whose lookup backward scatters to the density planes / lines (16-byte
//                       vector reductions); finishes d(rays) (vd = d/|d|, depth = sum(w z)/|d|).
//
// The math is the one pinned by oracle/lrf_oracle.c::orc_field_backward against the reference's
// autograd.  The shade step has two instantiations: bwd_shade_kernel<true> (default) runs its four
// per-sample matrix products on wgmma with bf16 hi/lo operands (the forward's arithmetic), the weight
// gradients on the CUDA cores; bwd_shade_kernel<false> (LRF_BWD_TC=0) is all fp32 on the CUDA cores.
#include "../../include/localrf_b200.h"
#include <cstdlib>

#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

// prepared block of the backward (floats): the forward's prepared block (lrf_common.cuh), whose bf16 images the
// tensor-core shade step reads and whose fp32 tail (b1, b2, W3, b3) both shade steps read, then folded layer 1
// and W2, both transposed (k-major), for the CUDA-core shade step
constexpr int BP_W1BT = PREP_BYTES / 4;         // [NF][FC]   (W1 @ basis)^T
constexpr int BP_W2T = BP_W1BT + NF * FC;       // [FC(k)][FC(n)]
constexpr int BP_FLOATS = BP_W2T + FC * FC;

struct BwdScratch {           // views into the caller's scratch block
  unsigned long long* count;  // number of shaded samples (zeroed per call)
  float* d_ovd;               // [n][6] position-gradient accumulators (zeroed per call)
  float* dpos;                // NULL, or [n][S][3] zeroed by the caller: each shaded sample's colour-branch position
                              // gradient in its own slot instead of d_ovd's atomics (a fixed summation order)
  float *alpha, *T, *w, *fe, *gw;   // [n][S]
  unsigned char* valid;       // [n][S]
  int *app_ray, *app_k;       // [n*S]
};

struct BwdArgs {
  long long n_rays;
  const float* rays;          // [n][6]
  const float* g_rgb;         // [n][3]
  const float* g_depth;       // [n]
  const float* bp;            // prepared block above
  int white_bg;
  float* d_rays;              // [n][6]
  float* d_dplane[3]; float* d_dline[3]; float* d_aplane[3]; float* d_aline[3];
  float* d_w1b; float* d_b1; float* d_w2; float* d_b2; float* d_w3; float* d_b3;
  BwdScratch s;
};

// each array 16-byte aligned; *zero_bytes: the leading bytes that hold count and d_ovd
inline BwdScratch carve(ScratchCarver& c, long long n, int S, size_t* zero_bytes = nullptr) {
  const size_t ns = (size_t)n * (size_t)S;
  BwdScratch s;
  s.count = c.take<unsigned long long>(16, 16);
  s.d_ovd = c.take<float>((size_t)n * 6 * sizeof(float), 16);
  if (zero_bytes) *zero_bytes = c.size(16);
  s.alpha = c.take<float>(ns * 4, 16);
  s.T = c.take<float>(ns * 4, 16);
  s.w = c.take<float>(ns * 4, 16);
  s.fe = c.take<float>(ns * 4, 16);
  s.gw = c.take<float>(ns * 4, 16);
  s.app_ray = c.take<int>(ns * 4, 16);
  s.app_k = c.take<int>(ns * 4, 16);
  s.valid = c.take(ns, 16);
  return s;
}

// ====================================================================================================
// 1. march
// ====================================================================================================
constexpr int MARCH_THREADS = 256;

__global__ void __launch_bounds__(MARCH_THREADS)
bwd_march_kernel(const FieldDev F, const BwdArgs A) {
  const int S = F.S;
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * MARCH_THREADS + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * MARCH_THREADS) >> 5;
  for (long long ray = warp0; ray < A.n_rays; ray += n_warps) {
    RaySm R;
    normalize_ray(A.rays + 6 * ray, A.rays + 6 * ray + 3, R);
    const float gsum = A.white_bg ? -(A.g_rgb[3 * ray] + A.g_rgb[3 * ray + 1] + A.g_rgb[3 * ray + 2]) : 0.0f;
    const float gd = A.g_depth[ray];
    const size_t base = (size_t)ray * S;
    float carry = 1.0f;
    for (int k0 = 0; k0 < S; k0 += 32) {
      const int k = k0 + lane;
      float alpha = 0.0f, fe, Tk, wk;
      bool valid;
      if (k < S) alpha = sample_alpha<false>(F, R, k, S, fe, valid);
      transmittance_step(alpha, k < S, lane, carry, Tk, wk);
      const bool on = (k < S) && (wk > F.weight_thres);                // tensorBase.py:622
      if (k < S) {
        A.s.alpha[base + k] = alpha; A.s.T[base + k] = Tk; A.s.w[base + k] = wk;
        A.s.fe[base + k] = fe; A.s.valid[base + k] = valid ? 1 : 0;
        A.s.gw[base + k] = gsum + gd * __fdiv_rn(__ldg(F.z + k), R.nrm);   // d rgb_map(white bg) + d depth
      }
      const unsigned m = __ballot_sync(0xffffffffu, on);
      if (m) {
        unsigned long long slot = 0;
        if (lane == 0) slot = atomicAdd(A.s.count, (unsigned long long)__popc(m));
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (on) {
          const unsigned long long e = slot + __popc(m & ((1u << lane) - 1u));
          A.s.app_ray[e] = (int)ray;
          A.s.app_k[e] = k;
        }
      }
    }
  }
}

// ====================================================================================================
// 2. shade: MLP forward + backward over tiles of 64 shaded samples
// ====================================================================================================
constexpr int SH_THREADS = 256;
constexpr int TS = 64;                 // samples per tile
constexpr int LDW = FC + 1;            // padded row of the transposed weights / activations
constexpr int LDX = NF + 1;            // padded row of the product tile

// TC = the four per-sample products (layer 1, layer 2, dh1 = dh2 W2, dprod = dh1 W1B) on wgmma: bf16 hi/lo
// images of W1B and W2 (the forward's operand block) replace the fp32 transposed weights, and one 32 KB
// scratch image holds the A operand of the product being run (x, h1, dh2, dh1 in turn).
constexpr int TC_IMG_BYTES = 2 * OPER1_BYTES + 2 * OPER2_BYTES;   // W1B hi | lo | W2 hi | lo
constexpr int TC_SCR_BYTES = 2 * TS * FC * 2;                     // one [64][128] hi | lo A image
template <bool TC>
struct ShadeSmemT {                    // float offsets
  static constexpr int w1bt = 0;                        // [NF][LDW] (TC: the weight images)
  static constexpr int w2t = w1bt + NF * LDW;           // [FC][LDW] (TC: unused)
  static constexpr int scr = TC_IMG_BYTES / 4;          // (TC) the A image
  static constexpr int x = TC ? scr + TC_SCR_BYTES / 4 : w2t + FC * LDW;   // [TS][LDX]  products, then their gradients
  static constexpr int h1 = x + TS * LDX;               // [TS][LDW]  h1, then dL/d(pre-activation 1)
  static constexpr int h2 = h1 + TS * LDW;              // [TS][LDW]  h2, then dL/d(pre-activation 2)
  static constexpr int w3 = h2 + TS * LDW;              // [3][W3_LD]
  static constexpr int b1 = w3 + 3 * W3_LD;
  static constexpr int b2 = b1 + FC;
  static constexpr int q = b2 + FC;                     // [TS][3] normalised grid coordinates
  static constexpr int praw = q + TS * 3;               // [TS][3] un-contracted sample position
  static constexpr int vd = praw + TS * 3;              // [TS][3]
  static constexpr int g = vd + TS * 3;                 // [TS][3] dL/d rgb_map of the sample's ray
  static constexpr int dpre = g + TS * 3;               // [TS][3] dL/d(layer-3 pre-sigmoid)
  static constexpr int wk = dpre + TS * 3;              // [TS]
  static constexpr int zk = wk + TS;                    // [TS]
  static constexpr int ray = zk + TS;                   // [TS] int
  static constexpr int kk = ray + TS;                   // [TS] int
  static constexpr int total = kk + TS;
};
using ShadeSmem = ShadeSmemT<false>;
static_assert(ShadeSmemT<true>::total * 4 <= 232448, "shared-memory budget of the tensor-core shade step");

// fp32 rows [TS][ld] (K columns used, zero beyond) -> the K-major hi / lo image pair at img (chunks K-chunks)
__device__ __forceinline__ void build_image(const float* src, int ld, int K, int chunks, unsigned char* img) {
  const int img_bytes = 16 * chunks * TS;
  for (int e = threadIdx.x; e < TS * chunks; e += SH_THREADS) {
    const int r = e / chunks, kc = e - r * chunks;
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = (kc * 8 + u < K) ? src[r * ld + kc * 8 + u] : 0.0f;
    store_chunk(img, img + img_bytes, r, kc, chunks, v);
  }
  fence_async_smem();      // generic-proxy writes -> visible to the tensor core
  __syncthreads();
}

// One warpgroup: D[64 x N] = A[64 x K] B^T with A the hi / lo image at a (a_chunks K-chunks), three products
// per K-step.  B: K-major image rows (TB = 0; lbo = 128, sbo = rows' chunks * 128) or read MN-major (TB = 1).
template <int N, int TB>
__device__ __forceinline__ void shade_gemm(float (&d)[N / 2], uint32_t a, int a_chunks, int ksteps, uint32_t b_hi,
                                           uint32_t b_lo, uint32_t b_kstep, uint32_t b_lbo, uint32_t b_sbo) {
  const uint32_t a_sbo = (uint32_t)a_chunks * 128u, a_lo = a + 16u * a_chunks * TS;
  wgmma_fence();
  for (int ks = 0; ks < ksteps; ++ks) {
    const uint64_t ah = gmma_desc(a + ks * 256u, 128u, a_sbo), al = gmma_desc(a_lo + ks * 256u, 128u, a_sbo);
    const uint64_t bh = gmma_desc(b_hi + ks * b_kstep, b_lbo, b_sbo), bl = gmma_desc(b_lo + ks * b_kstep, b_lbo, b_sbo);
    const uint32_t acc = ks > 0 ? 1u : 0u;
    if constexpr (N == 64) {
      wgmma_n64_ss_t<TB>(d, ah, bh, acc); wgmma_n64_ss_t<TB>(d, ah, bl, 1u); wgmma_n64_ss_t<TB>(d, al, bh, 1u);
    } else {
      wgmma_n40_ss_t<TB>(d, ah, bh, acc); wgmma_n40_ss_t<TB>(d, ah, bl, 1u); wgmma_n40_ss_t<TB>(d, al, bh, 1u);
    }
  }
  wgmma_commit();
  wgmma_wait_all();
  fence_regs(d);
}

template <bool TC>
__global__ void __launch_bounds__(SH_THREADS, 1)
bwd_shade_kernel(const FieldDev F, const BwdArgs A) {
  extern __shared__ __align__(1024) float sm[];
  using L = ShadeSmemT<TC>;
  float* W1BT_s = sm + L::w1bt;
  float* W2T_s = sm + L::w2t;
  float* X_s = sm + L::x;
  float* H1_s = sm + L::h1;
  float* H2_s = sm + L::h2;
  float* W3_s = sm + L::w3;
  float* b1_s = sm + L::b1;
  float* b2_s = sm + L::b2;
  float* q_s = sm + L::q;
  float* praw_s = sm + L::praw;
  float* vd_s = sm + L::vd;
  float* g_s = sm + L::g;
  float* dpre_s = sm + L::dpre;
  float* wk_s = sm + L::wk;
  float* zk_s = sm + L::zk;
  int* ray_s = reinterpret_cast<int*>(sm + L::ray);
  int* kk_s = reinterpret_cast<int*>(sm + L::kk);

  const int tid = threadIdx.x;
  const int tn = tid & 15, ts = tid >> 4;       // GEMM tiles: 4 samples x 8 units, or 8 x 8 weights
  const int S = F.S;

  // weights -> shared memory (padded rows: conflict-free both along n and along k; TC: the bf16 images)
  unsigned char* img = reinterpret_cast<unsigned char*>(sm);
  unsigned char* scr = reinterpret_cast<unsigned char*>(sm + L::scr);
  const uint32_t w1b_a = smem_u32(img), w2_a = w1b_a + 2 * OPER1_BYTES, scr_a = smem_u32(scr);
  const int wg = tid >> 7, q4 = tid & 3;
  if constexpr (TC) {
    const uint4* src = reinterpret_cast<const uint4*>(A.bp);
    for (int e = tid; e < TC_IMG_BYTES / 16; e += SH_THREADS) reinterpret_cast<uint4*>(img)[e] = __ldg(src + e);
  } else {
    for (int e = tid; e < NF * FC; e += SH_THREADS) W1BT_s[(e / FC) * LDW + (e % FC)] = __ldg(A.bp + BP_W1BT + e);
    for (int e = tid; e < FC * FC; e += SH_THREADS) W2T_s[(e / FC) * LDW + (e % FC)] = __ldg(A.bp + BP_W2T + e);
  }
  const float* tail = A.bp + PREP_TAIL / 4;
  for (int e = tid; e < 3 * W3_LD; e += SH_THREADS) W3_s[e] = __ldg(tail + TAIL_W3 + e);
  for (int e = tid; e < FC; e += SH_THREADS) { b1_s[e] = __ldg(tail + TAIL_B1 + e); b2_s[e] = __ldg(tail + TAIL_B2 + e); }
  const float b3r[3] = {__ldg(tail + TAIL_B3), __ldg(tail + TAIL_B3 + 1), __ldg(tail + TAIL_B3 + 2)};

  // per-thread gradient accumulators, kept for the whole launch
  float accW2[8][8];      // dW2[n = 8 ts + i][k = tn + 16 j]
  float accW1[8][5];      // dW1B[n = 8 ts + i][t = tn + 16 j], t < 72
  float accW3[3] = {0.f, 0.f, 0.f};   // tid < 128: dW3[c][n = tid]; 128..130: dW3[c][128 + a]; 131: db3
  float accB1 = 0.0f, accB2 = 0.0f;   // tid < 128
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) accW2[i][j] = 0.0f;
#pragma unroll
    for (int j = 0; j < 5; ++j) accW1[i][j] = 0.0f;
  }
  __syncthreads();

  const long long n_app = (long long)*A.s.count;
  const long long n_tiles = (n_app + TS - 1) / TS;
  const int ls = tid >> 2, cq = tid & 3;        // gather / scatter: sample ls, channels cq*6 .. cq*6+5

  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * TS;
    const int n_valid = (int)((n_app - e0) < TS ? (n_app - e0) : TS);
    // ---- 2a. tile header: ray data of each sample ---------------------------------------------------
    if (tid < TS) {
      int ray = 0, k = 0;
      float wk = 0.0f;
      if (tid < n_valid) { ray = A.s.app_ray[e0 + tid]; k = A.s.app_k[e0 + tid]; wk = A.s.w[(size_t)ray * S + k]; }
      ray_s[tid] = ray; kk_s[tid] = k; wk_s[tid] = wk;
      RaySm R;
      normalize_ray(A.rays + 6 * (size_t)ray, A.rays + 6 * (size_t)ray + 3, R);
      const float z = __ldg(F.z + k);
      zk_s[tid] = z;
      float p[3], q[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) praw_s[tid * 3 + a] = R.o[a] + R.vd[a] * z;
      sample_pos(F, R, z, p, q);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        q_s[tid * 3 + a] = q[a];
        vd_s[tid * 3 + a] = R.vd[a];
        g_s[tid * 3 + a] = tid < n_valid ? A.g_rgb[3 * (size_t)ray + a] : 0.0f;
      }
    }
    __syncthreads();
    // ---- 2b. the 72 products (compute_appfeature before basis_mat, tensoRF.py:153-195) --------------
    {
      const float qq[3] = {q_s[ls * 3], q_s[ls * 3 + 1], q_s[ls * 3 + 2]};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const VmTap t = vm_tap<CA>(F.g, i, qq);
        for (int grp = cq; grp < CA / 4; grp += 4) {                    // 4 components per 16-byte group
          float v[4];
          vm_products<4>(t, F.aplane[i], F.aline[i], grp * 4, v);
          float* xo = X_s + ls * LDX + i * CA + grp * 4;
          const bool ok = ls < n_valid;
#pragma unroll
          for (int e = 0; e < 4; ++e) xo[e] = ok ? v[e] : 0.0f;
        }
      }
    }
    __syncthreads();
    // ---- 2c. layer 1 (basis folded in) and layer 2, forward ----------------------------------------
    if constexpr (TC) {          // warpgroup wg: output units 64 wg .. 64 wg + 63 of both layers
      float d[32];
      build_image(X_s, LDX, NF, K1_CHUNKS, scr);
      shade_gemm<64, 0>(d, scr_a, K1_CHUNKS, K1 / 16, w1b_a + wg * 8 * K1_CHUNKS * 128, w1b_a + OPER1_BYTES + wg * 8 * K1_CHUNKS * 128,
                        256u, 128u, K1_CHUNKS * 128u);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 64 * wg + 8 * i + 2 * q4 + e;
            H1_s[wg_row(j) * LDW + n] = fmaxf(d[4 * i + 2 * j + e] + b1_s[n], 0.0f);
          }
      __syncthreads();                                                   // layer 1 has read the x image
      build_image(H1_s, LDW, FC, K2_CHUNKS, scr);
      shade_gemm<64, 0>(d, scr_a, K2_CHUNKS, FC / 16, w2_a + wg * 8 * K2_CHUNKS * 128, w2_a + OPER2_BYTES + wg * 8 * K2_CHUNKS * 128,
                        256u, 128u, K2_CHUNKS * 128u);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 64 * wg + 8 * i + 2 * q4 + e;
            H2_s[wg_row(j) * LDW + n] = fmaxf(d[4 * i + 2 * j + e] + b2_s[n], 0.0f);
          }
    } else {
      {
        float acc[4][8];
  #pragma unroll
        for (int i = 0; i < 4; ++i)
  #pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = b1_s[tn + 16 * j];
        for (int k = 0; k < NF; ++k) {
          float xv[4], wv[8];
  #pragma unroll
          for (int i = 0; i < 4; ++i) xv[i] = X_s[(4 * ts + i) * LDX + k];
  #pragma unroll
          for (int j = 0; j < 8; ++j) wv[j] = W1BT_s[k * LDW + tn + 16 * j];
  #pragma unroll
          for (int i = 0; i < 4; ++i)
  #pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
        }
  #pragma unroll
        for (int i = 0; i < 4; ++i)
  #pragma unroll
          for (int j = 0; j < 8; ++j) H1_s[(4 * ts + i) * LDW + tn + 16 * j] = fmaxf(acc[i][j], 0.0f);
      }
      __syncthreads();
      {
        float acc[4][8];
  #pragma unroll
        for (int i = 0; i < 4; ++i)
  #pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = b2_s[tn + 16 * j];
        for (int k = 0; k < FC; ++k) {
          float xv[4], wv[8];
  #pragma unroll
          for (int i = 0; i < 4; ++i) xv[i] = H1_s[(4 * ts + i) * LDW + k];
  #pragma unroll
          for (int j = 0; j < 8; ++j) wv[j] = W2T_s[k * LDW + tn + 16 * j];
  #pragma unroll
          for (int i = 0; i < 4; ++i)
  #pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
        }
  #pragma unroll
        for (int i = 0; i < 4; ++i)
  #pragma unroll
          for (int j = 0; j < 8; ++j) H2_s[(4 * ts + i) * LDW + tn + 16 * j] = fmaxf(acc[i][j], 0.0f);
      }
    }
    __syncthreads();
    // ---- 2d. layer 3 + sigmoid; dL/d(pre-sigmoid); g . rgb joins the sample's dL/dw ------------------
    {
      float s3[3] = {0.f, 0.f, 0.f};
      for (int m = 0; m < FC / 4; ++m) {
        const int n = cq + 4 * m;
        const float h = H2_s[ls * LDW + n];
#pragma unroll
        for (int c = 0; c < 3; ++c) s3[c] = fmaf(W3_s[c * W3_LD + n], h, s3[c]);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        s3[c] += __shfl_xor_sync(0xffffffffu, s3[c], 1);
        s3[c] += __shfl_xor_sync(0xffffffffu, s3[c], 2);
      }
      if (cq == 0) {
        float grgb = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float s = s3[c] + W3_s[c * W3_LD + FC] * vd_s[ls * 3] + W3_s[c * W3_LD + FC + 1] * vd_s[ls * 3 + 1] +
                          W3_s[c * W3_LD + FC + 2] * vd_s[ls * 3 + 2] + b3r[c];
          const float rgb = __fdiv_rn(1.0f, 1.0f + expf(-s));
          const float gc = g_s[ls * 3 + c];
          dpre_s[ls * 3 + c] = ls < n_valid ? gc * wk_s[ls] * rgb * (1.0f - rgb) : 0.0f;
          grgb += gc * rgb;
        }
        if (ls < n_valid) A.s.gw[(size_t)ray_s[ls] * S + kk_s[ls]] += grgb;
      }
    }
    __syncthreads();
    // ---- 2e. layer 3 backward --------------------------------------------------------------------------
    if (tid < FC) {
      for (int s = 0; s < TS; ++s) {
        const float h = H2_s[s * LDW + tid];
#pragma unroll
        for (int c = 0; c < 3; ++c) accW3[c] = fmaf(dpre_s[s * 3 + c], h, accW3[c]);
      }
    } else if (tid < FC + 3) {                   // view-direction columns (viewdirs detached, :628)
      const int a = tid - FC;
      for (int s = 0; s < TS; ++s) {
        const float v = vd_s[s * 3 + a];
#pragma unroll
        for (int c = 0; c < 3; ++c) accW3[c] = fmaf(dpre_s[s * 3 + c], v, accW3[c]);
      }
    } else if (tid == FC + 3) {                  // bias
      for (int s = 0; s < TS; ++s) {
#pragma unroll
        for (int c = 0; c < 3; ++c) accW3[c] += dpre_s[s * 3 + c];
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int s = 4 * ts + i;
      const float d0 = dpre_s[s * 3], d1 = dpre_s[s * 3 + 1], d2 = dpre_s[s * 3 + 2];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = tn + 16 * j;
        const float gsum = W3_s[n] * d0 + W3_s[W3_LD + n] * d1 + W3_s[2 * W3_LD + n] * d2;
        const float h = H2_s[s * LDW + n];
        H2_s[s * LDW + n] = h > 0.0f ? gsum : 0.0f;                     // dL/d(pre-activation 2)
      }
    }
    __syncthreads();
    // ---- 2f. layer 2 backward: db2, dW2 += dh2^T h1, dh1 = dh2 W2 ------------------------------------
    if (tid < FC) {
      float p0 = 0.0f, p1 = 0.0f, p2 = 0.0f, p3 = 0.0f;
#pragma unroll 4
      for (int s = 0; s < TS; s += 4) {
        p0 += H2_s[s * LDW + tid]; p1 += H2_s[(s + 1) * LDW + tid];
        p2 += H2_s[(s + 2) * LDW + tid]; p3 += H2_s[(s + 3) * LDW + tid];
      }
      accB2 += (p0 + p1) + (p2 + p3);
    }
    for (int s = 0; s < TS; ++s) {
      float dv[8], hv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) dv[i] = H2_s[s * LDW + 8 * ts + i];
#pragma unroll
      for (int j = 0; j < 8; ++j) hv[j] = H1_s[s * LDW + tn + 16 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) accW2[i][j] = fmaf(dv[i], hv[j], accW2[i][j]);
    }
    if constexpr (TC) {          // dh1[s][k] = dh2 W2: B = the W2 image read MN-major (k along N, n along K)
      float d[32];
      build_image(H2_s, LDW, FC, K2_CHUNKS, scr);
      shade_gemm<64, 1>(d, scr_a, K2_CHUNKS, FC / 16, w2_a + wg * 1024u, w2_a + OPER2_BYTES + wg * 1024u,
                        2u * K2_CHUNKS * 128u, K2_CHUNKS * 128u, 128u);
      __syncthreads();                                                   // every reader of h1 is done
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int o = wg_row(j) * LDW + 64 * wg + 8 * i + 2 * q4 + e;
            H1_s[o] = H1_s[o] > 0.0f ? d[4 * i + 2 * j + e] : 0.0f;       // dL/d(pre-activation 1)
          }
    } else {
      float acc[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
      for (int n = 0; n < FC; ++n) {
        float dv[4], wv[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) dv[i] = H2_s[(4 * ts + i) * LDW + n];
#pragma unroll
        for (int j = 0; j < 8; ++j) wv[j] = W2T_s[(tn + 16 * j) * LDW + n];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(dv[i], wv[j], acc[i][j]);
      }
      __syncthreads();                                                   // every reader of h1 is done
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int o = (4 * ts + i) * LDW + tn + 16 * j;
          H1_s[o] = H1_s[o] > 0.0f ? acc[i][j] : 0.0f;                   // dL/d(pre-activation 1)
        }
    }
    __syncthreads();
    // ---- 2g. layer 1 backward: db1, dW1B += dh1^T x, dprod = dh1 W1B -----------------------------------
    if (tid < FC) {
      float p0 = 0.0f, p1 = 0.0f, p2 = 0.0f, p3 = 0.0f;
#pragma unroll 4
      for (int s = 0; s < TS; s += 4) {
        p0 += H1_s[s * LDW + tid]; p1 += H1_s[(s + 1) * LDW + tid];
        p2 += H1_s[(s + 2) * LDW + tid]; p3 += H1_s[(s + 3) * LDW + tid];
      }
      accB1 += (p0 + p1) + (p2 + p3);
    }
    for (int s = 0; s < TS; ++s) {
      float dv[8], xv[5];
#pragma unroll
      for (int i = 0; i < 8; ++i) dv[i] = H1_s[s * LDW + 8 * ts + i];
#pragma unroll
      for (int j = 0; j < 5; ++j) xv[j] = (tn + 16 * j < NF) ? X_s[s * LDX + tn + 16 * j] : 0.0f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 5; ++j) accW1[i][j] = fmaf(dv[i], xv[j], accW1[i][j]);
    }
    if constexpr (TC) {          // dprod[s][t] = dh1 W1B: B = the W1B image read MN-major (t along N, n along K)
      float d[20];
      build_image(H1_s, LDW, FC, K2_CHUNKS, scr);
      shade_gemm<40, 1>(d, scr_a, K2_CHUNKS, FC / 16, w1b_a + wg * 640u, w1b_a + OPER1_BYTES + wg * 640u,
                        2u * K1_CHUNKS * 128u, K1_CHUNKS * 128u, 128u);
      __syncthreads();                                                   // every reader of x is done
#pragma unroll
      for (int i = 0; i < 5; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int t = 40 * wg + 8 * i + 2 * q4 + e;
            if (t < NF) X_s[wg_row(j) * LDX + t] = d[4 * i + 2 * j + e];
          }
    } else {
      float acc[4][5];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 5; ++j) acc[i][j] = 0.0f;
      for (int n = 0; n < FC; ++n) {
        float dv[4], wv[5];
#pragma unroll
        for (int i = 0; i < 4; ++i) dv[i] = H1_s[(4 * ts + i) * LDW + n];
#pragma unroll
        for (int j = 0; j < 5; ++j) wv[j] = (tn + 16 * j < NF) ? W1BT_s[(tn + 16 * j) * LDW + n] : 0.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 5; ++j) acc[i][j] = fmaf(dv[i], wv[j], acc[i][j]);
      }
      __syncthreads();                                                   // every reader of x is done
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 5; ++j)
          if (tn + 16 * j < NF) X_s[(4 * ts + i) * LDX + tn + 16 * j] = acc[i][j];
    }
    __syncthreads();
    // ---- 2h. products backward: appearance planes / lines (16-byte reductions), position -> ray -----
    {
      float dq0 = 0.0f, dq1 = 0.0f, dq2 = 0.0f;
      if (ls < n_valid) {
        const float qq[3] = {q_s[ls * 3], q_s[ls * 3 + 1], q_s[ls * 3 + 2]};
        float dq[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int i = 0; i < 3; ++i)                                       // this thread's 4-component groups cq, cq + 4
          vm_pair_backward<CA, 1>(F.g, i, F.aplane[i], F.aline[i], A.d_aplane[i], A.d_aline[i], qq,
                                  [&](int c) { return X_s[ls * LDX + i * CA + c]; }, dq, 4 * cq, 16);
        dq0 = dq[0]; dq1 = dq[1]; dq2 = dq[2];
      }
      dq0 += __shfl_xor_sync(0xffffffffu, dq0, 1); dq0 += __shfl_xor_sync(0xffffffffu, dq0, 2);
      dq1 += __shfl_xor_sync(0xffffffffu, dq1, 1); dq1 += __shfl_xor_sync(0xffffffffu, dq1, 2);
      dq2 += __shfl_xor_sync(0xffffffffu, dq2, 1); dq2 += __shfl_xor_sync(0xffffffffu, dq2, 2);
      if (cq == 0 && ls < n_valid) {
        float dp0, dp1, dp2;
        contract_bwd(praw_s[ls * 3], praw_s[ls * 3 + 1], praw_s[ls * 3 + 2], dq0 * F.ainv[0],
                     dq1 * F.ainv[1], dq2 * F.ainv[2], dp0, dp1, dp2);
        if (A.s.dpos) {          // one slot per (ray, sample): the density kernel sums them in a fixed order
          float* dst = A.s.dpos + 3 * ((size_t)ray_s[ls] * S + kk_s[ls]);
          dst[0] = dp0; dst[1] = dp1; dst[2] = dp2;
        } else {
          float* acc = A.s.d_ovd + 6 * (size_t)ray_s[ls];
          const float z = zk_s[ls];
          atomicAdd(acc + 0, dp0); atomicAdd(acc + 1, dp1); atomicAdd(acc + 2, dp2);
          atomicAdd(acc + 3, dp0 * z); atomicAdd(acc + 4, dp1 * z); atomicAdd(acc + 5, dp2 * z);
        }
      }
    }
    __syncthreads();
  }

  // ---- flush the per-thread accumulators -----------------------------------------------------------
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int n = 8 * ts + i;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (accW2[i][j] != 0.0f) atomicAdd(A.d_w2 + n * FC + tn + 16 * j, accW2[i][j]);
#pragma unroll
    for (int j = 0; j < 5; ++j)
      if (tn + 16 * j < NF && accW1[i][j] != 0.0f) atomicAdd(A.d_w1b + n * NF + tn + 16 * j, accW1[i][j]);
  }
  if (tid < FC + 3) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
      if (accW3[c] != 0.0f) atomicAdd(A.d_w3 + c * (FC + 3) + tid, accW3[c]);
  } else if (tid == FC + 3) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
      if (accW3[c] != 0.0f) atomicAdd(A.d_b3 + c, accW3[c]);
  }
  if (tid < FC) {
    if (accB1 != 0.0f) atomicAdd(A.d_b1 + tid, accB1);
    if (accB2 != 0.0f) atomicAdd(A.d_b2 + tid, accB2);
  }
}

// ====================================================================================================
// 3. density branch + rays
// ====================================================================================================
__global__ void __launch_bounds__(MARCH_THREADS)
bwd_density_kernel(const FieldDev F, const BwdArgs A) {
  const int S = F.S;
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * MARCH_THREADS + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * MARCH_THREADS) >> 5;
  const int n_chunks = (S + 31) / 32;
  for (long long ray = warp0; ray < A.n_rays; ray += n_warps) {
    RaySm R;
    normalize_ray(A.rays + 6 * ray, A.rays + 6 * ray + 3, R);
    const float gd = A.g_depth[ray];
    const size_t base = (size_t)ray * S;
    float d_o[3] = {0.0f, 0.0f, 0.0f}, d_vd[3] = {0.0f, 0.0f, 0.0f};   // lane-partial sums
    float dep_p = 0.0f;
    float suffix_carry = 0.0f;                                           // sum_{j in later chunks} gw_j w_j
    for (int ch = n_chunks - 1; ch >= 0; --ch) {
      const int k = ch * 32 + lane;
      const bool in = k < S;
      const float gwk = in ? A.s.gw[base + k] : 0.0f;
      const float wk = in ? A.s.w[base + k] : 0.0f;
      const float zk = in ? __ldg(F.z + k) : 0.0f;
      dep_p += wk * zk;
      const float term = gwk * wk;
      float inc = term;                                                  // inclusive suffix sum
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_down_sync(0xffffffffu, inc, o);
        if (lane + o < 32) inc += u;
      }
      const float excl = inc - term + suffix_carry;                      // sum_{j > k} gw_j w_j
      suffix_carry += __shfl_sync(0xffffffffu, inc, 0);
      if (in && A.s.dpos) {                                              // colour-branch part (zero if not shaded)
        const float* dp = A.s.dpos + 3 * (base + k);
#pragma unroll
        for (int a = 0; a < 3; ++a) { d_o[a] += dp[a]; d_vd[a] += dp[a] * zk; }
      }
      if (k < S - 1 && A.s.valid[base + k]) {                            // last / masked samples: constants
        const float al = A.s.alpha[base + k];
        const float dalpha = gwk * A.s.T[base + k] - __fdiv_rn(excl, (1.0f - al) + 1e-10f);
        const float dsigma = dalpha * (1.0f - al) * (__ldg(F.z + k + 1) - zk) * F.distance_scale;
        const float df = feature2density_grad(A.s.fe[base + k], F.density_shift, F.act, dsigma);
        if (df != 0.0f) {
          float p[3], q[3], dq[3] = {0.0f, 0.0f, 0.0f};
          sample_pos(F, R, zk, p, q);
#pragma unroll
          for (int i = 0; i < 3; ++i)
            vm_pair_backward<CD>(F.g, i, F.dplane[i], F.dline[i], A.d_dplane[i], A.d_dline[i], q,
                                 [&](int) { return df; }, dq);
          float dp0, dp1, dp2;
          contract_bwd(R.o[0] + R.vd[0] * zk, R.o[1] + R.vd[1] * zk, R.o[2] + R.vd[2] * zk,
                       dq[0] * F.ainv[0], dq[1] * F.ainv[1], dq[2] * F.ainv[2], dp0, dp1, dp2);
          d_o[0] += dp0; d_o[1] += dp1; d_o[2] += dp2;
          d_vd[0] += dp0 * zk; d_vd[1] += dp1 * zk; d_vd[2] += dp2 * zk;
        }
      }
    }
    // ---- rays: vd = d/|d| and depth = sum(w z)/|d| ----------------------------------------------------
#pragma unroll
    for (int a = 0; a < 3; ++a) { d_o[a] = warp_sum(d_o[a]); d_vd[a] = warp_sum(d_vd[a]); }
    const float depth = __fdiv_rn(warp_sum(dep_p), R.nrm);
    if (lane == 0) {
      const float* acc = A.s.d_ovd + 6 * (size_t)ray;                    // colour-branch part (zero with dpos)
#pragma unroll
      for (int a = 0; a < 3; ++a) { d_o[a] += acc[a]; d_vd[a] += acc[3 + a]; }
      const float dotv = R.vd[0] * d_vd[0] + R.vd[1] * d_vd[1] + R.vd[2] * d_vd[2];
      float* out = A.d_rays + 6 * ray;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        out[a] = d_o[a];
        out[3 + a] = __fdiv_rn(d_vd[a] - R.vd[a] * dotv, R.nrm) - gd * __fdiv_rn(depth, R.nrm) * R.vd[a];
      }
    }
  }
}

// the backward's part of its prepared block: folded layer 1 and W2, both transposed
__global__ void prepare_backward_kernel(const float* __restrict__ basis, const float* __restrict__ w1,
                                        const float* __restrict__ w2, float* __restrict__ bp) {
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  for (int e = t0; e < FC * NF; e += stride) {
    const int n = e / NF, t = e - n * NF;
    float s = 0.0f;
    for (int j = 0; j < APP_DIM; ++j) s = fmaf(w1[n * APP_DIM + j], basis[j * NF + t], s);
    bp[BP_W1BT + t * FC + n] = s;
  }
  for (int e = t0; e < FC * FC; e += stride) {
    const int n = e / FC, k = e - n * FC;
    bp[BP_W2T + k * FC + n] = w2[e];
  }
}

// ---- host-side launchers --------------------------------------------------------------------------
size_t backward_prepared_bytes() { return (size_t)BP_FLOATS * sizeof(float); }
size_t backward_scratch_bytes(long long n_rays, int S) {
  ScratchCarver c(nullptr);
  carve(c, n_rays, S);
  return c.size(16);
}
size_t backward_shade_smem_bytes(bool tc) { return (size_t)(tc ? ShadeSmemT<true>::total : ShadeSmem::total) * sizeof(float); }

cudaError_t launch_prepare_backward(const float* basis, const float* w1, const float* b1,
                                    const float* w2, const float* b2, const float* w3,
                                    const float* b3, float* bp, cudaStream_t stream) {
  prepare_backward_kernel<<<64, 256, 0, stream>>>(basis, w1, w2, bp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_prepare(basis, w1, b1, w2, b2, w3, b3, reinterpret_cast<unsigned char*>(bp), stream);
}

cudaError_t launch_render_backward(const FieldDev& F, BwdArgs A, void* scratch, float* dpos, int n_sms,
                                   cudaStream_t stream) {
  ScratchCarver c(scratch);
  size_t zero_bytes = 0;
  A.s = carve(c, A.n_rays, F.S, &zero_bytes);
  A.s.dpos = dpos;
  cudaError_t e = cudaMemsetAsync(scratch, 0, zero_bytes, stream);
  if (e != cudaSuccess) return e;
  // tensor-core shade step by default; LRF_BWD_TC=0 selects the CUDA-core kernel (the independent fp32
  // implementation the tensor-core one is tested against).  Read per call so tests can switch.
  const char* tc_env = getenv("LRF_BWD_TC");
  const bool use_tc = !(tc_env && tc_env[0] == '0');
  const size_t smem = backward_shade_smem_bytes(use_tc);
  e = set_max_dynamic_smem(use_tc ? (const void*)bwd_shade_kernel<true> : (const void*)bwd_shade_kernel<false>,
                           (int)smem);
  if (e != cudaSuccess) return e;
  const unsigned int grid = cta_count(A.n_rays, MARCH_THREADS / 32, n_sms, 8);   // a warp per ray
  bwd_march_kernel<<<grid, MARCH_THREADS, 0, stream>>>(F, A);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  if (use_tc) bwd_shade_kernel<true><<<n_sms, SH_THREADS, smem, stream>>>(F, A);
  else bwd_shade_kernel<false><<<n_sms, SH_THREADS, smem, stream>>>(F, A);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  bwd_density_kernel<<<grid, MARCH_THREADS, 0, stream>>>(F, A);
  return cudaGetLastError();
}

cudaError_t launch_render_backward_abi(const FieldDev& F, const float* rays, long long n_rays,
                                       int white_bg, const float* g_rgb, const float* g_depth,
                                       const float* bp, const LrfGradients& G, void* scratch,
                                       int n_sms, cudaStream_t stream, float* dpos) {
  BwdArgs A;
  A.n_rays = n_rays; A.rays = rays; A.g_rgb = g_rgb; A.g_depth = g_depth; A.bp = bp;
  A.white_bg = white_bg; A.d_rays = G.d_rays;
  for (int i = 0; i < 3; ++i) {
    A.d_dplane[i] = G.d_dplane[i]; A.d_dline[i] = G.d_dline[i];
    A.d_aplane[i] = G.d_aplane[i]; A.d_aline[i] = G.d_aline[i];
  }
  A.d_w1b = G.d_w1b; A.d_b1 = G.d_b1; A.d_w2 = G.d_w2; A.d_b2 = G.d_b2; A.d_w3 = G.d_w3; A.d_b3 = G.d_b3;
  return launch_render_backward(F, A, scratch, dpos, n_sms, stream);
}

}  // namespace lrf
