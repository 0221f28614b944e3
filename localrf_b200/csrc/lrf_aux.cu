// lrf_aux.cu -- the small kernels around the render kernel: the synchronous tensor-core MLP on
// explicit features (lrf_mlp_forward), weight preparation, stand-alone feature lookups, repack.
#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

constexpr int THREADS = 256;   // two warpgroups: one 64-row half of the 128-row tile each

// shared-memory carve-up of mlp_kernel
struct MlpSmem {
  int prep, a, rgb, vd, mbar, total;
};
__host__ __device__ inline MlpSmem mlp_smem() {
  MlpSmem L;
  int off = 0;
  L.prep = off;  off += PREP_BYTES;               // B operands (bf16 hi/lo) + fp32 tail
  off = (off + 1023) & ~1023;
  L.a = off;     off += 2 * OPER1_BYTES;          // A1 hi/lo (layer 2's A operand lives in registers)
  L.rgb = off;   off += TM * 4 * 4;
  L.vd = off;    off += TM * 3 * 4;
  L.mbar = off;  off += 16;                       // the weight-staging mbarrier
  L.total = off;
  return L;
}

// fused basis_mat + MLPRender_Fea_late_view on explicit plane x line products (one CTA per 128 rows):
// layers 1 + 2 on the tensor cores (mlp_gemm_n128 / mlp_layers23, the render kernel's code), layer 3 +
// sigmoid on the CUDA cores
__global__ void __launch_bounds__(THREADS, 1)
mlp_kernel(const float* __restrict__ prep_g, const float* __restrict__ feats,
           const float* __restrict__ viewdirs, long long M, float* __restrict__ rgb) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const MlpSmem L = mlp_smem();
  unsigned char* prep_s = smem + L.prep;
  unsigned char* a_s = smem + L.a;
  float* rgb_s = reinterpret_cast<float*>(smem + L.rgb);
  float* vd_s = reinterpret_cast<float*>(smem + L.vd);   // [TM][3] view directions
  const uint32_t bar_w = smem_u32(smem + L.mbar);
  const int tid = threadIdx.x, wg = tid >> 7, q = tid & 3;
  if (tid == 0) {
    mbar_init(bar_w, 1);
    constexpr uint32_t bytes = PREP_BYTES;
    mbar_expect_tx(bar_w, bytes);
    constexpr uint32_t CH = 32768;  // keep each bulk copy modest
    for (uint32_t o = 0; o < bytes; o += CH)
      tma_bulk_g2s(smem_u32(prep_s) + o, reinterpret_cast<const char*>(prep_g) + o, min(CH, bytes - o), bar_w);
  }
  __syncthreads();
  mbar_wait(bar_w, 0);
  const float* tail = reinterpret_cast<const float*>(prep_s + PREP_TAIL);
  const float* W3_s = tail + TAIL_W3;
  const float* b3_s = tail + TAIL_B3;
  const uint32_t prep_a = smem_u32(prep_s);
  const long long n_tiles = (M + TM - 1) / TM;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const long long base = t * TM;
    for (int item = tid; item < 3 * TM; item += THREADS) {
      const int pl = item / TM, m = item - pl * TM;
      float feat[CA];
#pragma unroll
      for (int c = 0; c < CA; ++c)
        feat[c] = (base + m < M) ? feats[(base + m) * NF + pl * CA + c] : 0.0f;
#pragma unroll
      for (int c8 = 0; c8 < CA / 8; ++c8)
        store_chunk(a_s, a_s + OPER1_BYTES, m, pl * (CA / 8) + c8, K1_CHUNKS, feat + 8 * c8);
      if (pl == 0) {
        const float zero[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        store_chunk(a_s, a_s + OPER1_BYTES, m, K1_CHUNKS - 1, K1_CHUNKS, zero);
#pragma unroll
        for (int c = 0; c < 3; ++c)
          vd_s[m * 3 + c] = (base + m < M) ? viewdirs[(base + m) * 3 + c] : 0.0f;
      }
    }
    fence_async_smem();   // generic-proxy writes of A1 -> visible to the tensor core
    __syncthreads();
    const uint32_t a_hi = smem_u32(a_s) + (uint32_t)wg * 8u * K1_CHUNKS * 128u;
    float acc[64];
    mlp_gemm_n128(acc, a_hi, a_hi + OPER1_BYTES, prep_a + PREP_B1HI, prep_a + PREP_B1LO, K1 / 16, K1_CHUNKS);
    float s[2][3];
    mlp_layers23(acc, tail, prep_a + PREP_B2HI, prep_a + PREP_B2LO, s);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row = 64 * wg + wg_row(j);
      if (q != 0) continue;
      const float* vd = vd_s + row * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = s[j][c] + W3_s[c * W3_LD + FC] * vd[0] + W3_s[c * W3_LD + FC + 1] * vd[1] +
                  W3_s[c * W3_LD + FC + 2] * vd[2];
        v += b3_s[c];
        rgb_s[row * 4 + c] = __fdiv_rn(1.0f, 1.0f + expf(-v));
      }
    }
    __syncthreads();
    for (int e = tid; e < TM * 3; e += THREADS) {
      const int m = e / 3, c = e - 3 * m;
      if (base + m < M) rgb[(base + m) * 3 + c] = rgb_s[m * 4 + c];
    }
    __syncthreads();
  }
}

// ---- small kernels ------------------------------------------------------------------------------
// element `off` (bytes) of a bf16 hi / lo operand image pair: v = hi + lo
__device__ __forceinline__ void put_hi_lo(unsigned char* hi_img, unsigned char* lo_img, int off, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
  *reinterpret_cast<__nv_bfloat16*>(hi_img + off) = hi;
  *reinterpret_cast<__nv_bfloat16*>(lo_img + off) = lo;
}

// the fp32 tail of a prepared block: b1, b2, the first n_w3 columns of each row of W3 [3][w3_ld] (zero
// beyond), b3; thread t of `stride`
__device__ __forceinline__ void fill_tail(float* tail, const float* b1, const float* b2, const float* w3, int w3_ld,
                                          int n_w3, const float* b3, int t, int stride) {
  for (int e = t; e < FC; e += stride) { tail[TAIL_B1 + e] = b1[e]; tail[TAIL_B2 + e] = b2[e]; }
  for (int e = t; e < 3 * W3_LD; e += stride) {
    const int c = e / W3_LD, n = e - c * W3_LD;
    tail[TAIL_W3 + e] = n < n_w3 ? w3[c * w3_ld + n] : 0.0f;
  }
  for (int e = t; e < 4; e += stride) tail[TAIL_B3 + e] = e < 3 ? b3[e] : 0.0f;
}

// prepared block: bf16 hi/lo operand images of W1B = W1 @ basis and W2, fp32 biases and W3
__global__ void prepare_kernel(const float* __restrict__ basis, const float* __restrict__ w1,
                               const float* __restrict__ b1, const float* __restrict__ w2,
                               const float* __restrict__ b2, const float* __restrict__ w3,
                               const float* __restrict__ b3, unsigned char* __restrict__ prep) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int stride = gridDim.x * blockDim.x;
  for (int e = t; e < FC * K1; e += stride) {
    const int n = e / K1, k = e - n * K1;
    float s = 0.0f;
    if (k < NF)
      for (int j = 0; j < APP_DIM; ++j) s = fmaf(w1[n * APP_DIM + j], basis[j * NF + k], s);
    put_hi_lo(prep + PREP_B1HI, prep + PREP_B1LO, oper_offset(n, k, K1_CHUNKS), s);
  }
  for (int e = t; e < FC * FC; e += stride) {
    const int n = e / FC, k = e - n * FC;
    put_hi_lo(prep + PREP_B2HI, prep + PREP_B2LO, oper_offset(n, k, K2_CHUNKS), w2[n * FC + k]);
  }
  fill_tail(reinterpret_cast<float*>(prep + PREP_TAIL), b1, b2, w3, FC + 3, FC + 3, b3, t, stride);
}

// prepared block of a field with positional encodings (layout: lrf_common.cuh)
__global__ void prepare_pe_kernel(const float* __restrict__ basis, const float* __restrict__ w1,
                                  const float* __restrict__ b1, const float* __restrict__ w2,
                                  const float* __restrict__ b2, const float* __restrict__ w3,
                                  const float* __restrict__ b3, int fea_pe, int view_pe,
                                  unsigned char* __restrict__ prep) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int stride = gridDim.x * blockDim.x;
  for (int e = t; e < PE_N0 * K1; e += stride) {
    const int n = e / K1, k = e - n * K1;
    put_hi_lo(prep + PE_B0HI, prep + PE_B0LO, oper_offset(n, k, K1_CHUNKS),
              (n < APP_DIM && k < NF) ? basis[n * NF + k] : 0.0f);
  }
  for (int e = t; e < FC * FC; e += stride) {
    const int n = e / FC, k = e - n * FC;
    put_hi_lo(prep + PE_B2HI, prep + PE_B2LO, oper_offset(n, k, K2_CHUNKS), w2[n * FC + k]);
  }
  const int in_dim = pe_in_dim(fea_pe), nch = pe_chunks(fea_pe);
  for (int e = t; e < nch * FC * PE_KC; e += stride) {
    const int c = e / (FC * PE_KC), r = e - c * FC * PE_KC, n = r / PE_KC, kk = r - n * PE_KC;
    const int k = c * PE_KC + kk;
    unsigned char* img = prep + PE_W1 + (size_t)c * 2 * PE_WC_BYTES;
    put_hi_lo(img, img + PE_WC_BYTES, oper_offset(n, kk, PE_KC / 8), k < in_dim ? w1[n * in_dim + k] : 0.0f);
  }
  // the view part of W3 is read from the module's own weight
  fill_tail(reinterpret_cast<float*>(prep + PE_TAIL), b1, b2, w3, FC + 3 * (1 + 2 * view_pe), FC, b3, t, stride);
}

template <bool H16>      // H16: bf16 grid storage (LrfField.grid_dtype)
__global__ void density_feature_kernel(const FieldDev F, const float* __restrict__ xyz,
                                       long long M, float* __restrict__ out) {
  long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float q[3] = {xyz[3 * m], xyz[3 * m + 1], xyz[3 * m + 2]};
  out[m] = density_feature_t<H16>(F, q);
}

// compute_appfeature: 72 products then basis_mat (unfolded: this entry returns the 27-vector)
template <bool H16>
__global__ void app_feature_kernel(const FieldDev F, const float* __restrict__ basis,
                                   const float* __restrict__ xyz, long long M,
                                   float* __restrict__ out) {
  long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  float q[3] = {xyz[3 * m], xyz[3 * m + 1], xyz[3 * m + 2]};
  float feat[NF];
  app_plane_features_t<H16>(F, 0, q, feat);
  app_plane_features_t<H16>(F, 1, q, feat + CA);
  app_plane_features_t<H16>(F, 2, q, feat + 2 * CA);
  for (int o = 0; o < APP_DIM; ++o) {
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < NF; ++k) s = fmaf(__ldg(basis + o * NF + k), feat[k], s);
    out[m * APP_DIM + o] = s;
  }
}

__global__ void repack_kernel(const float* __restrict__ src, float* __restrict__ dst, int C,
                              long long HW) {
  long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= HW * C) return;
  long long p = e / C;
  int c = (int)(e - p * C);
  dst[e] = src[(long long)c * HW + p];
}

// ---- host-side launchers (called from lrf_abi.cu) -----------------------------------------------
cudaError_t launch_mlp(const float* prep, const float* feats, const float* viewdirs, long long M,
                       float* rgb, int n_sms, cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  const size_t smem = (size_t)mlp_smem().total;
  const cudaError_t e = set_max_dynamic_smem((const void*)mlp_kernel, (int)smem);
  if (e != cudaSuccess) return e;
  mlp_kernel<<<cta_count(M, TM, n_sms, 1), THREADS, smem, stream>>>(prep, feats, viewdirs, M, rgb);
  return cudaGetLastError();
}

cudaError_t launch_prepare(const float* basis, const float* w1, const float* b1, const float* w2,
                           const float* b2, const float* w3, const float* b3, unsigned char* prep,
                           cudaStream_t stream) {
  prepare_kernel<<<64, 256, 0, stream>>>(basis, w1, b1, w2, b2, w3, b3, prep);
  return cudaGetLastError();
}

cudaError_t launch_prepare_pe(const float* basis, const float* w1, const float* b1, const float* w2,
                              const float* b2, const float* w3, const float* b3, int fea_pe, int view_pe,
                              unsigned char* prep, cudaStream_t stream) {
  prepare_pe_kernel<<<64, 256, 0, stream>>>(basis, w1, b1, w2, b2, w3, b3, fea_pe, view_pe, prep);
  return cudaGetLastError();
}

cudaError_t launch_density_feature(const FieldDev& F, const float* xyz, long long M, float* out,
                                   cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  if (F.grid16) density_feature_kernel<true><<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(F, xyz, M, out);
  else density_feature_kernel<false><<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(F, xyz, M, out);
  return cudaGetLastError();
}

cudaError_t launch_app_feature(const FieldDev& F, const float* basis, const float* xyz, long long M,
                               float* out, cudaStream_t stream) {
  if (M == 0) return cudaSuccess;
  if (F.grid16) app_feature_kernel<true><<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(F, basis, xyz, M, out);
  else app_feature_kernel<false><<<(unsigned)((M + 127) / 128), 128, 0, stream>>>(F, basis, xyz, M, out);
  return cudaGetLastError();
}

cudaError_t launch_repack(const float* src, float* dst, int C, long long HW, cudaStream_t stream) {
  long long n = HW * C;
  if (n == 0) return cudaSuccess;
  repack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, C, HW);
  return cudaGetLastError();
}

// fp32 -> bfloat16, round to nearest even (lrf_pack_bf16): the 16-bit copy of a plane / line tensor
__global__ void pack_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride)
    dst[e] = __float2bfloat16_rn(src[e]);
}

cudaError_t launch_pack_bf16(const float* src, void* dst, long long n, int n_sms, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  pack_bf16_kernel<<<cta_count(n, 256, n_sms, 8), 256, 0, stream>>>(
      src, static_cast<__nv_bfloat16*>(dst), n);
  return cudaGetLastError();
}

// ---- fused pixel exchange: step barrier over peer-mapped flags (include/localrf_b200.h) ----------
struct PeerFlags { unsigned long long* p[16]; };

__global__ void peer_barrier_kernel(const PeerFlags F, const int rank, const int world,
                                    const unsigned long long seq, const unsigned long long wait_seq) {
  const int t = threadIdx.x;
  if (t >= world) return;
  // the render kernel before us on this stream stored pixels into the peers' buffers: order those
  // stores before the flag for every observer in the system
  __threadfence_system();
  unsigned long long* remote = F.p[t] + rank;          // my slot in peer t's flag array
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(remote), "l"(seq) : "memory");
  const unsigned long long* local = F.p[rank] + t;     // peer t's slot in my flag array
  unsigned long long v = 0;
  do {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(local) : "memory");
  } while (v < wait_seq);
}

cudaError_t launch_peer_barrier(unsigned long long* const* peer_flags, int rank, int world,
                                unsigned long long seq, unsigned long long wait_seq, cudaStream_t stream) {
  PeerFlags F;
  for (int p = 0; p < 16; ++p) F.p[p] = p < world ? peer_flags[p] : nullptr;
  peer_barrier_kernel<<<1, 32, 0, stream>>>(F, rank, world, seq, wait_seq);
  return cudaGetLastError();
}

}  // namespace lrf
