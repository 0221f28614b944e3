// lrf_common.cuh -- device-side structures and small helpers shared by the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lrf {

constexpr int CD = 8;        // density components per plane   (opt.py:117 n_lamb_sigma)
constexpr int CA = 24;       // appearance components per plane (opt.py:118 n_lamb_sh)
constexpr int NF = 3 * CA;   // 72 appearance features per sample
constexpr int APP_DIM = 27;  // opt.py:119 data_dim_color
constexpr int FC = 128;      // opt.py:155 featureC

// matMode / vecMode of the reference (models/tensorBase.py:274-275)
__host__ __device__ constexpr int mat0(int i) { return i == 2 ? 1 : 0; }
__host__ __device__ constexpr int mat1(int i) { return i == 0 ? 1 : 2; }
__host__ __device__ constexpr int vecm(int i) { return 2 - i; }

// Layout of the per-field prepared block (BYTES).  The two dense layers are stored as bf16 hi/lo
// pairs (w = hi + lo to ~16 mantissa bits) already in the shared-memory image the tensor core reads:
// K-major, no swizzle, 8x8 core matrices ([row group][k chunk][8 rows][8 bf16 = 16 B]).
//   B1 : W1B[n][k] = (mlp[0].weight @ basis_mat.weight)[n][k], n < 128, k < 72 (+8 zero pad)
//   B2 : mlp[2].weight[n][k], n, k < 128
// followed by the fp32 tail: b1[128], b2[128], W3[3][132] (131 used), b3[4].
constexpr int K1 = 80;                       // layer-1 K padded to a multiple of 16
constexpr int K1_CHUNKS = K1 / 8;            // 10 16-byte chunks per row
constexpr int K2_CHUNKS = FC / 8;            // 16
constexpr int OPER1_BYTES = 16 * K1_CHUNKS * 128;   // one [128 x 80] bf16 operand   = 20480
constexpr int OPER2_BYTES = 16 * K2_CHUNKS * 128;   // one [128 x 128] bf16 operand  = 32768
constexpr int PREP_B1HI = 0;
constexpr int PREP_B1LO = PREP_B1HI + OPER1_BYTES;
constexpr int PREP_B2HI = PREP_B1LO + OPER1_BYTES;
constexpr int PREP_B2LO = PREP_B2HI + OPER2_BYTES;
constexpr int PREP_TAIL = PREP_B2LO + OPER2_BYTES;  // fp32 from here
constexpr int W3_LD = 132;
constexpr int TAIL_B1 = 0, TAIL_B2 = FC, TAIL_W3 = 2 * FC, TAIL_B3 = 2 * FC + 3 * W3_LD;
constexpr int TAIL_FLOATS = TAIL_B3 + 4;
constexpr int PREP_BYTES = PREP_TAIL + TAIL_FLOATS * 4;
static_assert(PREP_BYTES % 16 == 0, "prepared block must be a multiple of 16 bytes");

// ---- prepared block of a field WITH positional encodings (fea_pe > 0 or view_pe > 0) ------------------
// basis_mat cannot be folded into layer 1 (the encoding sits between them), and layer 1's operand
// [128][27 (1 + 2 fea_pe)] does not fit shared memory next to W2 for fea_pe up to 6, so it is cut into
// K-chunks of 64 that the kernel streams per tile:
//   B0 : basis_mat.weight[n][k], n < 32 (27 used), k < 80 (72 used)      bf16 hi | lo images
//   B2 : mlp[2].weight                                                    bf16 hi | lo images (as above)
//   tail (fp32, as above; W3 = the first 128 columns of mlp_view[0].weight, the view part is read from the
//   module's own weight by the producers)
//   W1 chunk c : mlp[0].weight[n][64 c .. 64 c + 63] (zero padded)       bf16 hi | lo images, 8 chunks per row
constexpr int PE_N0 = 32;                                  // layer-0 (basis) N, padded
constexpr int PE_B0_BYTES = 16 * K1_CHUNKS * PE_N0;        // one [32 x 80] operand = 5120
constexpr int PE_KC = 64;                                  // K elements per streamed layer-1 chunk
constexpr int PE_WC_BYTES = 16 * (PE_KC / 8) * 128;        // one [128 x 64] operand = 16384
constexpr int PE_B0HI = 0, PE_B0LO = PE_B0_BYTES;
constexpr int PE_B2HI = 2 * PE_B0_BYTES, PE_B2LO = PE_B2HI + OPER2_BYTES;
constexpr int PE_TAIL = PE_B2LO + OPER2_BYTES;
constexpr int PE_RESIDENT = PE_TAIL + TAIL_FLOATS * 4;     // what stays in shared memory (78 400 B)
constexpr int PE_W1 = (PE_RESIDENT + 1023) & ~1023;        // chunk c at PE_W1 + c * 2 * PE_WC_BYTES (hi | lo)
constexpr int PE_MAX_FEA = 8, PE_MAX_VIEW = 8;
__host__ __device__ constexpr int pe_in_dim(int fea_pe) { return APP_DIM * (1 + 2 * fea_pe); }
__host__ __device__ constexpr int pe_chunks(int fea_pe) { return (pe_in_dim(fea_pe) + PE_KC - 1) / PE_KC; }
__host__ __device__ constexpr int pe_prepared_bytes(int fea_pe) { return PE_W1 + pe_chunks(fea_pe) * 2 * PE_WC_BYTES; }

// byte offset of element (row, k) inside a core-matrix operand image with `chunks` k-chunks per row
__host__ __device__ constexpr int oper_offset(int row, int k, int chunks) {
  return (((row >> 3) * chunks + (k >> 3)) * 8 + (row & 7)) * 16 + (k & 7) * 2;
}

struct FieldDev {
  int g[3];
  float amin[3], ainv[3];     // aabb min, 2/(max-min)   (tensorBase.py:321,342-345)
  const float* dplane[3];
  const float* dline[3];
  const float* aplane[3];
  const float* aline[3];
  const float* prep;
  const float* alpha_vol;     // may be null
  int ad[3];                  // alpha dims D,H,W
  float aamin[3], aainv[3];   // alpha aabb min, invgridSize (tensorBase.py:45)
  float density_shift, distance_scale, weight_thres;
  int act;
  const float* z;
  int S;
  int fea_pe, view_pe;        // positional encodings of the MLP (tensorBase.py:14-21,115-125); 0, 0 = the folded fast path
  const float* w3;            // mlp_view[0].weight [3][128 + 3 (1 + 2 view_pe)] (the producers' view term)
  int grid16;                 // 1: the twelve plane / line pointers address bfloat16 texels (LrfField.grid_dtype)
};

// the mesh export's scene (LrfMeshScene): the fields' device views and stepSizes, the lattice and the owner rule
constexpr int MESH_MAX_FIELDS = 64;
struct MeshSceneDev {
  FieldDev f[MESH_MAX_FIELDS];
  float length[MESH_MAX_FIELDS];
  const float* w2rf;          // device [n_fields][3]
  int n_fields;
  float voxel, origin[3], max_norm, level;
};

struct BatchDev {
  long long n_rays;
  const float* rays;
  const long long* ray_ids;
  int W, H, fov360;
  float focal, cx, cy;
  const float* intrinsics;
  const float* c2w;
  long long rays_per_view;
  const float* w2rf;
  const float* blend;
  long long blend_stride;
  const float* exposure;
  int accumulate, finalize, white_bg;
  float floater_thresh;
  float* rgb;
  float* depth;
  int rgb_stride, depth_stride;   // floats between consecutive rays (3 / 1, or 4 / 4 for pix)
  float* weights;
  float* dirs;
  long long* ij;
  unsigned long long* stats;
  unsigned long long* sched;   // ray counter of this launch (library-owned, zeroed per launch)
  int n_peers;                 // fused pixel exchange: peers that receive this rank's pixels
  float* peer_pix[16];
  float* mc_pix;               // NVLS multicast address (one multimem store reaches every peer)
  unsigned long long* peer_flags[16];   // in-kernel step signalling (signal_seq > 0)
  int rank;
  unsigned long long signal_seq, wait_seq;
  unsigned int* done_ctr;      // CTAs of this launch that have finished (library-owned, zeroed per launch)
  int refine;                  // MLPRender_Fea_late_view's `refine` (tensorBase.py:118-124): 0 = zeros for the encoding
};

// ---- sampling helpers -------------------------------------------------------------------------

// ATen grid_sampler coordinate transform, align_corners=True, padding_mode="border"
// (call sites models/tensoRF.py:135-146): pixel = clamp((c+1)/2*(size-1), 0, size-1)
__device__ __forceinline__ void grid_coord(float c, int size, int& i0, int& i1, float& t) {
  float x = ((c + 1.0f) * 0.5f) * (float)(size - 1);
  x = fminf((float)(size - 1), fmaxf(x, 0.0f));
  float f = floorf(x);
  i0 = (int)f;
  i1 = min(i0 + 1, size - 1);
  t = x - f;
}

// utils/ray_utils.py:9-12
__device__ __forceinline__ void contract(float& x, float& y, float& z) {
  float n = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z));
  n = fmaxf(n, 1e-6f);
  if (!(n <= 1.0f)) {
    float s = __fdiv_rn(2.0f * n - 1.0f, n * n);
    x *= s; y *= s; z *= s;
  }
}

// d contract(p)/dp applied to dpc (ray_utils.py:9-12; amax routes the norm's gradient to the
// component of largest magnitude)
__device__ __forceinline__ void contract_bwd(float p0, float p1, float p2, float g0, float g1,
                                             float g2, float& o0, float& o1, float& o2) {
  float n = fmaxf(fmaxf(fabsf(p0), fabsf(p1)), fabsf(p2));
  n = fmaxf(n, 1e-6f);
  if (n <= 1.0f) { o0 = g0; o1 = g1; o2 = g2; return; }
  const float s = __fdiv_rn(2.0f * n - 1.0f, n * n);
  const float ds = -2.0f / (n * n) + 2.0f / (n * n * n);
  const float dot = g0 * p0 + g1 * p1 + g2 * p2;
  int j = 0;
  float best = fabsf(p0);
  if (fabsf(p1) > best) { j = 1; best = fabsf(p1); }
  if (fabsf(p2) > best) { j = 2; }
  o0 = s * g0; o1 = s * g1; o2 = s * g2;
  const float pj = j == 0 ? p0 : (j == 1 ? p1 : p2);
  const float extra = (pj >= 0.0f ? 1.0f : -1.0f) * ds * dot;
  if (j == 0) o0 += extra; else if (j == 1) o1 += extra; else o2 += extra;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

// models/tensorBase.py:495-499
__device__ __forceinline__ float feature2density(float f, float shift, int act) {
  if (act == 0) {
    float x = f + shift;
    return x > 20.0f ? x : log1pf(expf(x));  // F.softplus(beta=1, threshold=20)
  }
  return fmaxf(f, 0.0f);
}

// dL/df from g = dL/d(feature2density(f))
__device__ __forceinline__ float feature2density_grad(float f, float shift, int act, float g) {
  if (act == 0) {
    const float x = f + shift;
    return g * (x > 20.0f ? 1.0f : __fdiv_rn(1.0f, 1.0f + expf(-x)));
  }
  return f > 0.0f ? g : 0.0f;
}

}  // namespace lrf
