// Host emulation of the kernels' per-sample building blocks (TEST INFRASTRUCTURE; see shim/cuda_runtime.h).
// Compiles localrf_b200/csrc/lrf_common.cuh + lrf_device.cuh with g++ and exposes a few of their functions
// through a C ABI for tests/test_host_emul.py, which compares them with the oracle.  Nothing here is product code.
#include <cuda_runtime.h>
#include <cuda_bf16.h>

#include "../../localrf_b200/csrc/lrf_device.cuh"

using namespace lrf;

namespace {
FieldDev make_field(const int* grid, const float* aabb, const void* const* dplane, const void* const* dline,
                    const void* const* aplane, const void* const* aline, int grid16) {
  FieldDev F;
  memset(&F, 0, sizeof(F));
  for (int a = 0; a < 3; ++a) {
    F.g[a] = grid[a];
    F.amin[a] = aabb[a];
    F.ainv[a] = 2.0f / (aabb[3 + a] - aabb[a]);
    F.dplane[a] = static_cast<const float*>(dplane[a]); F.dline[a] = static_cast<const float*>(dline[a]);
    F.aplane[a] = static_cast<const float*>(aplane[a]); F.aline[a] = static_cast<const float*>(aline[a]);
  }
  F.grid16 = grid16;
  return F;
}
}  // namespace

extern "C" {

// compute_densityfeature on M normalised points, channel-last grids (fp32 or bf16 texels)
void emul_density_feature(const int* grid, const float* aabb, const void* const* dplane, const void* const* dline,
                          const void* const* aplane, const void* const* aline, int grid16, const float* xyz,
                          long long M, float* out) {
  const FieldDev F = make_field(grid, aabb, dplane, dline, aplane, aline, grid16);
  for (long long m = 0; m < M; ++m)
    out[m] = grid16 ? density_feature_t<true>(F, xyz + 3 * m) : density_feature_t<false>(F, xyz + 3 * m);
}

// the 72 plane x line products of compute_appfeature (before basis_mat), [M][72]
void emul_app_products(const int* grid, const float* aabb, const void* const* dplane, const void* const* dline,
                       const void* const* aplane, const void* const* aline, int grid16, const float* xyz,
                       long long M, float* out) {
  const FieldDev F = make_field(grid, aabb, dplane, dline, aplane, aline, grid16);
  for (long long m = 0; m < M; ++m)
    for (int i = 0; i < 3; ++i) {
      if (grid16) app_plane_features_t<true>(F, i, xyz + 3 * m, out + m * NF + i * CA);
      else app_plane_features_t<false>(F, i, xyz + 3 * m, out + m * NF + i * CA);
    }
}

// contract (utils/ray_utils.py:9-12) in place, then normalize_coord -> q; p [M][3] in, p (contracted) and q out
void emul_sample_pos(const float* aabb, const float* o, const float* vd, const float* z, long long M, float* p_out,
                     float* q_out) {
  FieldDev F;
  memset(&F, 0, sizeof(F));
  for (int a = 0; a < 3; ++a) { F.amin[a] = aabb[a]; F.ainv[a] = 2.0f / (aabb[3 + a] - aabb[a]); }
  RaySm R;
  for (int a = 0; a < 3; ++a) { R.o[a] = o[a]; R.vd[a] = vd[a]; }
  for (long long m = 0; m < M; ++m) sample_pos(F, R, z[m], p_out + 3 * m, q_out + 3 * m);
}

// AlphaGridMask.sample_alpha: trilinear lookup of vol [D][H][W] at world points p [M][3]
void emul_alpha_mask(const float* vol, const int* dims, const float* alpha_aabb, const float* p, long long M, float* out) {
  FieldDev F;
  memset(&F, 0, sizeof(F));
  F.alpha_vol = vol;
  for (int a = 0; a < 3; ++a) {
    F.ad[a] = dims[a];
    F.aamin[a] = alpha_aabb[a];
    F.aainv[a] = 1.0f / (alpha_aabb[3 + a] - alpha_aabb[a]) * 2.0f;
  }
  for (long long m = 0; m < M; ++m) out[m] = alpha_mask(F, p + 3 * m);
}

// feature2density (softplus with threshold 20 / relu)
void emul_feature2density(const float* f, long long M, float shift, int act, float* out) {
  for (long long m = 0; m < M; ++m) out[m] = feature2density(f[m], shift, act);
}

// contract_bwd: d contract(p)/dp applied to g, p and g [M][3]
void emul_contract_bwd(const float* p, const float* g, long long M, float* out) {
  for (long long m = 0; m < M; ++m) {
    const float* a = p + 3 * m;
    const float* b = g + 3 * m;
    contract_bwd(a[0], a[1], a[2], b[0], b[1], b[2], out[3 * m], out[3 * m + 1], out[3 * m + 2]);
  }
}

// sample_alpha over all S samples of n rays (origins o, directions d [n][3], normalised here) of a field with
// an alpha mask (fp32 grids): alpha, fe [n][S] and valid [n][S]
void emul_sample_alpha(const int* grid, const float* aabb, const void* const* dplane, const void* const* dline,
                       const void* const* aplane, const void* const* aline, const float* vol, const int* dims,
                       const float* alpha_aabb, float density_shift, float distance_scale, int act, const float* z,
                       int S, const float* o, const float* d, long long n, float* alpha, float* fe,
                       unsigned char* valid) {
  FieldDev F = make_field(grid, aabb, dplane, dline, aplane, aline, 0);
  F.alpha_vol = vol;
  for (int a = 0; a < 3; ++a) {
    F.ad[a] = dims[a];
    F.aamin[a] = alpha_aabb[a];
    F.aainv[a] = 1.0f / (alpha_aabb[3 + a] - alpha_aabb[a]) * 2.0f;
  }
  F.density_shift = density_shift; F.distance_scale = distance_scale; F.act = act;
  F.z = z; F.S = S;
  for (long long r = 0; r < n; ++r) {
    RaySm R;
    normalize_ray(o + 3 * r, d + 3 * r, R);
    for (int k = 0; k < S; ++k) {
      bool v;
      alpha[r * S + k] = sample_alpha<false>(F, R, k, S, fe[r * S + k], v);
      valid[r * S + k] = v ? 1 : 0;
    }
  }
}

// ray generation of LocalTensorfs.forward (ids2pixel, get_ray_directions_*, cam2rf, get_rays_lean, normalisation):
// out_o / out_vd [n][3], out_nrm [n], dirs [n][3] (camera space), ij [n][2]
void emul_setup_rays(const long long* ray_ids, long long n, long long n_views, int W, int H, int fov360, float focal,
                     float cx, float cy, const float* c2w, const float* w2rf, float* out_o, float* out_vd,
                     float* out_nrm, float* dirs, long long* ij) {
  BatchDev B;
  memset(&B, 0, sizeof(B));
  B.n_rays = n; B.ray_ids = ray_ids; B.W = W; B.H = H; B.fov360 = fov360;
  B.focal = focal; B.cx = cx; B.cy = cy; B.c2w = c2w; B.w2rf = w2rf;
  B.rays_per_view = n / n_views; B.dirs = dirs; B.ij = ij;
  for (long long r = 0; r < n; ++r) {
    RaySm R;
    setup_ray(B, r, R);
    for (int a = 0; a < 3; ++a) { out_o[3 * r + a] = R.o[a]; out_vd[3 * r + a] = R.vd[a]; }
    out_nrm[r] = R.nrm;
  }
}

// split2 / store_chunk: the bf16 hi/lo operand split of one row (8 values) -> reconstructed hi + lo as floats
void emul_split8(const float* v, float* hi, float* lo) {
  for (int j = 0; j < 8; j += 2) {
    uint32_t h, l;
    split2(v[j], v[j + 1], h, l);
    hi[j] = shim_bf2f((uint16_t)(h & 0xffff)); hi[j + 1] = shim_bf2f((uint16_t)(h >> 16));
    lo[j] = shim_bf2f((uint16_t)(l & 0xffff)); lo[j + 1] = shim_bf2f((uint16_t)(l >> 16));
  }
}

// byte offset of element (row, k) in a K-major, no-swizzle core-matrix operand image (lrf_common.cuh)
int emul_oper_offset(int row, int k, int chunks) { return oper_offset(row, k, chunks); }
// sizes of the prepared blocks as the headers compute them
int emul_prep_bytes(void) { return PREP_BYTES; }
int emul_pe_prepared_bytes(int fea_pe) { return pe_prepared_bytes(fea_pe); }

}  // extern "C"
