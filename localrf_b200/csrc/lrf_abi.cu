// lrf_abi.cu -- the C ABI declared in include/localrf_b200.h (validation + launches).
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "../../include/localrf_b200.h"
#include "lrf_common.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, const char* a = "") {
  snprintf(g_err, sizeof(g_err), fmt, a);
  return code;
}

int cuda_fail(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
  return LRF_ERR_CUDA;
}

// the status an entry point returns for the launch it ends with
int cuda_status(cudaError_t e, const char* where) { return e == cudaSuccess ? LRF_OK : cuda_fail(e, where); }

constexpr int MAX_DEVICES = 64;
constexpr unsigned int SCHED_RING = 256;

// what the launches need of a device, queried once, and its ring of per-launch ray counters
struct DevInfo {
  int n_sms = 0;
  int max_smem = 0;                      // the opt-in limit of dynamic shared memory per block
  int smem_per_sm = 0;                   // shared memory per SM
  int smem_reserved = 0;                 // shared memory the system reserves per block
  bool ok = false;
  unsigned long long* sched = nullptr;   // ring of per-launch ray counters (device memory)
  unsigned int next = 0;                 // the ring's slot lrf_render took last
};

// The shared-memory settings of the kernels that change them (a handful), per device.  An entry's kernel is set once
// and never changes, so a reader that finds its kernel's setting in place needs no lock.
struct KernelSmem {
  std::atomic<const void*> kernel{nullptr};
  std::atomic<int> max_dynamic[MAX_DEVICES] = {};   // the dynamic shared memory the kernel may use
  std::atomic<int> carveout_for[MAX_DEVICES] = {};  // the CTA size its carveout was chosen for (0: none chosen)
};

// Per-device launch state, process-global: each device's record is filled on first use by whichever host thread gets
// there first (the autograd engine's worker threads share it).  g_mu guards g_devices and the writers of g_kernels.
DevInfo g_devices[MAX_DEVICES];
KernelSmem g_kernels[16];
std::mutex g_mu;

// fills the record of device `dev` (in [0, MAX_DEVICES)) on its first use; on failure `where` names the call that
// failed.  Call with g_mu held.
cudaError_t fill_device(int dev, const char*& where) {
  DevInfo& d = g_devices[dev];
  if (d.ok) return cudaSuccess;
  cudaDeviceProp p;
  cudaError_t e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) { where = "cudaGetDeviceProperties"; return e; }
  d.n_sms = p.multiProcessorCount;
  d.max_smem = (int)p.sharedMemPerBlockOptin;
  d.smem_per_sm = (int)p.sharedMemPerMultiprocessor;
  d.smem_reserved = (int)p.reservedSharedMemPerBlock;
  e = cudaMalloc(&d.sched, 2 * SCHED_RING * sizeof(unsigned long long));
  if (e != cudaSuccess) { where = "cudaMalloc(ray counters)"; return e; }
  d.ok = true;
  return cudaSuccess;
}

// the current device's record.  take_slot: advance the ring for the render launch that asks (d.next is then its slot).
int device_info(DevInfo& d, bool take_slot = false) {
  std::lock_guard<std::mutex> lock(g_mu);
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  if (dev < 0 || dev >= MAX_DEVICES) return fail(LRF_ERR_INVALID, "device index out of range");
  const char* where = "";
  if ((e = fill_device(dev, where)) != cudaSuccess) return cuda_fail(e, where);
  if (take_slot) g_devices[dev].next = (g_devices[dev].next + 1) % SCHED_RING;
  d = g_devices[dev];
  return LRF_OK;
}

// the current device's SM count, for the entry points whose launch needs nothing else of the device
int sm_count(int& n_sms) {
  DevInfo d;
  const int rc = device_info(d);
  n_sms = d.n_sms;
  return rc;
}

// the kernel's entry, read without the lock; null when it has none
const KernelSmem* find_kernel(const void* kernel) {
  for (const KernelSmem& t : g_kernels)
    if (t.kernel.load(std::memory_order_acquire) == kernel) return &t;
  return nullptr;
}

// the kernel's entry, claimed on first use; null when the table is full.  Call with g_mu held.
KernelSmem* claim_kernel(const void* kernel) {
  for (KernelSmem& t : g_kernels) {
    const void* k = t.kernel.load(std::memory_order_relaxed);
    if (k == kernel) return &t;
    if (!k) {
      t.kernel.store(kernel, std::memory_order_release);
      return &t;
    }
  }
  return nullptr;
}

}  // namespace

cudaError_t lrf::set_max_dynamic_smem(const void* kernel, int bytes) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= MAX_DEVICES)
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  const KernelSmem* t = find_kernel(kernel);
  if (t && t->max_dynamic[dev].load(std::memory_order_acquire) >= bytes) return cudaSuccess;
  std::lock_guard<std::mutex> lock(g_mu);
  KernelSmem* w = claim_kernel(kernel);
  if (w && w->max_dynamic[dev].load(std::memory_order_relaxed) >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && w) w->max_dynamic[dev].store(bytes, std::memory_order_release);   // unless the table is full
  return e;
}

// The carveout is the smallest step of the SM's shared memory that holds the CTA and the memory reserved per block,
// so the L1 gets the rest; it is the code's choice, not the driver's.  A percentage that is not a step rounds up to
// the next step.
cudaError_t lrf::set_smem_carveout(const void* kernel, int cta_bytes) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= MAX_DEVICES) return cudaSuccess;   // no record of the device: the driver chooses
  const KernelSmem* t = find_kernel(kernel);
  if (t && t->carveout_for[dev].load(std::memory_order_acquire) == cta_bytes) return cudaSuccess;
  std::lock_guard<std::mutex> lock(g_mu);
  KernelSmem* w = claim_kernel(kernel);
  if (w && w->carveout_for[dev].load(std::memory_order_relaxed) == cta_bytes) return cudaSuccess;
  const char* where = "";
  if ((e = fill_device(dev, where)) != cudaSuccess) return e;
  const int per_sm = g_devices[dev].smem_per_sm, reserved = g_devices[dev].smem_reserved;
  static const int steps_kb[] = {0, 8, 16, 32, 64, 100, 132, 164, 196, 228};   // sm_90
  int pct = 100;
  for (int kb : steps_kb)
    if (kb * 1024 >= cta_bytes + reserved && kb * 1024 <= per_sm) { pct = (int)(kb * 1024LL * 100 / per_sm); break; }
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
  if (e == cudaSuccess && w) w->carveout_for[dev].store(cta_bytes, std::memory_order_release);   // unless the table is full
  return e;
}

namespace {

// validates the parts of a field every entry point needs and fills the device-side view
int make_field(const LrfField* f, bool need_mlp, bool need_table, const void* prepared,
               lrf::FieldDev& F, bool allow_pe = false, bool allow_bf16 = false) {
  if (!f) return fail(LRF_ERR_INVALID, "field is NULL");
  if (f->grid_dtype != LRF_GRID_F32 && f->grid_dtype != LRF_GRID_BF16)
    return fail(LRF_ERR_INVALID, "grid_dtype must be LRF_GRID_F32 or LRF_GRID_BF16");
  if (f->grid_dtype == LRF_GRID_BF16 && !allow_bf16)
    return fail(LRF_ERR_UNSUPPORTED, "bf16 grid storage is built for lrf_render (pe = 0), lrf_density_feature and "
                                     "lrf_app_feature only (inference); pass the fp32 parameters here");
  F.grid16 = f->grid_dtype == LRF_GRID_BF16 ? 1 : 0;
  if (f->n_dcomp != lrf::CD || f->n_acomp != lrf::CA)
    return fail(LRF_ERR_UNSUPPORTED, "only density_n_comp=8 / appearance_n_comp=24 per plane are built");
  for (int a = 0; a < 3; ++a) {
    if (f->grid[a] < 2) return fail(LRF_ERR_INVALID, "gridSize must be >= 2 on every axis");
    if (!(f->aabb[3 + a] > f->aabb[a])) return fail(LRF_ERR_INVALID, "aabb max must exceed aabb min");
    F.g[a] = f->grid[a];
    F.amin[a] = f->aabb[a];
    F.ainv[a] = 2.0f / (f->aabb[3 + a] - f->aabb[a]);
  }
  for (int i = 0; i < 3; ++i) {
    if (!f->dplane[i] || !f->dline[i] || !f->aplane[i] || !f->aline[i])
      return fail(LRF_ERR_INVALID, "plane/line pointer is NULL");
    if (((uintptr_t)f->dplane[i] | (uintptr_t)f->dline[i] | (uintptr_t)f->aplane[i] |
         (uintptr_t)f->aline[i]) & 15)
      return fail(LRF_ERR_INVALID, "plane/line pointers must be 16-byte aligned");
    F.dplane[i] = f->dplane[i]; F.dline[i] = f->dline[i];
    F.aplane[i] = f->aplane[i]; F.aline[i] = f->aline[i];
  }
  F.prep = static_cast<const float*>(prepared);
  F.alpha_vol = f->alpha_vol;
  if (f->alpha_vol) {
    for (int a = 0; a < 3; ++a) {
      if (f->alpha_dims[a] < 1) return fail(LRF_ERR_INVALID, "alpha mask dims must be >= 1");
      F.ad[a] = f->alpha_dims[a];
      F.aamin[a] = f->alpha_aabb[a];
      F.aainv[a] = 1.0f / (f->alpha_aabb[3 + a] - f->alpha_aabb[a]) * 2.0f;
    }
  } else {
    for (int a = 0; a < 3; ++a) { F.ad[a] = 1; F.aamin[a] = 0.f; F.aainv[a] = 0.f; }
  }
  F.density_shift = f->density_shift;
  F.distance_scale = f->distance_scale;
  F.weight_thres = f->weight_thres;
  if (f->act != 0 && f->act != 1) return fail(LRF_ERR_INVALID, "act must be 0 (softplus) or 1 (relu)");
  F.act = f->act;
  if (need_mlp) {
    if (f->app_dim != lrf::APP_DIM || f->featureC != lrf::FC)
      return fail(LRF_ERR_UNSUPPORTED, "only app_dim=27 / featureC=128 are built");
    if (f->fea_pe < 0 || f->view_pe < 0) return fail(LRF_ERR_INVALID, "fea_pe / view_pe must be >= 0");
    if ((f->fea_pe != 0 || f->view_pe != 0) && !allow_pe)
      return fail(LRF_ERR_UNSUPPORTED, "positional encodings (fea_pe/view_pe > 0) are built for lrf_render only");
    if (f->fea_pe > lrf::PE_MAX_FEA || f->view_pe > lrf::PE_MAX_VIEW)
      return fail(LRF_ERR_UNSUPPORTED, "fea_pe / view_pe above 8 are not built");
  }
  F.fea_pe = need_mlp ? f->fea_pe : 0;
  F.view_pe = need_mlp ? f->view_pe : 0;
  F.w3 = f->w3;
  F.z = f->z_vals;
  F.S = f->n_samples;
  if (need_table) {
    if (!f->z_vals) return fail(LRF_ERR_INVALID, "z_vals is NULL");
    if (f->n_samples < 2 || f->n_samples > 65535)
      return fail(LRF_ERR_INVALID, "n_samples must be in [2, 65535]");
  }
  return LRF_OK;
}

// n_rays >= 1 (>= 0 with allow_empty) rays split evenly into n_views >= 1 views
bool views_ok(long long n_rays, long long n_views, bool allow_empty) {
  return n_rays >= (allow_empty ? 0 : 1) && n_views >= 1 && n_rays % n_views == 0;
}

int check_views(long long n_rays, long long n_views, bool allow_empty) {
  if (views_ok(n_rays, n_views, allow_empty)) return LRF_OK;
  return fail(LRF_ERR_INVALID, allow_empty ? "n_rays must be a multiple of n_views >= 1"
                                           : "n_rays must be a positive multiple of n_views");
}

// a count of items the kernels index with 32-bit integers: [0, 2^31)
bool count_ok(int64_t n) { return n >= 0 && n <= 2147483647LL; }

// the ray count of a kernel that indexes rays with 32-bit integers (the callers have refused negative counts)
int check_31_bits(long long n_rays) {
  return count_ok(n_rays) ? LRF_OK : fail(LRF_ERR_INVALID, "n_rays must fit 31 bits");
}

// validates a batch of n_rays >= 1 -- its split into views when `per_view`, n_rays < 2^31 when `fit_31`, and in
// ray-generation mode (rays == NULL) its camera -- and fills the batch fields the render and its backward both read
int make_batch(const LrfBatch* b, bool per_view, bool fit_31, lrf::BatchDev& B) {
  memset(&B, 0, sizeof(B));
  int rc;
  if (per_view) {
    if ((rc = check_views(b->n_rays, b->n_views, false)) != LRF_OK) return rc;
    B.rays_per_view = b->n_rays / b->n_views;
  }
  if (fit_31 && (rc = check_31_bits(b->n_rays)) != LRF_OK) return rc;
  if (!b->rays) {
    if (!b->ray_ids || !b->cam2world) return fail(LRF_ERR_INVALID, "ray_ids/cam2world is NULL");
    if (b->W < 1 || b->H < 1) return fail(LRF_ERR_INVALID, "W/H must be positive");
    if (!b->fov360 && !b->intrinsics && !(b->focal != 0.0f))
      return fail(LRF_ERR_INVALID, "focal must be non-zero");
  }
  B.n_rays = b->n_rays;
  B.rays = b->rays;
  B.ray_ids = reinterpret_cast<const long long*>(b->ray_ids);
  B.W = b->W; B.H = b->H; B.fov360 = b->fov360;
  B.focal = b->focal; B.cx = b->cx; B.cy = b->cy;
  B.intrinsics = b->intrinsics;
  B.c2w = b->cam2world;
  B.w2rf = b->world2rf;
  B.exposure = b->exposure;
  B.white_bg = b->white_bg;
  return LRF_OK;
}

// the field's gradient buffers of lrf_render_backward (d_rays too) and lrf_render_backward_batch
int check_field_grads(const LrfGradients* g, bool need_d_rays) {
  if ((need_d_rays && !g->d_rays) || !g->d_w1b || !g->d_b1 || !g->d_w2 || !g->d_b2 || !g->d_w3 || !g->d_b3)
    return fail(LRF_ERR_INVALID, "gradient buffer is NULL");
  for (int i = 0; i < 3; ++i) {
    if (!g->d_dplane[i] || !g->d_dline[i] || !g->d_aplane[i] || !g->d_aline[i])
      return fail(LRF_ERR_INVALID, "gradient buffer is NULL");
    if (((uintptr_t)g->d_dplane[i] | (uintptr_t)g->d_dline[i] | (uintptr_t)g->d_aplane[i] |
         (uintptr_t)g->d_aline[i]) & 15)
      return fail(LRF_ERR_INVALID, "plane/line gradient buffers must be 16-byte aligned");
  }
  return LRF_OK;
}

// the MLP block lrf_field_prepare (allow_pe: fea_pe / view_pe up to 8) and lrf_field_prepare_backward (none) fold
int check_mlp_block(const LrfField* f, bool allow_pe) {
  if (f->app_dim != lrf::APP_DIM || f->featureC != lrf::FC || f->n_acomp != lrf::CA)
    return fail(LRF_ERR_UNSUPPORTED, "only app_dim=27 / featureC=128 / appearance_n_comp=24 are built");
  if (allow_pe && (f->fea_pe < 0 || f->view_pe < 0 || f->fea_pe > lrf::PE_MAX_FEA || f->view_pe > lrf::PE_MAX_VIEW))
    return fail(LRF_ERR_UNSUPPORTED, "fea_pe / view_pe must be in [0, 8]");
  if (!allow_pe && (f->fea_pe != 0 || f->view_pe != 0))
    return fail(LRF_ERR_UNSUPPORTED, "positional encodings (fea_pe/view_pe > 0) are not built yet");
  if (!f->basis || !f->w1 || !f->b1 || !f->w2 || !f->b2 || !f->w3 || !f->b3)
    return fail(LRF_ERR_INVALID, "MLP / basis pointer is NULL");
  return LRF_OK;
}

// a caller's scratch block: non-NULL, `align`-byte aligned (8 or 16) and at least `need` bytes
int check_scratch(const void* scratch, size_t bytes, size_t need, int align, const char* too_small) {
  if (!scratch || ((uintptr_t)scratch & (align - 1)))
    return fail(LRF_ERR_INVALID, "scratch is NULL or not %s-byte aligned", align == 16 ? "16" : "8");
  if (bytes < need) return fail(LRF_ERR_INVALID, "%s", too_small);
  return LRF_OK;
}

// how many of the flow group's four pointers (fwd_flow, fwd_mask, bwd_flow, bwd_mask) are set
template <typename T>
int flow_count(const T& x) {
  return !!x.fwd_flow + !!x.fwd_mask + !!x.bwd_flow + !!x.bwd_mask;
}

// the frame store of lrf_gather_rays and lrf_ingest_frame; n_flow: 4 when it holds the flow group, else 0
int check_store(const LrfFrameStore* s, int& n_flow) {
  if (s->n_px < 1) return fail(LRF_ERR_INVALID, "n_px must be >= 1");
  if (s->capacity < 1) return fail(LRF_ERR_INVALID, "capacity must be >= 1");
  if (!s->slot_frame || !s->rgb || !s->loss_weight)
    return fail(LRF_ERR_INVALID, "slot_frame / rgb / loss_weight of the store is NULL");
  n_flow = flow_count(*s);
  if (n_flow != 0 && n_flow != 4)
    return fail(LRF_ERR_INVALID, "the store's flow group is partly given: set all of fwd_flow, fwd_mask, bwd_flow, "
                                 "bwd_mask or none");
  return LRF_OK;
}

// the plane / line gradient buffers of the lookups' backward and lrf_density_l1_backward; `aligned16`: the lookups'
// backward adds into them with 16-byte vector atomics (lrf_density_l1_backward's scalar adds need float alignment only)
int check_grads(float* const d_plane[3], float* const d_line[3], bool aligned16) {
  if (!d_plane || !d_line) return fail(LRF_ERR_INVALID, "gradient pointer arrays are NULL");
  for (int i = 0; i < 3; ++i) {
    if (!d_plane[i] || !d_line[i]) return fail(LRF_ERR_INVALID, "gradient buffer is NULL");
    if (aligned16 && (((uintptr_t)d_plane[i] | (uintptr_t)d_line[i]) & 15))
      return fail(LRF_ERR_INVALID, "plane/line gradient buffers must be 16-byte aligned");
  }
  return LRF_OK;
}

// the batch and scratch block of lrf_supervision_losses and its backward
int check_loss_batch(const LrfLossBatch* b, const void* scratch, size_t scratch_bytes) {
  if (!b) return fail(LRF_ERR_INVALID, "batch is NULL");
  const int rc = check_views(b->n_rays, b->n_views, false);
  if (rc != LRF_OK) return rc;
  if (b->n_cams < 1) return fail(LRF_ERR_INVALID, "n_cams must be >= 1");
  if (!b->rgb_map || !b->rgb_train || !b->loss_weights)
    return fail(LRF_ERR_INVALID, "rgb_map / rgb_train / loss_weights is NULL");
  if (b->use_flow && (!b->view_ids || !b->depth_map || !b->directions || !b->ij || !b->cam2world || !b->focal ||
                      !b->center || !b->fwd_flow || !b->bwd_flow || !b->fwd_mask || !b->bwd_mask))
    return fail(LRF_ERR_INVALID, "a pointer of the flow term is NULL");
  if (b->use_depth && (!b->depth_map || !b->invdepths))
    return fail(LRF_ERR_INVALID, "a pointer of the depth term is NULL");
  if (b->n_rays / b->n_views > 4096) return fail(LRF_ERR_UNSUPPORTED, "more than 4096 rays per view");
  return check_scratch(scratch, scratch_bytes, lrf::losses_scratch_bytes(b->n_rays, b->n_views), 8,
                       "scratch_bytes is smaller than lrf_supervision_scratch_bytes(n_rays, n_views, n_cams)");
}

// the capacity of an export's open-addressing table (lrf_table.cuh): a power of two in [2, 2^30]
bool table_capacity_ok(int64_t capacity) {
  return capacity >= 2 && capacity <= (1LL << 30) && !(capacity & (capacity - 1));
}

int check_capacity(int64_t capacity) {
  return table_capacity_ok(capacity) ? LRF_OK : fail(LRF_ERR_INVALID, "capacity must be a power of two in [2, 2^30]");
}

// the origin of an export's lattice or cell grid
int check_origin(const float origin[3]) {
  if (!std::isfinite(origin[0]) || !std::isfinite(origin[1]) || !std::isfinite(origin[2]))
    return fail(LRF_ERR_INVALID, "origin must be finite");
  return LRF_OK;
}

// an extract's scratch block: non-NULL and 256-byte aligned, at least its buffers (known without a device), then at
// least the whole block (the sort-size query needs a device); `where` names a failed query
int check_extract_scratch(const void* scratch, size_t bytes, const lrf::ExtractScratch& x, const char* where,
                          const char* too_small) {
  if (!scratch || ((uintptr_t)scratch & 255)) return fail(LRF_ERR_INVALID, "scratch is NULL or not 256-byte aligned");
  size_t need = 0;
  x.bytes(need, false);
  if (bytes < need) return fail(LRF_ERR_INVALID, "%s", too_small);
  const cudaError_t e = x.bytes(need, true);
  if (e != cudaSuccess) return cuda_fail(e, where);
  if (bytes < need) return fail(LRF_ERR_INVALID, "%s", too_small);
  return LRF_OK;
}

// the voxel table of lrf_frame_points and lrf_voxel_extract
int check_voxel_table(const LrfVoxelTable* t) {
  if (!t) return fail(LRF_ERR_INVALID, "table is NULL");
  int rc = check_capacity(t->capacity);
  if (rc != LRF_OK) return rc;
  if (!(t->voxel_size > 0.0f) || !std::isfinite(t->voxel_size)) return fail(LRF_ERR_INVALID, "voxel_size must be > 0 and finite");
  if ((rc = check_origin(t->origin)) != LRF_OK) return rc;
  if (!t->keys || !t->sums || !t->stats) return fail(LRF_ERR_INVALID, "keys / sums / stats of the table is NULL");
  if (((uintptr_t)t->keys | (uintptr_t)t->sums | (uintptr_t)t->stats) & 7)
    return fail(LRF_ERR_INVALID, "keys / sums / stats of the table must be 8-byte aligned");
  return LRF_OK;
}

static_assert(LRF_MESH_MAX_FIELDS == lrf::MESH_MAX_FIELDS, "the header's field limit is the kernels'");

bool positive_finite(float x) { return x > 0.0f && std::isfinite(x); }

// the scene of the lrf_mesh_* entry points -> its device view
int make_mesh_scene(const LrfMeshScene* s, lrf::MeshSceneDev& S) {
  if (!s) return fail(LRF_ERR_INVALID, "scene is NULL");
  if (s->n_fields < 1 || s->n_fields > LRF_MESH_MAX_FIELDS)
    return fail(LRF_ERR_INVALID, "n_fields must be in [1, LRF_MESH_MAX_FIELDS]");
  if (!s->fields || !s->step_size || !s->world2rf)
    return fail(LRF_ERR_INVALID, "fields / step_size / world2rf of the scene is NULL");
  if (!positive_finite(s->voxel_size)) return fail(LRF_ERR_INVALID, "voxel_size must be > 0 and finite");
  if (!positive_finite(s->max_norm)) return fail(LRF_ERR_INVALID, "max_norm must be > 0 and finite");
  if (!positive_finite(s->level)) return fail(LRF_ERR_INVALID, "level must be > 0 and finite");
  int rc = check_origin(s->origin);
  if (rc != LRF_OK) return rc;
  for (int k = 0; k < s->n_fields; ++k) {
    if ((rc = make_field(s->fields + k, false, false, nullptr, S.f[k])) != LRF_OK) return rc;
    if (!positive_finite(s->step_size[k])) return fail(LRF_ERR_INVALID, "step_size must be > 0 and finite");
    S.length[k] = s->step_size[k];
  }
  S.w2rf = s->world2rf;
  S.n_fields = s->n_fields;
  S.voxel = s->voxel_size;
  for (int a = 0; a < 3; ++a) S.origin[a] = s->origin[a];
  S.max_norm = s->max_norm;
  S.level = s->level;
  return LRF_OK;
}

// a brick of lrf_mesh_lattice / lrf_mesh_cells: dims >= 2 points per axis, fewer than 2^31 points, every point's
// index in [-2^19, 2^19)
int check_brick(const int32_t lo[3], const int32_t dims[3]) {
  if (!lo || !dims) return fail(LRF_ERR_INVALID, "lo / dims is NULL");
  for (int a = 0; a < 3; ++a) {
    if (dims[a] < 2) return fail(LRF_ERR_INVALID, "a brick needs dims >= 2 on every axis");
    if (lo[a] < -(1 << 19) || (int64_t)lo[a] + dims[a] > (1 << 19))
      return fail(LRF_ERR_INVALID, "the brick's lattice indices must lie in [-2^19, 2^19)");
  }
  if ((int64_t)dims[0] * dims[1] * dims[2] > 2147483647LL) return fail(LRF_ERR_INVALID, "a brick must hold < 2^31 points");
  return LRF_OK;
}

// the edge and triangle table of lrf_mesh_cells and lrf_mesh_extract
int check_mesh_table(const LrfMeshTable* t) {
  if (!t) return fail(LRF_ERR_INVALID, "table is NULL");
  const int rc = check_capacity(t->capacity);
  if (rc != LRF_OK) return rc;
  if (t->max_triangles < 1 || t->max_triangles > 2147483647LL)
    return fail(LRF_ERR_INVALID, "max_triangles must be in [1, 2^31)");
  if (!t->keys || !t->verts || !t->tri_keys || !t->tri_slots || !t->stats)
    return fail(LRF_ERR_INVALID, "keys / verts / tri_keys / tri_slots / stats of the table is NULL");
  if ((((uintptr_t)t->keys | (uintptr_t)t->tri_keys | (uintptr_t)t->stats) & 7) ||
      (((uintptr_t)t->verts | (uintptr_t)t->tri_slots) & 3))
    return fail(LRF_ERR_INVALID, "the table's 64-bit arrays must be 8-byte and its 32-bit arrays 4-byte aligned");
  return LRF_OK;
}

// the panel size of lrf_test_panels: two W x H panels index with 32-bit integers
bool panel_size_ok(int32_t W, int32_t H) {
  return W >= 1 && H >= 1 && 2 * (int64_t)W * H <= 2147483647LL;
}

// a plane of ws x hs with `per_px` values per pixel and a row stride of `stride` elements
int check_plane(const void* p, int32_t ws, int32_t hs, int64_t stride, int per_px, const char* name) {
  if (!p) return fail(LRF_ERR_INVALID, "%s is NULL", name);
  if (ws < 1 || hs < 1) return fail(LRF_ERR_INVALID, "the %s plane's sizes must be >= 1", name);
  if (stride < (int64_t)per_px * ws) return fail(LRF_ERR_INVALID, "the %s plane's row stride is shorter than a row", name);
  return LRF_OK;
}

// the fused pixel exchange fields of lrf_render's outputs, for every batch: an empty one still publishes its step
int check_exchange(const LrfOutputs* o) {
  if (o->n_peers < 0 || o->n_peers > LRF_MAX_PEERS) return fail(LRF_ERR_INVALID, "n_peers out of range");
  if (o->n_peers > 0) {
    if (!o->pix) return fail(LRF_ERR_INVALID, "the fused pixel exchange needs the interleaved `pix` output");
    if (o->mc_pix) {
      if ((uintptr_t)o->mc_pix & 15) return fail(LRF_ERR_INVALID, "mc_pix must be 16-byte aligned");
    } else {
      for (int p = 0; p < o->n_peers; ++p)
        if (!o->peer_pix[p] || ((uintptr_t)o->peer_pix[p] & 15))
          return fail(LRF_ERR_INVALID, "peer_pix pointers must be non-NULL and 16-byte aligned");
    }
  }
  if (o->signal_seq) {
    if (o->n_peers < 1 || o->rank < 0 || o->rank >= o->n_peers || o->wait_seq > o->signal_seq)
      return fail(LRF_ERR_INVALID, "in-kernel signalling needs n_peers >= 1, 0 <= rank < n_peers, wait_seq <= signal_seq");
    for (int p = 0; p < o->n_peers; ++p)
      if (!o->peer_flags[p] || ((uintptr_t)o->peer_flags[p] & 7))
        return fail(LRF_ERR_INVALID, "peer_flags pointers must be non-NULL and 8-byte aligned");
  }
  return LRF_OK;
}

// the label and size outputs of lrf_mesh_components / lrf_point_components and their stats
int check_component_outputs(int64_t n, const int32_t* label, const int64_t* size, const int64_t* stats) {
  if (n > 0 && (!label || !size)) return fail(LRF_ERR_INVALID, "label / size is NULL");
  if (!stats) return fail(LRF_ERR_INVALID, "stats is NULL");
  if (((uintptr_t)label & 3) || (((uintptr_t)size | (uintptr_t)stats) & 7))
    return fail(LRF_ERR_INVALID, "label must be 4-byte and size / stats 8-byte aligned");
  return LRF_OK;
}

}  // namespace

extern "C" {

int lrf_version(void) { return 4; }

size_t lrf_sizeof(int32_t which) {
  switch (which) {
    case 0: return sizeof(LrfField);
    case 1: return sizeof(LrfBatch);
    case 2: return sizeof(LrfOutputs);
    case 3: return sizeof(LrfGradients);
    case 4: return sizeof(LrfLossBatch);
    case 5: return sizeof(LrfLossGrads);
    case 6: return sizeof(LrfAdamTensor);
    case 7: return sizeof(LrfCameraGrads);
    case 8: return sizeof(LrfFrameStore);
    case 9: return sizeof(LrfRayGather);
    case 10: return sizeof(LrfPanelFrame);
    case 11: return sizeof(LrfIngestFrame);
    case 12: return sizeof(LrfPointFrame);
    case 13: return sizeof(LrfVoxelTable);
    case 14: return sizeof(LrfMeshScene);
    case 15: return sizeof(LrfMeshTable);
    case 17: return sizeof(LrfColourFrame);
    default: return 0;
  }
}

const char* lrf_last_error(void) { return g_err; }

size_t lrf_prepared_bytes(void) { return (size_t)lrf::PREP_BYTES; }

size_t lrf_prepared_bytes_for(const LrfField* f) {
  if (!f || f->fea_pe < 0 || f->view_pe < 0 || f->fea_pe > lrf::PE_MAX_FEA || f->view_pe > lrf::PE_MAX_VIEW) return 0;
  if (f->fea_pe == 0 && f->view_pe == 0) return (size_t)lrf::PREP_BYTES;
  return (size_t)lrf::pe_prepared_bytes(f->fea_pe);
}

int lrf_field_prepare(const LrfField* f, void* prepared, lrf_stream_t stream) {
  if (!f || !prepared) return fail(LRF_ERR_INVALID, "field or prepared is NULL");
  if ((uintptr_t)prepared & 15) return fail(LRF_ERR_INVALID, "prepared must be 16-byte aligned");
  const int rc = check_mlp_block(f, /*allow_pe=*/true);
  if (rc != LRF_OK) return rc;
  if (f->fea_pe != 0 || f->view_pe != 0) {
    if ((uintptr_t)prepared & 1023) return fail(LRF_ERR_INVALID, "the prepared block of a field with positional encodings must be 1024-byte aligned");
    return cuda_status(lrf::launch_prepare_pe(f->basis, f->w1, f->b1, f->w2, f->b2, f->w3, f->b3, f->fea_pe, f->view_pe,
                                              static_cast<unsigned char*>(prepared),
                                              (cudaStream_t)stream), "prepare_pe_kernel");
  }
  return cuda_status(lrf::launch_prepare(f->basis, f->w1, f->b1, f->w2, f->b2, f->w3, f->b3,
                                         static_cast<unsigned char*>(prepared),
                                         (cudaStream_t)stream), "prepare_kernel");
}

int lrf_render(const LrfField* f, const void* prepared, const LrfBatch* b, const LrfOutputs* o,
               lrf_stream_t stream) {
  if (!b || !o) return fail(LRF_ERR_INVALID, "batch or outputs is NULL");
  if (!prepared) return fail(LRF_ERR_INVALID, "prepared is NULL (call lrf_field_prepare first)");
  lrf::FieldDev F;
  int rc = make_field(f, true, true, prepared, F, /*allow_pe=*/true, /*allow_bf16=*/true);
  if (rc != LRF_OK) return rc;
  if ((F.fea_pe || F.view_pe) && (!f->w3 || ((uintptr_t)prepared & 1023)))
    return fail(LRF_ERR_INVALID, "positional encodings need w3 and a 1024-byte aligned prepared block");
  if ((F.fea_pe || F.view_pe) && F.grid16)
    return fail(LRF_ERR_UNSUPPORTED, "bf16 grid storage is built for fields without positional encodings");
  if (b->n_rays < 0) return fail(LRF_ERR_INVALID, "n_rays < 0");
  if ((rc = check_exchange(o)) != LRF_OK) return rc;
  if (b->n_rays == 0) {
    // nothing to render; a rank with an empty shard must still publish its step to the peers (and waits for none)
    if (!o->signal_seq) return LRF_OK;
    return cuda_status(lrf::launch_peer_barrier(o->peer_flags, o->rank, o->n_peers, o->signal_seq, 0ull,
                                                (cudaStream_t)stream), "peer_barrier_kernel");
  }
  if (!o->pix && (!o->rgb || !o->depth)) return fail(LRF_ERR_INVALID, "rgb/depth output is NULL");
  lrf::BatchDev B;
  rc = make_batch(b, b->blend || b->exposure || !b->rays, /*fit_31=*/false, B);
  if (rc != LRF_OK) return rc;
  B.blend = b->blend;
  B.blend_stride = b->blend_stride;
  B.accumulate = b->accumulate; B.finalize = b->finalize;
  B.floater_thresh = b->floater_thresh;
  B.refine = b->refine;
  if (o->pix) {
    B.rgb = o->pix; B.depth = o->pix + 3; B.rgb_stride = 4; B.depth_stride = 4;
  } else {
    B.rgb = o->rgb; B.depth = o->depth; B.rgb_stride = 3; B.depth_stride = 1;
  }
  B.weights = o->weights;
  B.dirs = b->rays ? nullptr : o->directions;
  B.ij = b->rays ? nullptr : reinterpret_cast<long long*>(o->ij);
  B.stats = o->stats;
  B.n_peers = o->n_peers;                                            // (checked by check_exchange above)
  B.mc_pix = nullptr;
  if (o->n_peers > 0) {
    if (o->mc_pix) B.mc_pix = o->mc_pix;
    else
      for (int p = 0; p < o->n_peers; ++p) B.peer_pix[p] = o->peer_pix[p];
  }
  B.signal_seq = 0; B.wait_seq = 0; B.rank = 0;
  if (o->signal_seq) {
    for (int p = 0; p < o->n_peers; ++p) B.peer_flags[p] = o->peer_flags[p];
    B.signal_seq = o->signal_seq; B.wait_seq = o->wait_seq; B.rank = o->rank;
  }
  DevInfo d;
  rc = device_info(d, /*take_slot=*/true);
  if (rc != LRF_OK) return rc;
  const size_t smem = lrf::render_smem_bytes(F.S, B.floater_thresh > 0.0f, d.max_smem, F.fea_pe > 0 || F.view_pe > 0);
  if ((long long)smem > d.max_smem)
    return fail(LRF_ERR_UNSUPPORTED, "sample table too long for the shared-memory budget");
  B.sched = d.sched + 2 * d.next;                                   // [ray counter, finished-CTA counter]
  B.done_ctr = reinterpret_cast<unsigned int*>(d.sched + 2 * d.next + 1);
  return cuda_status(lrf::launch_render(F, B, d.n_sms, d.max_smem, (cudaStream_t)stream), "render_kernel");
}

int lrf_mlp_forward(const void* prepared, const float* feats, const float* viewdirs, int64_t M,
                    float* rgb, lrf_stream_t stream) {
  if (!prepared) return fail(LRF_ERR_INVALID, "prepared is NULL (call lrf_field_prepare first)");
  if ((uintptr_t)prepared & 15) return fail(LRF_ERR_INVALID, "prepared must be 16-byte aligned");
  if (M < 0 || (M > 0 && (!feats || !viewdirs || !rgb))) return fail(LRF_ERR_INVALID, "bad feats/viewdirs/rgb/M");
  if (M == 0) return LRF_OK;
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_mlp(static_cast<const float*>(prepared), feats, viewdirs, M, rgb,
                                     n_sms, (cudaStream_t)stream), "mlp_kernel");
}

int lrf_density_feature(const LrfField* f, const float* xyz, int64_t M, float* out,
                        lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F, false, /*allow_bf16=*/true);
  if (rc != LRF_OK) return rc;
  if (M < 0 || (M > 0 && (!xyz || !out))) return fail(LRF_ERR_INVALID, "bad xyz/out/M");
  return cuda_status(lrf::launch_density_feature(F, xyz, M, out, (cudaStream_t)stream), "density_feature_kernel");
}

int lrf_app_feature(const LrfField* f, const float* xyz, int64_t M, float* out,
                    lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F, false, /*allow_bf16=*/true);
  if (rc != LRF_OK) return rc;
  if (f->app_dim != lrf::APP_DIM) return fail(LRF_ERR_UNSUPPORTED, "only app_dim=27 is built");
  if (!f->basis) return fail(LRF_ERR_INVALID, "basis is NULL");
  if (M < 0 || (M > 0 && (!xyz || !out))) return fail(LRF_ERR_INVALID, "bad xyz/out/M");
  return cuda_status(lrf::launch_app_feature(F, f->basis, xyz, M, out, (cudaStream_t)stream), "app_feature_kernel");
}

int lrf_app_products(const LrfField* f, const float* xyz, int64_t M, float* out,
                     lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (M < 0 || (M > 0 && (!xyz || !out))) return fail(LRF_ERR_INVALID, "bad xyz/out/M");
  if ((uintptr_t)out & 15) return fail(LRF_ERR_INVALID, "out must be 16-byte aligned");
  return cuda_status(lrf::launch_app_products(F, xyz, M, out, (cudaStream_t)stream), "app_products_kernel");
}

int lrf_density_feature_backward(const LrfField* f, const float* xyz, const float* gout, int64_t M,
                                 float* const d_plane[3], float* const d_line[3], float* d_xyz,
                                 lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if ((rc = check_grads(d_plane, d_line, true)) != LRF_OK) return rc;
  if (M < 0 || (M > 0 && (!xyz || !gout))) return fail(LRF_ERR_INVALID, "bad xyz/grad_out/M");
  return cuda_status(lrf::launch_density_backward(F, d_plane, d_line, xyz, gout, M, d_xyz,
                                                  (cudaStream_t)stream), "density_backward_kernel");
}

int lrf_app_products_backward(const LrfField* f, const float* xyz, const float* gout, int64_t M,
                              float* const d_plane[3], float* const d_line[3], float* d_xyz,
                              lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if ((rc = check_grads(d_plane, d_line, true)) != LRF_OK) return rc;
  if (M < 0 || (M > 0 && (!xyz || !gout))) return fail(LRF_ERR_INVALID, "bad xyz/grad_out/M");
  return cuda_status(lrf::launch_app_products_backward(F, d_plane, d_line, xyz, gout, M, d_xyz,
                                                       (cudaStream_t)stream), "app_products_backward_kernel");
}

size_t lrf_prepared_backward_bytes(void) { return lrf::backward_prepared_bytes(); }

size_t lrf_backward_scratch_bytes(int64_t n_rays, int32_t n_samples) {
  if (n_rays < 0 || n_samples < 2) return 0;
  return lrf::backward_scratch_bytes(n_rays, n_samples);
}

int lrf_field_prepare_backward(const LrfField* f, void* prepared_bwd, lrf_stream_t stream) {
  if (!f || !prepared_bwd) return fail(LRF_ERR_INVALID, "field or prepared_bwd is NULL");
  if ((uintptr_t)prepared_bwd & 15) return fail(LRF_ERR_INVALID, "prepared_bwd must be 16-byte aligned");
  const int rc = check_mlp_block(f, /*allow_pe=*/false);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_prepare_backward(f->basis, f->w1, f->b1, f->w2, f->b2, f->w3, f->b3,
                                                  static_cast<float*>(prepared_bwd),
                                                  (cudaStream_t)stream), "prepare_backward_kernel");
}

int lrf_render_backward(const LrfField* f, const void* prepared_bwd, const float* rays,
                        int64_t n_rays, int32_t white_bg, const float* grad_rgb,
                        const float* grad_depth, const LrfGradients* g, void* scratch,
                        size_t scratch_bytes, lrf_stream_t stream) {
  if (!prepared_bwd) return fail(LRF_ERR_INVALID, "prepared_bwd is NULL (call lrf_field_prepare_backward first)");
  lrf::FieldDev F;
  int rc = make_field(f, true, true, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (n_rays < 0) return fail(LRF_ERR_INVALID, "n_rays < 0");
  if (n_rays == 0) return LRF_OK;
  if ((rc = check_31_bits(n_rays)) != LRF_OK) return rc;
  if (!rays || !grad_rgb || !grad_depth || !g) return fail(LRF_ERR_INVALID, "rays / grad_rgb / grad_depth / grads is NULL");
  if ((rc = check_field_grads(g, true)) != LRF_OK) return rc;
  if ((rc = check_scratch(scratch, scratch_bytes, lrf::backward_scratch_bytes(n_rays, F.S), 16,
                          "scratch is smaller than lrf_backward_scratch_bytes(n_rays, n_samples)")) != LRF_OK)
    return rc;
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_render_backward_abi(F, rays, n_rays, white_bg, grad_rgb, grad_depth,
                                                     static_cast<const float*>(prepared_bwd), *g, scratch,
                                                     n_sms, (cudaStream_t)stream), "render_backward");
}

int lrf_exposure_clamp(const float* x, const float* exposure, int64_t n_rays, int64_t n_views, float* rgb,
                       lrf_stream_t stream) {
  int rc = check_views(n_rays, n_views, true);
  if (rc != LRF_OK) return rc;
  if (n_rays > 0 && (!x || !rgb)) return fail(LRF_ERR_INVALID, "rgb_linear / rgb is NULL");
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_exposure_clamp(x, exposure, n_rays, n_views, rgb, n_sms,
                                                (cudaStream_t)stream), "exposure_clamp_kernel");
}

size_t lrf_backward_batch_scratch_bytes(int64_t n_rays, int32_t n_samples, int64_t n_views) {
  if (n_samples < 2 || !views_ok(n_rays, n_views, false)) return 0;
  return lrf::train_backward_scratch_bytes(n_rays, n_samples, n_views);
}

int lrf_render_backward_batch(const LrfField* f, const void* prepared_bwd, const LrfBatch* b, const float* x,
                              const float* grad_rgb, const float* grad_depth, const float* grad_directions,
                              const LrfGradients* g, const LrfCameraGrads* cg, void* scratch, size_t scratch_bytes,
                              lrf_stream_t stream) {
  if (!prepared_bwd) return fail(LRF_ERR_INVALID, "prepared_bwd is NULL (call lrf_field_prepare_backward first)");
  lrf::FieldDev F;
  int rc = make_field(f, true, true, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (!b || !g || !cg) return fail(LRF_ERR_INVALID, "batch / grads / cam_grads is NULL");
  if (b->rays) return fail(LRF_ERR_INVALID, "the batch backward generates its rays: batch->rays must be NULL");
  if (b->accumulate) return fail(LRF_ERR_INVALID, "accumulate is not supported by the batch backward");
  if (b->blend) return fail(LRF_ERR_INVALID, "a blend pointer is not supported by the batch backward");
  lrf::BatchDev B;
  if ((rc = make_batch(b, true, /*fit_31=*/true, B)) != LRF_OK) return rc;
  if (!x || !grad_rgb || !grad_depth) return fail(LRF_ERR_INVALID, "rgb_linear / grad_rgb / grad_depth is NULL");
  if ((rc = check_field_grads(g, false)) != LRF_OK) return rc;
  rc = check_scratch(scratch, scratch_bytes, lrf::train_backward_scratch_bytes(b->n_rays, F.S, b->n_views), 16,
                     "scratch is smaller than lrf_backward_batch_scratch_bytes(n_rays, n_samples, n_views)");
  if (rc != LRF_OK) return rc;
  if (b->floater_thresh > 0.0f) return fail(LRF_ERR_UNSUPPORTED, "the backward is built for floater_thresh = 0");
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_render_backward_batch(F, B, static_cast<const float*>(prepared_bwd), x, grad_rgb,
                                                       grad_depth, grad_directions, *g, *cg, scratch, b->n_views,
                                                       n_sms, (cudaStream_t)stream), "render_backward_batch");
}

int lrf_alpha_mask_build(const LrfField* f, const int32_t dims[3], float length, float thres,
                         float* alpha_scratch, float* mask, unsigned long long* kept, lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (!dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1) return fail(LRF_ERR_INVALID, "lattice dims must be >= 1");
  if (!alpha_scratch) return fail(LRF_ERR_INVALID, "alpha_scratch is NULL");
  if (mask && !kept) return fail(LRF_ERR_INVALID, "kept is NULL");
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  const int dd[3] = {dims[0], dims[1], dims[2]};
  return cuda_status(lrf::launch_alpha_mask_build(F, f->aabb + 3, dd, length, thres, alpha_scratch, mask, kept,
                                                  n_sms, (cudaStream_t)stream), "alpha_mask_build");
}

int lrf_upsample(const float* src, int32_t H, int32_t W, float* dst, int32_t H2, int32_t W2, int32_t C,
                 lrf_stream_t stream) {
  if (!src || !dst || H < 1 || W < 1 || H2 < 1 || W2 < 1 || C < 4 || (C & 3))
    return fail(LRF_ERR_INVALID, "bad upsample arguments (C must be a positive multiple of 4)");
  if (((uintptr_t)src | (uintptr_t)dst) & 15) return fail(LRF_ERR_INVALID, "upsample buffers must be 16-byte aligned");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_upsample(src, H, W, dst, H2, W2, C, n_sms, (cudaStream_t)stream), "upsample_kernel");
}

int lrf_density_l1(const LrfField* f, double* sum, lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (!sum) return fail(LRF_ERR_INVALID, "sum is NULL");
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_density_l1(F, sum, n_sms, (cudaStream_t)stream), "density_l1_fwd_kernel");
}

int lrf_density_l1_backward(const LrfField* f, const float* grad_out, float* const d_plane[3],
                            float* const d_line[3], lrf_stream_t stream) {
  lrf::FieldDev F;
  int rc = make_field(f, false, false, nullptr, F);
  if (rc != LRF_OK) return rc;
  if (!grad_out) return fail(LRF_ERR_INVALID, "grad_out is NULL");
  if ((rc = check_grads(d_plane, d_line, false)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_density_l1_backward(F, grad_out, d_plane, d_line,
                                                     (cudaStream_t)stream), "density_l1_bwd_kernel");
}

int lrf_tv_sums(const float* x, int32_t H, int32_t W, int32_t C, double* sums, lrf_stream_t stream) {
  if (!x || !sums || H < 1 || W < 1 || C < 1) return fail(LRF_ERR_INVALID, "bad tv arguments");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_tv(x, H, W, C, sums, n_sms, (cudaStream_t)stream), "tv_fwd_kernel");
}

int lrf_tv_sums_backward(const float* x, int32_t H, int32_t W, int32_t C, const float* grad_out, float kh,
                         float kw, float* dx, lrf_stream_t stream) {
  if (!x || !dx || !grad_out || H < 1 || W < 1 || C < 1) return fail(LRF_ERR_INVALID, "bad tv arguments");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_tv_backward(x, H, W, C, grad_out, kh, kw, dx, n_sms,
                                             (cudaStream_t)stream), "tv_bwd_kernel");
}

int lrf_sample_ray(const float* rays, const float* jitter, int64_t N, int32_t S, const float aabb[6],
                   float near, float far, float step, float* pts, float* z, unsigned char* inside,
                   lrf_stream_t stream) {
  if (N < 0 || S < 1 || !aabb) return fail(LRF_ERR_INVALID, "bad sample_ray sizes");
  if (N > 0 && (!rays || !pts || !z || !inside)) return fail(LRF_ERR_INVALID, "sample_ray buffer is NULL");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_sample_ray(rays, jitter, N, S, aabb, near, far, step, pts, z, inside, n_sms,
                                            (cudaStream_t)stream), "sample_ray_kernel");
}

int lrf_frame_to_u8(const float* rgb, int32_t rgb_stride, const float* depth, int32_t depth_stride, int64_t N,
                    double d_lo, double d_hi, const unsigned char* lut, unsigned char* rgb8, unsigned char* depth8,
                    lrf_stream_t stream) {
  if (N < 0) return fail(LRF_ERR_INVALID, "N < 0");
  if (rgb8 && (!rgb || rgb_stride < 3)) return fail(LRF_ERR_INVALID, "rgb8 requested without rgb / stride >= 3");
  if (depth8 && (!depth || depth_stride < 1 || !lut)) return fail(LRF_ERR_INVALID, "depth8 requested without depth / lut");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_frame_u8(rgb, rgb_stride, depth, depth_stride, N, d_lo, d_hi, lut, rgb8, depth8,
                                          n_sms, (cudaStream_t)stream), "frame_u8_kernel");
}

size_t lrf_image_metrics_scratch_bytes(int32_t H, int32_t W, int32_t filter_size) {
  if (filter_size < 1 || filter_size > 16 || H < filter_size || W < filter_size) return 0;
  return lrf::metrics_scratch_bytes(H, W);
}

int lrf_image_metrics(const float* img, int32_t img_stride, const float* gt, int32_t gt_stride, int32_t H, int32_t W,
                      double max_val, int32_t filter_size, double filter_sigma, double k1, double k2, double* out,
                      double* ssim_map, void* scratch, size_t scratch_bytes, lrf_stream_t stream) {
  if (!img) return fail(LRF_ERR_INVALID, "img is NULL");
  if (!gt) return fail(LRF_ERR_INVALID, "gt is NULL");
  if (!out) return fail(LRF_ERR_INVALID, "out is NULL");
  if (img_stride < 3) return fail(LRF_ERR_INVALID, "img_stride must be >= 3");
  if (gt_stride < 3) return fail(LRF_ERR_INVALID, "gt_stride must be >= 3");
  if (filter_size < 1 || filter_size > 16) return fail(LRF_ERR_UNSUPPORTED, "filter_size must be in [1, 16]");
  if (H < filter_size || W < filter_size)
    return fail(LRF_ERR_INVALID, "H and W must be >= filter_size (the reference's SSIM map would be empty)");
  const int rc = check_scratch(scratch, scratch_bytes, lrf::metrics_scratch_bytes(H, W), 8,
                               "scratch_bytes is smaller than lrf_image_metrics_scratch_bytes(H, W, filter_size)");
  if (rc != LRF_OK) return rc;
  const double c1 = (k1 * max_val) * (k1 * max_val), c2 = (k2 * max_val) * (k2 * max_val);
  return cuda_status(lrf::launch_image_metrics(img, img_stride, gt, gt_stride, H, W, filter_size, filter_sigma, c1, c2,
                                               out, ssim_map, scratch, (cudaStream_t)stream), "metrics_tile_kernel");
}

size_t lrf_supervision_scratch_bytes(int64_t n_rays, int64_t n_views, int64_t n_cams) {
  if (!views_ok(n_rays, n_views, false) || n_cams < 1) return 0;
  return lrf::losses_scratch_bytes(n_rays, n_views);
}

int lrf_supervision_losses(const LrfLossBatch* b, float* losses, void* scratch, size_t scratch_bytes,
                           lrf_stream_t stream) {
  const int rc = check_loss_batch(b, scratch, scratch_bytes);
  if (rc != LRF_OK) return rc;
  if (!losses) return fail(LRF_ERR_INVALID, "losses is NULL");
  return cuda_status(lrf::launch_supervision_losses(*b, losses, scratch, (cudaStream_t)stream), "supervision_losses");
}

int lrf_supervision_losses_backward(const LrfLossBatch* b, const float* grad_losses, const LrfLossGrads* g,
                                    void* scratch, size_t scratch_bytes, lrf_stream_t stream) {
  const int rc = check_loss_batch(b, scratch, scratch_bytes);
  if (rc != LRF_OK) return rc;
  if (!grad_losses || !g) return fail(LRF_ERR_INVALID, "grad_losses / grads is NULL");
  return cuda_status(lrf::launch_supervision_losses_backward(*b, grad_losses, *g, scratch,
                                                             (cudaStream_t)stream), "supervision_losses_backward");
}

int lrf_adam_step(const LrfAdamTensor* t, int64_t n, lrf_stream_t stream) {
  if (n < 0 || (n > 0 && !t)) return fail(LRF_ERR_INVALID, "bad tensor table / n");
  for (int64_t i = 0; i < n; ++i) {                 // every entry is checked before anything is launched
    if (t[i].numel < 0) return fail(LRF_ERR_INVALID, "a tensor has numel < 0");
    if (t[i].numel > 0 && (!t[i].param || !t[i].grad || !t[i].exp_avg || !t[i].exp_avg_sq))
      return fail(LRF_ERR_INVALID, "param / grad / exp_avg / exp_avg_sq of a tensor with elements is NULL");
  }
  return cuda_status(lrf::launch_adam_step(t, n, (cudaStream_t)stream), "adam_kernel");
}

int lrf_gather_rays(const LrfFrameStore* s, const LrfRayGather* g, lrf_stream_t stream) {
  if (!s || !g) return fail(LRF_ERR_INVALID, "store / gather is NULL");
  int n_flow = 0;
  int rc = check_store(s, n_flow);
  if (rc != LRF_OK) return rc;
  if ((rc = check_views(g->n_rays, g->n_views, true)) != LRF_OK) return rc;
  if ((rc = check_31_bits(g->n_rays)) != LRF_OK) return rc;
  if (!g->ids || !g->idx || !g->rgb || !g->loss_weight)
    return fail(LRF_ERR_INVALID, "ids / idx / rgb / loss_weight of the gather is NULL");
  if (!s->invdepth != !g->invdepth)
    return fail(LRF_ERR_INVALID, "the invdepth output must be set exactly when the store has invdepth");
  if (flow_count(*g) != n_flow)
    return fail(LRF_ERR_INVALID, "the flow outputs must be set exactly when the store has the flow group");
  return cuda_status(lrf::launch_gather_rays(*s, *g, (cudaStream_t)stream), "gather_rays_kernel");
}

int lrf_ray_opacity(const float* weights, int64_t n_rays, int32_t n_samples, int64_t n_views, const float* blend,
                    int64_t blend_stride, int32_t accumulate, float* acc, lrf_stream_t stream) {
  if (!weights || !acc) return fail(LRF_ERR_INVALID, "weights / acc is NULL");
  int rc = check_views(n_rays, n_views, true);
  if (rc != LRF_OK) return rc;
  if ((rc = check_31_bits(n_rays)) != LRF_OK) return rc;
  if (n_samples < 1) return fail(LRF_ERR_INVALID, "n_samples must be >= 1");
  return cuda_status(lrf::launch_ray_opacity(weights, n_rays, n_samples, n_views, blend, blend_stride, accumulate, acc,
                                             (cudaStream_t)stream), "ray_opacity_kernel");
}

int lrf_frame_points(const LrfPointFrame* f, const LrfVoxelTable* t, lrf_stream_t stream) {
  if (!f) return fail(LRF_ERR_INVALID, "frame is NULL");
  int rc = check_voxel_table(t);
  if (rc != LRF_OK) return rc;
  if (!count_ok(f->n_rays)) return fail(LRF_ERR_INVALID, "n_rays must lie in [0, 2^31)");
  if (f->n_fields < 1) return fail(LRF_ERR_INVALID, "n_fields must be >= 1");
  if (!f->rgb || !f->depth || !f->acc || !f->directions || !f->cam2world || !f->world2rf)
    return fail(LRF_ERR_INVALID, "rgb / depth / acc / directions / cam2world / world2rf of the frame is NULL");
  if (std::isnan(f->min_acc) || std::isnan(f->max_norm)) return fail(LRF_ERR_INVALID, "min_acc / max_norm is NaN");
  return cuda_status(lrf::launch_frame_points(*f, *t, (cudaStream_t)stream), "frame_points_kernel");
}

size_t lrf_voxel_extract_scratch_bytes(int64_t capacity) {
  if (!table_capacity_ok(capacity)) return 0;
  size_t bytes = 0;
  return lrf::voxel_extract_scratch(capacity).bytes(bytes, true) == cudaSuccess ? bytes : 0;
}

int lrf_voxel_extract(const LrfVoxelTable* t, int64_t min_count, float* xyz, uint8_t* rgb, int32_t* count,
                      int64_t* n_voxels, void* scratch, size_t scratch_bytes, lrf_stream_t stream) {
  int rc = check_voxel_table(t);
  if (rc != LRF_OK) return rc;
  if (min_count < 1) return fail(LRF_ERR_INVALID, "min_count must be >= 1");
  if (!xyz || !rgb || !count || !n_voxels) return fail(LRF_ERR_INVALID, "xyz / rgb / count / n_voxels is NULL");
  rc = check_extract_scratch(scratch, scratch_bytes, lrf::voxel_extract_scratch(t->capacity),
                             "voxel_extract (sort size)",
                             "scratch_bytes is smaller than lrf_voxel_extract_scratch_bytes(capacity)");
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_voxel_extract(*t, min_count, xyz, rgb, (int*)count, (long long*)n_voxels, scratch,
                                               (cudaStream_t)stream), "voxel_extract");
}

// the point count and sums of lrf_frame_colours and lrf_colour_extract
int check_colour_sums(const unsigned long long* sums, int64_t n) {
  if (!count_ok(n)) return fail(LRF_ERR_INVALID, "n must lie in [0, 2^31)");
  if (!sums || ((uintptr_t)sums & 7)) return fail(LRF_ERR_INVALID, "sums must be non-NULL and 8-byte aligned");
  return LRF_OK;
}

int lrf_frame_colours(const LrfColourFrame* f, const float* xyz, const float* normals, int64_t n,
                      unsigned long long* sums, lrf_stream_t stream) {
  if (!f) return fail(LRF_ERR_INVALID, "frame is NULL");
  int rc = check_colour_sums(sums, n);
  if (rc != LRF_OK) return rc;
  if (!xyz) return fail(LRF_ERR_INVALID, "xyz is NULL");
  if (f->W < 1 || f->H < 1 || (int64_t)f->W * f->H > 2147483647LL)
    return fail(LRF_ERR_INVALID, "W and H must be >= 1 with W H < 2^31");
  if (!f->intrinsics || !f->cam2world || !f->depth || !f->acc || !f->image)
    return fail(LRF_ERR_INVALID, "intrinsics / cam2world / depth / acc / image of the frame is NULL");
  if (std::isnan(f->min_acc)) return fail(LRF_ERR_INVALID, "min_acc is NaN");
  if (!positive_finite(f->depth_tol)) return fail(LRF_ERR_INVALID, "depth_tol must be > 0 and finite");
  if (!(f->min_cos > 0.0f && f->min_cos <= 1.0f)) return fail(LRF_ERR_INVALID, "min_cos must lie in (0, 1]");
  return cuda_status(lrf::launch_frame_colours(*f, xyz, normals, n, sums, (cudaStream_t)stream),
                     "frame_colours_kernel");
}

int lrf_colour_extract(const unsigned long long* sums, int64_t n, uint8_t* rgb, int32_t* count, lrf_stream_t stream) {
  const int rc = check_colour_sums(sums, n);
  if (rc != LRF_OK) return rc;
  if (!rgb || !count) return fail(LRF_ERR_INVALID, "rgb / count is NULL");
  return cuda_status(lrf::launch_colour_extract(sums, n, rgb, (int*)count, (cudaStream_t)stream),
                     "colour_extract_kernel");
}

// (the scene's device view is ~17 KB: static storage per host thread rather than stack)
int lrf_mesh_lattice(const LrfMeshScene* scene, const int32_t lo[3], const int32_t dims[3], float* values,
                     lrf_stream_t stream) {
  static thread_local lrf::MeshSceneDev S;
  int rc = make_mesh_scene(scene, S);
  if (rc != LRF_OK) return rc;
  if ((rc = check_brick(lo, dims)) != LRF_OK) return rc;
  if (!values) return fail(LRF_ERR_INVALID, "values is NULL");
  return cuda_status(lrf::launch_mesh_lattice(S, lo, dims, values, (cudaStream_t)stream), "mesh_lattice_kernel");
}

int lrf_mesh_cells(const LrfMeshScene* scene, const int32_t lo[3], const int32_t dims[3], const float* values,
                   const LrfMeshTable* table, lrf_stream_t stream) {
  static thread_local lrf::MeshSceneDev S;
  int rc = make_mesh_scene(scene, S);
  if (rc != LRF_OK) return rc;
  if ((rc = check_brick(lo, dims)) != LRF_OK) return rc;
  if (!values) return fail(LRF_ERR_INVALID, "values is NULL");
  if ((rc = check_mesh_table(table)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_mesh_cells(S, lo, dims, values, *table, (cudaStream_t)stream), "mesh_cells_kernel");
}

size_t lrf_mesh_extract_scratch_bytes(int64_t capacity, int64_t max_triangles) {
  if (!table_capacity_ok(capacity) || max_triangles < 1 || max_triangles > 2147483647LL) return 0;
  size_t bytes = 0;
  return lrf::mesh_extract_scratch(capacity, max_triangles).bytes(bytes, true) == cudaSuccess ? bytes : 0;
}

int lrf_mesh_extract(const LrfMeshTable* table, float* xyz, int32_t* faces, int64_t* counts, void* scratch,
                     size_t scratch_bytes, lrf_stream_t stream) {
  int rc = check_mesh_table(table);
  if (rc != LRF_OK) return rc;
  if (!xyz || !faces || !counts) return fail(LRF_ERR_INVALID, "xyz / faces / counts is NULL");
  rc = check_extract_scratch(scratch, scratch_bytes, lrf::mesh_extract_scratch(table->capacity, table->max_triangles),
                             "mesh_extract (sort size)",
                             "scratch_bytes is smaller than lrf_mesh_extract_scratch_bytes(capacity, max_triangles)");
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_mesh_extract(*table, xyz, (int*)faces, (long long*)counts, scratch,
                                              (cudaStream_t)stream), "mesh_extract");
}

int lrf_mesh_normals(const LrfMeshScene* scene, const float* xyz, int64_t n, float* normals, int32_t* owner,
                     lrf_stream_t stream) {
  static thread_local lrf::MeshSceneDev S;
  int rc = make_mesh_scene(scene, S);
  if (rc != LRF_OK) return rc;
  if (!count_ok(n)) return fail(LRF_ERR_INVALID, "n must lie in [0, 2^31)");
  if (n > 0 && (!xyz || !normals || !owner)) return fail(LRF_ERR_INVALID, "xyz / normals / owner is NULL");
  return cuda_status(lrf::launch_mesh_normals(S, xyz, n, normals, (int*)owner, (cudaStream_t)stream),
                     "mesh_normals_kernel");
}

int lrf_mesh_components(const int32_t* faces, int64_t n_triangles, int64_t n_vertices, int32_t* label, int64_t* size,
                        int64_t* stats, lrf_stream_t stream) {
  if (!count_ok(n_triangles) || !count_ok(n_vertices))
    return fail(LRF_ERR_INVALID, "n_triangles and n_vertices must lie in [0, 2^31)");
  if (n_triangles > 0 && (!faces || ((uintptr_t)faces & 3)))
    return fail(LRF_ERR_INVALID, "faces must be non-NULL and 4-byte aligned");
  const int rc = check_component_outputs(n_vertices, label, size, stats);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_mesh_components((const int*)faces, n_triangles, n_vertices, (int*)label,
                                                 (unsigned long long*)size, (unsigned long long*)stats,
                                                 (cudaStream_t)stream), "mesh_components");
}

int lrf_point_components(const float* xyz, int64_t n, const float origin[3], float cell_size, unsigned long long* keys,
                         int32_t* first, int64_t capacity, int32_t* label, int64_t* size, int64_t* stats,
                         lrf_stream_t stream) {
  if (!count_ok(n)) return fail(LRF_ERR_INVALID, "n must lie in [0, 2^31)");
  if (n > 0 && (!xyz || ((uintptr_t)xyz & 3))) return fail(LRF_ERR_INVALID, "xyz must be non-NULL and 4-byte aligned");
  if (!origin) return fail(LRF_ERR_INVALID, "origin is NULL");
  int rc = check_origin(origin);
  if (rc != LRF_OK) return rc;
  if (!positive_finite(cell_size)) return fail(LRF_ERR_INVALID, "cell_size must be > 0 and finite");
  if ((rc = check_capacity(capacity)) != LRF_OK) return rc;
  if (!keys || !first || ((uintptr_t)keys & 7) || ((uintptr_t)first & 3))
    return fail(LRF_ERR_INVALID, "keys must be non-NULL and 8-byte aligned, first non-NULL and 4-byte aligned");
  if ((rc = check_component_outputs(n, label, size, stats)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_point_components(xyz, n, origin, cell_size, keys, (int*)first, capacity, (int*)label,
                                                  (unsigned long long*)size, (unsigned long long*)stats,
                                                  (cudaStream_t)stream), "point_components");
}

size_t lrf_components_select_scratch_bytes(int64_t n) {
  size_t bytes = 0;
  return count_ok(n) && lrf::components_select_scratch(n).bytes(bytes, true) == cudaSuccess ? bytes : 0;
}

int lrf_components_select(const int32_t* label, const int64_t* size, int64_t n, int64_t keep, int64_t min_size,
                          int32_t* new_index, int32_t* rank, int64_t* sizes_sorted, int64_t* counts, void* scratch,
                          size_t scratch_bytes, lrf_stream_t stream) {
  if (!count_ok(n)) return fail(LRF_ERR_INVALID, "n must lie in [0, 2^31)");
  if (keep < 0 || min_size < 0) return fail(LRF_ERR_INVALID, "keep and min_size must be >= 0");
  if (!counts || ((uintptr_t)counts & 7)) return fail(LRF_ERR_INVALID, "counts must be non-NULL and 8-byte aligned");
  if (n > 0) {
    if (!label || !size || !new_index || !rank || !sizes_sorted)
      return fail(LRF_ERR_INVALID, "label / size / new_index / rank / sizes_sorted is NULL");
    if ((((uintptr_t)label | (uintptr_t)new_index | (uintptr_t)rank) & 3) ||
        (((uintptr_t)size | (uintptr_t)sizes_sorted) & 7))
      return fail(LRF_ERR_INVALID, "the 32-bit arrays must be 4-byte and the 64-bit arrays 8-byte aligned");
    const int rc = check_extract_scratch(scratch, scratch_bytes, lrf::components_select_scratch(n),
                                         "components_select (sort size)",
                                         "scratch_bytes is smaller than lrf_components_select_scratch_bytes(n)");
    if (rc != LRF_OK) return rc;
  }
  return cuda_status(lrf::launch_components_select((const int*)label, (const long long*)size, n, keep,
                                                   min_size, (int*)new_index, (int*)rank, (long long*)sizes_sorted,
                                                   (long long*)counts, scratch, (cudaStream_t)stream),
                     "components_select");
}

size_t lrf_test_panels_scratch_bytes(int32_t W, int32_t H) {
  return panel_size_ok(W, H) ? lrf::panels_scratch_bytes((long long)W * H) : 0;
}

int lrf_test_panels(const LrfPanelFrame* f, void* scratch, size_t scratch_bytes, lrf_stream_t stream) {
  if (!f) return fail(LRF_ERR_INVALID, "frame is NULL");
  if (!panel_size_ok(f->W, f->H)) return fail(LRF_ERR_INVALID, "W and H must be >= 1 with 2 W H < 2^31");
  if (f->h0 < 1 || f->w0 < 1) return fail(LRF_ERR_INVALID, "h0 and w0 must be >= 1");
  if (f->n_cams < 1) return fail(LRF_ERR_INVALID, "n_cams must be >= 1");
  if (f->idx < 0 || f->idx >= f->n_cams) return fail(LRF_ERR_INVALID, "idx must lie in [0, n_cams)");
  if (!f->depth) return fail(LRF_ERR_INVALID, "depth is NULL");
  const int n_flow = flow_count(*f);
  if (n_flow != 0 && n_flow != 4)
    return fail(LRF_ERR_INVALID, "the flow group is partly given: set all of fwd_flow, fwd_mask, bwd_flow, bwd_mask "
                                 "or none");
  if (n_flow && (!f->directions || !f->cam2world || !f->intrinsics))
    return fail(LRF_ERR_INVALID, "the flow panels need directions, cam2world and intrinsics");
  if (n_flow && (!f->fwd_panel || !f->bwd_panel)) return fail(LRF_ERR_INVALID, "fwd_panel / bwd_panel is NULL");
  if (f->invdepth && !f->depth_panel) return fail(LRF_ERR_INVALID, "depth_panel is NULL");
  int rc = check_scratch(scratch, scratch_bytes, lrf_test_panels_scratch_bytes(f->W, f->H), 8,
                         "scratch_bytes is smaller than lrf_test_panels_scratch_bytes(W, H)");
  if (rc != LRF_OK) return rc;
  int n_sms = 0;
  if ((rc = sm_count(n_sms)) != LRF_OK) return rc;
  return cuda_status(lrf::launch_test_panels(*f, scratch, n_sms, (cudaStream_t)stream), "test_panels");
}

size_t lrf_ingest_scratch_bytes(int64_t n_px) { return n_px >= 1 ? lrf::ingest_scratch_bytes(n_px) : 0; }

int lrf_ingest_frame(const LrfFrameStore* s, const LrfIngestFrame* f, void* scratch, size_t scratch_bytes,
                     lrf_stream_t stream) {
  if (!s || !f) return fail(LRF_ERR_INVALID, "store / frame is NULL");
  int n_flow = 0;
  int rc = check_store(s, n_flow);
  if (rc != LRF_OK) return rc;
  if (f->slot < 0 || f->slot >= s->capacity) return fail(LRF_ERR_INVALID, "slot must lie in [0, capacity)");
  if (f->w < 1 || f->h < 1 || (int64_t)f->w * f->h != s->n_px)
    return fail(LRF_ERR_INVALID, "w and h must be >= 1 with w h == the store's n_px");
  if ((rc = check_plane(f->image, f->w0, f->h0, f->image_stride, 3, "image")) != LRF_OK) return rc;
  if (!s->invdepth != !f->invdepth)
    return fail(LRF_ERR_INVALID, "invdepth must be set exactly when the store has invdepth");
  if (f->invdepth && (rc = check_plane(f->invdepth, f->wd, f->hd, f->invdepth_stride, 1, "invdepth")) != LRF_OK)
    return rc;
  if (!!f->fwd_flow != !!n_flow || !!f->bwd_flow != !!n_flow)
    return fail(LRF_ERR_INVALID, "fwd_flow and bwd_flow must be set exactly when the store has the flow group");
  if (n_flow && ((rc = check_plane(f->fwd_flow, f->wf, f->hf, f->flow_stride, 3, "fwd_flow")) != LRF_OK ||
                 (rc = check_plane(f->bwd_flow, f->wf, f->hf, f->flow_stride, 3, "bwd_flow")) != LRF_OK))
    return rc;
  if (f->mask && (rc = check_plane(f->mask, f->wm, f->hm, f->mask_stride, 1, "mask")) != LRF_OK) return rc;
  const size_t need = lrf_ingest_scratch_bytes(s->n_px);   // 0: too large, refused after the scratch checks
  if ((rc = check_scratch(scratch, scratch_bytes, need, 8,
                          "scratch_bytes is smaller than lrf_ingest_scratch_bytes(n_px)")) != LRF_OK)
    return rc;
  if (need == 0) return fail(LRF_ERR_UNSUPPORTED, "frames above 2^16 leaves of 128 pixels are not built");
  const int image_mode = lrf::ingest_resize_mode(f->w0, f->h0, f->w, f->h);
  if (image_mode < 1)
    return fail(LRF_ERR_UNSUPPORTED, "the image must be w x h or a reduction by 2 or 4 of it (k w x k h)");
  if (f->invdepth && lrf::ingest_resize_mode(f->wd, f->hd, f->w, f->h) < 0)
    return fail(LRF_ERR_UNSUPPORTED, "invdepth must be w x h, a reduction by 2 or 4 of it or at most w x h");
  const int flow_mode = n_flow ? lrf::ingest_resize_mode(f->wf, f->hf, f->w, f->h) : 1;
  if (flow_mode != 0 && flow_mode != 1)
    return fail(LRF_ERR_UNSUPPORTED, "the flows must be w x h or at most w x h on both axes (an enlargement)");
  if (f->mask && (f->wm != f->w || f->hm != f->h)) return fail(LRF_ERR_UNSUPPORTED, "the mask must be w x h");
  return cuda_status(lrf::launch_ingest_frame(*s, *f, scratch, (cudaStream_t)stream), "ingest_frame");
}

int lrf_resize_linear(const float* src, int32_t w0, int32_t h0, int64_t src_stride, float* dst, int32_t W, int32_t H,
                      int64_t dst_stride, lrf_stream_t stream) {
  if (!src || !dst) return fail(LRF_ERR_INVALID, "src / dst is NULL");
  if (w0 < 1 || h0 < 1 || W < 1 || H < 1) return fail(LRF_ERR_INVALID, "w0, h0, W and H must be >= 1");
  if ((int64_t)w0 * h0 >= 2147483648LL || (int64_t)W * H >= 2147483648LL)
    return fail(LRF_ERR_INVALID, "w0 h0 and W H must be below 2^31");
  if (src_stride < 3 * (int64_t)w0) return fail(LRF_ERR_INVALID, "src_stride must be >= 3 w0");
  if (dst_stride < 3 * (int64_t)W) return fail(LRF_ERR_INVALID, "dst_stride must be >= 3 W");
  return cuda_status(lrf::launch_resize_linear(src, w0, h0, src_stride, dst, W, H, dst_stride, (cudaStream_t)stream),
                     "resize_linear_kernel");
}

int lrf_peer_barrier(unsigned long long* const* peer_flags, int32_t rank, int32_t world,
                     unsigned long long seq, lrf_stream_t stream) {
  return lrf_peer_signal_wait(peer_flags, rank, world, seq, seq, stream);
}

int lrf_peer_signal_wait(unsigned long long* const* peer_flags, int32_t rank, int32_t world,
                         unsigned long long seq, unsigned long long wait_seq, lrf_stream_t stream) {
  if (wait_seq > seq) return fail(LRF_ERR_INVALID, "wait_seq must not exceed seq (a rank cannot wait for a step it has not signalled)");
  if (!peer_flags || world < 1 || world > LRF_MAX_PEERS || rank < 0 || rank >= world)
    return fail(LRF_ERR_INVALID, "bad peer_flags / rank / world");
  for (int p = 0; p < world; ++p)
    if (!peer_flags[p] || ((uintptr_t)peer_flags[p] & 7))
      return fail(LRF_ERR_INVALID, "peer flag arrays must be non-NULL and 8-byte aligned");
  return cuda_status(lrf::launch_peer_barrier(peer_flags, rank, world, seq, wait_seq,
                                              (cudaStream_t)stream), "peer_barrier_kernel");
}

int lrf_pack_bf16(const float* src, void* dst, int64_t n, lrf_stream_t stream) {
  if (n < 0 || (n > 0 && (!src || !dst))) return fail(LRF_ERR_INVALID, "bad src/dst/n");
  if ((uintptr_t)dst & 1) return fail(LRF_ERR_INVALID, "dst must be 2-byte aligned");
  int n_sms = 0;
  const int rc = sm_count(n_sms);
  if (rc != LRF_OK) return rc;
  return cuda_status(lrf::launch_pack_bf16(src, dst, n, n_sms, (cudaStream_t)stream), "pack_bf16_kernel");
}

int lrf_repack_nchw_to_nhwc(const float* src, float* dst, int32_t C, int32_t H, int32_t W,
                            lrf_stream_t stream) {
  if (!src || !dst || C < 1 || H < 1 || W < 1) return fail(LRF_ERR_INVALID, "bad repack arguments");
  return cuda_status(lrf::launch_repack(src, dst, C, (long long)H * W, (cudaStream_t)stream), "repack_kernel");
}

int lrf_launch_info(int32_t* n_sms, int32_t* threads_per_cta, int32_t* smem_bytes_per_cta) {
  DevInfo d;
  int rc = device_info(d);
  if (rc != LRF_OK) return rc;
  if (n_sms) *n_sms = d.n_sms;
  if (threads_per_cta) *threads_per_cta = lrf::render_threads();
  if (smem_bytes_per_cta) *smem_bytes_per_cta = (int32_t)lrf::render_smem_bytes(344, false, d.max_smem, false);
  return LRF_OK;
}

}  // extern "C"
