// lrf_launchers.cuh -- the host functions one .cu file defines and another calls: the launchers, the sizes of their
// scratch, prepared and shared-memory blocks, the ingest's resize rule and the extracts' sort.  Each defining file
// includes this header, so the compiler checks every definition against the declaration its callers use.
//
// Declarations, and one small host-side struct (KeySlotSort: the sort's buffer pointers and their accessors); no
// device code.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/localrf_b200.h"

namespace lrf {

struct FieldDev;
struct BatchDev;
struct MeshSceneDev;
struct ScratchCarver;

// lrf_render.cu
int render_threads();
size_t render_smem_bytes(int S, bool floater, int max_smem, bool pe);
cudaError_t launch_render(const FieldDev& F, const BatchDev& B, int n_sms, int max_smem, cudaStream_t stream);

// lrf_aux.cu
cudaError_t launch_prepare(const float* basis, const float* w1, const float* b1, const float* w2, const float* b2,
                           const float* w3, const float* b3, unsigned char* prep, cudaStream_t stream);
cudaError_t launch_prepare_pe(const float* basis, const float* w1, const float* b1, const float* w2, const float* b2,
                              const float* w3, const float* b3, int fea_pe, int view_pe, unsigned char* prep,
                              cudaStream_t stream);
cudaError_t launch_mlp(const float* prep, const float* feats, const float* viewdirs, long long M, float* rgb,
                       int n_sms, cudaStream_t stream);
cudaError_t launch_density_feature(const FieldDev& F, const float* xyz, long long M, float* out, cudaStream_t stream);
cudaError_t launch_app_feature(const FieldDev& F, const float* basis, const float* xyz, long long M, float* out,
                               cudaStream_t stream);
cudaError_t launch_repack(const float* src, float* dst, int C, long long HW, cudaStream_t stream);
cudaError_t launch_pack_bf16(const float* src, void* dst, long long n, int n_sms, cudaStream_t stream);
cudaError_t launch_peer_barrier(unsigned long long* const* peer_flags, int rank, int world, unsigned long long seq,
                                unsigned long long wait_seq, cudaStream_t stream);

// lrf_grad.cu
cudaError_t launch_app_products(const FieldDev& F, const float* xyz, long long M, float* out, cudaStream_t stream);
cudaError_t launch_density_backward(const FieldDev& F, float* const* d_plane, float* const* d_line, const float* xyz,
                                    const float* gout, long long M, float* dxyz, cudaStream_t stream);
cudaError_t launch_app_products_backward(const FieldDev& F, float* const* d_plane, float* const* d_line,
                                         const float* xyz, const float* gout, long long M, float* dxyz,
                                         cudaStream_t stream);

// lrf_backward.cu
size_t backward_prepared_bytes();
size_t backward_scratch_bytes(long long n_rays, int S);
cudaError_t launch_prepare_backward(const float* basis, const float* w1, const float* b1, const float* w2,
                                    const float* b2, const float* w3, const float* b3, float* bp, cudaStream_t stream);
// dpos: null, or [n_rays][S][3] zeroed by the caller, a slot for each shaded sample's colour-branch position gradient
// so that d_rays sums them in a fixed order (null: they are added atomically per ray)
cudaError_t launch_render_backward_abi(const FieldDev& F, const float* rays, long long n_rays, int white_bg,
                                       const float* g_rgb, const float* g_depth, const float* bp,
                                       const LrfGradients& G, void* scratch, int n_sms, cudaStream_t stream,
                                       float* dpos = nullptr);

// lrf_sched.cu
cudaError_t launch_alpha_mask_build(const FieldDev& F, const float* aabb_max, const int* dims, float length,
                                    float thres, float* alpha_scratch, float* mask, unsigned long long* kept,
                                    int n_sms, cudaStream_t stream);
cudaError_t launch_upsample(const float* src, int H, int W, float* dst, int H2, int W2, int C, int n_sms,
                            cudaStream_t stream);
cudaError_t launch_density_l1(const FieldDev& F, double* sum, int n_sms, cudaStream_t stream);
cudaError_t launch_density_l1_backward(const FieldDev& F, const float* gout, float* const* d_plane,
                                       float* const* d_line, cudaStream_t stream);
cudaError_t launch_tv(const float* x, int H, int W, int C, double* sums, int n_sms, cudaStream_t stream);
cudaError_t launch_tv_backward(const float* x, int H, int W, int C, const float* gout, float kh, float kw, float* dx,
                               int n_sms, cudaStream_t stream);
cudaError_t launch_sample_ray(const float* rays, const float* jitter, long long N, int S, const float* aabb,
                              float near, float far, float step, float* pts, float* z, unsigned char* inside,
                              int n_sms, cudaStream_t stream);
cudaError_t launch_frame_u8(const float* rgb, int rgb_stride, const float* depth, int depth_stride, long long N,
                            double d_lo, double d_hi, const unsigned char* lut, unsigned char* rgb8,
                            unsigned char* depth8, int n_sms, cudaStream_t stream);

// lrf_metrics.cu
size_t metrics_scratch_bytes(int H, int W);
cudaError_t launch_image_metrics(const float* img, int img_stride, const float* gt, int gt_stride, int H, int W,
                                 int fs, double sigma, double c1, double c2, double* out, double* ssim_map,
                                 void* scratch, cudaStream_t stream);

// lrf_losses.cu
size_t losses_scratch_bytes(long long N, long long V);
cudaError_t launch_supervision_losses(const LrfLossBatch& b, float* losses, void* scratch, cudaStream_t stream);
cudaError_t launch_supervision_losses_backward(const LrfLossBatch& b, const float* grad_losses, const LrfLossGrads& g,
                                               void* scratch, cudaStream_t stream);

// lrf_optim.cu
cudaError_t launch_adam_step(const LrfAdamTensor* t, long long n, cudaStream_t stream);

// lrf_train.cu
size_t train_backward_scratch_bytes(long long n, int S, long long V);
cudaError_t launch_exposure_clamp(const float* x, const float* E, long long n, long long V, float* rgb, int n_sms,
                                  cudaStream_t stream);
cudaError_t launch_render_backward_batch(const FieldDev& F, const BatchDev& B, const float* bp, const float* x,
                                         const float* g_rgb, const float* g_depth, const float* g_dirs,
                                         const LrfGradients& G, const LrfCameraGrads& CG, void* scratch,
                                         long long n_views, int n_sms, cudaStream_t stream);

// lrf_data.cu
cudaError_t launch_gather_rays(const LrfFrameStore& s, const LrfRayGather& g, cudaStream_t stream);

// lrf_panels.cu
size_t panels_scratch_bytes(long long n_px);
cudaError_t launch_test_panels(const LrfPanelFrame& f, void* scratch, int n_sms, cudaStream_t stream);

// lrf_ingest.cu
size_t ingest_scratch_bytes(long long n_px);
int ingest_resize_mode(int ws, int hs, int w, int h);
cudaError_t launch_ingest_frame(const LrfFrameStore& st, const LrfIngestFrame& f, void* scratch, cudaStream_t stream);
cudaError_t launch_resize_linear(const float* src, int w0, int h0, long long src_stride, float* dst, int W, int H,
                                 long long dst_stride, cudaStream_t stream);

// lrf_table.cu: the extracts' radix sort of n (64-bit key, 32-bit slot) pairs by key, the library's one use of CUB.
// carve() takes two key and two slot buffers of n from a scratch block, in that order; the caller writes the pairs to
// keys() / slots(), and after sort() they hold the sorted pairs.
struct KeySlotSort {
  unsigned long long* key_buf[2] = {};
  unsigned int* slot_buf[2] = {};
  int cur = 0;                                // the buffer of each pair that keys() / slots() return
  unsigned long long* keys() const { return key_buf[cur]; }
  unsigned int* slots() const { return slot_buf[cur]; }
  void carve(ScratchCarver& c, long long n);
  static cudaError_t temp_bytes(long long n, size_t& bytes);   // the sort's temporary storage for n pairs
  cudaError_t sort(long long n, void* temp, size_t temp_bytes, cudaStream_t stream);
};

// lrf_export.cu
cudaError_t launch_ray_opacity(const float* w, long long n, int S, long long n_views, const float* blend,
                               long long blend_stride, int accumulate, float* acc, cudaStream_t stream);
cudaError_t launch_frame_points(const LrfPointFrame& f, const LrfVoxelTable& t, cudaStream_t stream);
cudaError_t voxel_extract_scratch_bytes(long long cap, size_t& bytes);
cudaError_t launch_voxel_extract(const LrfVoxelTable& t, long long min_count, float* xyz, unsigned char* rgb,
                                 int* count, long long* n_out, void* scratch, cudaStream_t stream);
cudaError_t launch_frame_colours(const LrfColourFrame& f, const float* xyz, const float* normals, long long n,
                                 unsigned long long* sums, cudaStream_t stream);
cudaError_t launch_colour_extract(const unsigned long long* sums, long long n, unsigned char* rgb, int* count,
                                  cudaStream_t stream);

// lrf_mesh.cu
cudaError_t launch_mesh_lattice(const MeshSceneDev& S, const int* lo, const int* dims, float* values,
                                cudaStream_t stream);
cudaError_t launch_mesh_cells(const MeshSceneDev& S, const int* lo, const int* dims, const float* values,
                              const LrfMeshTable& t, cudaStream_t stream);
cudaError_t mesh_extract_scratch_bytes(long long cap, long long max_tri, size_t& bytes);
cudaError_t launch_mesh_extract(const LrfMeshTable& t, float* xyz, int* faces, long long* counts, void* scratch,
                                cudaStream_t stream);
cudaError_t launch_mesh_normals(const MeshSceneDev& S, const float* xyz, long long n, float* normals, int* owner,
                                cudaStream_t stream);

}  // namespace lrf
