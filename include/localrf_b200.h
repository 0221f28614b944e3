/*
 * localrf_b200.h -- C ABI of the B200-native render path of localrf.
 *
 * This is the drop-in boundary for the per-ray-batch volume-rendering hot path of
 * facebookresearch/localrf (reference at localTensoRF/, commit 3905e39):
 *
 *     LocalTensorfs.forward      local_tensorfs.py:382-499   (ray generation, per-field render,
 *                                                             blend, exposure, clamp)
 *     TensorBase.forward         models/tensorBase.py:567-636 (sample, contract, density,
 *                                                             alpha/T/weights, floater filter,
 *                                                             appearance, MLP, composite)
 *     compute_densityfeature     models/tensoRF.py:112-151
 *     compute_appfeature         models/tensoRF.py:153-196
 *
 * The reference has no FFI for this path: its "plugin API" is the two nn.Module classes.  The
 * Python mirror of those classes (localrf_b200/tensorf.py, localrf_b200/local_tensorfs.py) binds
 * these entry points through ctypes; INTEGRATION.md shows the stub a maintainer of the reference
 * would add.  Plain pointers and sizes only -- no torch types.
 *
 * All pointers are DEVICE pointers on the current CUDA device unless stated otherwise; all
 * floating-point data is fp32 (the plane / line grids optionally bfloat16, LrfField.grid_dtype); work is
 * enqueued on `stream` and never synchronises the host.
 * Every function returns LRF_OK (0) or a negative error code; lrf_last_error() gives the text.
 *
 * HBM layout of a field ("channel-last", one texel's components contiguous):
 *     plane i : [H_i][W_i][C]     W_i = grid[matMode[i][0]], H_i = grid[matMode[i][1]]
 *     line  i : [L_i][C]          L_i = grid[vecMode[i]]
 *     matMode = {{0,1},{0,2},{1,2}}, vecMode = {2,1,0}          (models/tensorBase.py:274-275)
 * This is exactly the memory of the reference's [1,C,H,W] / [1,C,L,1] parameters when they are
 * allocated with torch.channels_last; lrf_repack_nchw_to_nhwc() converts a contiguous NCHW tensor.
 * C = 8 (density) and 24 (appearance) per plane are the reference defaults (opt.py:117-119) and
 * the only component counts built so far; app_dim = 27, featureC = 128; positional encodings
 * fea_pe / view_pe 0..8 (0, 0 is the reference default and the fastest path; lrf_render only).
 */
#ifndef LOCALRF_B200_H
#define LOCALRF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LRF_OK 0
#define LRF_ERR_INVALID -1      /* bad argument (null pointer, size, unsupported configuration) */
#define LRF_ERR_UNSUPPORTED -2  /* valid reference configuration that this build does not cover */
#define LRF_ERR_CUDA -3         /* a CUDA runtime call failed */

typedef struct CUstream_st *lrf_stream_t; /* == cudaStream_t */

/* One radiance field (TensorVMSplit): the parameters TensorBase.forward reads.
 * replaces: TensorVMSplit attributes, models/tensorBase.py:232-287, models/tensoRF.py:18-50 */
typedef struct LrfField {
  int32_t grid[3];            /* gridSize (x,y,z)                       tensorBase.py:322 */
  float aabb[6];              /* aabb[0] = min xyz, aabb[1] = max xyz   tensorBase.py:259 */
  int32_t n_dcomp;            /* density components per plane (8)       tensorBase.py:256 */
  int32_t n_acomp;            /* appearance components per plane (24)   tensorBase.py:257 */
  const float *dplane[3];     /* [H_i][W_i][n_dcomp] */
  const float *dline[3];      /* [L_i][n_dcomp] */
  const float *aplane[3];     /* [H_i][W_i][n_acomp] */
  const float *aline[3];      /* [L_i][n_acomp] */
  int32_t app_dim;            /* 27 */
  const float *basis;         /* basis_mat.weight [app_dim][3*n_acomp]  tensoRF.py:25-27 */
  int32_t featureC;           /* 128 */
  int32_t fea_pe, view_pe;    /* positional encodings of the MLP inputs (tensorBase.py:14-21,115-125); 0..8 */
  const float *w1, *b1;       /* renderModule.mlp[0]      [featureC][app_dim (1 + 2 fea_pe)], [featureC] */
  const float *w2, *b2;       /* renderModule.mlp[2]      [featureC][featureC], [featureC] */
  const float *w3, *b3;       /* renderModule.mlp_view[0] [3][featureC + 3 (1 + 2 view_pe)], [3] */
  const float *alpha_vol;     /* AlphaGridMask.alpha_volume [D][H][W], or NULL  tensorBase.py:38-62 */
  int32_t alpha_dims[3];      /* D, H, W */
  float alpha_aabb[6];
  float density_shift;        /* tensorBase.py:263 */
  float distance_scale;       /* tensorBase.py:265 */
  float weight_thres;         /* rayMarch_weight_thres, tensorBase.py:266 */
  int32_t act;                /* 0 = softplus, 1 = relu                 tensorBase.py:495-499 */
  const float *z_vals;        /* [n_samples] per-batch distance table (tensorBase.py:419-437);
                                 the host builds it (it owns the RNG of the train-mode jitter) */
  int32_t n_samples;          /* S = 2*(nSamples/6) */
  int32_t grid_dtype;         /* storage type of the twelve plane / line tensors: LRF_GRID_F32 (0, default) or
                                 LRF_GRID_BF16: the dplane/dline/aplane/aline pointers then address bfloat16
                                 data in the SAME [H][W][C] / [L][C] layout (a density texel = one 16-byte
                                 load, an appearance texel three); arithmetic stays fp32 and the conversion
                                 is exact, so a field whose parameters are bf16-representable renders the same
                                 values from either storage.  Inference only: accepted by lrf_render (pe = 0),
                                 lrf_density_feature and lrf_app_feature; every other entry point returns
                                 LRF_ERR_UNSUPPORTED.  lrf_pack_bf16() makes the 16-bit copy. */
} LrfField;
#define LRF_GRID_F32 0
#define LRF_GRID_BF16 1

/* One ray batch.  Either explicit rays (TensorBase.forward's rays_chunk) or ray ids + cameras
 * (LocalTensorfs.forward; the kernel then generates origin/direction itself).
 * replaces: local_tensorfs.py:397-456 (ids2pixel, get_ray_directions_*, cam2rf, get_rays_lean) */
typedef struct LrfBatch {
  int64_t n_rays;
  const float *rays;          /* [n_rays][6] (o, d) or NULL -> generate from the fields below */
  const int64_t *ray_ids;     /* [n_rays]  col = id % W, row = (id / W) % H   local_tensorfs.py:23-29 */
  int32_t W, H;
  int32_t fov360;             /* 1: get_ray_directions_360, 0: get_ray_directions_lean */
  float focal, cx, cy;        /* LocalTensorfs.focal(W), .center(W,H)   local_tensorfs.py:377-380 */
  const float *intrinsics;    /* optional DEVICE [3] = {focal, cx, cy}; overrides the three values
                                 above so learnable intrinsics never round-trip through the host */
  const float *cam2world;     /* [n_views][3][4] */
  int64_t n_views;            /* ray r uses view r / (n_rays / n_views)  local_tensorfs.py:437 */
  const float *world2rf;      /* DEVICE [3] added to the camera translation (NULL = 0)  local_tensorfs.py:428 */
  const float *blend;         /* per-view blending weight of THIS field: blend[v*blend_stride], or
                                 NULL for weight 1                       local_tensorfs.py:438,452 */
  int64_t blend_stride;
  const float *exposure;      /* [n_views][3][3] or NULL; applied when `finalize` local_tensorfs.py:481-496 */
  int32_t accumulate;         /* 0: rgb/depth = w*result; 1: rgb/depth += w*result  (:467-474) */
  int32_t finalize;           /* 1: apply exposure (if any) and clamp(0,1) to rgb   (:481-497) */
  int32_t white_bg;           /* tensorBase.py:633-634 (the caller resolves the train-mode coin) */
  float floater_thresh;       /* tensorBase.py:617-620 */
  int32_t refine;             /* MLPRender_Fea_late_view's `refine` (tensorBase.py:118-124; LocalTensorfs passes
                                 is_refining, local_tensorfs.py:463): 0 = zeros instead of the feature encoding.
                                 Only read when fea_pe > 0. */
} LrfBatch;

typedef struct LrfOutputs {
  float *rgb;                 /* [n_rays][3] */
  float *depth;               /* [n_rays] */
  float *weights;             /* optional [n_rays][n_samples]: final per-sample weights of this field */
  float *directions;          /* optional [n_rays][3]: camera-space directions (ray-generation mode) */
  int64_t *ij;                /* optional [n_rays][2]: pixel (col, row) of every ray id (ray-generation mode) */
  float *pix;                 /* optional [n_rays][4]: when set, rgb and depth are written interleaved
                                 here (r,g,b,depth) instead of to rgb/depth -- the layout the multi-GPU
                                 path all-gathers in one collective */
  unsigned long long *stats;  /* optional [2]: += {density samples marched, appearance samples shaded} */
  /* ---- fused pixel exchange (multi-GPU, SURVEY.md 8e): when n_peers > 0 the thread that finishes a
   * ray on the `finalize` launch ALSO stores its (r,g,b,depth) as one 16-byte word into every
   * peer_pix[p] + 4*ray -- peer-mapped device memory of the other GPUs (NVLink P2P / symmetric
   * memory), each pointer already offset to where THIS rank's rays live in that peer's gathered
   * [total_rays][4] buffer -- so the all-gather of rendered pixels happens inside the render kernel,
   * store by store, instead of as a collective after it.  `pix` must be set (local copy).  If
   * mc_pix is set (NVLS multicast mapping of the same buffer) ONE multimem store reaches all peers
   * and peer_pix is ignored.  lrf_peer_barrier() then closes the step. */
  int32_t n_peers;            /* 0 = no exchange; <= LRF_MAX_PEERS */
  float *peer_pix[16];
  float *mc_pix;
  /* In-kernel step signalling (optional, signal_seq > 0): peer_flags[p] = peer p's [n_peers] uint64 flag
   * array (peer-mapped; peer_flags[rank] is this GPU's own).  Before its first peer store the launch waits
   * until all local flags have reached wait_seq (the peers are done with the buffer about to be overwritten;
   * 0 = no wait); the LAST CTA to finish release-stores signal_seq into slot `rank` of every peer's array,
   * after all pixel stores of the launch.  With wait_seq = signal_seq - lag (lag >= 1) this replaces
   * lrf_peer_signal_wait altogether: a step costs no extra launch.
   * These fields are checked for every batch, n_rays = 0 included (LRF_ERR_INVALID before any device work).  An
   * empty batch stores no pixels; with signal_seq > 0 it publishes the step as above and waits for nothing
   * (wait_seq is checked, not waited on). */
  unsigned long long *peer_flags[16];
  int32_t rank;
  unsigned long long signal_seq, wait_seq;
} LrfOutputs;
#define LRF_MAX_PEERS 16

int lrf_version(void);
const char *lrf_last_error(void);
/* sizeof() of the ABI structs as this library was compiled: 0 LrfField, 1 LrfBatch, 2 LrfOutputs,
 * 3 LrfGradients, 4 LrfLossBatch, 5 LrfLossGrads, 6 LrfAdamTensor, 7 LrfCameraGrads, 8 LrfFrameStore,
 * 9 LrfRayGather, 10 LrfPanelFrame, 11 LrfIngestFrame, 12 LrfPointFrame, 13 LrfVoxelTable, 14 LrfMeshScene,
 * 15 LrfMeshTable, 17 LrfColourFrame (0 for any other index; 16 is left unused and stays 0, as libraries
 * before LrfColourFrame answered).  Bindings compare these with their own mirrors at load time, so a stale library
 * or a drifted mirror fails loudly instead of mis-reading arguments. */
size_t lrf_sizeof(int32_t which);

/* Device bytes of the per-field "prepared" block (folded / re-laid-out MLP weights) of a field without
 * positional encodings; lrf_prepared_bytes_for() covers every field (fea_pe / view_pe in [0, 8]; 0 if not
 * built).  A field with encodings needs the block 1024-byte aligned (its layer-1 operand is streamed by TMA). */
size_t lrf_prepared_bytes(void);
size_t lrf_prepared_bytes_for(const LrfField *field);
/* Builds the prepared block from the field's current MLP / basis weights.  Call again whenever
 * those parameters change (every optimiser step while training). */
int lrf_field_prepare(const LrfField *field, void *prepared, lrf_stream_t stream);

/* The hot path: one fused launch per (field, ray batch).
 * replaces: TensorBase.forward (tensorBase.py:567-636) + the per-field body of
 * LocalTensorfs.forward's chunk loop (local_tensorfs.py:451-474) + :481-497 when finalize. */
int lrf_render(const LrfField *field, const void *prepared, const LrfBatch *batch,
               const LrfOutputs *out, lrf_stream_t stream);

/* basis_mat + MLPRender_Fea_late_view.forward (tensoRF.py:196 + tensorBase.py:115-135, pe = 0) on
 * explicit inputs: feats [M][72] = the plane x line products (tensoRF.py:192-194 order: plane-major,
 * channel-minor), viewdirs [M][3] normalised -> rgb [M][3].  Same tensor-core code as lrf_render.
 * `prepared` must be 16-byte aligned (it is staged by TMA bulk copies); feats / viewdirs / rgb may be NULL
 * when M = 0, which enqueues nothing.  M < 0 is LRF_ERR_INVALID. */
int lrf_mlp_forward(const void *prepared, const float *feats, const float *viewdirs, int64_t M,
                    float *rgb, lrf_stream_t stream);

/* The lookups below and their backward read F.grid_sample(align_corners=True, padding_mode="border") at
 * xyz_norm: a coordinate outside [-1, 1], +-inf included, clips to the border texel.  NaN reads texel 0 of
 * that axis (no NaN reaches the output) and, like a clipped coordinate, gets a zero position gradient.
 * xyz_norm / out / grad_out / d_xyz need only float alignment and may be NULL when M = 0 (nothing is
 * enqueued); M < 0 is LRF_ERR_INVALID. */
/* compute_densityfeature (tensoRF.py:112-151): xyz_norm [M][3] in [-1,1]^3 -> out [M] */
int lrf_density_feature(const LrfField *field, const float *xyz_norm, int64_t M, float *out,
                        lrf_stream_t stream);
/* compute_appfeature (tensoRF.py:153-196): xyz_norm [M][3] -> out [M][app_dim] */
int lrf_app_feature(const LrfField *field, const float *xyz_norm, int64_t M, float *out,
                    lrf_stream_t stream);

/* ---- differentiable lookups (the composed training path; SURVEY.md §8f rank 1) -------------------
 * The 72 plane x line products of compute_appfeature BEFORE basis_mat (tensoRF.py:174-194 order):
 * xyz_norm [M][3] -> out [M][3*n_acomp].  `out` must be 16-byte aligned (float4 stores). */
int lrf_app_products(const LrfField *field, const float *xyz_norm, int64_t M, float *out,
                     lrf_stream_t stream);
/* Backward of lrf_density_feature (autograd of F.grid_sample x6 + product-sum, tensoRF.py:112-151):
 * grad_out [M]; d_plane[i] / d_line[i] have the layout of the parameters, must be 16-byte aligned (float4
 * atomic adds) and are ACCUMULATED into (zero them first); d_xyz [M][3] is overwritten (may be NULL). */
int lrf_density_feature_backward(const LrfField *field, const float *xyz_norm,
                                 const float *grad_out, int64_t M, float *const d_plane[3],
                                 float *const d_line[3], float *d_xyz, lrf_stream_t stream);
/* Backward of lrf_app_products: grad_out [M][3*n_acomp]; same conventions. */
int lrf_app_products_backward(const LrfField *field, const float *xyz_norm, const float *grad_out,
                              int64_t M, float *const d_plane[3], float *const d_line[3],
                              float *d_xyz, lrf_stream_t stream);

/* ---- backward of the whole render (SURVEY.md §8f rank 1) -----------------------------------------
 * What torch autograd computes through TensorBase.forward (tensorBase.py:567-636, the training path
 * local_tensorfs.py:417-452 takes per field) with floater_thresh = 0: given dL/d(rgb_map) [n][3] and
 * dL/d(depth_map) [n] for a batch of explicit rays, ACCUMULATES dL/d(parameter) into buffers laid
 * out like the parameters (zero them first) and overwrites d_rays [n][6].
 *   d_w1b is dL/d(mlp[0].weight @ basis_mat.weight) [featureC][3*n_acomp]; the caller finishes
 *   dL/d(mlp[0].weight) = d_w1b @ basis^T and dL/d(basis_mat.weight) = mlp[0].weight^T @ d_w1b.
 * `prepared_bwd`: lrf_prepared_backward_bytes() bytes filled by lrf_field_prepare_backward (redo after
 * a parameter update).  `scratch`: lrf_backward_scratch_bytes(n_rays, n_samples) bytes of device
 * memory, contents irrelevant.  white_bg as in LrfBatch.  PE > 0 is LRF_ERR_UNSUPPORTED. */
typedef struct LrfGradients {
  float *d_rays;                                /* [n][6]                                  */
  float *d_dplane[3], *d_dline[3];              /* [H][W][n_dcomp], [L][n_dcomp]           */
  float *d_aplane[3], *d_aline[3];              /* [H][W][n_acomp], [L][n_acomp]           */
  float *d_w1b;                                 /* [featureC][3*n_acomp]                   */
  float *d_b1, *d_w2, *d_b2, *d_w3, *d_b3;      /* shapes of mlp[0].bias .. mlp_view[0].bias */
} LrfGradients;
size_t lrf_prepared_backward_bytes(void);
size_t lrf_backward_scratch_bytes(int64_t n_rays, int32_t n_samples);
int lrf_field_prepare_backward(const LrfField *field, void *prepared_bwd, lrf_stream_t stream);
int lrf_render_backward(const LrfField *field, const void *prepared_bwd, const float *rays,
                        int64_t n_rays, int32_t white_bg, const float *grad_rgb,
                        const float *grad_depth, const LrfGradients *grads, void *scratch,
                        size_t scratch_bytes, lrf_stream_t stream);

/* ---- the training call of LocalTensorfs.forward with camera gradients ------------------------------------
 * replaces: local_tensorfs.py:397-499 with is_train, one field, under autograd -- ids2pixel,
 * get_ray_directions_lean / _360, cam2rf, get_rays_lean, the render, exposure (bmm) and clamp -- forward and
 * backward.  Forward: lrf_render in ray-generation mode with finalize = 0 and exposure = NULL writes rgb_linear,
 * then lrf_exposure_clamp writes rgb = clamp(E_v rgb_linear, 0, 1) with the render kernel's own finalize
 * arithmetic (bitwise the rgb of a finalize = 1 launch).  exposure [n_views][3][3] may be NULL (identity); ray r
 * uses view r / (n_rays / n_views). */
int lrf_exposure_clamp(const float *rgb_linear, const float *exposure, int64_t n_rays, int64_t n_views, float *rgb,
                       lrf_stream_t stream);

/* Camera-side gradients of lrf_render_backward_batch.  Each may be NULL (not wanted); each is OVERWRITTEN. */
typedef struct LrfCameraGrads {
  float *d_cam2world;         /* [n_views][3][4] */
  float *d_intrinsics;        /* [3] focal, cx, cy (zero for fov360: its directions do not use them) */
  float *d_exposure;          /* [n_views][3][3]: sum over the view's rays of g' x^T (also when batch->exposure
                                 is NULL: the gradient at the identity) */
  float *d_world2rf;          /* [3] */
} LrfCameraGrads;

/* Scratch bytes of lrf_render_backward_batch; 0 if n_rays < 1, n_samples < 2, n_views < 1 or n_rays % n_views.
 * The block holds, in this order and each part starting 16-byte aligned: the generated rays [n_rays][6] fp32
 * (o, d: exactly what lrf_render marched) at byte 0, the camera-space directions [n_rays][3], g_lin [n_rays][3],
 * g' [n_rays][3], d_rays [n_rays][6] (used when grads->d_rays is NULL), per-view fp64 partials, one slot
 * [n_rays][n_samples][3] per sample for the colour branch's position gradient, and the block of lrf_render_backward. */
size_t lrf_backward_batch_scratch_bytes(int64_t n_rays, int32_t n_samples, int64_t n_views);

/* Backward of the training call above.  `batch` is the forward's LrfBatch in ray-generation mode (rays, blend
 * and accumulate unset; its white_bg is the one the forward used); rgb_linear [n][3] the forward's pre-exposure
 * colour; grad_rgb [n][3] = dL/d(rgb) of the CLAMPED output, grad_depth [n], grad_directions [n][3] or NULL
 * (dL/d of the camera-space directions, e.g. from the flow loss).  Three stages:
 *   1. per ray: the generated rays go to scratch; g' = grad_rgb [0 <= E x <= 1] (both ends pass the gradient,
 *      as torch's clamp backward does); g_lin = E_v^T g';
 *   2. lrf_render_backward on the scratch rays with g_lin: the field gradients are ACCUMULATED into `grads` as
 *      there (atomic adds), d_rays (may be NULL here) overwritten -- summed in a fixed order (each sample's colour
 *      term in its own scratch slot), unlike lrf_render_backward's d_rays;
 *   3. per view: d_cam2world = [d_rays_d dir^T | d_rays_o], d_exposure = sum g' x^T, d_world2rf = sum d_rays_o,
 *      and with d_dir = R_v^T d_rays_d + grad_directions: d focal = sum -d_dir . dir / focal,
 *      d cx = sum -d_dir_x / focal, d cy = sum d_dir_y / focal.
 * No float atomics in d_rays or in stages 1 and 3, and a fixed summation order (fp64): the camera gradients
 * are bitwise repeatable.  LRF_ERR_INVALID before any device work for explicit rays, accumulate, a blend pointer,
 * n_rays % n_views != 0, a NULL field-gradient pointer or too little scratch; floater_thresh > 0 and fields
 * with positional encodings are LRF_ERR_UNSUPPORTED. */
int lrf_render_backward_batch(const LrfField *field, const void *prepared_bwd, const LrfBatch *batch,
                              const float *rgb_linear, const float *grad_rgb, const float *grad_depth,
                              const float *grad_directions, const LrfGradients *grads,
                              const LrfCameraGrads *cam_grads, void *scratch, size_t scratch_bytes,
                              lrf_stream_t stream);

/* Closes a fused pixel exchange: enqueues on `stream` a one-CTA kernel that (1) makes this GPU's
 * earlier peer stores visible system-wide, (2) writes `seq` into slot `rank` of every peer's flag
 * array (peer_flags[p] = peer p's [world] uint64 array, peer-mapped; peer_flags[rank] is this GPU's
 * own), (3) waits until all `world` slots of the local array have reached `seq`.  When the kernel
 * ends, every rank's pixels of step `seq` are in this GPU's gathered buffer.  `seq` must increase by
 * one per step, starting at 1 (flags zero-initialised).  replaces: the ncclAllGather of SURVEY.md 8e. */
int lrf_peer_barrier(unsigned long long *const *peer_flags, int32_t rank, int32_t world,
                     unsigned long long seq, lrf_stream_t stream);
/* The same with the two halves decoupled: signals `seq`, waits until every peer has signalled `wait_seq`
 * (<= seq).  wait_seq = seq - 1 is the double-buffered exchange: step i's pixels are pushed while the
 * consumer works on step i-1's, so a step never waits for the slowest peer of the SAME step. */
int lrf_peer_signal_wait(unsigned long long *const *peer_flags, int32_t rank, int32_t world,
                         unsigned long long seq, unsigned long long wait_seq, lrf_stream_t stream);

/* ---- schedule-time operators on the field's tensors (SURVEY.md 8f ranks 2-3) ---------------------------
 * Occupancy-mask rebuild.  replaces: getDenseAlpha + updateAlphaMask (models/tensorBase.py:501-536), which
 * move the model to the CPU and loop over slabs.  dims = (gx,gy,gz) of the lattice (the caller passes
 * gridSize/2, local_tensorfs.py:264-266); `length` = stepSize.  alpha_scratch [gx][gy][gz] receives
 * getDenseAlpha()'s alpha (an existing mask in `field` culls as compute_alpha does, :538-558); mask
 * [gz][gy][gx] receives {0,1} = max_pool3d(3, pad 1)(clamp(alpha,0,1)) >= thres; *kept += #ones.
 * mask may be NULL (dense alpha only). */
int lrf_alpha_mask_build(const LrfField *field, const int32_t dims[3], float length, float thres,
                         float *alpha_scratch, float *mask, unsigned long long *kept,
                         lrf_stream_t stream);
/* Grid upsampling.  replaces: F.interpolate(bilinear, align_corners=True) of up_sampling_VM
 * (models/tensoRF.py:198-221) on one channel-last tensor: src [H][W][C] -> dst [H2][W2][C] (lines: W = W2 = 1).
 * C must be a multiple of 4. */
int lrf_upsample(const float *src, int32_t H, int32_t W, float *dst, int32_t H2, int32_t W2, int32_t C,
                 lrf_stream_t stream);
/* density_L1 (models/tensoRF.py:83-92) without the 8*G^3 intermediate: *sum += sum_n sqrt(clamp(
 * feature2density(f[n]), 1e-5)) over the G^3 flat indices (the caller divides by G^3).  The backward
 * ACCUMULATES d(mean)/d(plane_i, line_i) * (*grad_out) into buffers laid out like the parameters. */
int lrf_density_l1(const LrfField *field, double *sum, lrf_stream_t stream);
int lrf_density_l1_backward(const LrfField *field, const float *grad_out, float *const d_plane[3],
                            float *const d_line[3], lrf_stream_t stream);
/* TVLoss (utils/utils.py:293-312) pieces on one channel-last [H][W][C] tensor: sums[0] += sum of squared
 * differences along H, sums[1] += along W.  Backward: dx += (*grad_out) * (kh * d sums[0]/dx + kw * d sums[1]/dx). */
int lrf_tv_sums(const float *x, int32_t H, int32_t W, int32_t C, double *sums, lrf_stream_t stream);
int lrf_tv_sums_backward(const float *x, int32_t H, int32_t W, int32_t C, const float *grad_out, float kh,
                         float kw, float *dx, lrf_stream_t stream);
/* sample_ray (models/tensorBase.py:396-417): ray-AABB entry distance clamped to [near, far], S uniform steps
 * of `step` from there (+ jitter[r] steps when jitter != NULL: the train-mode draw, one per ray), points and
 * the inside-the-box mask.  rays [N][6]; aabb = {min xyz, max xyz}; pts [N][S][3], z [N][S], inside [N][S]. */
int lrf_sample_ray(const float *rays, const float *jitter, int64_t N, int32_t S, const float aabb[6],
                   float near, float far, float step, float *pts, float *z, unsigned char *inside,
                   lrf_stream_t stream);

/* Frame post-processing on the device.  replaces: the host-side conversions of renderer.py:126-131,173-176
 * (rgb_map.cpu() ... cv2.imwrite(255 * rgb[..., ::-1]); visualize_depth -> cv2.applyColorMap, utils/utils.py:
 * 179-197).  rgb [N] x 3 floats `rgb_stride` apart, depth [N] floats `depth_stride` apart (3 / 1, or 4 / 4 for the
 * interleaved pix layout) -> rgb8 [N][3] 8-bit BGR and depth8 [N][3] = lut[(uint8)(255 * clip((d - d_lo) /
 * (d_hi - d_lo + 1e-8), 0, 1))] with lut [256][3] (the caller's colour map, e.g. cv2.COLORMAP_JET).  NaN depths
 * count as 0.  The bounds are doubles, as visualize_depth's Python numbers are: the denominator d_hi - d_lo + 1e-8
 * is formed in double and rounded to float once, d_lo is rounded to float, and the rest is fp32, which is what numpy
 * does with a float32 frame.  Either output may be NULL.  Outputs may live in pinned host memory (zero-copy).
 * Difference from the reference: rgb values with 255 * v >= 2^31 (and +inf) give 255, where OpenCV's float -> 8-bit
 * conversion on x86-64 gives 0; below that, NaN and -inf give what OpenCV gives (NaN and -inf give 0).  The renderer
 * clamps rgb to [0, 1] before this step. */
int lrf_frame_to_u8(const float *rgb, int32_t rgb_stride, const float *depth, int32_t depth_stride, int64_t N,
                    double d_lo, double d_hi, const unsigned char *lut, unsigned char *rgb8, unsigned char *depth8,
                    lrf_stream_t stream);

/* Test-frame metrics on the device.  replaces: renderer.py:162-163, `mse = ((gt_rgb - rgb_map) ** 2).mean()` and
 * `rgb_ssim(gt_rgb, rgb_map, 1)` with rgb_ssim of utils/utils.py:232-287 (numpy + scipy.signal.convolve2d).
 * img and gt are H x W x 3 fp32 frames, pixel (row, col) channel c at ptr[(row * W + col) * stride + c] (stride 3
 * for [N][3], 4 for the interleaved pix layout).  Inputs and `out` may be device or pinned host memory.
 * out[0] = mean of (gt - img)^2 over all H * W * 3 values (fp32 terms summed in fp64); out[1] = SSIM: a "valid"
 * separable Gaussian filter (filter_size taps, filter_sigma) of the five moments, the squares and the cross
 * product formed in fp32 as the reference's float32 arrays do, everything else in fp64, and the mean of the map.
 * ssim_map, when non-NULL, receives the fp64 map [H - filter_size + 1][W - filter_size + 1][3].
 * scratch: at least lrf_image_metrics_scratch_bytes(H, W, filter_size) bytes of device memory, 8-byte aligned.
 * Bitwise deterministic, no host synchronisation.  filter_size outside [1, 16] is LRF_ERR_UNSUPPORTED.
 * Difference from the reference: H or W below filter_size is LRF_ERR_INVALID (the reference averages an empty
 * map and returns NaN). */
size_t lrf_image_metrics_scratch_bytes(int32_t H, int32_t W, int32_t filter_size); /* 0 if invalid */
int lrf_image_metrics(const float *img, int32_t img_stride, const float *gt, int32_t gt_stride, int32_t H, int32_t W,
                      double max_val, int32_t filter_size, double filter_sigma, double k1, double k2, double *out,
                      double *ssim_map, void *scratch, size_t scratch_bytes, lrf_stream_t stream);

/* Supervision losses of one training step on the device.  replaces: train.py:369-423 -- the loss-weighted L1
 * rgb term, the optical-flow reprojection term (get_fwd_bwd_cam2cams / get_pred_flow / pts2px, utils/utils.py:
 * 15-48) cut per view above its 0.9 quantile, and the monocular-depth term (compute_depth_loss, utils/utils.py:
 * 50-59) cut per view above its 0.8 quantile.  The batch is view-major: rays v*R .. v*R+R-1 belong to view v
 * (R = n_rays / n_views).  Device pointers, fp32 unless stated. */
typedef struct LrfLossBatch {
  int64_t n_rays;              /* N = n_views * R, R <= 4096 */
  int64_t n_views;             /* V */
  int64_t n_cams;              /* rows of cam2world (>= 1) */
  int64_t starting_id;         /* absolute frame id of cam2world[0]; view v uses camera view_ids[v] - starting_id */
  int32_t use_flow, use_depth; /* which regularisers are on (the rgb term always is) */
  float flow_weight;           /* L_flow = mean(cut e) * flow_weight (the caller folds train.py's factors) */
  float depth_weight;          /* L_depth = mean(cut d) * depth_weight */
  const float *rgb_map;        /* [N][3] */
  const float *rgb_train;      /* [N][3] */
  const float *loss_weights;   /* [N] */
  const int64_t *view_ids;     /* [V] absolute frame ids (flow) */
  const float *depth_map;      /* [N] (flow, depth) */
  const float *directions;     /* [N][3] camera-space ray directions (flow) */
  const int64_t *ij;           /* [N][2] pixel (column, row) (flow) */
  const float *cam2world;      /* [n_cams][3][4] (flow) */
  const float *focal;          /* [1] (flow) */
  const float *center;         /* [2] cx, cy (flow) */
  const float *fwd_flow, *bwd_flow;  /* [N][2] (flow) */
  const float *fwd_mask, *bwd_mask;  /* [N] (flow) */
  const float *invdepths;      /* [N] (depth) */
} LrfLossBatch;

/* Gradients of lrf_supervision_losses_backward; each may be NULL (not wanted).  All are OVERWRITTEN, also when a
 * term is off (d_directions, d_cam2world, d_focal and d_center are then zero without the flow term). */
typedef struct LrfLossGrads {
  float *d_rgb;                /* [N][3] */
  float *d_depth;              /* [N] */
  float *d_directions;         /* [N][3] */
  float *d_cam2world;          /* [n_cams][3][4]: the per-view cam2cam gradients chained in view order */
  float *d_focal;              /* [1] */
  float *d_center;             /* [2] */
} LrfLossGrads;

/* Device scratch bytes of one forward + its backward (8-byte aligned).  0 if the sizes are invalid. */
size_t lrf_supervision_scratch_bytes(int64_t n_rays, int64_t n_views, int64_t n_cams);
/* losses[3] = {L_rgb, L_flow, L_depth} (a term that is off gives 0).  Per view: e = the flow residual of each ray
 * (backward flow first, then forward; the forward mask is zero for every ray of a view whose ABSOLUTE id equals
 * n_cams - 1, as in the reference), x = 1 / max(depth, 1e-6) and g = invdepths normalised by their lower medians
 * and mean absolute deviations, d = (xn - gn)^2; each of e and d is zeroed above its torch.quantile (linear, bit
 * for bit).  A view whose camera id view_ids[v] - starting_id lies outside [0, n_cams) gets NaN flow residuals
 * (the id cannot be checked on the host without a synchronisation).  A MAD of 0 gives NaN/inf, as in the
 * reference.  The scratch keeps the forward's decisions for the backward; its leading part is, in bytes:
 * e [N] fp32 at 0, d [N] fp32 at 4N (both before the cut), tau [2][V] fp32 at 8N (flow, then depth thresholds),
 * median ray indices [V][2] int32 at 8N + 8V (x, then g: the lowest ray index holding the median value, which is
 * NaN when the view holds a NaN, as torch.median's).  Entries of a term that is off are not written.
 * No atomics, no host synchronisation: bitwise repeatable.  R > 4096 is LRF_ERR_UNSUPPORTED. */
int lrf_supervision_losses(const LrfLossBatch *batch, float *losses, void *scratch, size_t scratch_bytes,
                           lrf_stream_t stream);
/* Backward of the same batch, after lrf_supervision_losses on the same scratch: grad_losses [3] (device) are the
 * upstream gradients of the three losses.  Cut entries and the thresholds carry no gradient; each median passes
 * its gradient to the ray the forward selected.  A view with an out-of-range camera id gives NaN gradients
 * through its flow term and adds nothing to d_cam2world. */
int lrf_supervision_losses_backward(const LrfLossBatch *batch, const float *grad_losses, const LrfLossGrads *grads,
                                    void *scratch, size_t scratch_bytes, lrf_stream_t stream);

/* One Adam step over many fp32 tensors in one launch.  replaces: torch.optim.Adam.step with its default options
 * (torch 2.11's _multi_tensor_adam, non-capturable) for every optimiser of a training step, local_tensorfs.py:
 * 245,272-284.  The caller increments the step counters and folds the per-tensor scalars in double precision, as
 * torch does, rounding each to float where ATen's opmath cast does.  Per element, in fp32 with one rounding each:
 *   exp_avg = lerp(exp_avg, grad, one_minus_beta1); exp_avg_sq = exp_avg_sq * beta2;
 *   exp_avg_sq = fma(one_minus_beta2, grad * grad, exp_avg_sq); d = sqrt(exp_avg_sq) / bc2_sqrt + eps;
 *   param = fma(step_size, exp_avg / d, param).
 * The four arrays of one entry have numel elements each and one dense layout; entries must not overlap (a parameter
 * listed twice is updated once, from the values before the launch).  16-byte aligned entries use vector accesses. */
typedef struct LrfAdamTensor {
  float *param;
  const float *grad;
  float *exp_avg;
  float *exp_avg_sq;
  int64_t numel;               /* 0 = skipped */
  float one_minus_beta1;       /* float(1 - beta1) */
  float beta2;                 /* float(beta2) */
  float one_minus_beta2;       /* float(1 - beta2) */
  float eps;                   /* float(eps) */
  float step_size;             /* float((lr / (1 - beta1 ** step)) * -1) */
  float bc2_sqrt;              /* float((1 - beta2 ** step) ** 0.5) */
} LrfAdamTensor;

/* t: HOST array of n entries, read before the call returns.  One launch per 448 tensors; no atomics, no host
 * synchronisation, bitwise repeatable.  n == 0 does nothing. */
int lrf_adam_step(const LrfAdamTensor *t, int64_t n, lrf_stream_t stream);

/* Training rays from device-resident frames.  replaces: the numpy gather of LocalRFDataset.sample
 * (dataLoader/localrf_dataset.py:273-315, `self.all_*[idx_sample]`) and the uploads of train.py:352-356.  The host
 * keeps drawing the view and pixel ids (the reference's RNG); the frames stay on the device.
 * A ring of frame slots, one fp32 array per quantity; frame f lives in slot f % capacity. */
typedef struct LrfFrameStore {
  int64_t n_px;                /* pixels per frame */
  int64_t capacity;            /* slots */
  const int64_t *slot_frame;   /* [capacity] frame id each slot holds (anything negative = empty) */
  const float *rgb;            /* [capacity][n_px][3] */
  const float *loss_weight;    /* [capacity][n_px] */
  const float *invdepth;       /* [capacity][n_px], or NULL (no depth) */
  const float *fwd_flow;       /* [capacity][n_px][2] \                                          */
  const float *fwd_mask;       /* [capacity][n_px]     | the flow group: all four, or all NULL   */
  const float *bwd_flow;       /* [capacity][n_px][2]  | (no flow)                               */
  const float *bwd_mask;       /* [capacity][n_px]    /                                          */
} LrfFrameStore;

/* One batch: view-major rays, ray r belongs to view r / (n_rays / n_views), as the reference orders them.  Outputs
 * of a group the store has must be set; those of a group it lacks must be NULL. */
typedef struct LrfRayGather {
  int64_t n_rays;
  int64_t n_views;             /* n_rays % n_views == 0 */
  const int64_t *ids;          /* [n_views + n_rays]: the views' frame ids, then each ray's pixel within its frame */
  int64_t *idx;                /* [n_rays] view * n_px + pixel (the reference's `idx`) */
  float *rgb;                  /* [n_rays][3] */
  float *loss_weight;          /* [n_rays] */
  float *invdepth;             /* [n_rays] */
  float *fwd_flow;             /* [n_rays][2] */
  float *fwd_mask;             /* [n_rays] */
  float *bwd_flow;             /* [n_rays][2] */
  float *bwd_mask;             /* [n_rays] */
} LrfRayGather;

/* One launch, one thread per ray.  A ray whose view is not the frame its slot holds, or whose pixel is negative or
 * >= n_px, gets NaN in every output row (its idx is still written); no other frame's data is read.  The ids are
 * never read on the host.  No atomics, no host synchronisation. */
int lrf_gather_rays(const LrfFrameStore *store, const LrfRayGather *g, lrf_stream_t stream);

/* One frame into a slot of the store, from its files' decoded pixels.  replaces: the per-frame conversions of
 * LocalRFDataset.read_meta (dataLoader/localrf_dataset.py:143-258) after cv2.imread, bit for bit.  The output frame
 * is w x h = store->n_px pixels.  Planes are device memory, row-major with row strides in elements.  INTER_AREA
 * resizes to w x h in three forms: the same size is a copy; a reduction by k in {2, 4} (source k w x k h) sums each
 * block in a fixed order (k = 2: ((a + b) + c) + d in row-major order; k = 4: each row in order, then the rows in
 * order), times 1 / k^2, as cv2 does for 3-channel float32 images; an enlargement (source <= w x h on both axes) is
 * cv2's separable area-weighted linear rule in fp32, horizontal then vertical, rounded to nearest even and saturated
 * for uint16; its weights are formed in double as cv2 forms them, the product and the difference each rounded once
 * (never fused), so a weight that is exactly 0 there is exactly 0 here.  An enlargement by an integer factor has
 * only such weights: it repeats the source pixel.  Any other ratio is LRF_ERR_UNSUPPORTED. */
typedef struct LrfIngestFrame {
  int64_t slot;                /* 0 <= slot < store->capacity; the caller tags slot_frame */
  int32_t w, h;                /* the frame's size: w h == store->n_px */
  const uint8_t *image;        /* [h0][image_stride] BGR, 3 per pixel: rgb = (float)v / 255, reduced when k > 1 */
  int32_t w0, h0;              /* (w, h) or (k w, k h), k in {2, 4} */
  int64_t image_stride;        /* >= 3 w0 */
  const uint16_t *invdepth;    /* [hd][invdepth_stride]: (float)v, resized; set exactly when the store has invdepth */
  int32_t wd, hd;              /* same size, reduction or enlargement */
  int64_t invdepth_stride;     /* >= wd */
  const uint16_t *fwd_flow;    /* [hf][flow_stride], 3 per pixel, the file's channel order: resized as uint16, then */
  const uint16_t *bwd_flow;    /* flow = (e0,1 - 32768) / 256 * flow_scale, mask = e2 > 32768 (1 or 0); both set   */
                               /* exactly when the store has the flow group */
  int32_t wf, hf;              /* both flows: same size or enlargement */
  int64_t flow_stride;         /* >= 3 wf */
  float flow_scale;            /* float32(h / hf_of_the_forward_file) */
  const uint8_t *mask;         /* [h][mask_stride] motion mask (> 0 keeps the pixel), or NULL (every pixel kept) */
  int32_t wm, hm;              /* (w, h): a mask of another size is LRF_ERR_UNSUPPORTED */
  int64_t mask_stride;         /* >= wm */
} LrfIngestFrame;

/* Device scratch bytes of one frame of n_px pixels (8-byte aligned); 0 if n_px < 1 or the frame is too large: the
 * variance's summation tree is built for 16 halvings of numpy's recursion, which splits a run at half its length
 * rounded down to a multiple of 8.  2^16 leaves of 128 pixels (8 388 608) is the largest frame taken; an uneven split
 * leaves the longer half up to 7 values more at each level, so some smaller frames need a 17th halving and are
 * refused as well (4096 x 2048 - 1 is one; 3840 x 2160 is taken; every frame up to 7 864 328 pixels is, 7 864 329
 * is the smallest refused). */
size_t lrf_ingest_scratch_bytes(int64_t n_px);
/* Writes rgb, loss_weight and, when the store has them, invdepth, the flows and the flow masks of slot `slot`
 * (through the store's pointers, which must be writable here).  loss_weight = the variance of the 4-neighbour
 * Laplacian (reflect-101 borders, fp32) of cv2's 15-bit RGB2GRAY of (uint8)(rgb * 255), as numpy's float32 var()
 * computes it (pairwise summation of the mean, then of the squared deviations, each divided by n), times the mask.
 * The variance is summed by a fixed tree in the scratch: no atomics, no host synchronisation, bitwise repeatable.
 * Nine launches on `stream`.  LRF_ERR_INVALID before any device work for NULL store / frame / scratch, a store
 * without slot_frame, rgb or loss_weight, a partly given flow group, a slot outside [0, capacity), w h != n_px, a
 * plane sized below 1 or with a short stride, a NULL plane of a group the store has or a plane of a group it lacks,
 * and scratch not 8-byte aligned or smaller than lrf_ingest_scratch_bytes(n_px); LRF_ERR_UNSUPPORTED for the
 * ratios above and frames too large for the scratch.  Rows may be further apart than their width and planes need
 * not start their allocation; only the slot's rows of the store and the first lrf_ingest_scratch_bytes(n_px) bytes
 * of the scratch are written, and a scratch last used for another frame or size gives the same bits as a fresh one. */
int lrf_ingest_frame(const LrfFrameStore *store, const LrfIngestFrame *frame, void *scratch, size_t scratch_bytes,
                     lrf_stream_t stream);

/* A held-out frame's ground truth at the render size.  replaces: renderer.py:157, `gt_rgb = cv2.resize(gt_rgb, (W,
 * H))` (INTER_LINEAR) of the test split's float32 rgb.  src is w0 x h0, dst W x H, 3 floats per pixel, row strides
 * in floats; both device or pinned host memory, not overlapping.  dst equals OpenCV's portable implementation,
 * cv2.resize(src, (W, H)) with IPP disabled (and on builds without IPP), bit for bit:
 *   - the same size is a copy;
 *   - w0 == 2 W and h0 == 2 H is INTER_AREA, as OpenCV switches it: (((a + b) + c) + d) * 0.25 in row-major order,
 *     the 2x block sum of lrf_ingest_frame;
 *   - anything else is separable linear: per column, scale_x = 1 / ((double)W / w0), fx = (float)((x + 0.5) scale_x
 *     - 0.5) in double, sx = floor(fx), fx -= sx in float; sx < 0 gives sx = 0, fx = 0; a column with sx + 1 >= w0
 *     copies pixel min(sx, w0 - 1) of the row, the others are S[sx] (1 - fx) + S[sx + 1] fx.  Rows take fy the same
 *     way without the reset: rows clamp(sy) and clamp(sy + 1) into [0, h0) blended by (1 - fy, fy), the horizontal
 *     results rounded to float first.  Every product and sum rounds once (no FMA).
 * Difference from an IPP build (the opencv-python wheels; IPP picks its code path from the host CPU), measured with
 * IPP 2022.2.0's AVX-512 path on values in [0, 1): at 2x, at most 2 ulp (5.96e-8) on about a fifth of the values at
 * 960x540 -> 480x270; at other ratios up to 3.3e-5 (963x541 -> 481x270) and 6.9e-5 (1921x1081 -> 960x540).
 * One launch, one thread per output pixel, no host synchronisation, bitwise repeatable.  LRF_ERR_INVALID before any
 * device work for a NULL pointer, a size below 1, w0 h0 or W H at or above 2^31, and a stride below 3 times its
 * width. */
int lrf_resize_linear(const float *src, int32_t w0, int32_t h0, int64_t src_stride, float *dst, int32_t W,
                      int32_t H, int64_t dst_stride, lrf_stream_t stream);

/* Flow and depth comparison panels of one held-out frame.  replaces: renderer.py:79-124, the TensorBoard panels
 * render(test=True) builds for every test frame (get_fwd_bwd_cam2cams / get_pred_flow / compute_depth_loss of
 * utils/utils.py:15-59 and the inline numpy / cv2 lines around them).  The frame is rendered at W x H with
 * rays_ids = arange(W H), so pixel p is (column p % W, row p / W).  The ground truth is h0 x w0 and is resized with
 * OpenCV's INTER_NEAREST rule (flow values are not rescaled, as in the reference).  Pointers are device or pinned
 * host memory, fp32 unless stated. */
typedef struct LrfPanelFrame {
  int32_t W, H;                /* render size */
  int32_t h0, w0;              /* ground-truth size */
  int64_t n_cams;              /* rows of cam2world = get_cam2world() (every frame, from 0) */
  int64_t idx;                 /* the frame's camera, 0 <= idx < n_cams */
  const float *depth;          /* [H W] rendered depth */
  const float *directions;     /* [H W][3] camera-space ray directions (flow) */
  const float *cam2world;      /* [n_cams][3][4] (flow) */
  const float *intrinsics;     /* [3] focal(W), center(W, H) (flow) */
  const float *fwd_flow;       /* [h0][w0][2] \                                          */
  const float *fwd_mask;       /* [h0][w0]     | the flow group: all four, or all NULL  */
  const float *bwd_flow;       /* [h0][w0][2]  | (no flow panels)                       */
  const float *bwd_mask;       /* [h0][w0]    /                                          */
  const float *invdepth;       /* [h0][w0], or NULL (no depth panel) */
  float *fwd_panel;            /* [3H][2W] (flow) */
  float *bwd_panel;            /* [3H][2W] (flow) */
  float *depth_panel;          /* [3H][W] (depth) */
  float *fwd_pred, *bwd_pred;  /* optional [H][W][2]: the predicted flows before scaling (flow) */
  float *stats;                /* optional [8]: the 0.9 quantiles of fwd channel 0, 1 and bwd channel 0, 1, then
                                  median and mean absolute deviation of x, then of g (NaN for a branch that is off) */
} LrfPanelFrame;

/* Device scratch bytes of one frame (8-byte aligned); 0 if W H is out of range. */
size_t lrf_test_panels_scratch_bytes(int32_t W, int32_t H);
/* Flow panel (per direction, cam2cam from camera idx to camera clamp(idx +- 1), the forward mask is kept also for
 * the last camera): pred = pts2px(Rcc (directions * depth) + tcc) - (column, row); gt = the resized flow; per
 * channel c, rows [0, H) = pred_c / q_c, rows [H, 2H) = gt_c / q_c with q_c = np.quantile([pred_c; gt_c], 0.9)
 * (numpy 2.x's float32 arithmetic, bit for bit), rows [2H, 3H) = |pred_c - gt_c| * mask / W; channel c fills
 * columns [c W, c W + W).  Depth panel: x = 1 / max(depth, 1e-6), g = the resized invdepth, each normalised as
 * (v - t) / s with t its lower median (torch.median) and s the mean of |v - t| (fp64, fixed order, rounded once);
 * rows 0.5 xn, 0.5 gn, (xn - gn)^2.  Every value is clamped to [0, 1] with NaN and -0 passed through.  One exception
 * to "bit for bit": numpy and torch select by comparison, where -0 == +0, so the sign of a zero quantile or median
 * depends on where the zeros lie in their input; this kernel orders -0 before +0.  A zero quantile then turns rows of
 * nonzero values into infinities of the other sign, which clamp to the other bound.  A quantile <= 0
 * gives inf or NaN rows and a NaN in an array gives a NaN statistic, as in the reference.  With neither group given
 * nothing is launched.  LRF_ERR_INVALID before any device work for W or H < 1, 2 W H >= 2^31, h0 or w0 < 1, n_cams
 * < 1, idx outside [0, n_cams), a NULL depth, a flow group partly given, a NULL input or panel of a branch that is
 * on, and scratch that is NULL, not 8-byte aligned or too small.  No atomics on floats, no host synchronisation:
 * bitwise repeatable. */
int lrf_test_panels(const LrfPanelFrame *frame, void *scratch, size_t scratch_bytes, lrf_stream_t stream);

/* ---- point-cloud export: the training views rendered, back-projected and voxel-merged on the device ----------------
 * A ray's point is its normalised expected depth along its camera-space direction, in the world frame of cam2world
 * (the frame transforms.json is written in): s = depth / acc, c = dir s, p_a = ((R_a0 c_0 + R_a1 c_1) + R_a2 c_2) + t_a.
 * Points are merged per voxel of a world-space grid as 64-bit integer sums, so the cloud is bitwise repeatable
 * whatever the ray chunking, frame order or thread scheduling. */

/* Blended opacity of a batch's rays, called after each field's lrf_render with LrfOutputs.weights set:
 * acc_k = (float) sum_s (double) weights[r][s] in sample order, then acc[r] = b acc_k (accumulate = 0, the first field)
 * or acc[r] += b acc_k (later fields) in fp32 without FMA, b = blend[(r / (n_rays / n_views)) blend_stride] (1 when
 * blend is NULL), the batch's own LrfBatch.blend.  weights is [n_rays][n_samples] device memory.  One launch, no
 * atomics.  LRF_ERR_INVALID before any device work for NULL weights / acc, n_rays < 0 or at least 2^31, n_rays not a
 * multiple of n_views >= 1, and n_samples < 1. */
int lrf_ray_opacity(const float *weights, int64_t n_rays, int32_t n_samples, int64_t n_views, const float *blend,
                    int64_t blend_stride, int32_t accumulate, float *acc, lrf_stream_t stream);

/* The rendered rays of one view (LocalTensorfs.forward's outputs with the opacity above).  Device memory. */
typedef struct LrfPointFrame {
  int64_t n_rays;
  const float *rgb;            /* [n_rays][3] */
  const float *depth;          /* [n_rays] */
  const float *acc;            /* [n_rays] blended opacity (lrf_ray_opacity) */
  const float *directions;     /* [n_rays][3] camera-space directions */
  const float *cam2world;      /* [3][4] the view's camera */
  const float *world2rf;       /* [n_fields][3] */
  const float *blend;          /* [n_fields] the view's blending weights, or NULL (every field weight 1) */
  int32_t n_fields;
  float min_acc;               /* a ray is kept when acc >= min_acc, acc > 0 and depth is finite ... */
  float max_norm;              /* ... and max_a |p_a + world2rf_k_a| <= max_norm for a field k with blend > 0 */
} LrfPointFrame;

/* An open-addressing table of voxels (linear probing from splitmix64 of the key, key claimed by atomicCAS).  Zero
 * keys, sums and stats before the first frame.  The table holds at most capacity / 2 voxels (probes stay short):
 * stats[2] > capacity / 2 means it overflowed, and its content is then incomplete. */
typedef struct LrfVoxelTable {
  int64_t capacity;            /* slots: a power of two in [2, 2^30] */
  float voxel_size;            /* > 0, finite */
  float origin[3];             /* finite */
  unsigned long long *keys;    /* [capacity] voxel key + 1, 0 = empty */
  unsigned long long *sums;    /* [capacity][7] count, sum f_x, f_y, f_z, sum r, g, b */
  unsigned long long *stats;   /* [3] += points merged, points whose key is out of range; occupied slots */
} LrfVoxelTable;

/* Adds one view's kept rays to the table.  q_a = (p_a - origin_a) / voxel_size, k_a = floor(q_a), f_a = q_a - k_a
 * (fp32, round to nearest, in this order).  A k_a outside [-2^20, 2^20) drops the point into stats[1]; otherwise the
 * key (k_x + 2^20) << 42 | (k_y + 2^20) << 21 | (k_z + 2^20) gets count += 1, sum f_a += min((uint64)(f_a 2^32),
 * 2^32 - 1), sum c += (uint32)(clamp(rgb_c, 0, 1) 2^24).  Once the table has overflowed, rays are skipped.  One
 * launch, one thread per ray, no host synchronisation.  LRF_ERR_INVALID before any device work for a NULL frame,
 * table or pointer (blend excepted), n_rays < 0 or at least 2^31, n_fields < 1, a NaN min_acc or max_norm, and a table
 * whose capacity, voxel_size or origin is out of range or whose arrays are not 8-byte aligned. */
int lrf_frame_points(const LrfPointFrame *frame, const LrfVoxelTable *table, lrf_stream_t stream);

/* Device scratch bytes of lrf_voxel_extract (256-byte aligned); 0 for a capacity lrf_frame_points refuses or when the
 * device cannot be queried (the sort's temporary storage depends on it). */
size_t lrf_voxel_extract_scratch_bytes(int64_t capacity);
/* One point per voxel with count >= min_count, in ascending key order (x-major): rows [0, *n_voxels) of xyz
 * [capacity][3], rgb [capacity][3] and count [capacity] (int32, saturated), computed in fp64 and rounded once:
 * xyz_a = (float)(origin_a + (k_a + sum f_a / (count 2^32)) voxel_size), rgb_c = (uint8)floor(sum c / (count 2^24) 255
 * + 0.5).  *n_voxels (device) is written.  Three launches and CUB's radix sort; no atomics, no host synchronisation.
 * LRF_ERR_INVALID before any device work for a NULL table or output, a table lrf_frame_points refuses, min_count < 1,
 * and scratch that is NULL, not 256-byte aligned or smaller than lrf_voxel_extract_scratch_bytes(capacity). */
int lrf_voxel_extract(const LrfVoxelTable *table, int64_t min_count, float *xyz, uint8_t *rgb, int32_t *count,
                      int64_t *n_voxels, void *scratch, size_t scratch_bytes, lrf_stream_t stream);

/* ---- colours from the frames: points projected into the rendered views that see them, blended on the device -------
 * One rendered view and its photo, all in device memory. */
typedef struct LrfColourFrame {
  int32_t W, H;                /* >= 1, W H < 2^31 */
  int32_t fov360;              /* nonzero: equirectangular (get_ray_directions_360), else pinhole */
  const float *intrinsics;     /* [3] focal, cx, cy, as LrfBatch.intrinsics (not read for fov360) */
  const float *cam2world;      /* [3][4] the view's camera */
  const float *depth;          /* [H W] the view's eval render (LrfOutputs.depth) */
  const float *acc;            /* [H W] its blended opacity (lrf_ray_opacity) */
  const float *image;          /* [H][W][3] the frame, fp32 RGB */
  float min_acc;               /* a pixel counts when acc >= min_acc (not NaN) ... */
  float depth_tol;             /* ... and |d_v - s| <= depth_tol s (> 0, finite) ... */
  float min_cos;               /* ... and, with normals, w >= min_cos (in (0, 1]) */
} LrfColourFrame;

/* Adds one view's pixels to the points that view sees.  Per point p (xyz [n][3]), fp32 round to nearest in this order,
 * no FMA, with R = cam2world[:, :3], t = cam2world[:, 3]:
 *   1. c_b = (R_0b (p_0 - t_0) + R_1b (p_1 - t_1)) + R_2b (p_2 - t_2).
 *   2. pinhole (needs c_2 < 0): d_v = -c_2, i = floor(c_0 / d_v f + cx), j = floor(-c_1 / d_v f + cy); the pixel must
 *      lie in [0, W) x [0, H).  d_v is the planar depth, which the render's depth is for get_ray_directions_lean's
 *      z = -1 directions.
 *   3. fov360 (inverts get_ray_directions_360): d_v = r = sqrt((c_0 c_0 + c_1 c_1) + c_2 c_2) (needs 0 < r < inf),
 *      phi = asinf(clamp(c_1 / r, -1, 1)), theta = atan2f(c_0, c_2), j = floor((phi + pi/2) H / pi) clamped to
 *      [0, H - 1], i = floor((theta - pi) W / (2 pi)) mod W (fp32 pi; asinf and atan2f are CUDA's, within their ulp
 *      bounds).  d_v is the range, since those directions are unit vectors.
 *   4. depth test at k = j W + i: a = acc[k], s = depth[k] / a; the pixel counts only if a >= min_acc, a > 0, s is
 *      finite, s > 0 and |d_v - s| <= depth_tol s.
 *   5. weight: w = 1 when normals is NULL; else w = ((n_0 e_0 + n_1 e_1) + n_2 e_2) / sqrt((e_0 e_0 + e_1 e_1) + e_2 e_2)
 *      with e = t - p, and the point needs w >= min_cos (a zero normal never passes).
 *   6. a pixel with a non-finite channel adds nothing; else q = (uint32)(min(w, 1) 2^16), c24_ch =
 *      (uint32)(clamp(image[k][ch], 0, 1) 2^24) and sums[p] += {1, q, q c24_r, q c24_g, q c24_b} (atomics).
 * The sums are integers, so they are bitwise the same whatever the frame order or thread scheduling; w is capped at 1
 * so that each view adds at most 2^40 to a sum.  Zero sums [n][5] before the first view.  One launch, one thread per
 * point, no host synchronisation.  LRF_ERR_INVALID before any device work for a NULL frame, xyz, sums or frame
 * pointer (normals may be NULL), n < 0 or n >= 2^31, W or H < 1 or W H >= 2^31, sums not 8-byte aligned, a NaN
 * min_acc, a depth_tol that is not > 0 and finite, and a min_cos outside (0, 1]. */
int lrf_frame_colours(const LrfColourFrame *frame, const float *xyz, const float *normals, int64_t n,
                      unsigned long long *sums, lrf_stream_t stream);
/* Per point of sums [n][5]: count[p] = sums[p][0] (the views that coloured it; int32, saturated) and rgb[p][ch] =
 * (uint8)floor(sum q c24_ch / (sum q 2^24) 255 + 0.5) in fp64, rounded once; rgb is 0 where sum q is 0 (count 0
 * included).  rgb [n][3] and count [n] are device memory.  One launch, no atomics.  LRF_ERR_INVALID before any device
 * work for a NULL sums, rgb or count, n < 0 or n >= 2^31, and sums not 8-byte aligned. */
int lrf_colour_extract(const unsigned long long *sums, int64_t n, uint8_t *rgb, int32_t *count, lrf_stream_t stream);

/* ---- mesh export: marching cubes over the fields' density on a world-space lattice, on the device -----------------
 * Lattice point i = (ix, iy, iz) sits at p_a = origin_a + i_a voxel_size (fp32, round to nearest).  The scalar field at
 * a world point p is A(p): the owner is the field k with the smallest max_a |p_a + world2rf_k_a| (fp32 adds; ties to
 * the lowest k); A = 0 when that norm is above max_norm or no field has a finite one; else A is getDenseAlpha's value
 * (1 - exp(-sigma stepSize), an alpha mask culling) of the owner at contract(p + world2rf_owner). */
#define LRF_MESH_MAX_FIELDS 64

typedef struct LrfMeshScene {
  int32_t n_fields;            /* [1, LRF_MESH_MAX_FIELDS] */
  const LrfField *fields;      /* host array [n_fields]: fp32 grids (LRF_GRID_F32); the MLP pointers are not read */
  const float *step_size;      /* host array [n_fields]: each field's stepSize (getDenseAlpha's length) */
  const float *world2rf;       /* device [n_fields][3] */
  float voxel_size;            /* > 0, finite */
  float origin[3];             /* finite */
  float max_norm;              /* > 0, finite */
  float level;                 /* > 0, finite: a lattice point is inside when A >= level (NaN is outside) */
} LrfMeshScene;

/* The cut edges (an open-addressing table keyed like LrfVoxelTable's) and the triangles of a mesh.  Zero keys and stats
 * before the first brick.  The table holds at most capacity / 2 vertices and max_triangles triangles: stats[0] >
 * capacity / 2 or stats[1] > max_triangles means it overflowed, and its content is then incomplete. */
typedef struct LrfMeshTable {
  int64_t capacity;            /* slots: a power of two in [2, 2^30] */
  int64_t max_triangles;       /* [1, 2^31) */
  unsigned long long *keys;    /* [capacity] edge key + 1, 0 = empty */
  float *verts;                /* [capacity][3] the vertex of each claimed slot */
  unsigned long long *tri_keys;/* [max_triangles] sort key of each triangle: cell key << 3 | index within its case */
  int32_t *tri_slots;          /* [max_triangles][3] the slots of its three edges */
  unsigned long long *stats;   /* [2] claimed slots (vertices), appended triangles */
} LrfMeshTable;

/* A at every point of one brick: values[(x dims_y + y) dims_z + z] = A(lattice point lo + (x, y, z)).  The brick's
 * points must lie in [-2^19, 2^19) on every axis.  One launch, no atomics.  LRF_ERR_INVALID before any device work for
 * a NULL scene, field array, step array, world2rf or values, n_fields outside [1, LRF_MESH_MAX_FIELDS], a field
 * lrf_alpha_mask_build refuses or one with bf16 grid storage, a voxel_size, max_norm or level that is not > 0 and
 * finite, an origin that is not finite, dims < 2 on some axis, a brick outside the key range, and more than 2^31
 * points. */
int lrf_mesh_lattice(const LrfMeshScene *scene, const int32_t lo[3], const int32_t dims[3], float *values,
                     lrf_stream_t stream);
/* Marching cubes over each cell of the brick lrf_mesh_lattice wrote (the same scene, lo and dims): a corner is inside
 * when its value >= level.  Each cut edge is keyed (i_x + 2^19) << 42 | (i_y + 2^19) << 22 | (i_z + 2^19) << 2 | axis by
 * its lower point i; the first cell to reach it claims its slot and stores the vertex: t = (level - v_lo) / (v_hi -
 * v_lo) (fp32, round to nearest; 0 when not finite, clamped to [0, 1]) moves the lower point along the axis by t
 * voxel_size (pa + t (pb - pa)).  Every cell computes the same bits for an edge.  Triangles of the 256-case table are
 * appended with their three slots, wound counter-clockwise seen from outside (the right-hand normal points to lower
 * A).  Bricks that share a face share its points, so consecutive bricks overlap by one point.  One launch, no host
 * synchronisation.  LRF_ERR_INVALID as lrf_mesh_lattice, and for a NULL table or a table whose capacity or
 * max_triangles is out of range or whose arrays are NULL or misaligned. */
int lrf_mesh_cells(const LrfMeshScene *scene, const int32_t lo[3], const int32_t dims[3], const float *values,
                   const LrfMeshTable *table, lrf_stream_t stream);
/* Device scratch bytes of lrf_mesh_extract (256-byte aligned); 0 for sizes lrf_mesh_cells refuses or when the device
 * cannot be queried. */
size_t lrf_mesh_extract_scratch_bytes(int64_t capacity, int64_t max_triangles);
/* The mesh in a canonical order: vertices in ascending edge-key order (rows [0, counts[0]) of xyz [capacity / 2][3]),
 * triangles in ascending sort-key order as vertex indices (rows [0, counts[1]) of faces [max_triangles][3] int32).
 * counts (device, [2]) receive the claimed slots and appended triangles; past either limit nothing is written beyond
 * the buffers, and the caller must treat the mesh as incomplete.  The output is bitwise the same whatever the brick
 * size, the brick order or the thread scheduling.  CUB radix sorts; no host synchronisation.  LRF_ERR_INVALID for a
 * table lrf_mesh_cells refuses, NULL outputs, and scratch that is NULL, not 256-byte aligned or too small. */
int lrf_mesh_extract(const LrfMeshTable *table, float *xyz, int32_t *faces, int64_t *counts, void *scratch,
                     size_t scratch_bytes, lrf_stream_t stream);
/* Per vertex: g_a = A(x + h e_a) - A(x - h e_a), h = voxel_size / 2 (fp32); normals = -g / |g| (outward), (0, 0, 0)
 * when |g| is 0 or not finite; owner = the field of smallest max-norm at x (without the max_norm cut; -1 when none is
 * finite).  xyz, normals [n][3] and owner [n] are device memory.  LRF_ERR_INVALID as lrf_mesh_lattice for the scene,
 * n < 0 or at least 2^31, and NULL arrays with n > 0. */
int lrf_mesh_normals(const LrfMeshScene *scene, const float *xyz, int64_t n, float *normals, int32_t *owner,
                     lrf_stream_t stream);

/* fp32 -> bfloat16 (round to nearest even), n elements: the 16-bit copy of a channel-last plane / line
 * tensor for LrfField.grid_dtype = LRF_GRID_BF16.  dst must be 16-byte aligned when used as a grid. */
int lrf_pack_bf16(const float *src, void *dst, int64_t n, lrf_stream_t stream);

/* [C][H][W] (contiguous NCHW parameter of the reference) -> [H][W][C]; float alignment suffices */
int lrf_repack_nchw_to_nhwc(const float *src, float *dst, int32_t C, int32_t H, int32_t W,
                            lrf_stream_t stream);

/* Launch configuration used by lrf_render on this device (for the bench's roofline record). */
int lrf_launch_info(int32_t *n_sms, int32_t *threads_per_cta, int32_t *smem_bytes_per_cta);

#ifdef __cplusplus
}
#endif
#endif /* LOCALRF_B200_H */
