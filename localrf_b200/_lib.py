"""ctypes binding of the C ABI (include/localrf_b200.h) + the in-tree nvcc build.

The product path has NO fallback: if the shared library is missing or cannot be loaded,
`lib()` raises.  Nothing here imports oracle/.
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_CSRC, "liblrf_b200.so")
SOURCES = ["lrf_render.cu", "lrf_aux.cu", "lrf_grad.cu", "lrf_backward.cu", "lrf_sched.cu", "lrf_metrics.cu",
           "lrf_losses.cu", "lrf_optim.cu", "lrf_train.cu", "lrf_data.cu", "lrf_panels.cu", "lrf_ingest.cu",
           "lrf_table.cu", "lrf_export.cu", "lrf_mesh.cu", "lrf_components.cu", "lrf_abi.cu"]
HEADERS = ["lrf_common.cuh", "lrf_device.cuh", "lrf_launch.cuh", "lrf_launchers.cuh", "lrf_reproject.cuh",
           "lrf_select.cuh", "lrf_table.cuh", os.path.join("..", "..", "include", "localrf_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]

_fp = C.POINTER(C.c_float)
_vp = C.c_void_p


class LrfField(C.Structure):
    _fields_ = [
        ("grid", C.c_int32 * 3),
        ("aabb", C.c_float * 6),
        ("n_dcomp", C.c_int32), ("n_acomp", C.c_int32),
        ("dplane", _vp * 3), ("dline", _vp * 3), ("aplane", _vp * 3), ("aline", _vp * 3),
        ("app_dim", C.c_int32),
        ("basis", _vp),
        ("featureC", C.c_int32), ("fea_pe", C.c_int32), ("view_pe", C.c_int32),
        ("w1", _vp), ("b1", _vp), ("w2", _vp), ("b2", _vp), ("w3", _vp), ("b3", _vp),
        ("alpha_vol", _vp),
        ("alpha_dims", C.c_int32 * 3),
        ("alpha_aabb", C.c_float * 6),
        ("density_shift", C.c_float), ("distance_scale", C.c_float), ("weight_thres", C.c_float),
        ("act", C.c_int32),
        ("z_vals", _vp),
        ("n_samples", C.c_int32),
        ("grid_dtype", C.c_int32),       # GRID_F32 / GRID_BF16
    ]


GRID_F32, GRID_BF16 = 0, 1


class LrfLossBatch(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int64), ("n_views", C.c_int64), ("n_cams", C.c_int64), ("starting_id", C.c_int64),
        ("use_flow", C.c_int32), ("use_depth", C.c_int32),
        ("flow_weight", C.c_float), ("depth_weight", C.c_float),
        ("rgb_map", _vp), ("rgb_train", _vp), ("loss_weights", _vp), ("view_ids", _vp), ("depth_map", _vp),
        ("directions", _vp), ("ij", _vp), ("cam2world", _vp), ("focal", _vp), ("center", _vp),
        ("fwd_flow", _vp), ("bwd_flow", _vp), ("fwd_mask", _vp), ("bwd_mask", _vp), ("invdepths", _vp),
    ]


class LrfLossGrads(C.Structure):
    _fields_ = [("d_rgb", _vp), ("d_depth", _vp), ("d_directions", _vp), ("d_cam2world", _vp), ("d_focal", _vp),
                ("d_center", _vp)]


class LrfAdamTensor(C.Structure):
    _fields_ = [("param", _vp), ("grad", _vp), ("exp_avg", _vp), ("exp_avg_sq", _vp), ("numel", C.c_int64),
                ("one_minus_beta1", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float),
                ("eps", C.c_float), ("step_size", C.c_float), ("bc2_sqrt", C.c_float)]


class LrfFrameStore(C.Structure):
    _fields_ = [("n_px", C.c_int64), ("capacity", C.c_int64), ("slot_frame", _vp), ("rgb", _vp), ("loss_weight", _vp),
                ("invdepth", _vp), ("fwd_flow", _vp), ("fwd_mask", _vp), ("bwd_flow", _vp), ("bwd_mask", _vp)]


class LrfRayGather(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("n_views", C.c_int64), ("ids", _vp), ("idx", _vp), ("rgb", _vp),
                ("loss_weight", _vp), ("invdepth", _vp), ("fwd_flow", _vp), ("fwd_mask", _vp), ("bwd_flow", _vp),
                ("bwd_mask", _vp)]


class LrfPanelFrame(C.Structure):
    _fields_ = [("W", C.c_int32), ("H", C.c_int32), ("h0", C.c_int32), ("w0", C.c_int32),
                ("n_cams", C.c_int64), ("idx", C.c_int64),
                ("depth", _vp), ("directions", _vp), ("cam2world", _vp), ("intrinsics", _vp),
                ("fwd_flow", _vp), ("fwd_mask", _vp), ("bwd_flow", _vp), ("bwd_mask", _vp), ("invdepth", _vp),
                ("fwd_panel", _vp), ("bwd_panel", _vp), ("depth_panel", _vp), ("fwd_pred", _vp), ("bwd_pred", _vp),
                ("stats", _vp)]


class LrfIngestFrame(C.Structure):
    _fields_ = [("slot", C.c_int64), ("w", C.c_int32), ("h", C.c_int32),
                ("image", _vp), ("w0", C.c_int32), ("h0", C.c_int32), ("image_stride", C.c_int64),
                ("invdepth", _vp), ("wd", C.c_int32), ("hd", C.c_int32), ("invdepth_stride", C.c_int64),
                ("fwd_flow", _vp), ("bwd_flow", _vp), ("wf", C.c_int32), ("hf", C.c_int32), ("flow_stride", C.c_int64),
                ("flow_scale", C.c_float),
                ("mask", _vp), ("wm", C.c_int32), ("hm", C.c_int32), ("mask_stride", C.c_int64)]


class LrfPointFrame(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("rgb", _vp), ("depth", _vp), ("acc", _vp), ("directions", _vp),
                ("cam2world", _vp), ("world2rf", _vp), ("blend", _vp), ("n_fields", C.c_int32),
                ("min_acc", C.c_float), ("max_norm", C.c_float)]


class LrfVoxelTable(C.Structure):
    _fields_ = [("capacity", C.c_int64), ("voxel_size", C.c_float), ("origin", C.c_float * 3), ("keys", _vp),
                ("sums", _vp), ("stats", _vp)]


class LrfMeshScene(C.Structure):
    _fields_ = [("n_fields", C.c_int32), ("fields", C.POINTER(LrfField)), ("step_size", _fp), ("world2rf", _vp),
                ("voxel_size", C.c_float), ("origin", C.c_float * 3), ("max_norm", C.c_float), ("level", C.c_float)]


class LrfMeshTable(C.Structure):
    _fields_ = [("capacity", C.c_int64), ("max_triangles", C.c_int64), ("keys", _vp), ("verts", _vp),
                ("tri_keys", _vp), ("tri_slots", _vp), ("stats", _vp)]


class LrfColourFrame(C.Structure):
    _fields_ = [("W", C.c_int32), ("H", C.c_int32), ("fov360", C.c_int32), ("intrinsics", _vp), ("cam2world", _vp),
                ("depth", _vp), ("acc", _vp), ("image", _vp), ("min_acc", C.c_float), ("depth_tol", C.c_float),
                ("min_cos", C.c_float)]


MESH_MAX_FIELDS = 64


class LrfBatch(C.Structure):
    _fields_ = [
        ("n_rays", C.c_int64),
        ("rays", _vp),
        ("ray_ids", _vp),
        ("W", C.c_int32), ("H", C.c_int32),
        ("fov360", C.c_int32),
        ("focal", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("intrinsics", _vp),
        ("cam2world", _vp),
        ("n_views", C.c_int64),
        ("world2rf", _vp),
        ("blend", _vp),
        ("blend_stride", C.c_int64),
        ("exposure", _vp),
        ("accumulate", C.c_int32), ("finalize", C.c_int32), ("white_bg", C.c_int32),
        ("floater_thresh", C.c_float), ("refine", C.c_int32),
    ]


class LrfOutputs(C.Structure):
    _fields_ = [("rgb", _vp), ("depth", _vp), ("weights", _vp), ("directions", _vp),
                ("ij", _vp), ("pix", _vp), ("stats", _vp),
                ("n_peers", C.c_int32), ("peer_pix", _vp * 16), ("mc_pix", _vp),
                ("peer_flags", _vp * 16), ("rank", C.c_int32), ("signal_seq", C.c_uint64), ("wait_seq", C.c_uint64)]


class LrfGradients(C.Structure):
    _fields_ = [("d_rays", _vp), ("d_dplane", _vp * 3), ("d_dline", _vp * 3), ("d_aplane", _vp * 3),
                ("d_aline", _vp * 3), ("d_w1b", _vp), ("d_b1", _vp), ("d_w2", _vp), ("d_b2", _vp),
                ("d_w3", _vp), ("d_b3", _vp)]


class LrfCameraGrads(C.Structure):
    _fields_ = [("d_cam2world", _vp), ("d_intrinsics", _vp), ("d_exposure", _vp), ("d_world2rf", _vp)]


EXPORTS = ["lrf_version", "lrf_sizeof", "lrf_last_error", "lrf_prepared_bytes", "lrf_prepared_bytes_for", "lrf_field_prepare",
           "lrf_render", "lrf_mlp_forward", "lrf_app_products", "lrf_density_feature_backward",
           "lrf_app_products_backward", "lrf_density_feature", "lrf_app_feature", "lrf_repack_nchw_to_nhwc",
           "lrf_launch_info", "lrf_prepared_backward_bytes", "lrf_backward_scratch_bytes",
           "lrf_field_prepare_backward", "lrf_render_backward", "lrf_peer_barrier", "lrf_peer_signal_wait",
           "lrf_alpha_mask_build", "lrf_upsample", "lrf_density_l1", "lrf_density_l1_backward", "lrf_tv_sums",
           "lrf_tv_sums_backward", "lrf_sample_ray", "lrf_frame_to_u8", "lrf_pack_bf16",
           "lrf_image_metrics_scratch_bytes", "lrf_image_metrics", "lrf_supervision_scratch_bytes",
           "lrf_supervision_losses", "lrf_supervision_losses_backward", "lrf_adam_step",
           "lrf_exposure_clamp", "lrf_backward_batch_scratch_bytes", "lrf_render_backward_batch", "lrf_gather_rays",
           "lrf_test_panels_scratch_bytes", "lrf_test_panels", "lrf_ingest_scratch_bytes", "lrf_ingest_frame",
           "lrf_resize_linear", "lrf_ray_opacity", "lrf_frame_points", "lrf_voxel_extract_scratch_bytes",
           "lrf_voxel_extract", "lrf_mesh_lattice", "lrf_mesh_cells", "lrf_mesh_extract_scratch_bytes",
           "lrf_mesh_extract", "lrf_mesh_normals", "lrf_frame_colours", "lrf_colour_extract", "lrf_mesh_components",
           "lrf_point_components", "lrf_components_select_scratch_bytes", "lrf_components_select"]


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(os.path.join(_CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """nvcc -gencode arch=compute_90a,code=sm_90a ... -> localrf_b200/csrc/liblrf_b200.so"""
    if not force and not _stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    extra = os.environ.get("LRF_NVCC_EXTRA", "").split()          # extra nvcc flags (e.g. -Xptxas -warn-spills)
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + SOURCES
    env = dict(os.environ)
    env.pop("CC", None); env.pop("CXX", None)  # the image's CC points at a gcc without libgomp
    r = subprocess.run(cmd, cwd=_CSRC, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout + r.stderr)
    return LIB_PATH


_lib = None


ABI_VERSION = 4


def lib():
    """Loads the shared library (building it if sources are newer).  Raises if it is missing, if a
    needed rebuild fails (a stale binary is never loaded silently), or if the binary's ABI version or
    struct sizes differ from the ctypes mirrors in this file."""
    global _lib
    if _lib is not None:
        return _lib
    if _stale():
        try:
            build()
        except (RuntimeError, FileNotFoundError) as e:
            raise RuntimeError(
                "localrf_b200: the CUDA library is missing or older than its sources and rebuilding "
                f"it failed; there is no CPU fallback and no stale binary is loaded ({e})") from e
    L = C.CDLL(LIB_PATH)
    if not hasattr(L, "lrf_sizeof") or L.lrf_version() != ABI_VERSION:
        raise RuntimeError(f"localrf_b200: {LIB_PATH} has a different ABI version than this binding; "
                           "rebuild it (python -c 'import localrf_b200; localrf_b200.build(force=True)')")
    L.lrf_sizeof.restype = C.c_size_t
    L.lrf_sizeof.argtypes = [C.c_int32]
    mirrors = list(enumerate((LrfField, LrfBatch, LrfOutputs, LrfGradients, LrfLossBatch, LrfLossGrads,
                              LrfAdamTensor, LrfCameraGrads, LrfFrameStore, LrfRayGather, LrfPanelFrame,
                              LrfIngestFrame, LrfPointFrame, LrfVoxelTable, LrfMeshScene, LrfMeshTable)))
    for which, mirror in mirrors + [(17, LrfColourFrame)]:
        if L.lrf_sizeof(which) != C.sizeof(mirror):
            raise RuntimeError(f"localrf_b200: struct {mirror.__name__} is {L.lrf_sizeof(which)} bytes in "
                               f"{LIB_PATH} but {C.sizeof(mirror)} in the ctypes mirror -- stale build")
    L.lrf_version.restype = C.c_int
    L.lrf_last_error.restype = C.c_char_p
    L.lrf_prepared_bytes.restype = C.c_size_t
    L.lrf_prepared_bytes_for.restype = C.c_size_t
    L.lrf_prepared_bytes_for.argtypes = [C.POINTER(LrfField)]
    L.lrf_field_prepare.argtypes = [C.POINTER(LrfField), _vp, _vp]
    L.lrf_render.argtypes = [C.POINTER(LrfField), _vp, C.POINTER(LrfBatch), C.POINTER(LrfOutputs), _vp]
    L.lrf_mlp_forward.argtypes = [_vp, _vp, _vp, C.c_int64, _vp, _vp]
    L.lrf_density_feature.argtypes = [C.POINTER(LrfField), _vp, C.c_int64, _vp, _vp]
    L.lrf_app_feature.argtypes = [C.POINTER(LrfField), _vp, C.c_int64, _vp, _vp]
    L.lrf_app_products.argtypes = [C.POINTER(LrfField), _vp, C.c_int64, _vp, _vp]
    for name in ("lrf_density_feature_backward", "lrf_app_products_backward"):
        getattr(L, name).argtypes = [C.POINTER(LrfField), _vp, _vp, C.c_int64, _vp * 3, _vp * 3, _vp, _vp]
    L.lrf_repack_nchw_to_nhwc.argtypes = [_vp, _vp, C.c_int32, C.c_int32, C.c_int32, _vp]
    L.lrf_pack_bf16.argtypes = [_vp, _vp, C.c_int64, _vp]
    L.lrf_launch_info.argtypes = [C.POINTER(C.c_int32)] * 3
    L.lrf_prepared_backward_bytes.restype = C.c_size_t
    L.lrf_backward_scratch_bytes.restype = C.c_size_t
    L.lrf_backward_scratch_bytes.argtypes = [C.c_int64, C.c_int32]
    L.lrf_field_prepare_backward.argtypes = [C.POINTER(LrfField), _vp, _vp]
    L.lrf_render_backward.argtypes = [C.POINTER(LrfField), _vp, _vp, C.c_int64, C.c_int32, _vp, _vp,
                                      C.POINTER(LrfGradients), _vp, C.c_size_t, _vp]
    L.lrf_exposure_clamp.argtypes = [_vp, _vp, C.c_int64, C.c_int64, _vp, _vp]
    L.lrf_backward_batch_scratch_bytes.restype = C.c_size_t
    L.lrf_backward_batch_scratch_bytes.argtypes = [C.c_int64, C.c_int32, C.c_int64]
    L.lrf_render_backward_batch.argtypes = [C.POINTER(LrfField), _vp, C.POINTER(LrfBatch), _vp, _vp, _vp, _vp,
                                            C.POINTER(LrfGradients), C.POINTER(LrfCameraGrads), _vp, C.c_size_t, _vp]
    L.lrf_alpha_mask_build.argtypes = [C.POINTER(LrfField), C.c_int32 * 3, C.c_float, C.c_float, _vp, _vp, _vp, _vp]
    L.lrf_upsample.argtypes = [_vp, C.c_int32, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp]
    L.lrf_density_l1.argtypes = [C.POINTER(LrfField), _vp, _vp]
    L.lrf_density_l1_backward.argtypes = [C.POINTER(LrfField), _vp, _vp * 3, _vp * 3, _vp]
    L.lrf_tv_sums.argtypes = [_vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp]
    L.lrf_tv_sums_backward.argtypes = [_vp, C.c_int32, C.c_int32, C.c_int32, _vp, C.c_float, C.c_float, _vp, _vp]
    L.lrf_sample_ray.argtypes = [_vp, _vp, C.c_int64, C.c_int32, C.c_float * 6, C.c_float, C.c_float, C.c_float,
                                 _vp, _vp, _vp, _vp]
    L.lrf_frame_to_u8.argtypes = [_vp, C.c_int32, _vp, C.c_int32, C.c_int64, C.c_double, C.c_double, _vp, _vp, _vp,
                                  _vp]
    L.lrf_image_metrics_scratch_bytes.restype = C.c_size_t
    L.lrf_image_metrics_scratch_bytes.argtypes = [C.c_int32] * 3
    L.lrf_image_metrics.argtypes = [_vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32,
                                    C.c_double, C.c_double, C.c_double, _vp, _vp, _vp, C.c_size_t, _vp]
    L.lrf_supervision_scratch_bytes.restype = C.c_size_t
    L.lrf_supervision_scratch_bytes.argtypes = [C.c_int64] * 3
    L.lrf_supervision_losses.argtypes = [C.POINTER(LrfLossBatch), _vp, _vp, C.c_size_t, _vp]
    L.lrf_supervision_losses_backward.argtypes = [C.POINTER(LrfLossBatch), _vp, C.POINTER(LrfLossGrads), _vp,
                                                  C.c_size_t, _vp]
    L.lrf_adam_step.argtypes = [_vp, C.c_int64, _vp]        # LrfAdamTensor array: a ctypes array or packed bytes
    L.lrf_gather_rays.argtypes = [C.POINTER(LrfFrameStore), C.POINTER(LrfRayGather), _vp]
    L.lrf_test_panels_scratch_bytes.restype = C.c_size_t
    L.lrf_test_panels_scratch_bytes.argtypes = [C.c_int32, C.c_int32]
    L.lrf_test_panels.argtypes = [C.POINTER(LrfPanelFrame), _vp, C.c_size_t, _vp]
    L.lrf_ingest_scratch_bytes.restype = C.c_size_t
    L.lrf_ingest_scratch_bytes.argtypes = [C.c_int64]
    L.lrf_ingest_frame.argtypes = [C.POINTER(LrfFrameStore), C.POINTER(LrfIngestFrame), _vp, C.c_size_t, _vp]
    L.lrf_resize_linear.argtypes = [_vp, C.c_int32, C.c_int32, C.c_int64, _vp, C.c_int32, C.c_int32, C.c_int64, _vp]
    L.lrf_ray_opacity.argtypes = [_vp, C.c_int64, C.c_int32, C.c_int64, _vp, C.c_int64, C.c_int32, _vp, _vp]
    L.lrf_frame_points.argtypes = [C.POINTER(LrfPointFrame), C.POINTER(LrfVoxelTable), _vp]
    L.lrf_voxel_extract_scratch_bytes.restype = C.c_size_t
    L.lrf_voxel_extract_scratch_bytes.argtypes = [C.c_int64]
    L.lrf_voxel_extract.argtypes = [C.POINTER(LrfVoxelTable), C.c_int64, _vp, _vp, _vp, _vp, _vp, C.c_size_t, _vp]
    L.lrf_mesh_lattice.argtypes = [C.POINTER(LrfMeshScene), C.c_int32 * 3, C.c_int32 * 3, _vp, _vp]
    L.lrf_mesh_cells.argtypes = [C.POINTER(LrfMeshScene), C.c_int32 * 3, C.c_int32 * 3, _vp, C.POINTER(LrfMeshTable),
                                 _vp]
    L.lrf_mesh_extract_scratch_bytes.restype = C.c_size_t
    L.lrf_mesh_extract_scratch_bytes.argtypes = [C.c_int64, C.c_int64]
    L.lrf_mesh_extract.argtypes = [C.POINTER(LrfMeshTable), _vp, _vp, _vp, _vp, C.c_size_t, _vp]
    L.lrf_mesh_normals.argtypes = [C.POINTER(LrfMeshScene), _vp, C.c_int64, _vp, _vp, _vp]
    L.lrf_frame_colours.argtypes = [C.POINTER(LrfColourFrame), _vp, _vp, C.c_int64, _vp, _vp]
    L.lrf_colour_extract.argtypes = [_vp, C.c_int64, _vp, _vp, _vp]
    L.lrf_mesh_components.argtypes = [_vp, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp]
    L.lrf_point_components.argtypes = [_vp, C.c_int64, C.c_float * 3, C.c_float, _vp, _vp, C.c_int64, _vp, _vp, _vp,
                                       _vp]
    L.lrf_components_select_scratch_bytes.restype = C.c_size_t
    L.lrf_components_select_scratch_bytes.argtypes = [C.c_int64]
    L.lrf_components_select.argtypes = [_vp, _vp, C.c_int64, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp, _vp,
                                        C.c_size_t, _vp]
    L.lrf_peer_barrier.argtypes = [C.POINTER(_vp), C.c_int32, C.c_int32, C.c_uint64, _vp]
    L.lrf_peer_signal_wait.argtypes = [C.POINTER(_vp), C.c_int32, C.c_int32, C.c_uint64, C.c_uint64, _vp]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError if the header and the library ever drift apart
    _lib = L
    return L


class LrfError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        msg = lib().lrf_last_error().decode()
        if rc == -2:
            raise NotImplementedError(f"localrf_b200: {msg}")
        if rc == -1:
            raise ValueError(f"localrf_b200: {msg}")
        raise LrfError(f"localrf_b200 (code {rc}): {msg}")
