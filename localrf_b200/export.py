"""The reconstruction's geometry as a coloured point cloud, in the world frame of `LocalTensorfs.get_cam2world()` (the
frame train.py's `save_transforms` writes transforms.json in), for tools that take the poses further: Gaussian
splatting initialisation, meshing, measuring the scene.

Each training view is rendered through the eval path (the fused render of `LocalTensorfs.forward`, which also writes
its per-sample weights), each ray's normalised expected depth is back-projected along its direction, and the points
are merged into a world-space voxel grid on the device as integer sums (include/localrf_b200.h, lrf_ray_opacity /
lrf_frame_points / lrf_voxel_extract): the cloud is bitwise repeatable whatever the view order or chunking.

    cloud = point_cloud(local_tensorfs, W, H)
    write_ply("points.ply", cloud["xyz"], cloud["rgb"])
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .tensorf import _stream

_TABLE_WORDS = 8          # per slot: the key, then count, sum f_x, f_y, f_z, sum r, g, b


def point_cloud(local_tensorfs, W, H, view_ids=None, test_ids=(), voxel_size=1 / 256, origin=(0, 0, 0), min_acc=0.5,
                max_norm=1.0, min_count=1, capacity=1 << 24, weights_budget=256 << 20, _frames=None):
    """Renders every view of `view_ids` (default: every frame of r_c2w, each with its own pose and blending row) at
    W x H (focal and center scale with W, H as in forward) and merges the kept rays into voxels of `voxel_size` on the
    grid through `origin`.

    A ray is kept when its blended opacity is >= `min_acc`, its depth is finite and its point lies within `max_norm`
    (max-norm) of the centre of a field that renders the view.  Views in `test_ids` use the neighbour-averaged exposure
    of held-out frames (forward's test_id).  Voxels with fewer than `min_count` points are dropped.  The voxel table has
    `capacity` slots (a power of two) and holds at most capacity / 2 voxels; a scene with more raises RuntimeError.  A
    view renders in chunks of at most weights_budget / (4 S) rays, S the longest eval distance table of the fields
    (`TensorBase.sample_table`, 2 (nSamples // 6) samples: the weights each ray's render writes).  W or H below 1
    raises ValueError.

    -> dict(xyz [P,3] float32, rgb [P,3] uint8, count [P] int32 (CUDA tensors, one row per voxel in ascending voxel-key
    order: x, then y, then z), n_rays (rays rendered), n_kept (points merged), n_out_of_range (points whose voxel index
    lies outside [-2^20, 2^20) on some axis)).  The only host read is the voxel count at the end.

    `_frames`, when a list, receives (view, first ray, rgb, depth, acc, directions) of every chunk (tests)."""
    lt = local_tensorfs
    dev = lt.blending_weights.device
    if dev.type != "cuda":
        raise RuntimeError("localrf_b200: the scene model is on the CPU; the export runs only on a CUDA device")
    views = list(range(len(lt.r_c2w))) if view_ids is None else [int(v) for v in view_ids]
    tests = {int(v) for v in test_ids}
    if not tests <= set(views):
        raise ValueError("test_ids must be among the exported view_ids")
    W, H = int(W), int(H)
    if W < 1 or H < 1:
        raise ValueError(f"W and H must be >= 1 (got W={W}, H={H})")
    S = max(rf.sample_table(False, -1, dev).numel() for rf in lt.tensorfs)
    per_chunk = int(weights_budget) // (4 * S)
    if per_chunk < 1:
        raise ValueError(f"weights_budget must hold one ray's weights ({4 * S} bytes)")
    n = W * H
    per_chunk = min(per_chunk, n)
    capacity = int(capacity)
    if capacity < 2 or capacity > 1 << 30 or capacity & (capacity - 1):
        raise ValueError("capacity must be a power of two in [2, 2^30]")
    lib = _lib.lib()

    store = torch.zeros(_TABLE_WORDS * capacity + 4, dtype=torch.int64, device=dev)
    table = _lib.LrfVoxelTable(capacity=capacity, voxel_size=float(voxel_size), keys=store.data_ptr(),
                               sums=store.data_ptr() + 8 * capacity, stats=store.data_ptr() + 8 * _TABLE_WORDS * capacity)
    table.origin[:] = [float(v) for v in origin]
    stats = store[_TABLE_WORDS * capacity:]
    n_fields = len(lt.tensorfs)
    w2rf = torch.stack([w.detach().to(dev, torch.float32) for w in lt.world2rf]).contiguous()
    blend_rows = lt.blending_weights.detach().to(dev, torch.float32).contiguous()
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    weights = torch.empty(per_chunk * S, dtype=torch.float32, device=dev)
    n_rays = 0
    with torch.no_grad(), torch.cuda.device(dev):
        stream = _stream(dev)
        for v in views:
            for lo in range(0, n, per_chunk):
                m = min(per_chunk, n - lo)
                plan = lt._eval_plan(v, m, W, H, v in tests, dev)
                if plan is None:
                    break
                outs = lt._alloc_outputs(m, dev, None, None)
                acc = torch.empty(m, dtype=torch.float32, device=dev)
                rgb, depth, dirs, _ = lt._run_weights(plan, ids.data_ptr() + 8 * lo, outs, weights, acc)
                f = _lib.LrfPointFrame(n_rays=m, rgb=rgb.data_ptr(), depth=depth.data_ptr(), acc=acc.data_ptr(),
                                       directions=dirs.data_ptr(), cam2world=plan.keep[0].data_ptr(),
                                       world2rf=w2rf.data_ptr(), blend=blend_rows[v].data_ptr(), n_fields=n_fields,
                                       min_acc=float(min_acc), max_norm=float(max_norm))
                _lib.check(lib.lrf_frame_points(C.byref(f), C.byref(table), stream))
                n_rays += m
                if _frames is not None:
                    _frames.append((v, lo, rgb, depth, acc, dirs))
        scratch_bytes = lib.lrf_voxel_extract_scratch_bytes(capacity)
        if scratch_bytes == 0:
            raise RuntimeError("localrf_b200: the voxel extract's scratch size could not be determined")
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
        xyz = torch.empty(capacity, 3, dtype=torch.float32, device=dev)
        rgb8 = torch.empty(capacity, 3, dtype=torch.uint8, device=dev)
        count = torch.empty(capacity, dtype=torch.int32, device=dev)
        _lib.check(lib.lrf_voxel_extract(C.byref(table), int(min_count), xyz.data_ptr(), rgb8.data_ptr(),
                                         count.data_ptr(), stats.data_ptr() + 24, scratch.data_ptr(), scratch_bytes,
                                         stream))
        kept, out_of_range, occupied, P = stats.tolist()
    if occupied > capacity // 2:
        raise RuntimeError(f"localrf_b200: the scene has more voxels than the table holds (capacity / 2 = "
                           f"{capacity // 2}); raise `capacity` or `voxel_size`")
    return dict(xyz=xyz[:P].clone(), rgb=rgb8[:P].clone(), count=count[:P].clone(), n_rays=n_rays, n_kept=kept,
                n_out_of_range=out_of_range)


def write_ply(path, xyz, rgb):
    """Writes a binary little-endian PLY with one `vertex` element: float x, y, z and uchar red, green, blue.  xyz
    [P,3] and rgb [P,3] are numpy arrays or tensors (on any device)."""
    as_np = lambda a: a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    xyz, rgb = as_np(xyz), as_np(rgb)
    if xyz.ndim != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape:
        raise ValueError("xyz and rgb must both be [P, 3]")
    rec = np.empty(xyz.shape[0], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"),
                                        ("blue", "u1")])
    for i, name in enumerate(("x", "y", "z")):
        rec[name] = xyz[:, i]
    for i, name in enumerate(("red", "green", "blue")):
        rec[name] = rgb[:, i]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {xyz.shape[0]}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(rec.tobytes())
