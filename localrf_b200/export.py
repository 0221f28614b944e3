"""The reconstruction's geometry as a coloured point cloud, in the world frame of `LocalTensorfs.get_cam2world()` (the
frame train.py's `save_transforms` writes transforms.json in), for tools that take the poses further: Gaussian
splatting initialisation, meshing, measuring the scene.

Each training view is rendered through the eval path (the fused render of `LocalTensorfs.forward`, which also writes
its per-sample weights), each ray's normalised expected depth is back-projected along its direction, and the points
are merged into a world-space voxel grid on the device as integer sums (include/localrf_b200.h, lrf_ray_opacity /
lrf_frame_points / lrf_voxel_extract): the cloud is bitwise repeatable whatever the view order or chunking.

    cloud = point_cloud(local_tensorfs, W, H)
    write_ply("points.ply", cloud["xyz"], cloud["rgb"])

The surface as a triangle mesh, in the same frame: marching cubes over the fields' density on a world-space lattice
(include/localrf_b200.h, lrf_mesh_lattice / lrf_mesh_cells / lrf_mesh_extract / lrf_mesh_normals), each lattice point
read from the field whose centre is nearest, so overlapping fields give one surface:

    m = mesh(local_tensorfs)
    write_ply("mesh.ply", m["xyz"], m["rgb"], faces=m["faces"], normals=m["normals"])

Colours of any such points from the video's own frames: each point projected into the rendered views that see it,
tested against the view's rendered depth, and the frame's pixels blended on the device as integer sums
(include/localrf_b200.h, lrf_frame_colours / lrf_colour_extract):

    fc = frame_colours(local_tensorfs, m["xyz"], frames, normals=m["normals"])
    rgb = torch.where(fc["count"][:, None] > 0, fc["rgb"], m["rgb"])

Floaters removed: the mesh's or cloud's connected components found on the device (include/localrf_b200.h,
lrf_mesh_components / lrf_point_components / lrf_components_select), and only the large ones kept:

    clean = keep_components(m, keep=1)                                   # mesh: size = triangles
    clean = keep_components(cloud, min_size=50, cell_size=1 / 256)       # cloud: size = points
"""
import ctypes as C
import math
import operator

import numpy as np
import torch

from . import _lib
from .ray_utils import contract
from .tensorf import _stream

def _cuda_device(local_tensorfs):
    dev = local_tensorfs.blending_weights.device
    if dev.type != "cuda":
        raise RuntimeError("localrf_b200: the scene model is on the CPU; the export runs only on a CUDA device")
    return dev


def _table_capacity(capacity):
    """`capacity` of an export's open-addressing table (csrc/lrf_table.cuh): a power of two in [2, 2^30]."""
    capacity = int(capacity)
    if capacity < 2 or capacity > 1 << 30 or capacity & (capacity - 1):
        raise ValueError("capacity must be a power of two in [2, 2^30]")
    return capacity


def _extract_scratch(nbytes, what, dev):
    """The scratch block of an extract, `nbytes` from its *_extract_scratch_bytes (0: the size query failed)."""
    if nbytes == 0:
        raise RuntimeError(f"localrf_b200: the {what}'s scratch size could not be determined")
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


def _check_overflow(n, limit, what, param, size):
    """RuntimeError when an export's table overflowed (n > limit, `what` with {} the limit), naming `param` to raise."""
    if n > limit:
        raise RuntimeError(f"localrf_b200: the {what.format(limit)}; raise `{param}` or `{size}`")


# (stats, counts) at the end of each export's int64 block: the voxel table's stats (kept, out of range, occupied) and
# lrf_voxel_extract's voxel count; the mesh table's (edge claims, triangles appended) and lrf_mesh_extract's vertex and
# triangle counts; the components' stats and lrf_components_select's counts
_VOXEL_TAIL, _MESH_TAIL, _COMPONENTS_TAIL = (3, 1), (2, 2), (2, 4)


def _int64_block(dev, words):
    """One zeroed int64 device block cut into consecutive views of `words` words each -> (block, views)."""
    block = torch.zeros(sum(words), dtype=torch.int64, device=dev)
    return block, block.split(words)


def _tail(block, tail):
    """The (stats, counts) `tail` at the end of `block` -> (both, to read with one .tolist(); stats; counts)."""
    words = block[block.numel() - sum(tail):]
    return words, words[:tail[0]], words[tail[0]:]


def _voxel_table(capacity, voxel_size, origin, dev):
    """A zeroed LrfVoxelTable in one int64 device block: keys [capacity], sums [capacity][7] (count, sum f_x, f_y,
    f_z, sum r, g, b), then _VOXEL_TAIL -> (struct, block)."""
    block, (keys, sums, stats, _) = _int64_block(dev, (capacity, 7 * capacity) + _VOXEL_TAIL)
    table = _lib.LrfVoxelTable(capacity=capacity, voxel_size=float(voxel_size), keys=keys.data_ptr(),
                               sums=sums.data_ptr(), stats=stats.data_ptr())
    table.origin[:] = [float(v) for v in origin]
    return table, block


def _mesh_table(capacity, max_triangles, dev):
    """A zeroed LrfMeshTable in one int64 device block: edge keys [capacity], vertices [capacity][3] float32,
    triangle keys [max_triangles], triangle slots [max_triangles][3] int32, then _MESH_TAIL -> (struct, block)."""
    words = (capacity, (3 * capacity + 1) // 2, max_triangles, (3 * max_triangles + 1) // 2) + _MESH_TAIL
    block, views = _int64_block(dev, words)
    keys, verts, tri_keys, tri_slots, stats, _ = (v.data_ptr() for v in views)
    table = _lib.LrfMeshTable(capacity=capacity, max_triangles=max_triangles, keys=keys, verts=verts,
                              tri_keys=tri_keys, tri_slots=tri_slots, stats=stats)
    return table, block


def _chunk_rays(lt, weights_budget, dev):
    """(S, rays per chunk): S the longest eval distance table of the fields (`TensorBase.sample_table`, the weights
    each ray's render writes), and the most rays whose weights fit in `weights_budget` bytes (ValueError below one)."""
    S = max(rf.sample_table(False, -1, dev).numel() for rf in lt.tensorfs)
    per_chunk = int(weights_budget) // (4 * S)
    if per_chunk < 1:
        raise ValueError(f"weights_budget must hold one ray's weights ({4 * S} bytes)")
    return S, per_chunk


def _render_view(lt, v, W, H, test, per_chunk, ids, weights, dev, frame=None):
    """The eval render of view `v` at W x H (forward's render with its per-sample weights into `weights`, then
    lrf_ray_opacity's blended opacity) in chunks of at most `per_chunk` rays, ray r = ids[r] (`ids` an int64 arange of
    at least W H on `dev`).  Yields (first ray, plan, rgb, depth, acc, directions) per chunk: fresh tensors, or rows of
    frame = (rgb [W H, 3], depth [W H], acc [W H]) when given.  Yields nothing when no field renders the view."""
    n = W * H
    for lo in range(0, n, per_chunk):
        m = min(per_chunk, n - lo)
        plan = lt._eval_plan(v, m, W, H, test, dev)
        if plan is None:
            return
        if frame is None:
            outs = lt._alloc_outputs(m, dev, None, None)
            acc = torch.empty(m, dtype=torch.float32, device=dev)
        else:
            outs = lt._alloc_outputs(m, dev, None, (frame[0][lo:lo + m], frame[1][lo:lo + m]))
            acc = frame[2][lo:lo + m]
        rgb, depth, dirs, _ = lt._run_weights(plan, ids.data_ptr() + 8 * lo, outs, weights, acc)
        yield lo, plan, rgb, depth, acc, dirs


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
    dev = _cuda_device(lt)
    views = list(range(len(lt.r_c2w))) if view_ids is None else [int(v) for v in view_ids]
    tests = {int(v) for v in test_ids}
    if not tests <= set(views):
        raise ValueError("test_ids must be among the exported view_ids")
    W, H = int(W), int(H)
    if W < 1 or H < 1:
        raise ValueError(f"W and H must be >= 1 (got W={W}, H={H})")
    S, per_chunk = _chunk_rays(lt, weights_budget, dev)
    n = W * H
    per_chunk = min(per_chunk, n)
    capacity = _table_capacity(capacity)
    lib = _lib.lib()

    table, store = _voxel_table(capacity, voxel_size, origin, dev)
    tail, _, counts = _tail(store, _VOXEL_TAIL)
    n_fields = len(lt.tensorfs)
    w2rf = torch.stack([w.detach().to(dev, torch.float32) for w in lt.world2rf]).contiguous()
    blend_rows = lt.blending_weights.detach().to(dev, torch.float32).contiguous()
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    weights = torch.empty(per_chunk * S, dtype=torch.float32, device=dev)
    n_rays = 0
    with torch.no_grad(), torch.cuda.device(dev):
        stream = _stream(dev)
        for v in views:
            for lo, plan, rgb, depth, acc, dirs in _render_view(lt, v, W, H, v in tests, per_chunk, ids, weights, dev):
                m = acc.numel()
                f = _lib.LrfPointFrame(n_rays=m, rgb=rgb.data_ptr(), depth=depth.data_ptr(), acc=acc.data_ptr(),
                                       directions=dirs.data_ptr(), cam2world=plan.keep[0].data_ptr(),
                                       world2rf=w2rf.data_ptr(), blend=blend_rows[v].data_ptr(), n_fields=n_fields,
                                       min_acc=float(min_acc), max_norm=float(max_norm))
                _lib.check(lib.lrf_frame_points(C.byref(f), C.byref(table), stream))
                n_rays += m
                if _frames is not None:
                    _frames.append((v, lo, rgb, depth, acc, dirs))
        scratch_bytes = lib.lrf_voxel_extract_scratch_bytes(capacity)
        scratch = _extract_scratch(scratch_bytes, "voxel extract", dev)
        xyz = torch.empty(capacity, 3, dtype=torch.float32, device=dev)
        rgb8 = torch.empty(capacity, 3, dtype=torch.uint8, device=dev)
        count = torch.empty(capacity, dtype=torch.int32, device=dev)
        _lib.check(lib.lrf_voxel_extract(C.byref(table), int(min_count), xyz.data_ptr(), rgb8.data_ptr(),
                                         count.data_ptr(), counts.data_ptr(), scratch.data_ptr(),
                                         scratch_bytes, stream))
        kept, out_of_range, occupied, P = tail.tolist()
    _check_overflow(occupied, capacity // 2, "scene has more voxels than the table holds (capacity / 2 = {})",
                    "capacity", "voxel_size")
    return dict(xyz=xyz[:P].clone(), rgb=rgb8[:P].clone(), count=count[:P].clone(), n_rays=n_rays, n_kept=kept,
                n_out_of_range=out_of_range)


def _mesh_bricks(w2rf, voxel_size, origin, max_norm, brick):
    """The bricks (lattice index of the lower corner, multiples of `brick` cells) whose cells meet some field's max_norm
    cube, widened by one lattice step so that a surface cut by the cube's boundary closes outside it.  A field whose
    world2rf has a NaN or infinite component owns no point (the owner rule of lrf_mesh_*), so it adds no brick."""
    out = set()
    for w in w2rf:
        if not all(math.isfinite(x) for x in w):
            continue
        lo, hi = [], []
        for a in range(3):
            lo.append(math.floor((-w[a] - max_norm - origin[a]) / voxel_size) - 1)
            hi.append(math.ceil((-w[a] + max_norm - origin[a]) / voxel_size) + 1)
        rng = [range(lo[a] // brick, (hi[a] - 1) // brick + 1) for a in range(3)]
        out.update((bx * brick, by * brick, bz * brick) for bx in rng[0] for by in rng[1] for bz in rng[2])
    return sorted(out)


def mesh(local_tensorfs, voxel_size=1 / 128, level=0.005, origin=(0, 0, 0), max_norm=1.0, capacity=1 << 24,
         max_triangles=1 << 25, _brick=64):
    """The iso-surface A = `level` of the scene's density as a triangle mesh, in the world frame of get_cam2world().

    A is sampled on the lattice origin + i voxel_size: at each point, the field whose centre is nearest (smallest
    max-norm of p + world2rf_k, ties to the lowest k) gives getDenseAlpha's value (1 - exp(-sigma stepSize)) at its
    contracted local position, and A = 0 beyond `max_norm` of every centre.  Marching cubes runs over the cells of the
    bricks (`_brick` cells per axis, tests only) that meet some field's cube.  The table holds at most capacity / 2
    vertices (`capacity` a power of two) and `max_triangles` triangles; a larger mesh raises RuntimeError naming the
    parameter to raise (`capacity` first when both overflow).  A field whose world2rf is not finite owns no point;
    with no finite one the mesh is empty.  The default level is the one TensoRF's mesh export passes with getDenseAlpha.

    -> dict(xyz [V,3] float32, normals [V,3] float32 (outward: -grad A / |grad A|, central differences of half a
    voxel; 0 where the gradient vanishes), rgb [V,3] uint8, faces [T,3] int32 (counter-clockwise seen from outside)),
    CUDA tensors: vertices in ascending edge-key order, triangles in ascending cell order, the same bits whatever the
    brick size.  Colours: each vertex's owner field's appearance at the vertex, shaded by its renderModule looking at
    the surface head-on (viewdirs = -normal, (0, 0, -1) where the normal is 0), without exposure, floor(255 c + 0.5).
    The only host reads are world2rf and the stepSizes at the start and the counts at the end."""
    lt = local_tensorfs
    dev = _cuda_device(lt)
    n_fields = len(lt.tensorfs)
    if n_fields > _lib.MESH_MAX_FIELDS:
        raise NotImplementedError(f"localrf_b200: the mesh export is built for at most {_lib.MESH_MAX_FIELDS} fields")
    capacity, max_triangles, brick = _table_capacity(capacity), int(max_triangles), int(_brick)
    if max_triangles < 1 or max_triangles >= 1 << 31:
        raise ValueError("max_triangles must be in [1, 2^31)")
    if brick < 1:
        raise ValueError("_brick must be >= 1")
    voxel_size, level, max_norm = float(voxel_size), float(level), float(max_norm)
    origin = [float(v) for v in origin]
    lib = _lib.lib()
    w2rf = torch.stack([w.detach().to(dev, torch.float32).reshape(3) for w in lt.world2rf]).contiguous()
    w_host = w2rf.tolist()
    steps = (C.c_float * n_fields)(*[float(rf.stepSize) for rf in lt.tensorfs])
    fields = (_lib.LrfField * n_fields)(*[rf._field() for rf in lt.tensorfs])
    scene = _lib.LrfMeshScene(n_fields=n_fields, fields=fields, step_size=steps, world2rf=w2rf.data_ptr(),
                              voxel_size=voxel_size, max_norm=max_norm, level=level)
    scene.origin[:] = origin
    bricks = _mesh_bricks(w_host, voxel_size, origin, max_norm, brick)
    key_lim = 1 << 19
    if bricks and (min(min(b) for b in bricks) < -key_lim or max(max(b) for b in bricks) + brick >= key_lim):
        raise ValueError("the lattice indices exceed [-2^19, 2^19): raise `voxel_size` or move `origin`")

    table, store = _mesh_table(capacity, max_triangles, dev)
    _, _, counts = _tail(store, _MESH_TAIL)
    values = torch.empty((brick + 1) ** 3, dtype=torch.float32, device=dev)
    dims = (C.c_int32 * 3)(brick + 1, brick + 1, brick + 1)
    with torch.no_grad(), torch.cuda.device(dev):
        stream = _stream(dev)
        for b in bricks:
            lo = (C.c_int32 * 3)(*b)
            _lib.check(lib.lrf_mesh_lattice(C.byref(scene), lo, dims, values.data_ptr(), stream))
            _lib.check(lib.lrf_mesh_cells(C.byref(scene), lo, dims, values.data_ptr(), C.byref(table), stream))
        scratch_bytes = lib.lrf_mesh_extract_scratch_bytes(capacity, max_triangles)
        scratch = _extract_scratch(scratch_bytes, "mesh extract", dev)
        xyz = torch.empty(capacity // 2, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(max_triangles, 3, dtype=torch.int32, device=dev)
        _lib.check(lib.lrf_mesh_extract(C.byref(table), xyz.data_ptr(), faces.data_ptr(), counts.data_ptr(),
                                        scratch.data_ptr(), scratch_bytes, stream))
        del scratch
        n_vert, n_tri = counts.tolist()
        _check_overflow(n_vert, capacity // 2, "mesh has more vertices than the table holds (capacity / 2 = {})",
                        "capacity", "voxel_size")
        _check_overflow(n_tri, max_triangles, "mesh has more than max_triangles = {} triangles", "max_triangles",
                        "voxel_size")
        xyz, faces = xyz[:n_vert].clone(), faces[:n_tri].clone()
        del store
        normals = torch.empty(n_vert, 3, dtype=torch.float32, device=dev)
        owner = torch.empty(n_vert, dtype=torch.int32, device=dev)
        _lib.check(lib.lrf_mesh_normals(C.byref(scene), xyz.data_ptr(), n_vert, normals.data_ptr(),
                                        owner.data_ptr(), stream))
        rgb = _mesh_colours(lt, xyz, normals, owner, w2rf)
    return dict(xyz=xyz, normals=normals, rgb=rgb, faces=faces)


def _mesh_colours(lt, xyz, normals, owner, w2rf):
    """Each vertex's colour from its owner field: compute_appfeature at the normalised, contracted vertex, then the
    field's renderModule with viewdirs = -normal ((0, 0, -1) where the normal is 0) and refine = is_refining, as the
    eval render shades; no exposure.  -> [V, 3] uint8."""
    rgb = torch.zeros(xyz.shape[0], 3, dtype=torch.uint8, device=xyz.device)
    view = -normals
    view[(normals == 0).all(-1)] = torch.tensor([0.0, 0.0, -1.0], device=xyz.device)
    for k, rf in enumerate(lt.tensorfs):
        sel = (owner == k).nonzero().reshape(-1)
        if sel.numel() == 0:
            continue
        x =rf.normalize_coord(contract(xyz[sel] + w2rf[k]))
        c = rf.renderModule(None, view[sel], rf.compute_appfeature(x), bool(lt.is_refining))
        rgb[sel] = torch.floor(255 * c + 0.5).clamp(0, 255).to(torch.uint8)
    return rgb


def _points_arg(a, name, dev):
    """`a` ([P, 3] float32, a tensor on any device or a numpy array, P < 2^31) as a contiguous tensor on `dev`."""
    t = torch.from_numpy(a) if isinstance(a, np.ndarray) else a
    if not torch.is_tensor(t) or t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3 or t.shape[0] >= 1 << 31:
        raise ValueError(f"{name} must be a [P, 3] float32 tensor or array with P < 2^31")
    return t.detach().to(dev).contiguous()


def _frame_image(image, dev):
    """A frame's image ([h, w, 3] float32: a numpy array, a pinned tensor or a tensor on `dev`) as a contiguous tensor
    on `dev`, enqueued on the current stream without blocking: arrays are staged through pinned memory (the caching
    host allocator keeps each staging block until its copy has run)."""
    host = isinstance(image, np.ndarray)
    shape = image.shape if host or torch.is_tensor(image) else None
    dtype_ok = (image.dtype == np.float32) if host else (torch.is_tensor(image) and image.dtype == torch.float32)
    if (not dtype_ok or len(shape) != 3 or shape[2] != 3 or shape[0] < 1 or shape[1] < 1
            or shape[0] * shape[1] >= 1 << 31):
        raise ValueError("each frame's image must be [h, w, 3] float32 (a numpy array or a tensor) with w h < 2^31")
    if host:
        staged = torch.empty(shape, dtype=torch.float32, pin_memory=True)
        staged.numpy()[...] = image
        return staged.to(dev, non_blocking=True)
    if image.is_cuda:
        if image.device != dev:
            raise ValueError(f"a CUDA image must be on the scene's device ({dev})")
        return image.contiguous()
    if not image.is_pinned():
        raise ValueError("a host tensor image must be pinned (page-locked); pass a numpy array to have it staged")
    return image.to(dev, non_blocking=True).contiguous()


def frame_colours(local_tensorfs, xyz, frames, normals=None, min_acc=0.5, depth_tol=0.02, min_cos=0.1,
                  weights_budget=256 << 20):
    """Colours of the points `xyz` [P, 3] (world frame of get_cam2world(): a mesh's vertices, a cloud's points) from the
    video's frames.  `frames` is an iterable of (view, image): `view` indexes r_c2w and `image` is that frame's photo,
    [h, w, 3] float32 RGB in [0, 1] (a numpy array, a pinned tensor or a CUDA tensor).  Each view renders through the
    eval path at its image's size (focal(w) and center(w, h) as forward scales them), in chunks of at most
    weights_budget / (4 S) rays as in point_cloud, and each point it sees takes the pixel it projects to
    (lrf_frame_colours): the point must lie within `depth_tol` (relative) of the pixel's normalised expected depth
    depth / acc, and the pixel's acc must be >= `min_acc`.  With `normals` [P, 3] a view's pixel is weighted by the
    cosine between the normal and the direction to the camera, and a view with cosine below `min_cos` does not count;
    without them every view that passes the depth test weighs 1.  Views no field renders add nothing.

    -> dict(rgb [P,3] uint8 (the weighted mean of the pixels, floor(255 c + 0.5), exact; 0 where no view counted),
    count [P] int32 (the views that gave each point a positive weight), n_rays (rays rendered)); rgb and count are CUDA tensors,
    bitwise the same whatever the frame order.  A malformed xyz or normals or an option out of range raises ValueError
    before any launch; each (view, image) pair is checked before its view renders, and a malformed one (a view outside
    r_c2w, an image of the wrong shape, type or device) raises ValueError.  With no points (P = 0) the pairs are
    checked but nothing renders (n_rays 0).  Nothing is read back from the device; host images do not block the
    loop."""
    lt = local_tensorfs
    dev = _cuda_device(lt)
    xyz = _points_arg(xyz, "xyz", dev)
    P = xyz.shape[0]
    if normals is not None:
        normals = _points_arg(normals, "normals", dev)
        if normals.shape[0] != P:
            raise ValueError("normals must have one row per point of xyz")
    min_acc, depth_tol, min_cos = float(min_acc), float(depth_tol), float(min_cos)
    if math.isnan(min_acc):
        raise ValueError("min_acc must not be NaN")
    if not (depth_tol > 0 and math.isfinite(depth_tol)):
        raise ValueError("depth_tol must be > 0 and finite")
    if not 0 < min_cos <= 1:
        raise ValueError("min_cos must lie in (0, 1]")
    S, per_chunk = _chunk_rays(lt, weights_budget, dev)
    n_views = len(lt.r_c2w)
    fov360 = int(lt.fov == 360)
    lib = _lib.lib()
    sums = torch.zeros(P, 5, dtype=torch.int64, device=dev)
    ids = torch.empty(0, dtype=torch.int64, device=dev)
    weights = torch.empty(0, dtype=torch.float32, device=dev)
    n_rays = 0
    with torch.no_grad(), torch.cuda.device(dev):
        stream = _stream(dev)
        for view, image in frames:
            view = operator.index(view)
            if not 0 <= view < n_views:
                raise ValueError(f"view {view} lies outside r_c2w (0 <= view < {n_views})")
            image = _frame_image(image, dev)
            if P == 0:                                   # nothing to colour: the pair is checked, nothing renders
                continue
            h, w = image.shape[0], image.shape[1]
            n = w * h
            chunk = min(per_chunk, n)
            if ids.numel() < n:
                ids = torch.arange(n, dtype=torch.int64, device=dev)
            if weights.numel() < chunk * S:
                weights = torch.empty(chunk * S, dtype=torch.float32, device=dev)
            rendered = tuple(torch.empty(shape, dtype=torch.float32, device=dev) for shape in ((n, 3), n, n))
            plan = None
            for _, plan, *_ in _render_view(lt, view, w, h, False, chunk, ids, weights, dev, rendered):
                pass
            if plan is None:
                continue
            n_rays += n
            f = _lib.LrfColourFrame(W=w, H=h, fov360=fov360, intrinsics=plan.keep[1].data_ptr(),
                                    cam2world=plan.keep[0].data_ptr(), depth=rendered[1].data_ptr(),
                                    acc=rendered[2].data_ptr(), image=image.data_ptr(), min_acc=min_acc,
                                    depth_tol=depth_tol, min_cos=min_cos)
            n_ptr = None if normals is None else normals.data_ptr()
            _lib.check(lib.lrf_frame_colours(C.byref(f), xyz.data_ptr(), n_ptr, P, sums.data_ptr(), stream))
        rgb = torch.empty(P, 3, dtype=torch.uint8, device=dev)
        count = torch.empty(P, dtype=torch.int32, device=dev)
        if P:
            _lib.check(lib.lrf_colour_extract(sums.data_ptr(), P, rgb.data_ptr(), count.data_ptr(), stream))
    return dict(rgb=rgb, count=count, n_rays=n_rays)


def _rows_at(pos, n):
    """The rows r with pos[r] >= 0 ordered by pos (each of 0 .. n - 1 taken once), as int64 [n] on pos's device,
    without a host read: row r is scattered to slot pos[r], the others to a spare slot past the end."""
    m = pos.numel()
    rows = torch.empty(m + 1, dtype=torch.int64, device=pos.device)
    rows.scatter_(0, torch.where(pos >= 0, pos.long(), m), torch.arange(m, dtype=torch.int64, device=pos.device))
    return rows[:n]


def keep_components(geometry, keep=0, min_size=0, cell_size=None, origin=(0, 0, 0), capacity=None):
    """The large connected parts of an exported mesh or point cloud: `geometry` is a dict as mesh() or point_cloud()
    returns it.  With `faces`, two vertices are connected when a triangle joins them and a component's size is its
    triangles.  Without, `cell_size` is required: each point falls in the cell floor((xyz - origin) / cell_size) (as
    point_cloud's voxels, so cell_size = its voxel_size connects neighbouring voxels), points in the same or adjacent
    cells (the 26 around a cell) are connected, and a component's size is its points; a point that is not finite or
    whose cell index lies outside [-2^20, 2^20) is a component of its own.  The components are ranked by size
    (descending, ties to the one holding the lowest row), and those with size >= `min_size` are kept, only the `keep`
    largest of them unless keep is 0.

    keep=1 keeps the largest part alone: every part of the scene not connected to it goes, separate real objects as
    well as floaters.  Use `min_size` to drop only small debris.

    -> a dict with the same keys: every tensor entry but `faces` (one row per vertex: xyz, normals, rgb, count) holds
    the kept rows in their original order, `faces` the kept triangles in their original order with their vertex
    indices renumbered, and other entries are copied; plus component ([V'] int32: the rank of each kept row's
    component, 0 the largest) and sizes ([K] int64: the size of every component, kept or not, in rank order).  The
    input is not modified.  The cell table of a cloud holds capacity / 2 cells (`capacity` a power of two; default the
    smallest holding one cell per point, up to 2^30): more raises RuntimeError naming `capacity`.  A malformed dict
    or option raises ValueError before any launch; a face index outside [0, V) raises ValueError.  The only host read
    is the counts at the end."""
    if not isinstance(geometry, dict) or "xyz" not in geometry:
        raise ValueError("geometry must be a dict as mesh() or point_cloud() returns it, with an `xyz` entry")
    xyz = geometry["xyz"]
    if (not torch.is_tensor(xyz) or not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.dim() != 2
            or xyz.shape[1] != 3 or xyz.shape[0] >= 1 << 31):
        raise ValueError("geometry['xyz'] must be a [V, 3] float32 CUDA tensor with V < 2^31")
    dev, V = xyz.device, xyz.shape[0]
    for k, v in geometry.items():
        if k not in ("faces", "sizes") and torch.is_tensor(v) and (v.dim() < 1 or v.shape[0] != V or v.device != dev):
            raise ValueError(f"geometry[{k!r}] must have one row per vertex of xyz, on its device")
    keep, min_size = operator.index(keep), operator.index(min_size)
    if keep < 0 or min_size < 0:
        raise ValueError("keep and min_size must be >= 0")
    faces = geometry.get("faces")
    if faces is not None:
        if cell_size is not None:
            raise ValueError("cell_size is for a point cloud; a mesh is connected by its faces")
        if (not torch.is_tensor(faces) or faces.device != dev or faces.dtype != torch.int32 or faces.dim() != 2
                or faces.shape[1] != 3 or faces.shape[0] >= 1 << 31):
            raise ValueError("geometry['faces'] must be a [T, 3] int32 tensor on the device of xyz with T < 2^31")
        faces = faces.contiguous()
    else:
        if cell_size is None:
            raise ValueError("a point cloud (a dict without `faces`) needs cell_size")
        cell_size = float(cell_size)
        if not (cell_size > 0 and math.isfinite(cell_size)):
            raise ValueError("cell_size must be > 0 and finite")
        origin = [float(v) for v in origin]
        if len(origin) != 3 or not all(math.isfinite(v) for v in origin):
            raise ValueError("origin must be three finite numbers")
        if capacity is None:
            capacity = min(max(2, 1 << (2 * V - 1).bit_length()), 1 << 30)
        capacity = _table_capacity(capacity)
    lib = _lib.lib()
    with torch.no_grad(), torch.cuda.device(dev):
        stream = _stream(dev)
        xyz = xyz.contiguous()
        label = torch.empty(V, dtype=torch.int32, device=dev)
        size = torch.empty(V, dtype=torch.int64, device=dev)
        tail, stats, counts = _tail(_int64_block(dev, _COMPONENTS_TAIL)[0], _COMPONENTS_TAIL)
        if faces is not None:
            _lib.check(lib.lrf_mesh_components(faces.data_ptr(), faces.shape[0], V, label.data_ptr(), size.data_ptr(),
                                               stats.data_ptr(), stream))
        else:
            keys = torch.empty(capacity, dtype=torch.int64, device=dev)
            first = torch.empty(capacity, dtype=torch.int32, device=dev)
            _lib.check(lib.lrf_point_components(xyz.data_ptr(), V, (C.c_float * 3)(*origin), cell_size, keys.data_ptr(),
                                                first.data_ptr(), capacity, label.data_ptr(), size.data_ptr(),
                                                stats.data_ptr(), stream))
            del keys, first
        scratch_bytes = lib.lrf_components_select_scratch_bytes(V) if V else 0
        scratch = _extract_scratch(scratch_bytes, "component select", dev) if V else None
        new_index = torch.empty(V, dtype=torch.int32, device=dev)
        rank = torch.empty(V, dtype=torch.int32, device=dev)
        sizes = torch.empty(V, dtype=torch.int64, device=dev)
        _lib.check(lib.lrf_components_select(label.data_ptr(), size.data_ptr(), V, keep, min_size, new_index.data_ptr(),
                                             rank.data_ptr(), sizes.data_ptr(), counts.data_ptr(),
                                             None if scratch is None else scratch.data_ptr(), scratch_bytes, stream))
        del scratch
        stat0, _, n_rows, _, n_comp, kept_size = tail.tolist()
        if faces is not None and stat0:
            raise ValueError(f"geometry['faces'] has {stat0} triangles with a vertex index outside [0, {V})")
        if faces is None:
            _check_overflow(stat0, capacity // 2, "cloud has more cells than the table holds (capacity / 2 = {})",
                            "capacity", "cell_size")
        rows = _rows_at(new_index, n_rows)
        out = {}
        for k, v in geometry.items():
            if k == "faces":
                remapped = new_index[faces.long()]
                kept = remapped[:, 0] >= 0
                out[k] = remapped[_rows_at(torch.where(kept, torch.cumsum(kept, 0) - 1, -1), kept_size)]
            elif k != "sizes":
                out[k] = v[rows] if torch.is_tensor(v) else v
        out["component"] = rank[:n_rows].clone()
        out["sizes"] = sizes[:n_comp].clone()
    return out


def write_ply(path, xyz, rgb, faces=None, normals=None):
    """Writes a binary little-endian PLY with one `vertex` element: float x, y, z (then float nx, ny, nz when `normals`
    is given) and uchar red, green, blue; with `faces` [T,3], a `face` element of `property list uchar int
    vertex_indices`.  xyz [P,3], rgb [P,3], normals [P,3] and faces are numpy arrays or tensors (on any device)."""
    as_np = lambda a: a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    xyz, rgb = as_np(xyz), as_np(rgb)
    if xyz.ndim != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape:
        raise ValueError("xyz and rgb must both be [P, 3]")
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if normals is not None else [])
    rec = np.empty(xyz.shape[0], dtype=[(n, "<f4") for n in names] + [("red", "u1"), ("green", "u1"), ("blue", "u1")])
    for i, name in enumerate(("x", "y", "z")):
        rec[name] = xyz[:, i]
    if normals is not None:
        normals = as_np(normals)
        if normals.shape != xyz.shape:
            raise ValueError("normals must be [P, 3]")
        for i, name in enumerate(("nx", "ny", "nz")):
            rec[name] = normals[:, i]
    for i, name in enumerate(("red", "green", "blue")):
        rec[name] = rgb[:, i]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {xyz.shape[0]}\n"
              + "".join(f"property float {n}\n" for n in names) +
              "property uchar red\nproperty uchar green\nproperty uchar blue\n")
    body = rec.tobytes()
    if faces is not None:
        faces = as_np(faces)
        if faces.ndim != 2 or faces.shape[1] != 3:
            raise ValueError("faces must be [T, 3]")
        frec = np.empty(faces.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
        frec["n"] = 3
        frec["v"] = faces
        header += f"element face {faces.shape[0]}\nproperty list uchar int vertex_indices\n"
        body += frec.tobytes()
    with open(path, "wb") as fh:
        fh.write((header + "end_header\n").encode("ascii"))
        fh.write(body)
