"""-m gpu: the mesh export at the edges of its C ABI (include/localrf_b200.h lrf_mesh_lattice / lrf_mesh_cells /
lrf_mesh_extract / lrf_mesh_normals, localrf_b200.export.mesh).  The kernels equal the numpy restatement
(tests/mesh_oracle.py) bit for bit, with canaries past every output: tables filled to exactly capacity / 2 vertices
and max_triangles triangles and one past either, an overflow in a later brick, forced probe collisions that wrap from
the last slot to 0, more than 2^24 vertices and triangles, bricks one point thick and at the key limits, scenes of up
to 64 fields with NaN, infinite and tied world2rf rows, points on the max_norm boundary, normals, and the extract on a
dirty scratch block, a side stream and a table extracted twice."""
import contextlib
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import export_oracle as eo
import localrf_b200 as L
import mesh_oracle as mo
import render64 as r64
from localrf_b200 import _lib
from localrf_b200.export import _mesh_table, mesh

pytestmark = pytest.mark.gpu

CANARY = -12345.0
PAD = 64
H = mo.HALF


def _lt(n_fields=1, grid=48, density_shift=2.0):
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", grid, n_init_frames=2, density_shift=density_shift)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(2):
            lt.t_c2w[i].add_(0.3 * torch.randn(3, generator=g))
    for _ in range(n_fields - 1):
        lt.append_rf(2)
    return lt.to("cuda")


@pytest.fixture(scope="module")
def field_set():
    """Three single-field scenes: grids 48, 32 (with an alpha mask) and 64 (density_shift 1)."""
    a, b, c = _lt(grid=48), _lt(grid=32), _lt(grid=64, density_shift=1.0)
    b.tensorfs[0].updateAlphaMask((16, 16, 16))
    return [a, b, c]


@pytest.fixture(scope="module")
def two_fields():
    return _lt(2)


def _scene(rfs, w2rf, voxel=0.25, origin=(0.0, 0.0, 0.0), max_norm=1.0, level=0.5):
    """An LrfMeshScene over the field modules `rfs` (one may appear several times) -> (struct, what it points at)."""
    n = len(rfs)
    keep = dict(w2rf=torch.as_tensor(np.asarray(w2rf, np.float32).reshape(n, 3)).cuda().contiguous(),
                fields=(_lib.LrfField * n)(*[rf._field() for rf in rfs]),
                steps=(C.c_float * n)(*[float(rf.stepSize) for rf in rfs]))
    s = _lib.LrfMeshScene(n_fields=n, fields=keep["fields"], step_size=keep["steps"],
                          world2rf=keep["w2rf"].data_ptr(), voxel_size=voxel, max_norm=max_norm, level=level)
    s.origin[:] = [float(o) for o in origin]
    return s, keep


def _lattice(s, lo, dims):
    n = int(np.prod(dims, dtype=np.int64))
    v = torch.full((n + PAD,), CANARY, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().lrf_mesh_lattice(C.byref(s), (C.c_int32 * 3)(*lo), (C.c_int32 * 3)(*dims), v.data_ptr(),
                                           None))
    torch.cuda.synchronize()
    assert bool((v[n:] == CANARY).all()), "lrf_mesh_lattice wrote past values"
    return v[:n]


@contextlib.contextmanager
def _on(stream):
    """Work queued on `stream` (a torch.cuda.Stream; None: the current stream) after everything the current stream
    has queued, behind a spin of ~10 ms there: a kernel that ignored the stream argument and ran on the legacy default
    stream would not wait for the stream's later copies and would read stale inputs."""
    if stream is None:
        yield
        return
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        torch.cuda._sleep(20_000_000)
        yield


def _cells(s, lo, dims, values, t, stream=None):
    """lrf_mesh_cells of a brick whose values (a numpy array or a flat device tensor) sit before a canary tail; on
    `stream` (a torch.cuda.Stream), the canaries and the values are written there, after a spin, before the launch."""
    n = int(np.prod(dims, dtype=np.int64))
    if isinstance(values, np.ndarray):
        values = torch.from_numpy(np.ascontiguousarray(values, np.float32).reshape(-1)).cuda()
    with _on(stream):
        buf = torch.full((n + PAD,), CANARY, dtype=torch.float32, device="cuda")
        buf[:n] = values.reshape(-1)
        _lib.check(_lib.lib().lrf_mesh_cells(C.byref(s), (C.c_int32 * 3)(*lo), (C.c_int32 * 3)(*dims),
                                             buf.data_ptr(), C.byref(t),
                                             None if stream is None else C.c_void_p(stream.cuda_stream)))
    torch.cuda.synchronize()
    assert bool((buf[n:] == CANARY).all())


def _stats(store):
    """(edge claims, triangles appended) of a table built by _mesh_table."""
    return tuple(store[-4:-2].tolist())


def _extract(t, fill=0x5A, stream=None, before=None):
    """lrf_mesh_extract into canary-padded outputs -> (xyz [min(V, half)], faces [min(T, max_triangles)], (V, T)).
    On `stream` (a torch.cuda.Stream) the outputs and the scratch are filled there, after a spin, then `before()`
    runs there, then the extract."""
    lib = _lib.lib()
    nb = lib.lrf_mesh_extract_scratch_bytes(t.capacity, t.max_triangles)
    assert nb > 0
    half, mt = t.capacity // 2, t.max_triangles
    with _on(stream):
        scratch = torch.full((nb,), fill, dtype=torch.uint8, device="cuda")
        xyz = torch.full((half + PAD, 3), CANARY, dtype=torch.float32, device="cuda")
        faces = torch.full((mt + PAD, 3), -7, dtype=torch.int32, device="cuda")
        counts = torch.full((2 + PAD,), -9, dtype=torch.int64, device="cuda")
        if before is not None:
            before()
        _lib.check(lib.lrf_mesh_extract(C.byref(t), xyz.data_ptr(), faces.data_ptr(), counts.data_ptr(),
                                        scratch.data_ptr(), nb,
                                        None if stream is None else C.c_void_p(stream.cuda_stream)))
    torch.cuda.synchronize()
    nv, nt = counts[:2].tolist()
    assert bool((counts[2:] == -9).all()), "a count was written past counts[1]"
    assert bool((xyz[half:] == CANARY).all()) and bool((faces[mt:] == -7).all()), "an output was written past its end"
    v, f = min(nv, half), min(nt, mt)
    assert bool((xyz[v:half] == CANARY).all()) and bool((faces[f:mt] == -7).all())
    return xyz[:v].cpu().numpy(), faces[:f].cpu().numpy(), (nv, nt)


def _same(got, want):
    return got[0].shape == want[0].shape and np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and \
        np.array_equal(got[1], want[1])


def _random(dims, seed, special=True):
    rng = np.random.default_rng(seed)
    v = rng.random(dims, dtype=np.float32)
    if special:
        v[rng.random(dims) < 0.03] = 0.5
        v[rng.random(dims) < 0.01] = np.nan
        v[rng.random(dims) < 0.01] = np.inf
        v[rng.random(dims) < 0.01] = -np.inf
    return v


ORIGIN, VOX = (0.1, -0.2, 0.3), 0.03125


# ---- 1. table limits and probing -------------------------------------------------------------------------------
def _isolated(V):
    """A zero lattice with isolated inside points (1, level 0.5) on even coordinates that cut exactly V >= 3 edges: a
    point cuts 3 edges at a lattice corner, 4 on a lattice edge, 5 on a face and 6 inside."""
    extra = {0: [], 1: [3, 4], 2: [4, 4], 3: [3], 4: [4], 5: [5]}[V % 6]
    a = (V - sum(extra)) // 6
    assert a >= 0 and 6 * a + sum(extra) == V
    c = 2
    while c ** 3 < a:
        c += 1
    n = 2 * c + 3
    v = np.zeros((n, n, n), np.float32)
    i = np.stack(np.unravel_index(np.arange(a), (c, c, c)), 1) * 2 + 2
    v[i[:, 0], i[:, 1], i[:, 2]] = 1.0
    spots = {3: [(0, 0, 0)], 4: [(2, 0, 0), (4, 0, 0)], 5: [(2, 2, 0)]}
    for d in extra:
        v[spots[d].pop()] = 1.0
    return v


def _fresh(cap, max_t):
    return _mesh_table(cap, max_t, "cuda")


@pytest.mark.parametrize("cap", [8, 16, 1024, 1 << 21, 1 << 26])
def test_exactly_half_full_then_one_past(field_set, cap):
    """capacity / 2 vertices fill the table and extract in full, equal to the restatement; one more cut edge
    overflows: the count exceeds capacity / 2 and nothing is written past xyz or faces."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    half = cap // 2
    lo = (-3, 5, -(1 << 18))
    v = _isolated(half)
    want = mo.cells_np(v, lo, 0.5, ORIGIN, VOX)
    assert len(want[0]) == half
    mt = max(len(want[1]), 1)
    t, store = _fresh(cap, mt)
    _cells(s, lo, v.shape, v, t)
    assert _stats(store) == (half, len(want[1]))
    got = _extract(t)
    assert got[2] == (half, len(want[1])) and _same(got, want)
    del t, store
    v = _isolated(half + 1)
    t, store = _fresh(cap, 4 * (half + 1) // 3 + 16)             # at most 8 triangles per 6 cut edges, and a few
    _cells(s, lo, v.shape, v, t)
    nv, nt = _extract(t)[2]
    assert nv > half and _stats(store)[0] == nv


@pytest.mark.parametrize("cap", [2, 4])
def test_capacity_below_one_point_overflows(field_set, cap):
    """A lone inside corner point (3 edges, 1 triangle).  At capacity 4 (half 2) the third claim finds the counter at
    half: it returns -1, so the cell appends nothing and the counts are exactly (3, 0)."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    v = np.zeros((2, 2, 2), np.float32)
    v[0, 0, 0] = 1.0
    t, store = _fresh(cap, 4)
    _cells(s, (0, 0, 0), (2, 2, 2), v, t)
    xyz, faces, counts = _extract(t)
    if cap == 4:
        assert counts == (3, 0) and _stats(store) == (3, 0)
    else:
        assert counts[0] > 1 and counts[1] == 0
    assert len(faces) == 0


@pytest.mark.parametrize("max_t", [1, 7])
def test_exactly_max_triangles_then_one_past_by_hand(field_set, max_t):
    """Isolated points give 1 (lattice corner), 2 (lattice edge) or 4 (face) triangles: exactly max_triangles
    triangles extract in full; one more is counted and not written."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    v = np.zeros((7, 7, 7), np.float32)
    v[0, 0, 0] = 1.0
    if max_t == 7:
        v[2, 2, 0] = v[4, 0, 0] = 1.0
    want = mo.cells_np(v, (1, 2, 3), 0.5, ORIGIN, VOX)
    assert len(want[1]) == max_t
    t, store = _fresh(64, max_t)
    _cells(s, (1, 2, 3), v.shape, v, t)
    got = _extract(t)
    assert got[2] == (len(want[0]), max_t) and _same(got, want)
    v[6, 6, 6] = 1.0
    t, store = _fresh(64, max_t)
    _cells(s, (1, 2, 3), v.shape, v, t)
    got = _extract(t)
    assert got[2] == (len(want[0]) + 3, max_t + 1) and len(got[1]) == max_t


def test_exactly_max_triangles_then_one_past_random(field_set):
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    v = _random((64, 65, 66), 5)
    lo = (-30, -2, 7)
    want = mo.cells_np(v, lo, 0.5, ORIGIN, VOX)
    T = len(want[1])
    assert T > 500000
    for mt in (T, T - 1):
        t, store = _fresh(1 << 21, mt)
        _cells(s, lo, v.shape, v, t)
        got = _extract(t)
        assert got[2] == (len(want[0]), T)
        if mt == T:
            assert _same(got, want)
        else:
            assert len(got[1]) == T - 1 and np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32))


def test_overflow_in_a_later_brick(field_set):
    """Brick 1 leaves the counter at exactly capacity / 2.  Brick 2 re-covers cells of brick 1, so every cut edge it
    meets is in the table: it finds them and appends its triangles without overflowing (the result is the
    restatement's merge of both bricks).  Brick 3 has new edges and overflows; brick 4, run after it, appends
    nothing."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    cap = 1024
    v = _isolated(cap // 2)
    lo = (4, -9, 0)
    t, store = _fresh(cap, 1 << 12)
    _cells(s, lo, v.shape, v, t)
    p1 = mo.cells_parts(v, lo, 0.5, ORIGIN, VOX)
    assert _stats(store) == (cap // 2, len(p1[2]))
    sub = v[2:7, 1:9]                                    # the cells around two layers of interior points
    lo2 = (lo[0] + 2, lo[1] + 1, lo[2])
    p2 = mo.cells_parts(sub, lo2, 0.5, ORIGIN, VOX)
    assert len(p2[2]) > 50
    _cells(s, lo2, sub.shape, sub, t)
    assert _stats(store) == (cap // 2, len(p1[2]) + len(p2[2]))
    got = _extract(t)
    assert _same(got, mo.extract_np([p1, p2]))
    lone = np.zeros((3, 3, 3), np.float32)
    lone[1, 1, 1] = 1.0
    _cells(s, (100, 100, 100), lone.shape, lone, t)
    after3 = _stats(store)
    assert after3[0] > cap // 2
    _cells(s, lo2, sub.shape, sub, t)
    assert _stats(store) == after3


def _wrapping_lo(v, cap, base):
    """The first lo = base + (x, 0, 0) whose cut-edge keys include one that starts probing at slot capacity - 1 and
    whose chain wraps through slot 0 (slot 0 occupied, no key starting there) -> (lo, keys)."""
    for x in range(4096):
        lo = (base[0] + x, base[1], base[2])
        keys = mo.cells_parts(v, lo, 0.5, ORIGIN, VOX)[0]
        starts = set((eo.mix64(keys) & np.uint64(cap - 1)).tolist())
        if cap - 1 in starts and 0 not in starts and 0 in mo.probe_slots(keys.tolist(), cap):
            return lo, keys
    raise AssertionError("no wrapping lo found")


@pytest.mark.parametrize("cap, n_points", [(64, 5), (1024, 80)])
def test_forced_collisions_wrap_through_slot_zero(field_set, cap, n_points):
    """The occupied slots equal the linear-probing simulation, the tags are the cut-edge keys + 1, and the mesh is
    the restatement's."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    v = np.zeros((13, 13, 13), np.float32)
    i = np.stack(np.unravel_index(np.arange(n_points), (5, 5, 5)), 1) * 2 + 2
    v[i[:, 0], i[:, 1], i[:, 2]] = 1.0
    lo, keys = _wrapping_lo(v, cap, (-H, 77, -5))
    keys = np.unique(keys)
    assert len(keys) == 6 * n_points <= cap // 2
    t, store = _fresh(cap, 1 << 10)
    _cells(s, lo, v.shape, v, t)
    tags = store[:cap].cpu().numpy().view(np.uint64)
    occupied = set(np.nonzero(tags)[0].tolist())
    assert occupied == mo.probe_slots(keys.tolist(), cap) and {0, cap - 1} <= occupied
    assert np.array_equal(np.sort(tags[tags != 0] - np.uint64(1)), keys)
    assert _same(_extract(t), mo.cells_np(v, lo, 0.5, ORIGIN, VOX))


def test_240_cubed_more_than_2e24_vertices(field_set):
    """A random 240^3 lattice: 2.07e7 vertices (> 2^24) and 4.37e7 triangles (> 2^25) in one brick and in uneven
    bricks, equal to the restatement bit for bit."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], 1 / 256, ORIGIN)
    n = 240
    v = np.random.default_rng(9).random((n, n, n), dtype=np.float32)
    lo = (-120, -7, 3)
    want = mo.cells_np(v, lo, 0.5, ORIGIN, 1 / 256)
    assert len(want[0]) > 1 << 24 and len(want[1]) > 1 << 25
    t, store = _fresh(1 << 26, 1 << 26)
    vt = torch.from_numpy(v).cuda()
    _cells(s, lo, v.shape, vt, t)
    assert _same(_extract(t), want)
    store.zero_()
    cuts = [(0, 96), (96, 160), (160, 239)]                    # cells; each brick holds its last cell's far points
    for x0, x1 in cuts:
        for y0, y1 in cuts:
            for z0, z1 in cuts:
                sub = vt[x0:x1 + 1, y0:y1 + 1, z0:z1 + 1].contiguous()
                _cells(s, (lo[0] + x0, lo[1] + y0, lo[2] + z0), sub.shape, sub, t)
    assert _same(_extract(t), want)


# ---- 2. bricks and keys ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(2, 2, 2), (2, 2, 41), (2, 41, 2), (41, 2, 2), (2, 33, 65), (65, 2, 33),
                                  (33, 65, 2), (7, 9, 11), (31, 3, 17)])
def test_brick_shapes(field_set, dims):
    """Thin and odd bricks: the lattice's last partial block writes nothing past values, and the cells of a brick one
    cell thick cover every case it holds, equal to the restatement."""
    s, keep = _scene(field_set[0].tensorfs, [[0.1, 0.0, -0.1]], VOX, ORIGIN)
    lo = (-13, 0, 11)
    _lattice(s, lo, dims)
    v = _random(dims, sum(dims))
    want = mo.cells_np(v, lo, 0.5, ORIGIN, VOX)
    t, store = _fresh(1 << 14, 1 << 14)
    _cells(s, lo, dims, v, t)
    assert _same(_extract(t), want)


def test_brick_of_more_than_2e24_points(field_set):
    """A 2 x 4097 x 4097 brick (3.4e7 points): the lattice fills it and nothing past it, and the cells of a sparse
    lattice there equal the restatement."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], 1 / 1024, ORIGIN)
    dims = (2, 4097, 4097)
    lo = (0, -2048, -2048)
    got = _lattice(s, lo, dims)
    assert bool(torch.isfinite(got).all()) and float(got.max()) > 0
    del got
    rng = np.random.default_rng(1)
    v = np.zeros(dims, np.float32)
    idx = rng.integers(0, dims, (20000, 3))
    v[idx[:, 0], idx[:, 1], idx[:, 2]] = 1.0
    v[1, -1, -1] = 1.0                                         # the brick's last point
    want = mo.cells_np(v, lo, 0.5, ORIGIN, 1 / 1024)
    t, store = _fresh(1 << 18, 1 << 18)
    _cells(s, lo, dims, v, t)
    assert _same(_extract(t), want)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_key_limits_and_sign(field_set, axis):
    """Bricks at lo = -2^19 and at lo + dims = 2^19 on each axis (the largest accepted), and one across 0: the edge and
    cell keys order negative indices before positive ones, as the restatement does."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    dims = [9, 10, 11]
    for lo_a in (-H, H - dims[axis], -4):
        lo = [3, -6, 5]
        lo[axis] = lo_a
        v = _random(tuple(dims), lo_a & 0xFFFF)
        _lattice(s, lo, dims)
        t, store = _fresh(1 << 12, 1 << 12)
        _cells(s, lo, dims, v, t)
        assert _same(_extract(t), mo.cells_np(v, lo, 0.5, ORIGIN, VOX))
    bad = [3, -6, 5]
    bad[axis] = H - dims[axis] + 1
    vals = torch.zeros(int(np.prod(dims)), dtype=torch.float32, device="cuda")      # a real brick: refused, not read
    rc = _lib.lib().lrf_mesh_cells(C.byref(s), (C.c_int32 * 3)(*bad), (C.c_int32 * 3)(*dims), vals.data_ptr(),
                                   C.byref(t), None)
    assert rc == -1 and b"[-2^19, 2^19)" in _lib.lib().lrf_last_error()


def test_mesh_at_the_key_limits():
    """Through mesh() with one-cell bricks: a lattice whose top brick ends at index 2^19 - 1, or whose bottom brick
    starts at -2^19, is accepted; one step further raises ValueError."""
    lt = _lt()
    with torch.no_grad():
        lt.world2rf[0].zero_()
    kw = dict(voxel_size=0.5, level=0.05, _brick=1, capacity=1 << 12, max_triangles=1 << 12)
    for m, ok in ((H - 4, True), (H - 3, False)):              # top brick's last point: m + 3
        if ok:
            mesh(lt, origin=(-0.5 * m, 0.0, 0.0), **kw)
        else:
            with pytest.raises(ValueError, match="2\\^19"):
                mesh(lt, origin=(-0.5 * m, 0.0, 0.0), **kw)
    for q, ok in ((H - 3, True), (H - 2, False)):              # bottom brick's first point: -q - 3
        if ok:
            mesh(lt, origin=(0.0, 0.5 * q, 0.0), **kw)
        else:
            with pytest.raises(ValueError, match="2\\^19"):
                mesh(lt, origin=(0.0, 0.5 * q, 0.0), **kw)


# ---- 3. scene and fields ---------------------------------------------------------------------------------------
def _points(lo, dims, voxel, origin):
    ax = [np.float32(origin[a]) + np.arange(lo[a], lo[a] + dims[a]).astype(np.float32) * np.float32(voxel)
          for a in range(3)]
    return np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3)


def _owners(s, xyz):
    """lrf_mesh_normals' owner (and normals) of points xyz [M, 3] float32."""
    x = torch.from_numpy(np.ascontiguousarray(xyz, np.float32)).cuda()
    n = len(xyz)
    nrm = torch.full((n + PAD, 3), CANARY, dtype=torch.float32, device="cuda")
    own = torch.full((n + PAD,), -77, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().lrf_mesh_normals(C.byref(s), x.data_ptr(), n, nrm.data_ptr(), own.data_ptr(), None))
    torch.cuda.synchronize()
    assert bool((nrm[n:] == CANARY).all()) and bool((own[n:] == -77).all())
    return own[:n].cpu().numpy(), nrm[:n].cpu().numpy()


def _check_lattice(rfs, w2rf, lo, dims, voxel, origin, max_norm):
    """The lattice's A within float64 tolerance of mesh_value64 where the point is not flagged (rows with a
    non-finite component left out of the float64 scene, which is what the owner rule does), and the owners of
    lrf_mesh_normals equal to owner32 bit for bit -> owners."""
    s, keep = _scene(rfs, w2rf, voxel, origin, max_norm)
    got = _lattice(s, lo, dims).double().cpu()
    pts = _points(lo, dims, voxel, origin)
    own, _ = _owners(s, pts)
    want_own, _ = mo.owner32(pts, w2rf)
    assert np.array_equal(own, want_own)
    finite = [k for k in range(len(rfs)) if np.isfinite(np.asarray(w2rf[k], np.float32)).all()]
    if not finite:
        assert (got == 0).all() and (own == -1).all()
        return own
    fields = {id(rf): r64.Field64.from_module(rf) for rf in rfs}
    A, o64, flagged = mo.mesh_value64([fields[id(rfs[k])] for k in finite], [float(rfs[k].stepSize) for k in finite],
                                      np.asarray(w2rf, np.float32)[finite], torch.from_numpy(pts.astype(np.float64)),
                                      max_norm)
    ok = ~flagged
    assert int(flagged.sum()) < 0.02 * len(A)
    assert float((got - A)[ok].abs().max()) <= 2e-5 + 1e-5 * float(A.abs().max())
    inside = (o64 >= 0).numpy() & ok.numpy()
    assert np.array_equal(np.asarray(finite)[o64.numpy()[inside]], own[inside])
    assert (got[(o64 == -1) & ok] == 0).all()
    return own


@pytest.mark.parametrize("n_fields", [3, 17, 64])
def test_many_fields(field_set, n_fields):
    """Fields of three grid sizes (one with an alpha mask), cycled, with centres spread over the lattice and the last
    centre alone in a corner, so that the last field owns part of it (MeshSceneDev read up to field 63)."""
    rfs = [field_set[k % 3].tensorfs[0] for k in range(n_fields)]
    rng = np.random.default_rng(n_fields)
    centres = rng.uniform(-0.7, 0.3, (n_fields, 3)).astype(np.float32)
    centres[-1] = [0.9, 0.9, 0.9]
    w2rf = -centres
    own = _check_lattice(rfs, w2rf, (-18, -18, -18), (37, 37, 37), 1 / 16, (0.0, 0.0, 0.0), 0.75)
    assert (own == n_fields - 1).sum() > 100 and len(np.unique(own)) >= min(n_fields, 3)


@pytest.mark.parametrize("rows", ["nan", "inf", "tie", "all_nan"])
def test_nonfinite_and_tied_world2rf_rows(field_set, rows):
    """A row with one NaN component, a +inf component or a copy of an earlier row never owns a point; with every row
    NaN, A = 0 and owner = -1 everywhere."""
    a, c = field_set[0].tensorfs[0], field_set[2].tensorfs[0]
    # no sum or difference of their components, nor 1 - or -1 - one, is a multiple of the voxel: no near-ties
    w0, w1 = [0.21, 0.03, -0.13], [-0.31, 0.11, 0.17]
    bad = {"nan": [0.25, np.nan, 0.0], "inf": [np.inf, 0.0, 0.0], "tie": w0}[rows] if rows != "all_nan" else None
    if rows == "all_nan":
        rfs, w2rf = [a, c, a], [[np.nan, 0.0, 0.0], [0.0, np.nan, 0.0], [np.nan] * 3]
    else:
        rfs, w2rf = [a, c, a, c], [w0, bad, w1, bad]
    w2rf = np.asarray(w2rf, np.float32)
    own = _check_lattice(rfs, w2rf, (-20, -20, -20), (41, 41, 41), 1 / 16, (0.0, 0.0, 0.0), 1.0)
    if rows == "all_nan":
        assert (own == -1).all()
    else:
        assert set(np.unique(own).tolist()) == {0, 2}


def test_points_on_the_max_norm_boundary(field_set):
    """Lattice points whose fp32 norm is exactly max_norm are inside (A uses <=); with max_norm one ulp below they are
    0, and no other point changes."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], 0.25, (0.0, 0.0, 0.0), 0.75)
    lo, dims = (-4, -4, -4), (9, 9, 9)
    a = _lattice(s, lo, dims).cpu().numpy()
    s2, keep2 = _scene(field_set[0].tensorfs, [[0, 0, 0]], 0.25, (0.0, 0.0, 0.0),
                       float(np.nextafter(np.float32(0.75), np.float32(0))))
    b = _lattice(s2, lo, dims).cpu().numpy()
    norm = np.abs(_points(lo, dims, 0.25, (0, 0, 0))).max(1)
    on = norm == 0.75
    assert on.sum() == 7 ** 3 - 5 ** 3 and (a[on] > 0).all() and (b[on] == 0).all()
    assert (a[norm > 0.75] == 0).all() and np.array_equal(a[norm < 0.75].view(np.uint32), b[norm < 0.75].view(np.uint32))


# ---- 4. normals ------------------------------------------------------------------------------------------------
def test_normals_owner_and_gradient(two_fields):
    """On a mesh's vertices, with a tied and a NaN row added: the owner equals owner32 bit for bit, the normals match
    a float64 central difference (also within h of the max_norm cube and of an owner seam, where neither difference
    is flagged), and a constant-A plateau gives (0, 0, 0) exactly."""
    lt = two_fields
    m = mesh(lt, voxel_size=1 / 32, level=0.05, capacity=1 << 18, max_triangles=1 << 19)
    xyz = m["xyz"].cpu().numpy()
    w = torch.stack([x.detach().float() for x in lt.world2rf]).cpu().numpy()
    rfs = [lt.tensorfs[0], lt.tensorfs[1], lt.tensorfs[0], lt.tensorfs[1]]
    w2rf = np.concatenate([w, w[:1], [[np.nan, 0.0, 0.0]]]).astype(np.float32)
    s, keep = _scene(rfs, w2rf, 1 / 32, (0.0, 0.0, 0.0), 1.0, 0.05)
    far = np.array([[5.0, 5.0, 5.0], [-7.0, 0.0, 0.0], [0.0, 9.0, -9.0]], np.float32)   # A = 0 around them
    own, nrm = _owners(s, np.concatenate([xyz, far]))
    assert np.array_equal(own, mo.owner32(np.concatenate([xyz, far]), w2rf)[0]) and set(own.tolist()) <= {0, 1}
    assert (nrm[-3:] == 0).all() and not np.signbit(nrm[-3:]).any()
    assert np.array_equal(nrm[:-3].view(np.uint32), m["normals"].cpu().numpy().view(np.uint32))
    x = torch.from_numpy(xyz.astype(np.float64))
    fields = [r64.Field64.from_module(rf) for rf in lt.tensorfs]
    steps = [float(rf.stepSize) for rf in lt.tensorfs]
    h = (1 / 32) / 2
    g = torch.zeros_like(x)
    bad = torch.zeros(len(x), dtype=torch.bool)
    for a in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[a] = h
        hi, _, f1 = mo.mesh_value64(fields, steps, w, x + e, 1.0)
        lo, _, f2 = mo.mesh_value64(fields, steps, w, x - e, 1.0)
        g[:, a] = hi - lo
        bad |= f1 | f2
    gn = g.norm(dim=1)
    ok = ~bad & (gn > 1e-2)
    n64 = -g / gn[:, None]
    assert float((torch.from_numpy(nrm[:-3]).double() - n64)[ok].abs().max()) <= 1e-3
    xd = x.numpy()
    near_cube = np.abs(np.abs(xd[:, None] + w[None].astype(np.float64)).max(-1) - 1.0).min(1) <= h
    nk = np.sort(np.abs(xd[:, None] + w[None].astype(np.float64)).max(-1), 1)
    near_seam = nk[:, 1] - nk[:, 0] <= h
    assert int((ok.numpy() & near_cube).sum()) > 20 and int((ok.numpy() & near_seam).sum()) > 0


def test_normals_of_none_and_of_more_than_2e24_vertices(two_fields):
    lt = two_fields
    w = torch.stack([x.detach().float() for x in lt.world2rf]).cpu().numpy()
    s, keep = _scene(list(lt.tensorfs), w, 1 / 32, (0.0, 0.0, 0.0), 1.0, 0.05)
    assert _lib.lib().lrf_mesh_normals(C.byref(s), None, 0, None, None, None) == 0
    n = (1 << 24) + 1000
    xyz = np.random.default_rng(2).uniform(-1.5, 1.5, (n, 3)).astype(np.float32)
    own, nrm = _owners(s, xyz)
    assert np.array_equal(own, mo.owner32(xyz, w)[0])
    tail = xyz[-5000:]
    own_t, nrm_t = _owners(s, tail)
    assert np.array_equal(nrm[-5000:].view(np.uint32), nrm_t.view(np.uint32)) and np.array_equal(own[-5000:], own_t)
    assert (np.abs(nrm[-5000:]).sum(1) > 0).any()


# ---- 5. extract conditions -------------------------------------------------------------------------------------
def test_extract_scratch_stream_and_repeats(field_set):
    """A scratch block of 0xFF, a side stream and a second extract of the same table give the same bits; cells of a
    new brick after an extract, then a second extract, give the one-pass mesh."""
    s, keep = _scene(field_set[0].tensorfs, [[0, 0, 0]], VOX, ORIGIN)
    v = _random((40, 41, 42), 11)
    lo = (-20, -20, -20)
    bricks = [((0, 21), (0, 41), (0, 42)), ((20, 40), (0, 41), (0, 42))]
    want = mo.cells_np(v, lo, 0.5, ORIGIN, VOX)
    t, store = _fresh(1 << 18, 1 << 18)
    (x0, x1), (y0, y1), (z0, z1) = bricks[0]
    _cells(s, (lo[0] + x0, lo[1] + y0, lo[2] + z0), (x1 - x0, y1 - y0, z1 - z0), v[x0:x1, y0:y1, z0:z1], t)
    first = _extract(t)
    assert _same(first, mo.cells_np(v[x0:x1], lo, 0.5, ORIGIN, VOX))
    assert _same(_extract(t, fill=0xFF), first)
    # On a non-blocking stream, behind a spin there: the table is zeroed on the current stream and restored on the
    # side stream just before the extract, and the second brick's values are copied there just before the cells, so
    # a launch that ignored the stream argument would read an empty table or stale values.
    side = torch.cuda.Stream()
    snap = store.clone()
    store.zero_()
    assert _same(_extract(t, fill=0xFF, stream=side, before=lambda: store.copy_(snap)), first)
    (x0, x1), (y0, y1), (z0, z1) = bricks[1]
    sub = v[x0:x1, y0:y1, z0:z1]
    _cells(s, (lo[0] + x0, lo[1] + y0, lo[2] + z0), sub.shape, sub, t, stream=side)
    got = _extract(t, fill=0xFF, stream=side)
    assert _same(got, want) and _same(_extract(t), want)


# ---- 6. mesh() -------------------------------------------------------------------------------------------------
def test_mesh_level_above_every_value_is_empty(two_fields):
    m = mesh(two_fields, voxel_size=1 / 32, level=1.5, capacity=1 << 16, max_triangles=1 << 16)
    for k, dt in (("xyz", torch.float32), ("normals", torch.float32), ("rgb", torch.uint8), ("faces", torch.int32)):
        assert m[k].shape == (0, 3) and m[k].dtype == dt and m[k].is_cuda


def _bytes(m):
    return b"".join(m[k].cpu().numpy().tobytes() for k in ("xyz", "normals", "rgb", "faces"))


@pytest.mark.parametrize("where", [0, 1, 2])
@pytest.mark.parametrize("value", [math.nan, math.inf, -math.inf])
def test_mesh_skips_a_non_finite_world2rf_row(two_fields, where, value):
    """A field whose world2rf row has a NaN or infinite component gives the mesh of the scene without it; with no
    finite row the mesh is empty."""
    lt = two_fields
    rfs, ws = list(lt.tensorfs), [x.detach() for x in lt.world2rf]
    scene = lambda r, w: types.SimpleNamespace(tensorfs=r, world2rf=w, blending_weights=lt.blending_weights,
                                               is_refining=lt.is_refining)
    kw = dict(voxel_size=1 / 32, level=0.05, capacity=1 << 18, max_triangles=1 << 19)
    want = mesh(scene(rfs, ws), **kw)
    assert len(want["faces"]) > 1000
    row = torch.zeros(3, device="cuda")
    row[where] = value
    got = mesh(scene(rfs[:1] + [rfs[0]] + rfs[1:], ws[:1] + [row] + ws[1:]), **kw)
    assert _bytes(got) == _bytes(want)
    got = mesh(scene(rfs + [rfs[1]], ws + [row]), **kw)
    assert _bytes(got) == _bytes(want)
    empty = mesh(scene(rfs, [row, row]), **kw)
    assert all(empty[k].shape == (0, 3) for k in ("xyz", "normals", "rgb", "faces"))


def test_mesh_reports_capacity_first_when_both_limits_overflow(two_fields):
    with pytest.raises(RuntimeError, match="capacity / 2 = 32"):
        mesh(two_fields, voxel_size=1 / 32, level=0.05, capacity=64, max_triangles=64)
