"""CPU-only: the mesh export's numpy restatement (tests/mesh_oracle.py) on every marching-cubes case and on sampled
solids whose topology and volume are known, localrf_b200.export.write_ply with faces and normals read back, the
LrfMeshScene / LrfMeshTable mirrors, and lrf_mesh_* refusing bad arguments with LRF_ERR_INVALID and a message before
they touch a device (the non-NULL pointers below are never dereferenced)."""
import ctypes as C
import math

import numpy as np
import pytest

import export_oracle as eo
import mesh_oracle as mo
from localrf_b200 import _lib
from localrf_b200.export import write_ply

INVALID = -1
FAKE = 0x10000                       # never read


def _cut_edges(case, cell=(0, 0, 0)):
    """{edge key: edge} of the cut edges of a cell whose inside corners are the set bits of `case`."""
    out = {}
    for e, (a, b) in enumerate(mo.EDGES):
        if ((case >> a) ^ (case >> b)) & 1:
            pa, pb = np.add(cell, mo.CORNERS[a]), np.add(cell, mo.CORNERS[b])
            lo = np.minimum(pa, pb)
            out[mo.edge_key(lo, int(np.argmax(np.abs(pb - pa))))] = e
    return out


@pytest.mark.parametrize("case", range(256))
def test_every_case_cuts_exactly_its_edges(case):
    """A cell alone (values 1 inside, 0 outside, level 0.5): its triangles' vertices are the midpoints of its cut
    edges, every cut edge is used, and nothing else is."""
    v = np.zeros((2, 2, 2), np.float32)
    for c, (x, y, z) in enumerate(mo.CORNERS):
        v[x, y, z] = 1.0 if (case >> c) & 1 else 0.0
    edges, tris = mo.cells(v, (3, -2, 5), 0.5, (0.0, 0.0, 0.0), 0.25)
    want = _cut_edges(case, (3, -2, 5))
    assert set(edges) == set(want)
    assert {k for t in tris for k in t[1:]} == set(want)
    assert len(tris) == mo.N_TRI[case] and [t[0] & 7 for t in tris] == list(range(len(tris)))
    for k, e in want.items():
        a, b = mo.EDGES[e]
        mid = (np.add((3, -2, 5), mo.CORNERS[a]) + np.add((3, -2, 5), mo.CORNERS[b])) * 0.5 * 0.25
        assert np.array_equal(edges[k], mid.astype(np.float32))


@pytest.mark.parametrize("seed", range(12))
def test_random_lattices_mesh_closed_and_oriented(seed):
    """Random lattices whose border is outside: every directed edge is used once and its reverse once.  This is what
    validates the copied table (all 256 cases occur in these lattices)."""
    rng = np.random.default_rng(seed)
    n = 12
    v = rng.random((n, n, n)).astype(np.float32)
    v[[0, -1]] = v[:, [0, -1]] = v[:, :, [0, -1]] = 0.0
    level = np.float32(rng.uniform(0.3, 0.7))
    xyz, faces = mo.mesh_lattice(v, (-5, 0, 7), level, (0.5, -0.25, 0.0), 0.125)
    assert len(faces) > 100 and mo.is_closed_oriented(faces)
    assert faces.min() >= 0 and faces.max() < len(xyz) and len(np.unique(faces)) == len(xyz)
    assert mo.signed_volume(xyz, faces) > 0


def test_random_lattices_cover_every_case():
    seen = set()
    for seed in range(12):
        rng = np.random.default_rng(seed)
        v = rng.random((12, 12, 12)) >= rng.uniform(0.3, 0.7)
        idx = np.zeros((11, 11, 11), np.int64)
        for c, (x, y, z) in enumerate(mo.CORNERS):
            idx |= v[x:x + 11, y:y + 11, z:z + 11].astype(np.int64) << c
        seen |= set(np.unique(idx).tolist())
    assert len(seen) == 256


def _sampled(fn, n, vox, org):
    g = np.stack(np.meshgrid(*[np.float32(org[a]) + np.arange(n, dtype=np.float32) * np.float32(vox) for a in range(3)],
                             indexing="ij"), -1).astype(np.float64)
    return fn(g).astype(np.float32)


def test_ball_has_euler_characteristic_two_and_its_volume():
    r, vox, n, org = 0.8, 0.05, 40, (-1.0, -1.0, -1.0)
    v = _sampled(lambda g: 1.0 - np.linalg.norm(g, axis=-1) / r, n, vox, org)      # >= 0 inside the ball
    xyz, faces = mo.mesh_lattice(v, (0, 0, 0), 1e-6, org, vox)
    assert mo.is_closed_oriented(faces) and mo.euler_characteristic(xyz, faces) == 2
    vol, want = mo.signed_volume(xyz, faces), 4 / 3 * math.pi * r ** 3
    assert 0 < vol and abs(vol - want) <= 4 * math.pi * r ** 2 * vox ** 2 / r    # chords: O(h^2 / r) per area
    assert np.abs(np.linalg.norm(xyz.astype(np.float64), axis=1) - r).max() <= vox


def test_torus_has_euler_characteristic_zero_and_its_volume():
    R, r, vox, n, org = 0.6, 0.25, 0.04, 50, (-1.0, -1.0, -1.0)
    v = _sampled(lambda g: r - np.hypot(np.hypot(g[..., 0], g[..., 1]) - R, g[..., 2]), n, vox, org)
    xyz, faces = mo.mesh_lattice(v, (0, 0, 0), 1e-7, org, vox)
    assert mo.is_closed_oriented(faces) and mo.euler_characteristic(xyz, faces) == 0
    vol, want = mo.signed_volume(xyz, faces), 2 * math.pi ** 2 * R * r ** 2
    assert 0 < vol and abs(vol - want) <= 4 * math.pi ** 2 * R * r * vox ** 2 / r


def test_values_on_the_level_and_nan():
    """A corner exactly on the level is inside (t = 1 from below, 0 from above); a NaN corner is outside and its
    edges' t is not finite, so their vertex sits on the lower point."""
    v = np.zeros((2, 2, 2), np.float32)
    v[1, 0, 0] = 0.5
    edges, _ = mo.cells(v, (0, 0, 0), 0.5, (0, 0, 0), 1.0)
    assert np.array_equal(edges[mo.edge_key((0, 0, 0), 0)], np.float32([1, 0, 0]))
    v[1, 0, 0], v[0, 0, 0] = np.nan, 1.0
    edges, _ = mo.cells(v, (0, 0, 0), 0.5, (0, 0, 0), 1.0)
    assert np.array_equal(edges[mo.edge_key((0, 0, 0), 0)], np.float32([0, 0, 0]))
    assert mo.case_index(v[[0, 1, 1, 0, 0, 1, 1, 0], [0, 0, 1, 1, 0, 0, 1, 1], [0, 0, 0, 0, 1, 1, 1, 1]], 0.5) == 1


def test_ply_round_trip_with_faces_and_normals(tmp_path):
    rng = np.random.default_rng(0)
    xyz = rng.standard_normal((9, 3)).astype(np.float32)
    nrm = rng.standard_normal((9, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (9, 3)).astype(np.uint8)
    faces = rng.integers(0, 9, (5, 3)).astype(np.int32)
    p = tmp_path / "m.ply"
    write_ply(p, xyz, rgb, faces=faces, normals=nrm)
    x, n, c, f = mo.read_mesh_ply(p.read_bytes())
    assert np.array_equal(x, xyz) and np.array_equal(n, nrm) and np.array_equal(c, rgb) and np.array_equal(f, faces)
    write_ply(p, xyz, rgb, faces=faces)
    x, n, c, f = mo.read_mesh_ply(p.read_bytes())
    assert n is None and np.array_equal(f, faces)


def test_ply_without_faces_or_normals_is_unchanged(tmp_path):
    """The bytes of a point cloud's PLY: the header and records the point-cloud export has always written."""
    rng = np.random.default_rng(1)
    xyz = rng.standard_normal((7, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (7, 3)).astype(np.uint8)
    p = tmp_path / "c.ply"
    write_ply(p, xyz, rgb)
    head = (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty float x\nproperty float y\n"
            b"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    body = b"".join(xyz[i].tobytes() + rgb[i].tobytes() for i in range(7))
    assert p.read_bytes() == head + body
    x, c = eo.read_ply(p.read_bytes())
    assert np.array_equal(x, xyz) and np.array_equal(c, rgb)


def test_struct_mirrors():
    L = _lib.lib()
    assert L.lrf_sizeof(14) == C.sizeof(_lib.LrfMeshScene) == 56
    assert L.lrf_sizeof(15) == C.sizeof(_lib.LrfMeshTable) == 56
    assert L.lrf_sizeof(16) == 0


def _scene(**kw):
    fields = (_lib.LrfField * 2)()
    steps = (C.c_float * 2)(0.01, 0.01)
    s = _lib.LrfMeshScene(n_fields=2, fields=fields, step_size=steps, world2rf=FAKE, voxel_size=0.25, max_norm=1.0,
                          level=0.005)
    for k, v in kw.items():
        setattr(s, k, v)
    return s, fields, steps


def _table(**kw):
    t = _lib.LrfMeshTable(capacity=1 << 10, max_triangles=1 << 10, keys=FAKE, verts=FAKE, tri_keys=FAKE,
                          tri_slots=FAKE, stats=FAKE)
    for k, v in kw.items():
        setattr(t, k, v)
    return t


def _err(rc, text):
    assert rc == INVALID, rc
    assert text in _lib.lib().lrf_last_error().decode()


@pytest.mark.parametrize("kw, text", [
    (dict(n_fields=0), "n_fields"), (dict(n_fields=65), "n_fields"), (dict(world2rf=None), "world2rf"),
    (dict(voxel_size=0.0), "voxel_size"), (dict(voxel_size=math.inf), "voxel_size"),
    (dict(max_norm=-1.0), "max_norm"), (dict(level=0.0), "level"), (dict(level=math.nan), "level"),
])
def test_scene_refusals(kw, text):
    L = _lib.lib()
    s, keep, keep2 = _scene(**kw)
    lo, d = (C.c_int32 * 3)(0, 0, 0), (C.c_int32 * 3)(4, 4, 4)
    _err(L.lrf_mesh_lattice(C.byref(s), lo, d, FAKE, None), text)
    _err(L.lrf_mesh_cells(C.byref(s), lo, d, FAKE, C.byref(_table()), None), text)
    _err(L.lrf_mesh_normals(C.byref(s), FAKE, 1, FAKE, FAKE, None), text)


def test_null_scene_origin_and_step_refusals():
    L = _lib.lib()
    lo, d = (C.c_int32 * 3)(0, 0, 0), (C.c_int32 * 3)(4, 4, 4)
    _err(L.lrf_mesh_lattice(None, lo, d, FAKE, None), "scene is NULL")
    s, keep, keep2 = _scene()
    s.origin[1] = math.nan
    _err(L.lrf_mesh_lattice(C.byref(s), lo, d, FAKE, None), "origin")
    s.origin[1] = 0.0
    assert L.lrf_mesh_lattice(C.byref(s), lo, d, FAKE, None) == -2        # a zeroed LrfField: 0 components
    assert b"density_n_comp" in L.lrf_last_error()


def _valid_field():
    """A field make_field accepts (pointers never dereferenced)."""
    f = _lib.LrfField()
    f.n_dcomp, f.n_acomp = 8, 24
    for a in range(3):
        f.grid[a] = 4
        f.aabb[a], f.aabb[3 + a] = -2.0, 2.0
    for i in range(3):
        f.dplane[i] = f.dline[i] = f.aplane[i] = f.aline[i] = FAKE
    return f


def test_brick_table_and_output_refusals():
    L = _lib.lib()
    fields = (_lib.LrfField * 1)(_valid_field())
    steps = (C.c_float * 1)(0.01)
    s = _lib.LrfMeshScene(n_fields=1, fields=fields, step_size=steps, world2rf=FAKE, voxel_size=0.25, max_norm=1.0,
                          level=0.005)
    lo = (C.c_int32 * 3)(0, 0, 0)
    for d, text in [((1, 4, 4), "dims >= 2"), ((4, 4, (1 << 19) + 1), "[-2^19, 2^19)"),
                    ((2048, 2048, 2048), "< 2^31")]:
        _err(L.lrf_mesh_lattice(C.byref(s), lo, (C.c_int32 * 3)(*d), FAKE, None), text)
    _err(L.lrf_mesh_lattice(C.byref(s), (C.c_int32 * 3)(-(1 << 19) - 1, 0, 0), (C.c_int32 * 3)(4, 4, 4), FAKE, None),
         "[-2^19, 2^19)")
    d = (C.c_int32 * 3)(4, 4, 4)
    _err(L.lrf_mesh_lattice(C.byref(s), lo, d, None, None), "values is NULL")
    _err(L.lrf_mesh_cells(C.byref(s), lo, d, FAKE, None, None), "table is NULL")
    for kw, text in [(dict(capacity=3), "capacity"), (dict(capacity=1 << 31), "capacity"),
                     (dict(max_triangles=0), "max_triangles"), (dict(max_triangles=1 << 31), "max_triangles"),
                     (dict(tri_slots=None), "NULL"), (dict(keys=FAKE + 4), "aligned"), (dict(verts=FAKE + 2), "aligned")]:
        _err(L.lrf_mesh_cells(C.byref(s), lo, d, FAKE, C.byref(_table(**kw)), None), text)
        _err(L.lrf_mesh_extract(C.byref(_table(**kw)), FAKE, FAKE, FAKE, FAKE, 1 << 30, None), text)
    _err(L.lrf_mesh_extract(C.byref(_table()), None, FAKE, FAKE, FAKE, 1 << 30, None), "NULL")
    _err(L.lrf_mesh_extract(C.byref(_table()), FAKE, FAKE, FAKE, FAKE + 8, 1 << 30, None), "256-byte")
    assert L.lrf_mesh_extract_scratch_bytes(3, 16) == 0 and L.lrf_mesh_extract_scratch_bytes(16, 0) == 0
    assert L.lrf_mesh_extract_scratch_bytes(16, 1 << 31) == 0
    # a block smaller than its buffers (the cell sort's 24 bytes per slot, 4 per slot of the extract's own, the
    # triangle sort's 24 per triangle, each array from a 256-byte boundary) is refused before the sort-size query,
    # which needs a device; alignment is checked first
    buffers = 24 * 1024 + 4 * 1024 + 24 * 1024
    for nbytes in (0, 24 * 1024, buffers - 1):
        _err(L.lrf_mesh_extract(C.byref(_table()), FAKE, FAKE, FAKE, FAKE, nbytes, None),
             "scratch_bytes is smaller than lrf_mesh_extract_scratch_bytes(capacity, max_triangles)")
    _err(L.lrf_mesh_extract(C.byref(_table()), FAKE, FAKE, FAKE, FAKE + 8, buffers - 1, None), "256-byte")
    _err(L.lrf_mesh_normals(C.byref(s), FAKE, -1, FAKE, FAKE, None), "n must")
    _err(L.lrf_mesh_normals(C.byref(s), None, 3, FAKE, FAKE, None), "NULL")
    bad = _valid_field()
    bad.grid_dtype = _lib.GRID_BF16
    s.fields = (_lib.LrfField * 1)(bad)
    assert L.lrf_mesh_lattice(C.byref(s), lo, d, FAKE, None) == -2
    s.fields = fields
    steps[0] = 0.0
    _err(L.lrf_mesh_lattice(C.byref(s), lo, d, FAKE, None), "step_size")


def test_mesh_bricks_skip_non_finite_world2rf_rows():
    """A world2rf row with a NaN or infinite component owns no lattice point, so it adds no brick; with no finite row
    there is none."""
    from localrf_b200.export import _mesh_bricks
    args = (0.25, [0.0, 0.5, -0.5], 1.0, 4)
    want = _mesh_bricks([[0.0, 0.0, 0.0], [0.5, -0.25, 0.0]], *args)
    assert len(want) > 8
    rows = [[math.nan, 0.0, 0.0], [0.0, math.inf, 0.0], [0.0, 0.0, -math.inf], [math.nan] * 3]
    assert _mesh_bricks([rows[0], [0.0, 0.0, 0.0], rows[1], [0.5, -0.25, 0.0], rows[2], rows[3]], *args) == want
    assert _mesh_bricks(rows, *args) == []
