"""CPU-only: the connected-components restatement (tests/components_oracle.py) on hand-built meshes and clouds, and
lrf_mesh_components / lrf_point_components / lrf_components_select refusing bad arguments with LRF_ERR_INVALID and a
message before they touch a device (the non-NULL pointers below are never dereferenced).  The entries take plain
arguments, so no struct is added: lrf_sizeof 16, 18 and 19 stay 0."""
import ctypes as C
import math

import numpy as np
import pytest

import components_oracle as co
from localrf_b200 import _lib

INVALID = -1
FAKE = 0x10000                       # never read
ORIGIN = (C.c_float * 3)(0.0, 0.0, 0.0)


def test_mesh_oracle_on_hand_built_graphs():
    # two triangles sharing an edge, one apart, an unused vertex, a degenerate triangle, an out-of-range one
    faces = [[4, 5, 6], [2, 1, 0], [1, 3, 2], [7, 7, 8], [10, 0, 1], [-1, 2, 3]]
    label, size, bad = co.mesh_components(faces, 10)
    assert label.tolist() == [0, 0, 0, 0, 4, 4, 4, 7, 7, 9] and bad == 2
    assert size.tolist() == [2, 0, 0, 0, 1, 0, 0, 1, 0, 0]
    s = co.select(label, size)
    assert s["sizes"].tolist() == [2, 1, 1, 0] and s["counts"] == [10, 4, 4, 4]
    assert s["new_index"].tolist() == list(range(10)) and s["rank"].tolist() == [0, 0, 0, 0, 1, 1, 1, 2, 2, 3]
    s = co.select(label, size, keep=1)
    assert s["new_index"].tolist() == [0, 1, 2, 3] + [-1] * 6 and s["counts"] == [4, 1, 4, 2]
    s = co.select(label, size, min_size=1)                       # the tie 4 / 7 ranks the lower label first
    assert s["new_index"].tolist() == [0, 1, 2, 3, 4, 5, 6, 7, 8, -1]
    assert s["rank"].tolist() == [0] * 4 + [1] * 3 + [2] * 2
    s = co.select(label, size, keep=2, min_size=2)
    assert s["counts"] == [4, 1, 4, 2]
    xyz = np.arange(30, dtype=np.float32).reshape(10, 3)
    valid = [f for f in faces if 0 <= min(f) and max(f) < 10]
    kx, kf, _ = co.keep_mesh(xyz, valid, co.select(label, size, min_size=1)["new_index"])
    assert len(kx) == 9 and kf.tolist() == [[4, 5, 6], [2, 1, 0], [1, 3, 2], [7, 7, 8]]


def test_mesh_oracle_without_faces_and_vertices():
    label, size, bad = co.mesh_components(np.zeros((0, 3), np.int32), 5)
    assert label.tolist() == list(range(5)) and size.tolist() == [0] * 5 and bad == 0
    label, size, bad = co.mesh_components([[0, 1, 2]], 0)
    assert len(label) == 0 and bad == 1
    assert co.select(label, size)["counts"] == [0, 0, 0, 0]


def test_point_oracle_cells_and_neighbours():
    h = 0.5
    pts = np.array([[0.1, 0.1, 0.1], [0.4, 0.2, 0.3],          # one cell
                    [0.6, 0.6, 0.6],                             # its corner neighbour
                    [2.1, 0.1, 0.1],                             # cell (4, 0, 0): apart
                    [1.5, 0.0, 0.0],                             # exactly on a boundary: cell (3, 0, 0), next to [3]
                    [np.nan, 0, 0], [np.inf, 0, 0],              # not finite
                    [-0.01, -0.01, -0.01],                       # cell (-1, -1, -1): corner of the first
                    [h * (1 << 20), 0, 0], [-h * (1 << 20), 0, 0]], np.float32)   # out of range / the lowest cell
    ok, ki, _ = co.cells(pts, (0, 0, 0), h)
    assert ok.tolist() == [True] * 5 + [False, False, True, False, True]
    assert ki[4].tolist() == [3, 0, 0] and ki[7].tolist() == [-1, -1, -1] and ki[9].tolist() == [-(1 << 20), 0, 0]
    label, size, n_cells, n_out = co.point_components(pts, (0, 0, 0), h)
    assert label.tolist() == [0, 0, 0, 3, 3, 5, 6, 0, 8, 9] and n_out == 3 and n_cells == 6
    assert size.tolist() == [4, 0, 0, 2, 0, 1, 1, 0, 1, 1]
    s = co.select(label, size, keep=1)
    assert s["new_index"].tolist() == [0, 1, 2, -1, -1, -1, -1, 3, -1, -1] and s["counts"] == [4, 1, 6, 4]


def test_struct_ids_stay_free():
    L = _lib.lib()
    assert L.lrf_sizeof(16) == 0 and L.lrf_sizeof(18) == 0 and L.lrf_sizeof(19) == 0
    for name in ("lrf_mesh_components", "lrf_point_components", "lrf_components_select_scratch_bytes",
                 "lrf_components_select"):
        assert name in _lib.EXPORTS


def _err(rc, text):
    assert rc == INVALID, rc
    assert text in _lib.lib().lrf_last_error().decode()


def _mesh(faces=FAKE, T=10, V=10, label=FAKE, size=FAKE, stats=FAKE):
    return _lib.lib().lrf_mesh_components(faces, T, V, label, size, stats, None)


@pytest.mark.parametrize("kw, text", [
    (dict(T=-1), "n_triangles and n_vertices"), (dict(T=1 << 31), "n_triangles and n_vertices"),
    (dict(V=-1), "n_triangles and n_vertices"), (dict(V=1 << 31), "n_triangles and n_vertices"),
    (dict(faces=None), "faces"), (dict(faces=FAKE + 2), "faces"), (dict(label=None), "label / size"),
    (dict(size=None), "label / size"), (dict(stats=None), "stats"), (dict(stats=None, V=0, T=0), "stats"),
    (dict(label=FAKE + 2), "aligned"), (dict(size=FAKE + 4), "aligned"), (dict(stats=FAKE + 4), "aligned"),
])
def test_mesh_refusals(kw, text):
    _err(_mesh(**kw), text)


def _points(xyz=FAKE, n=10, origin=ORIGIN, cell=0.5, keys=FAKE, first=FAKE, cap=16, label=FAKE, size=FAKE, stats=FAKE):
    return _lib.lib().lrf_point_components(xyz, n, origin, cell, keys, first, cap, label, size, stats, None)


def _origin(*v):
    return (C.c_float * 3)(*v)


@pytest.mark.parametrize("kw, text", [
    (dict(n=-1), "n must"), (dict(n=1 << 31), "n must"), (dict(xyz=None), "xyz"), (dict(xyz=FAKE + 2), "xyz"),
    (dict(origin=_origin(math.nan, 0, 0)), "origin"), (dict(origin=_origin(0, math.inf, 0)), "origin"),
    (dict(cell=0.0), "cell_size"), (dict(cell=-1.0), "cell_size"), (dict(cell=math.inf), "cell_size"),
    (dict(cell=math.nan), "cell_size"), (dict(cap=0), "capacity"), (dict(cap=1), "capacity"),
    (dict(cap=12), "capacity"), (dict(cap=1 << 31), "capacity"), (dict(cap=-16), "capacity"),
    (dict(keys=None), "keys"), (dict(first=None), "keys"), (dict(keys=FAKE + 4), "keys"),
    (dict(first=FAKE + 2), "keys"), (dict(label=None), "label / size"), (dict(size=None), "label / size"),
    (dict(stats=None), "stats"), (dict(size=FAKE + 4), "aligned"),
])
def test_point_refusals(kw, text):
    _err(_points(**kw), text)


def test_point_origin_pointer():
    L = _lib.lib()
    L2 = C.CDLL(_lib.LIB_PATH)                                  # a NULL origin, which the bound argtypes cannot pass
    L2.lrf_last_error.restype = C.c_char_p
    rc = L2.lrf_point_components(C.c_void_p(FAKE), C.c_int64(10), None, C.c_float(0.5), C.c_void_p(FAKE),
                                 C.c_void_p(FAKE), C.c_int64(16), C.c_void_p(FAKE), C.c_void_p(FAKE), C.c_void_p(FAKE),
                                 None)
    assert rc == INVALID and b"origin" in L.lrf_last_error()


def _select(label=FAKE, size=FAKE, n=10, keep=0, min_size=0, new_index=FAKE, rank=FAKE, sizes=FAKE, counts=FAKE,
            scratch=0x100000, nbytes=1 << 20):
    return _lib.lib().lrf_components_select(label, size, n, keep, min_size, new_index, rank, sizes, counts, scratch,
                                            nbytes, None)


@pytest.mark.parametrize("kw, text", [
    (dict(n=-1), "n must"), (dict(n=1 << 31), "n must"), (dict(keep=-1), "keep and min_size"),
    (dict(min_size=-1), "keep and min_size"), (dict(counts=None), "counts"), (dict(counts=FAKE + 4), "counts"),
    (dict(counts=None, n=0), "counts"), (dict(label=None), "NULL"), (dict(size=None), "NULL"),
    (dict(new_index=None), "NULL"), (dict(rank=None), "NULL"), (dict(sizes=None), "NULL"),
    (dict(label=FAKE + 2), "aligned"), (dict(rank=FAKE + 2), "aligned"), (dict(sizes=FAKE + 4), "aligned"),
    (dict(size=FAKE + 4), "aligned"), (dict(scratch=None), "scratch"), (dict(scratch=0x100000 + 128), "256-byte"),
    (dict(nbytes=0), "scratch_bytes"), (dict(nbytes=16 * 10), "scratch_bytes"),
    (dict(n=1 << 20, nbytes=1 << 20), "scratch_bytes"),
])
def test_select_refusals(kw, text):
    _err(_select(**kw), text)


def test_select_scratch_bytes_refuses_out_of_range_counts():
    L = _lib.lib()
    assert L.lrf_components_select_scratch_bytes(-1) == 0 and L.lrf_components_select_scratch_bytes(1 << 31) == 0
