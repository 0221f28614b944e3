"""CPU-only: the point-cloud export's numpy restatement (tests/export_oracle.py) on hand-built rays whose keys, fractions
and means are known, localrf_b200.export.write_ply read back by a small parser, the LrfPointFrame / LrfVoxelTable
mirrors, and lrf_ray_opacity / lrf_frame_points / lrf_voxel_extract refusing bad arguments with LRF_ERR_INVALID and a
message before they touch a device (the non-NULL pointers below are never dereferenced)."""
import ctypes as C

import numpy as np
import pytest

import export_oracle as eo
from localrf_b200 import _lib
from localrf_b200.export import write_ply

INVALID = -1
FAKE = 0x10000                       # never read
EYE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)


def _points(p, acc=None, depth=None, rgb=None, world2rf=((0, 0, 0),), blend=None, min_acc=0.5, max_norm=1.0,
            voxel_size=0.25, origin=(0, 0, 0)):
    """Rays of an identity camera whose points are p [n,3] (direction p, depth 1, acc 1 unless given)."""
    p = np.asarray(p, np.float32)
    n = len(p)
    acc = np.ones(n, np.float32) if acc is None else np.asarray(acc, np.float32)
    depth = acc.copy() if depth is None else np.asarray(depth, np.float32)
    rgb = np.full((n, 3), 0.5, np.float32) if rgb is None else np.asarray(rgb, np.float32)
    return eo.ray_points(rgb, depth, acc, p, EYE, world2rf, blend, min_acc, max_norm, voxel_size, origin)


def _k(key):
    return tuple(((int(key) >> (21 * (2 - a))) & ((1 << 21) - 1)) - (1 << 20) for a in range(3))


def test_voxel_boundaries_and_negative_coordinates():
    keep, out, key, fu, cu = _points([[0.5, 0.25, 0.0], [-0.1, -0.75, 0.2]])
    assert keep.all() and not out.any()
    assert _k(key[0]) == (2, 1, 0) and fu[0].tolist() == [0, 0, 0]        # a boundary belongs to the voxel above
    assert _k(key[1]) == (-1, -3, 0)
    q = np.float32(-0.1) / np.float32(0.25)
    assert fu[1, 0] == int((q - np.floor(q)) * np.float32(2 ** 32)) and fu[1, 1] == 0
    assert cu[0].tolist() == [2 ** 23] * 3


def test_fraction_rounding_to_one_saturates():
    keep, _, key, fu, _ = _points([[-1e-10, 0.1, 0.1]], voxel_size=1.0)
    assert keep[0] and _k(key[0]) == (-1, 0, 0)
    assert fu[0, 0] == 2 ** 32 - 1                                        # f = 1.0 in fp32


def test_out_of_range_keys():
    vs = 1 / 256
    lim = 2 ** 20 * vs                                                    # 4096
    keep, out, key, _, _ = _points([[lim - vs, 0, 0], [lim, 0, 0], [-lim, 0, 0], [-lim - vs, 0, 0]],
                                   voxel_size=vs, max_norm=1e5)
    assert keep.tolist() == [True, False, True, False] and out.tolist() == [False, True, False, True]
    assert _k(key[0])[0] == 2 ** 20 - 1 and _k(key[2])[0] == -2 ** 20


def test_depth_and_opacity_rules():
    p = np.full((6, 3), 0.1, np.float32)
    acc = np.array([1, 1, 1, 0.5, np.nextafter(np.float32(0.5), np.float32(0)), 0], np.float32)
    depth = np.array([np.nan, np.inf, -np.inf, 0.5, 0.5, 0.0], np.float32)
    keep, out, _, _, _ = _points(p, acc=acc, depth=depth)
    assert keep.tolist() == [False, False, False, True, False, False] and not out.any()
    keep, _, _, _, _ = _points(p[:1], acc=[0.0], depth=[0.0], min_acc=0.0)   # acc > 0 is required as well
    assert not keep[0]


def test_field_cubes():
    p = [[0.0, 0.0, 0.0], [1.5, 0.0, 0.0], [3.5, 0.0, 0.0], [1.0, 1.0, -1.0]]
    w2 = [[0, 0, 0], [-2, 0, 0], [-4, 0, 0]]
    keep, _, _, _, _ = _points(p, world2rf=w2, max_norm=1.0)
    assert keep.tolist() == [True, True, True, True]
    keep, _, _, _, _ = _points(p, world2rf=w2, blend=[0.3, 0.7, 0.0], max_norm=1.0)
    assert keep.tolist() == [True, True, False, True]
    keep, _, _, _, _ = _points(p, world2rf=w2, blend=[0.0, 1.0, 0.0], max_norm=0.6)
    assert keep.tolist() == [False, True, False, False]


def test_merge_and_extract():
    t = eo.new_table()
    rgb = np.array([[0, 0.5, 1], [1, 1, 1], [0.25, 0.25, 0.25]], np.float32)
    eo.frame_points(t, rgb, np.ones(3, np.float32), np.ones(3, np.float32),
                    np.array([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [-0.1, 0.1, 0.1]], np.float32), EYE, [[0, 0, 0]], None,
                    0.5, 1.0, 0.25, (0, 0, 0))
    assert t["kept"] == 3 and len(t["voxels"]) == 2
    xyz, rgb8, count = eo.extract(t, 1, 0.25, (0, 0, 0))
    assert count.tolist() == [1, 2]                                       # key order: x = -1 first
    assert rgb8.tolist() == [[64, 64, 64], [128, 191, 255]]
    np.testing.assert_allclose(xyz[1], [0.15, 0.15, 0.15], atol=1e-6)
    xyz, _, count = eo.extract(t, 2, 0.25, (0, 0, 0))
    assert count.tolist() == [2] and len(xyz) == 1


def test_ray_opacity_sequential_sum():
    w = np.array([[1.0, 2.0 ** -30, -1.0, 2.0 ** -30]], np.float32)
    assert eo.ray_opacity(w, np.float32(1))[0] == np.float32(2.0 ** -29)
    acc = eo.ray_opacity(w, np.float32(0.5))
    assert eo.ray_opacity(w, np.float32(0.5), acc)[0] == np.float32(2.0 ** -29)


def test_write_ply_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    xyz = rng.standard_normal((37, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (37, 3)).astype(np.uint8)
    path = tmp_path / "cloud.ply"
    write_ply(str(path), xyz, rgb)
    got_xyz, got_rgb = eo.read_ply(path.read_bytes())
    assert np.array_equal(got_xyz, xyz) and np.array_equal(got_rgb, rgb)
    write_ply(str(path), xyz[:0], rgb[:0])
    assert eo.read_ply(path.read_bytes())[0].shape == (0, 3)
    with pytest.raises(ValueError):
        write_ply(str(path), xyz, rgb[:5])


def test_struct_mirrors():
    L = _lib.lib()
    assert L.lrf_sizeof(12) == C.sizeof(_lib.LrfPointFrame) == 8 + 7 * 8 + 3 * 4 + 4
    assert L.lrf_sizeof(13) == C.sizeof(_lib.LrfVoxelTable) == 8 + 4 * 4 + 3 * 8
    assert _lib.LrfPointFrame.max_norm.offset == 72 and _lib.LrfVoxelTable.keys.offset == 24
    for name in ("lrf_ray_opacity", "lrf_frame_points", "lrf_voxel_extract_scratch_bytes", "lrf_voxel_extract"):
        assert name in _lib.EXPORTS
    assert "lrf_export.cu" in _lib.SOURCES


def _table():
    t = _lib.LrfVoxelTable(capacity=1024, voxel_size=0.25, keys=FAKE, sums=FAKE, stats=FAKE)
    return t


def _frame():
    return _lib.LrfPointFrame(n_rays=64, rgb=FAKE, depth=FAKE, acc=FAKE, directions=FAKE, cam2world=FAKE,
                              world2rf=FAKE, blend=None, n_fields=2, min_acc=0.5, max_norm=1.0)


def _refused(rc, text):
    L = _lib.lib()
    assert rc == INVALID
    assert text in L.lrf_last_error(), L.lrf_last_error()


def test_ray_opacity_invalid():
    L = _lib.lib()
    call = lambda w=FAKE, n=64, S=8, V=4, acc=FAKE: L.lrf_ray_opacity(w, n, S, V, None, 0, 0, acc, None)
    _refused(call(w=None), b"weights / acc is NULL")
    _refused(call(acc=None), b"weights / acc is NULL")
    for n, V in ((65, 4), (64, 0), (-4, 4)):
        _refused(call(n=n, V=V), b"multiple of n_views")
    _refused(call(n=2 ** 31, V=1), b"31 bits")
    _refused(call(S=0), b"n_samples")


def test_frame_points_invalid():
    L = _lib.lib()
    _refused(L.lrf_frame_points(None, C.byref(_table()), None), b"frame is NULL")
    _refused(L.lrf_frame_points(C.byref(_frame()), None, None), b"table is NULL")
    for name in ("rgb", "depth", "acc", "directions", "cam2world", "world2rf"):
        f = _frame()
        setattr(f, name, None)
        _refused(L.lrf_frame_points(C.byref(f), C.byref(_table()), None), b"of the frame is NULL")
    for n in (-1, 2 ** 31):
        f = _frame()
        f.n_rays = n
        _refused(L.lrf_frame_points(C.byref(f), C.byref(_table()), None), b"n_rays")
    f = _frame()
    f.n_fields = 0
    _refused(L.lrf_frame_points(C.byref(f), C.byref(_table()), None), b"n_fields")
    for name in ("min_acc", "max_norm"):
        f = _frame()
        setattr(f, name, float("nan"))
        _refused(L.lrf_frame_points(C.byref(f), C.byref(_table()), None), b"is NaN")
    for cap in (0, 1, 3, 1000, 2 ** 31):
        t = _table()
        t.capacity = cap
        _refused(L.lrf_frame_points(C.byref(_frame()), C.byref(t), None), b"power of two")
    for vs in (0.0, -1.0, float("nan"), float("inf")):
        t = _table()
        t.voxel_size = vs
        _refused(L.lrf_frame_points(C.byref(_frame()), C.byref(t), None), b"voxel_size")
    t = _table()
    t.origin[1] = float("inf")
    _refused(L.lrf_frame_points(C.byref(_frame()), C.byref(t), None), b"origin")
    for name in ("keys", "sums", "stats"):
        t = _table()
        setattr(t, name, None)
        _refused(L.lrf_frame_points(C.byref(_frame()), C.byref(t), None), b"of the table is NULL")
        t = _table()
        setattr(t, name, FAKE + 4)
        _refused(L.lrf_frame_points(C.byref(_frame()), C.byref(t), None), b"8-byte aligned")


def test_voxel_extract_invalid():
    L = _lib.lib()
    call = lambda t, mc=1, xyz=FAKE, rgb=FAKE, cnt=FAKE, nv=FAKE, s=FAKE: \
        L.lrf_voxel_extract(C.byref(t) if t is not None else None, mc, xyz, rgb, cnt, nv, s, 1 << 30, None)
    _refused(call(None), b"table is NULL")
    t = _table()
    t.capacity = 6
    _refused(call(t), b"power of two")
    _refused(call(_table(), mc=0), b"min_count")
    for k in ("xyz", "rgb", "cnt", "nv"):
        _refused(call(_table(), **{k: None}), b"is NULL")
    _refused(call(_table(), s=None), b"scratch")
    _refused(call(_table(), s=FAKE + 16), b"256-byte aligned")
    assert L.lrf_voxel_extract_scratch_bytes(6) == 0 and L.lrf_voxel_extract_scratch_bytes(2 ** 31) == 0


def test_voxel_extract_refuses_scratch_smaller_than_its_buffers_without_a_device():
    """A block smaller than the sort's key and slot buffers (two of 8 and two of 4 bytes per slot, each from a 256-byte
    boundary) is refused before the sort-size query, which needs a device; alignment is checked first."""
    L = _lib.lib()
    buffers = 24 * 1024                                             # the table's 1024 slots
    call = lambda s, nbytes: L.lrf_voxel_extract(C.byref(_table()), 1, FAKE, FAKE, FAKE, FAKE, s, nbytes, None)
    for nbytes in (0, 256, buffers - 1):
        _refused(call(FAKE, nbytes), b"scratch_bytes is smaller than lrf_voxel_extract_scratch_bytes(capacity)")
    _refused(call(FAKE + 16, 0), b"256-byte aligned")
    _refused(call(FAKE + 16, buffers - 1), b"256-byte aligned")


def test_point_cloud64_agrees_with_ray_points():
    """The float64 reference on hand-built rays of a rotated, translated camera: the same rays kept and the same
    voxels as the float32 restatement, with no ray near a boundary (so none is ambiguous)."""
    rng = np.random.default_rng(5)
    n = 400
    a, b = 0.4, -0.7
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    c2w = np.concatenate([Rx @ Ry, [[0.1], [-0.2], [0.3]]], 1).astype(np.float32)
    w2rf = np.array([[-0.1, 0.2, -0.3], [-5.0, 0.0, 0.0]], np.float32)
    dirs = np.concatenate([rng.uniform(-0.6, 0.6, (n, 2)), -np.ones((n, 1))], 1).astype(np.float32)
    depth = rng.uniform(0.1, 0.9, n).astype(np.float32)
    acc = rng.uniform(0.0, 1.0, n).astype(np.float32)
    rgb = rng.uniform(-0.2, 1.2, (n, 3)).astype(np.float32)
    depth[:5] = np.nan
    acc[5:10] = 0.0
    blend = np.array([1.0, 0.0], np.float32)
    args = (rgb, depth, acc, dirs)
    vs, origin, min_acc, max_norm = 1 / 32, (0.0, 0.0, 0.0), 0.25, 0.8
    keep, _, key, _, _ = eo.ray_points(*args, c2w, w2rf, blend, min_acc, max_norm, vs, origin)
    ref = eo.point_cloud64([(0, *args)], c2w[None], w2rf, blend[None], min_acc, max_norm, vs, origin)
    assert not ref["ambiguous"] and ref["n_rays"] == n
    assert ref["kept"] == int(keep.sum()) > 100
    want = {}
    for k in key[keep].tolist():
        want[k] = want.get(k, 0) + 1
    assert {k: v[0] for k, v in ref["voxels"].items()} == want
    # x = 0.75 (1 / 3) lies on the face x = 8 voxels in float64; float32's 1 / 3 may put it in voxel 7: ambiguous
    near = eo.point_cloud64([(0, rgb[:1], np.ones(1, np.float32), np.full(1, 3.0, np.float32),
                              np.array([[0.75, 0.9, -1.2]], np.float32))], EYE[None], [[0, 0, 0]], [[1.0]], 0.5, 1.0,
                            vs, origin)
    assert near["ambiguous"] == {(0, 0)}
    assert {eo.pack_key([k, 9, -13]) for k in (7, 8)} <= near["ambiguous_keys"]


def test_probe_table_wraps_at_the_last_slot():
    cap = 64
    cand = np.arange(1, 200000, dtype=np.uint64)
    last = cand[(eo.mix64(cand) & np.uint64(cap - 1)) == cap - 1][:5]
    assert len(last) == 5
    assert eo.probe_table(last, cap) == {63, 0, 1, 2, 3}                  # 63, then wrapped to 0, 1, 2, 3
    assert eo.probe_table(last[::-1], cap) == {63, 0, 1, 2, 3}
    mid = cand[(eo.mix64(cand) & np.uint64(cap - 1)) == 1][:2]
    assert eo.probe_table(np.concatenate([last, mid]), cap) == {63, 0, 1, 2, 3, 4, 5}
    assert int(eo.mix64(np.uint64(0))) == 0 and int(eo.mix64(np.uint64(1))) == 0x5692161d100b05e5
    assert eo.pack_key([-(1 << 20), 0, (1 << 20) - 1]) == (1 << 41) | (1 << 21) - 1
