"""-m gpu: the point-cloud export at the edges of its C ABI (include/localrf_b200.h lrf_ray_opacity / lrf_frame_points /
lrf_voxel_extract, localrf_b200.export.point_cloud).  The kernels equal their numpy restatement (tests/export_oracle.py)
bit for bit, with canaries around every output, at the tile and CTA edges of the opacity sum, on hand-built rays at the
value edges of the back-projection and the key, on tables at exactly half full, one voxel past it, with forced probe
collisions and wrap-around, under heavy atomic contention, and on tables written word by word.  On scenes of every
kind the exporter supports, the cloud also agrees with an independent float64 reference (export_oracle.point_cloud64)
that shares none of the kernels' conventions, and slabs seen from rotated cameras and through offset fields export onto
their planes."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import export_oracle as eo
import localrf_b200 as L
from localrf_b200 import _lib
from localrf_b200.export import _voxel_table, point_cloud
from test_gpu_export import CANARY_F, PAD, _extract, _frame_points, _padded, _rot

pytestmark = pytest.mark.gpu

EYE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)
LIM = 1 << 20


def _bits_equal(a, b):
    """float32 arrays equal bit for bit, except that any NaN equals any NaN (payloads are not specified)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and \
        np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


# ---- 1. lrf_ray_opacity ------------------------------------------------------------------------------------------
def _opacity(w, n_views, blend, stride, acc0=None, offset=0):
    """One lrf_ray_opacity launch into a canary-padded acc (pre-filled with acc0 when accumulating) -> acc [n]."""
    n, S = w.shape
    acc = _padded(n, 0, torch.float32, CANARY_F)
    if acc0 is not None:
        acc[PAD:PAD + n] = torch.from_numpy(acc0).cuda()
    wd = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    bd = None if blend is None else torch.from_numpy(np.ascontiguousarray(blend, np.float32)).cuda()
    _lib.check(_lib.lib().lrf_ray_opacity(wd.data_ptr(), n, S, n_views, None if bd is None else bd.data_ptr() + 4 * offset,
                                          stride, int(acc0 is not None), acc[PAD:].data_ptr(), None))
    torch.cuda.synchronize()
    assert bool((acc[:PAD] == CANARY_F).all()) and bool((acc[PAD + n:] == CANARY_F).all()), "a canary was overwritten"
    return acc[PAD:PAD + n].cpu().numpy()


def _weights(n, S, seed):
    rng = np.random.default_rng(seed)
    w = (rng.uniform(0, 1, (n, S)) ** 6).astype(np.float32)
    w[rng.uniform(size=(n, S)) < 0.2] = 0.0
    return w


@pytest.mark.parametrize("S", [1, 31, 32, 33, 64, 65, 1065])
@pytest.mark.parametrize("n", [1, 127, 128, 129])
@pytest.mark.parametrize("mode", ["per_ray", "one_view", "null_blend", "stride0"])
def test_ray_opacity_tiles_ctas_and_blends(S, n, mode):
    w = _weights(n, S, 7 * S + n)
    rng = np.random.default_rng(n)
    if mode == "per_ray":                       # n views of one ray, the blend column 1 of [n, 3] rows
        V, blend, stride, off = n, rng.uniform(0, 1, (n, 3)).astype(np.float32), 3, 1
        b = blend[:, 1]
    elif mode == "one_view":
        V, blend, stride, off = 1, np.array([0.375, 0.8125], np.float32), 0, 1
        b = np.full(n, blend[1], np.float32)
    elif mode == "null_blend":                  # blend taken as 1
        V, blend, stride, off = 1, None, 0, 0
        b = np.ones(n, np.float32)
    else:                                       # every view reads blend[0]
        V, blend, stride, off = n, np.array([0.625], np.float32), 0, 0
        b = np.full(n, blend[0], np.float32)
    got = _opacity(w, V, blend, stride, offset=off)
    assert _bits_equal(got, eo.ray_opacity(w, b))
    if mode == "null_blend":
        assert _bits_equal(got, np.cumsum(w.astype(np.float64), 1)[:, -1].astype(np.float32))


@pytest.mark.parametrize("S", [1, 33, 65])
def test_ray_opacity_2e20_rays(S):
    n = (1 << 20) + 1
    w = _weights(n, S, S)
    blend = np.array([0.7], np.float32)
    assert _bits_equal(_opacity(w, 1, blend, 0), eo.ray_opacity(w, blend[0]))
    assert _bits_equal(_opacity(w, 1, None, 0), eo.ray_opacity(w, np.float32(1)))


def test_ray_opacity_accumulates_fields_of_different_sample_counts():
    n, V = 640, 5
    rng = np.random.default_rng(3)
    blend = rng.uniform(0, 1, (V, 8)).astype(np.float32)
    blend[2, 3] = 0.0
    acc = want = None
    for k, S in enumerate([1, 31, 32, 33, 64, 65, 344, 1065]):
        w = _weights(n, S, S + k)
        acc = _opacity(w, V, blend, 8, acc0=acc, offset=k)
        want = eo.ray_opacity(w, blend[:, k].repeat(n // V), want)
        assert _bits_equal(acc, want)


def test_ray_opacity_special_values():
    """Subnormals, -0, negative weights, +inf and NaN: the fp64 sum in sample order propagates them as np.cumsum does
    (a row of -0 sums to -0; inf - inf and anything with NaN is NaN; a subnormal survives the conversion)."""
    tiny = np.float32(1e-45)
    rows = [[-0.0], [-0.0, -0.0, -0.0], [0.0, -0.0], [tiny], [tiny] * 40, [1.0, -1.0], [-0.25, 0.125],
            [np.inf, 1.0], [np.inf, -np.inf], [np.nan, 1.0], [1.0] * 32 + [np.nan], [3e38, 3e38, -3e38],
            [1.0, 2.0 ** -30, -1.0, 2.0 ** -30], [-np.inf], [np.float32(1.1754942e-38), -tiny]]
    for S in (1, 3, 33, 70):
        w = np.zeros((len(rows) * 3, S), np.float32)
        for i, r in enumerate(rows):
            w[i, :min(len(r), S)] = r[:S]
            w[len(rows) + i, S - min(len(r), S):] = r[:S]        # at the end of the row
        w[2 * len(rows):] = -0.0
        for b in (np.float32(1), np.float32(0.5), np.float32(-2)):
            got = _opacity(w, 1, np.array([b], np.float32), 0)
            assert _bits_equal(got, eo.ray_opacity(w, b)), (S, b)
        got = _opacity(w, 1, None, 0)
        want = eo.ray_opacity(w, np.float32(1))
        assert _bits_equal(got, want)
        assert np.signbit(got[2 * len(rows):]).all() and (got[2 * len(rows):] == 0).all()      # -0 stays -0


# ---- 2. lrf_frame_points at value edges ----------------------------------------------------------------------------
def _on_device(rgb, depth, acc, dirs, c2w=EYE, w2rf=((0, 0, 0),), blend=None, min_acc=0.5, max_norm=1.0, vs=0.25,
               origin=(0, 0, 0), cap=1024, min_count=1):
    """Runs one frame through lrf_frame_points and lrf_voxel_extract and the restatement; asserts they agree bit
    for bit, stats included -> (keep, out, cloud)."""
    n = len(acc)
    args = [np.ascontiguousarray(a, np.float32) for a in (rgb, depth, acc, dirs, c2w)]
    w2 = np.asarray(w2rf, np.float32).reshape(-1, 3)
    bl = None if blend is None else np.asarray(blend, np.float32)
    t, store = _voxel_table(cap, vs, origin, "cuda")
    _frame_points(t, *args, w2, bl, min_acc, max_norm)
    table = eo.new_table()
    eo.frame_points(table, *args, w2, bl, min_acc, max_norm, vs, origin)
    keep, out, _, _, _ = eo.ray_points(*args, w2, bl, min_acc, max_norm, vs, origin)
    xyz, rgb8, count, stats = _extract(t, store, min_count)
    want = eo.extract(table, min_count, vs, origin)
    assert stats[0] == table["kept"] == int(keep.sum()) and stats[1] == table["out_of_range"] == int(out.sum())
    assert stats[2] == len(table["voxels"]) and n == len(keep)
    assert _bits_equal(xyz, want[0]) and np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2])
    return keep, out, (xyz, rgb8, count)


def _rays(p, acc=None, depth=None, rgb=None):
    """rgb, depth, acc, dirs of identity-camera rays whose points are p (direction p, depth = acc = 1 unless given)."""
    p = np.asarray(p, np.float32)
    acc = np.ones(len(p), np.float32) if acc is None else np.asarray(acc, np.float32)
    depth = acc.copy() if depth is None else np.asarray(depth, np.float32)
    rgb = np.full((len(p), 3), 0.5, np.float32) if rgb is None else np.asarray(rgb, np.float32)
    return rgb, depth, acc, p


def test_frame_points_hand_built_cases():
    """Every hand-built case of test_export_cpu.py, on the device."""
    keep, out, (xyz, _, count) = _on_device(*_rays([[0.5, 0.25, 0.0], [-0.1, -0.75, 0.2]]))
    assert keep.all() and len(count) == 2
    keep, _, (xyz, _, _) = _on_device(*_rays([[-1e-10, 0.1, 0.1]]), vs=1.0)
    assert keep[0] and xyz[0, 0] == np.float32(-1.0 + (2 ** 32 - 1) / 2 ** 32)          # the saturated fraction
    vs = 1 / 256
    lim = LIM * vs
    keep, out, _ = _on_device(*_rays([[lim - vs, 0, 0], [lim, 0, 0], [-lim, 0, 0], [-lim - vs, 0, 0]]), vs=vs,
                              max_norm=1e5)
    assert keep.tolist() == [True, False, True, False] and out.tolist() == [False, True, False, True]
    p = np.full((6, 3), 0.1, np.float32)
    acc = np.array([1, 1, 1, 0.5, np.nextafter(np.float32(0.5), np.float32(0)), 0], np.float32)
    depth = np.array([np.nan, np.inf, -np.inf, 0.5, 0.5, 0.0], np.float32)
    keep, _, _ = _on_device(*_rays(p, acc=acc, depth=depth))
    assert keep.tolist() == [False, False, False, True, False, False]
    keep, _, _ = _on_device(*_rays(p[:1], acc=[0.0], depth=[0.0]), min_acc=0.0)
    assert not keep[0]
    pc = [[0.0, 0.0, 0.0], [1.5, 0.0, 0.0], [3.5, 0.0, 0.0], [1.0, 1.0, -1.0]]
    w2 = [[0, 0, 0], [-2, 0, 0], [-4, 0, 0]]
    for blend, mn, want in ((None, 1.0, [True] * 4), ([0.3, 0.7, 0.0], 1.0, [True, True, False, True]),
                            ([0.0, 1.0, 0.0], 0.6, [False, True, False, False])):
        keep, _, _ = _on_device(*_rays(pc), w2rf=w2, blend=blend, max_norm=mn)
        assert keep.tolist() == want
    rgb = np.array([[0, 0.5, 1], [1, 1, 1], [0.25, 0.25, 0.25]], np.float32)
    _, _, (_, rgb8, count) = _on_device(*_rays([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [-0.1, 0.1, 0.1]], rgb=rgb))
    assert count.tolist() == [1, 2] and rgb8.tolist() == [[64, 64, 64], [128, 191, 255]]
    _, _, (_, _, count) = _on_device(*_rays([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [-0.1, 0.1, 0.1]]), min_count=2)
    assert count.tolist() == [2]


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_frame_points_key_limits(axis):
    """Keys at -2^20 and 2^20 - 1 on each axis (kept) and one voxel beyond either (out of range)."""
    vs = 1 / 256
    ks = [-LIM, LIM - 1, -LIM - 1, LIM, 0]
    p = np.zeros((len(ks), 3), np.float32)
    p[:, axis] = (np.array(ks, np.float64) + 0.5) * vs
    p[:, (axis + 1) % 3] = 0.3
    keep, out, (xyz, _, count) = _on_device(*_rays(p), vs=vs, max_norm=np.inf)
    assert keep.tolist() == [True, True, False, False, True] and out.tolist() == [False, False, True, True, False]
    assert len(count) == 3 and sorted(xyz[:, axis].tolist()) == [(-LIM + 0.5) * vs, 0.5 * vs, (LIM - 0.5) * vs]


def test_frame_points_value_edges():
    rng = np.random.default_rng(11)
    n = 64
    p = rng.uniform(-0.9, 0.9, (n, 3)).astype(np.float32)
    base = _rays(p, rgb=rng.uniform(0, 1, (n, 3)))
    for min_acc in (-np.inf, np.inf, 0.0, 1.0):
        acc = rng.uniform(0, 1, n).astype(np.float32)
        acc[:3] = [np.inf, 0.0, 1.0]
        keep, _, _ = _on_device(base[0], base[1], acc, base[3], min_acc=min_acc)
        assert keep[0] and not keep[1]                    # acc = inf: s = 0, the camera centre, kept even at +inf
    for max_norm in (np.inf, 0.0, -1.0, 0.5):
        pp = p.copy()
        pp[0] = 0.0
        pp[1] = [1e30, 0, 0]
        keep, out, _ = _on_device(*_rays(pp), max_norm=max_norm, vs=1 / 64, cap=256)
        assert keep[0] == (max_norm >= 0) and not keep[1] and out[1] == (max_norm == np.inf)
        assert keep.sum() == {np.inf: n - 1, 0.0: 1, -1.0: 0}.get(max_norm, keep.sum())
    w2 = np.zeros((4, 3), np.float32)
    for blend in ([np.nan, 1.0, -0.0, -1.0], [np.nan, np.nan, np.nan, np.nan], [-0.0, -0.0, -0.0, 1e-45],
                  [-1.0, 0.0, np.inf, 0.0]):
        _on_device(*base, w2rf=w2, blend=blend)
    keep, _, _ = _on_device(*base, w2rf=w2, blend=[np.nan, -0.0, -1.0, 0.0])
    assert not keep.any()
    # 64 fields, the point inside only the last field's cube
    w2 = np.tile(np.array([[50.0, 0, 0]], np.float32), (64, 1))
    w2[-1] = [-0.25, 0.0, 0.0]
    keep, _, _ = _on_device(*_rays([[0.25, 0.1, 0.1], [-0.95, 0, 0]]), w2rf=w2, max_norm=0.5)
    assert keep.tolist() == [True, False]
    keep, _, _ = _on_device(*_rays([[0.25, 0.1, 0.1]]), w2rf=w2, blend=[1.0] * 63 + [0.0], max_norm=0.5)
    assert not keep[0]


def test_frame_points_non_finite_inputs():
    rng = np.random.default_rng(12)
    n = 96
    p = rng.uniform(-0.9, 0.9, (n, 3)).astype(np.float32)
    p[:8] = [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.inf, np.inf, np.inf], [np.nan] * 3,
             [0, 0, 0], [0.1, 0, 0], [1e-45, 0, 0]]
    acc = rng.uniform(0.5, 1, n).astype(np.float32)
    acc[5:8] = [1e-45, 1e-42, 1e-45]                      # subnormal: depth / acc overflows (or not, for 0 / a)
    depth = acc.copy()
    depth[5] = 0.0
    depth[6] = 0.5
    rgb = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    rgb[8:16] = [[np.nan, 0.5, 0.5], [np.inf, -np.inf, 1.0], [1.0, 1.0, 1.0], [-1e-30, -0.0, 0.0],
                 [np.nextafter(np.float32(1), np.float32(2)), 0.5, np.nan], [-np.inf, np.nan, np.inf],
                 [0.0, np.nextafter(np.float32(0), np.float32(-1)), 1.0], [2.0 ** -25, 1 - 2.0 ** -24, 0.5]]
    for max_norm in (1.0, np.inf):
        keep, out, _ = _on_device(rgb, depth, acc, p, max_norm=max_norm, vs=1 / 32, min_acc=0.0)
        assert keep[8:16].all() and not keep[[0, 1, 2, 3, 4, 6]].any()
    for bad in (np.nan, np.inf, -np.inf):
        for i in (0, 5, 11):                              # a rotation entry, the x and z translations
            M = EYE.copy()
            M.flat[i] = bad
            keep, out, _ = _on_device(rgb, depth, acc, p, c2w=M, max_norm=np.inf, vs=1 / 32)
            assert not keep[:5].any()


# ---- 3. the table at its limits ------------------------------------------------------------------------------------
def _centres(k, vs):
    """identity-camera rays at the centres of voxels k [n,3] (exact in float32 for a power-of-two vs)."""
    return ((np.asarray(k, np.float64) + 0.5) * vs).astype(np.float32)


def _distinct_voxels(m, seed):
    rng = np.random.default_rng(seed)
    flat = rng.choice(256 ** 3, size=m, replace=False)
    return np.stack([flat // 65536 - 128, (flat // 256) % 256 - 128, flat % 256 - 128], 1)


def _rgb(n, seed):
    return np.random.default_rng(seed).uniform(0, 1, (n, 3)).astype(np.float32)


def _occupied_slots(store, cap):
    return set(np.nonzero(store[:cap].cpu().numpy())[0].tolist())


@pytest.mark.parametrize("cap", [2, 4, 1024, 1 << 21])
def test_exactly_half_and_one_past(cap):
    """capacity / 2 distinct voxels fill the table exactly and extract in full; one more overflows, and the claim
    that overflows adds nothing (its slot stays at count 0)."""
    half = cap // 2
    vs = 1 / 64
    k = _distinct_voxels(half + 1, cap)
    p = _centres(k, vs)
    rgb = _rgb(half + 1, cap)
    for m in (half, half + 1):
        t, store = _voxel_table(cap, vs, (0, 0, 0), "cuda")
        _frame_points(t, rgb[:m], np.ones(m, np.float32), np.ones(m, np.float32), p[:m], EYE,
                      np.zeros((1, 3), np.float32), None, 0.5, np.inf)
        xyz, rgb8, count, stats = _extract(t, store, 1)
        assert stats[0] == m and stats[1] == 0 and stats[2] == m
        assert len(_occupied_slots(store, cap)) == m
        if m == half:
            table = eo.new_table()
            eo.frame_points(table, rgb[:m], np.ones(m, np.float32), np.ones(m, np.float32), p[:m], EYE,
                            np.zeros((1, 3), np.float32), None, 0.5, np.inf, vs, (0, 0, 0))
            want = eo.extract(table, 1, vs, (0, 0, 0))
            assert np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
            assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2]) and stats[3] == half
        else:
            assert stats[2] > half and stats[3] == half and (count == 1).all()


def test_overflow_in_a_later_frame():
    cap, vs = 1024, 1 / 64
    half = cap // 2
    k = _distinct_voxels(half + 1, 5)
    p, rgb = _centres(k, vs), _rgb(half + 1, 5)
    t, store = _voxel_table(cap, vs, (0, 0, 0), "cuda")
    one = lambda a, b: _frame_points(t, rgb[a:b], np.ones(b - a, np.float32), np.ones(b - a, np.float32), p[a:b], EYE,
                                     np.zeros((1, 3), np.float32), None, 0.5, np.inf)
    one(0, half)
    assert store[8 * cap + 2].item() == half
    one(0, 1)                                             # an existing voxel is still added at exactly half
    one(half, half + 1)                                   # a new one overflows
    one(1, 2)                                             # and once overflowed, nothing is added
    xyz, rgb8, count, stats = _extract(t, store, 1)
    assert stats[2] == half + 1 and stats[0] == half + 2 and stats[3] == half
    assert sorted(count.tolist()) == [1] * (half - 1) + [2]


def _keys_to_slot(cap, slot, m, lo=-40, hi=40):
    """m voxel indices in [lo, hi)^3 whose keys start their probe at `slot`."""
    r = np.arange(lo, hi)
    k = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
    hit = k[(eo.mix64(eo.pack_key(k).astype(np.uint64)) & np.uint64(cap - 1)) == slot]
    assert len(hit) >= m
    return hit[:m]


@pytest.mark.parametrize("cap", [64, 1024])
def test_forced_collisions_and_wrap_around(cap):
    vs = 1 / 32
    n_last, n_mid = min(cap // 4, 40), min(cap // 8, 20)
    k = np.concatenate([_keys_to_slot(cap, cap - 1, n_last), _keys_to_slot(cap, cap // 2 - 3, n_mid)])
    keys = eo.pack_key(k)
    want_slots = eo.probe_table(keys, cap)
    assert {cap - 1, 0, n_last - 2} <= want_slots and cap // 2 - 3 + n_mid - 1 in want_slots     # wrapped, chained
    rep = np.repeat(k, 3, axis=0)                          # three rays per voxel, interleaved across the warp
    rep = np.concatenate([rep[0::3], rep[1::3], rep[2::3]])
    p, rgb = _centres(rep, vs), _rgb(len(rep), cap)
    n = len(rep)
    t, store = _voxel_table(cap, vs, (0, 0, 0), "cuda")
    _frame_points(t, rgb, np.ones(n, np.float32), np.ones(n, np.float32), p, EYE, np.zeros((1, 3), np.float32), None,
                  0.5, np.inf)
    assert _occupied_slots(store, cap) == want_slots
    tags = store[:cap].cpu().numpy().view(np.uint64)
    assert sorted(int(x) - 1 for x in tags if x) == sorted(keys.tolist())
    xyz, rgb8, count, stats = _extract(t, store, 1)
    table = eo.new_table()
    eo.frame_points(table, rgb, np.ones(n, np.float32), np.ones(n, np.float32), p, EYE, np.zeros((1, 3), np.float32),
                    None, 0.5, np.inf, vs, (0, 0, 0))
    want = eo.extract(table, 1, vs, (0, 0, 0))
    assert np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2]) and (count == 3).all()


@pytest.mark.parametrize("voxels", [1, 2])
def test_contention_past_2e24_points(voxels):
    """Frames of 2^22 rays into one voxel (or alternating between two within each warp): counts past 2^24, where a
    float32 count would stop counting, and the means still equal the restatement's bit for bit."""
    n, vs = 1 << 22, 1 / 16
    rng = np.random.default_rng(voxels)
    org = np.array([0.01, -0.02, 0.03])
    t, store = _voxel_table(1024, vs, org, "cuda")
    table = eo.new_table()
    centres = org + (np.array([[4, -3, 1], [4, -3, 2]]) + 0.5) * vs
    frames = 4 * voxels + 1
    for f in range(frames):
        which = np.arange(n) % voxels
        p = (centres[which] + rng.uniform(-0.4 * vs, 0.4 * vs, (n, 3))).astype(np.float32)
        rgb = rng.uniform(-0.1, 1.1, (n, 3)).astype(np.float32)
        args = (rgb, np.ones(n, np.float32), np.ones(n, np.float32), p, EYE, np.zeros((1, 3), np.float32), None, 0.5,
                np.inf)
        _frame_points(t, *args)
        eo.frame_points(table, *args, vs, org)
    xyz, rgb8, count, stats = _extract(t, store, 1)
    want = eo.extract(table, 1, vs, org)
    assert stats[0] == frames * n and len(count) == voxels and count.sum() == frames * n and count.min() > 1 << 24
    assert np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2])


# ---- 4. lrf_voxel_extract on tables written word by word -----------------------------------------------------------
def _written(cap, slots, vs=0.25, origin=(0.5, -1.0, 2.0)):
    """A table whose slot i holds key `key` and sums `sums` for each (i, key, sums) of `slots`, and the same voxels
    as a restatement table."""
    t, store = _voxel_table(cap, vs, origin, "cuda")
    words = np.zeros(8 * cap + 4, np.uint64)
    table = eo.new_table()
    for i, key, sums in slots:
        words[i] = key + 1
        words[cap + 7 * i: cap + 7 * i + 7] = sums
        table["voxels"][key] = list(sums)
    words[8 * cap + 2] = len(slots)
    words[8 * cap + 3] = 777                               # n_voxels: must be written
    store.copy_(torch.from_numpy(words.view(np.int64)))
    return t, store, table


def _sums(count, frac=0.5, col=0.5):
    return [count, int(count * frac * 2 ** 32), int(count * frac * 2 ** 32) // 2, 0,
            int(count * col * 2 ** 24), 0, count * 2 ** 24]


def _check_extract(t, store, table, min_count, vs=0.25, origin=(0.5, -1.0, 2.0)):
    xyz, rgb8, count, stats = _extract(t, store, min_count)
    want = eo.extract(table, min_count, vs, origin)
    assert stats[3] == len(want[0])
    assert np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2])
    return xyz, rgb8, count


def test_extract_count_saturation_and_min_count():
    key = lambda kx, ky, kz: int(eo.pack_key([kx, ky, kz]))
    big = [(3, key(1, 2, 3), _sums(2 ** 31 - 1)), (9, key(-5, 0, 0), _sums(2 ** 31)),
           (1, key(0, 0, 0), [2 ** 40, 2 ** 40 * 2 ** 20, 0, 2 ** 40 * 2 ** 22, 2 ** 40 * 2 ** 23, 2 ** 40, 0]),
           (12, key(7, 7, 7), _sums(5)), (13, key(7, 7, 8), _sums(6)), (0, key(9, 9, 9), [0] * 7)]
    t, store, table = _written(16, big)
    _, _, count = _check_extract(t, store, table, 1)
    assert sorted(count.tolist()) == [5, 6] + [2 ** 31 - 1] * 3           # saturated; the count-0 slot is dropped
    for mc, n in ((5, 5), (6, 4), (2 ** 31, 2), (2 ** 40, 1), (2 ** 40 + 1, 0), (2 ** 62, 0)):
        _, _, count = _check_extract(t, store, table, mc)
        assert len(count) == n


def test_extract_full_and_empty_tables():
    cap = 1024
    k = _distinct_voxels(cap, 9)
    keys = eo.pack_key(k).tolist()
    rng = np.random.default_rng(9)
    slots = [(i, keys[i], _sums(int(rng.integers(1, 100)), rng.uniform(), rng.uniform())) for i in range(cap)]
    t, store, table = _written(cap, slots)
    _, _, count = _check_extract(t, store, table, 1)
    assert len(count) == cap                               # P == capacity: the last row writes n_voxels
    _, _, count = _check_extract(t, store, table, 50)
    assert 0 < len(count) < cap
    t, store, table = _written(cap, [])
    xyz, _, count = _check_extract(t, store, table, 1)     # n_voxels 0 written over 777, every canary intact
    assert len(count) == 0 and store[8 * cap + 3].item() == 0


def test_extract_key_extremes_and_high_bits():
    """Keys 0 and 2^63 - 1 and keys that differ only above bit 32, placed in reverse order in the slots: the sort must
    run over all 64 bits."""
    kk = [0, 2 ** 63 - 1, 5 << 40, 3 << 40, (1 << 33) | 7, 7, (1 << 62) | 7, (1 << 45) | 7]
    slots = [(60 - 3 * i, key, _sums(i + 1, 0.25 * (i % 4), 0.1 * i)) for i, key in enumerate(sorted(kk, reverse=True))]
    t, store, table = _written(64, slots)
    xyz, _, _ = _check_extract(t, store, table, 1)
    assert xyz[0, 0] == np.float32(0.5 + (-LIM + 0.25 * 3) * 0.25)       # key 0 first: every index at -2^20


def test_extract_colour_on_the_half_boundary():
    """Colour sums whose mean times 255 is exactly k + 0.5 in fp64: rounded up, as floor(x + 0.5) does."""
    found = []
    for cnt in (2, 6, 10, 30, 34, 102, 170, 510):
        for k in range(255):
            v = round((k + 0.5) / 255 * cnt * 2 ** 24)
            if 0 < v <= cnt * 2 ** 24 and v / (cnt * 16777216.0) * 255.0 == k + 0.5:
                found.append((cnt, v, k))
    assert len(found) >= 8
    found = found[:200]
    slots = [(i, int(eo.pack_key([i, 0, 0])), [cnt, 0, 0, 0, v, v, v]) for i, (cnt, v, k) in enumerate(found)]
    t, store, table = _written(512, slots)
    _, rgb8, _ = _check_extract(t, store, table, 1)
    assert rgb8[:, 0].tolist() == [k + 1 for _, _, k in found]


def test_extract_dirty_scratch_and_a_stream():
    cap = 4096
    k = _distinct_voxels(1500, 4)
    rng = np.random.default_rng(4)
    slots = [(int(s), int(key), _sums(int(rng.integers(1, 9)), rng.uniform(), rng.uniform()))
             for s, key in zip(rng.choice(cap, 1500, replace=False), eo.pack_key(k))]
    t, store, table = _written(cap, slots)
    lib = _lib.lib()
    nb = lib.lrf_voxel_extract_scratch_bytes(cap)
    scratch = torch.full((nb + 4096,), 0xFF, dtype=torch.uint8, device="cuda")
    xyz = _padded(cap, 3, torch.float32, CANARY_F)
    rgb = _padded(cap, 3, torch.uint8, 0xA5)
    cnt = _padded(cap, 0, torch.int32, -7)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        _lib.check(lib.lrf_voxel_extract(C.byref(t), 1, xyz[PAD:].data_ptr(), rgb[PAD:].data_ptr(), cnt[PAD:].data_ptr(),
                                         store.data_ptr() + 8 * (8 * cap + 3), scratch.data_ptr(), nb + 4096,
                                         s.cuda_stream))
    s.synchronize()
    want = eo.extract(table, 1, 0.25, (0.5, -1.0, 2.0))
    P = store[8 * cap + 3].item()
    assert P == 1500
    assert np.array_equal(xyz[PAD:PAD + P].cpu().numpy().view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb[PAD:PAD + P].cpu().numpy(), want[1])
    assert np.array_equal(cnt[PAD:PAD + P].cpu().numpy(), want[2])
    for a, fill in ((xyz, CANARY_F), (rgb, 0xA5), (cnt, -7)):
        assert bool((a[:PAD] == fill).all()) and bool((a[PAD + P:] == fill).all())


def test_extract_at_capacity_2e26():
    cap = 1 << 26
    need = 64 * cap + _lib.lib().lrf_voxel_extract_scratch_bytes(cap) + 16 * (cap + 2 * PAD) + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    rng = np.random.default_rng(26)
    k = _distinct_voxels(3000, 26)
    slots = [(int(s), int(key), _sums(int(rng.integers(1, 9)), rng.uniform(), rng.uniform()))
             for s, key in zip(rng.choice(cap, 3000, replace=False), eo.pack_key(k))]
    slots.append((cap - 1, int(eo.pack_key([-LIM, -LIM, -LIM])), _sums(3)))
    t, store, table = _written(cap, slots)
    _check_extract(t, store, table, 1)
    del store
    torch.cuda.empty_cache()



# ---- 5. point_cloud on scenes of every kind, against the restatement and the float64 reference --------------------
W, H = 48, 40


def _scene(kind):
    """Small scenes over the bench's field: poses jittered, density_shift 2 so views see surfaces."""
    import bench
    over = dict(fea_pe=2, view_pe=2) if kind == "pe" else {}
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", 48, n_init_frames=3, density_shift=2.0, **over)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(3):
            lt.r_c2w[i].add_(0.1 * torch.randn(3, 2, generator=g))
            lt.t_c2w[i].add_(0.1 * torch.randn(3, generator=g))
            lt.exposure[i].add_(0.05 * torch.randn(3, 3, generator=g))
    if kind in ("two_counts", "zero_row"):
        torch.manual_seed(1)
        lt.append_rf(2)                                      # rows [1, 0], [0.5, 0.5], [0, 1]
    if kind == "two_counts":
        lt.tensorfs[1].upsample_volume_grid([80, 80, 80])
    lt = lt.to("cuda")
    if kind == "bf16":
        lt.set_grid_storage("bf16")
    elif kind == "alpha":
        with torch.no_grad():
            lt.tensorfs[0].density_line[1][:, :, :20] = -20.0     # carve a region empty, then mask it out
        lt.tensorfs[0].updateAlphaMask((32, 32, 32))
        assert lt.tensorfs[0].alphaMask is not None
    elif kind == "two_counts":
        S = [rf.sample_table(False, -1, "cuda").numel() for rf in lt.tensorfs]
        assert S[0] != S[1], S
    elif kind == "zero_row":
        torch.manual_seed(2)
        lt.append_rf(1)
        with torch.no_grad():
            lt.blending_weights[1] = 0.0
        assert len(lt.tensorfs) == 3 and lt.blending_weights.detach()[1].abs().sum() == 0
    return lt


def _checked_cloud(lt, vs, origin, min_acc, max_norm, min_count=1, test_ids=(), view_ids=None, **kw):
    """point_cloud with its renders checked against forward, its cloud against the restatement bit for bit and
    against the float64 reference within the float32 pipeline's error -> (cloud, frames, restatement table)."""
    frames = []
    cloud = point_cloud(lt, W, H, view_ids=view_ids, test_ids=test_ids, voxel_size=vs, origin=origin, min_acc=min_acc,
                        max_norm=max_norm, min_count=min_count, _frames=frames, **kw)
    w2rf = torch.stack([w.detach() for w in lt.world2rf]).cpu().numpy()
    bw = lt.blending_weights.detach().cpu().numpy()
    c2w = np.stack([lt.get_cam2world([v])[0].detach().cpu().numpy() for v in range(len(lt.r_c2w))])
    table = eo.new_table()
    with torch.no_grad():
        for v, lo, rgb, depth, acc, dirs in frames:
            m = rgb.shape[0]
            r_rgb, r_depth, r_dirs, _ = lt(torch.arange(lo, lo + m, device="cuda"), [v], W, H, is_train=False,
                                           test_id=v in test_ids)
            assert torch.equal(rgb, r_rgb) and torch.equal(depth, r_depth) and torch.equal(dirs, r_dirs)
            eo.frame_points(table, *[a.cpu().numpy() for a in (rgb, depth, acc, dirs)], c2w[v], w2rf, bw[v], min_acc,
                            max_norm, vs, origin)
    want = eo.extract(table, min_count, vs, origin)
    got = [cloud[k].cpu().numpy() for k in ("xyz", "rgb", "count")]
    assert cloud["n_kept"] == table["kept"] and cloud["n_out_of_range"] == table["out_of_range"]
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])

    fr = [(v, *(a.cpu().numpy() for a in (rgb, depth, acc, dirs))) for v, lo, rgb, depth, acc, dirs in frames]
    ref = eo.point_cloud64(fr, c2w.astype(np.float64), w2rf, bw, min_acc, max_norm, vs, origin, min_count)
    assert ref["n_rays"] == cloud["n_rays"]
    assert len(ref["ambiguous"]) < 1e-3 * ref["n_rays"], (len(ref["ambiguous"]), ref["n_rays"])
    assert abs(ref["kept"] - cloud["n_kept"]) <= len(ref["ambiguous"])
    rows = {key: i for i, key in enumerate(sorted(k for k, v in table["voxels"].items() if v[0] >= min_count))}
    compared = 0
    for key, v in ref["voxels"].items():
        if key in ref["ambiguous_keys"]:
            continue
        i = rows[key]
        assert got[2][i] == v[0]
        mean = np.array(v[1:4]) / v[0]
        bound = v[7] + vs * 2.0 ** -31 + 2.0 ** -23 * np.abs(mean).max()
        assert np.abs(got[0][i].astype(np.float64) - mean).max() <= bound, (got[0][i], mean, bound)
        col = np.floor(np.array(v[4:7]) / v[0] * 255.0 + 0.5)
        assert np.abs(got[1][i].astype(np.float64) - col).max() <= 1
        compared += 1
    assert all(key in ref["voxels"] or key in ref["ambiguous_keys"] for key in rows)
    assert compared > 0.9 * len(rows) and compared > 50
    return cloud, frames, table


@pytest.mark.parametrize("kind", ["bench", "pe", "bf16", "alpha", "two_counts", "zero_row"])
def test_scene_against_float64(kind):
    lt = _scene(kind)
    cloud, frames, _ = _checked_cloud(lt, 1 / 64, (0.01, -0.02, 0.0), 0.05, 0.9, test_ids=[2])
    views = {v for v, *_ in frames}
    if kind == "zero_row":
        assert views == {0, 2} and cloud["n_rays"] == 2 * W * H           # the all-zero row is skipped
    else:
        assert views == {0, 1, 2} and cloud["n_rays"] == 3 * W * H
    assert cloud["n_kept"] > 0.2 * cloud["n_rays"]


# ---- 6. geometry that does not depend on the code's conventions -------------------------------------------------
G = 64


def _slab(rf, idx):
    """density that depends on the field's local z only: opaque one grid cell around z = idx / (G - 1) 4 - 2."""
    with torch.no_grad():
        for i in range(3):
            rf.density_plane[i].fill_(1.0 / 8 if i == 0 else 0.0)
            rf.density_line[i].fill_(0.0)
        rf.density_line[0].fill_(-30.0)
        rf.density_line[0][:, :, idx] = 30.0
    return idx / (G - 1) * 4.0 - 2.0


def test_rotated_camera_exports_onto_the_plane():
    """The thin slab from cameras rotated 30 degrees about x and y: every point lies within cell + step + voxel of
    the plane.  A transposed rotation in the back-projection moves points off it."""
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", G, n_init_frames=2).to("cuda")
    rf = lt.tensorfs[0]
    c = _slab(rf, 36)
    R = torch.from_numpy(_rot([math.radians(30), math.radians(30), 0.0])).float()
    with torch.no_grad():
        for i in range(2):
            Ri = R if i == 0 else torch.from_numpy(_rot([math.radians(-30), math.radians(20), 0.5])).float()
            lt.r_c2w[i].copy_(Ri[:, :2].cuda())
            lt.t_c2w[i].copy_(torch.tensor([0.05 * i, -0.1, 0.8]).cuda())
    vs = 1 / 256
    cloud = point_cloud(lt, 64, 48, voxel_size=vs, capacity=1 << 16)
    z = cloud["xyz"][:, 2].double().cpu()
    assert len(z) > 500 and cloud["n_kept"] > 0.5 * 2 * 64 * 48
    assert float((z - c).abs().max()) <= 4.0 / (G - 1) + float(rf.stepSize) + vs, (float(z.min()), float(z.max()), c)


def test_offset_fields_export_onto_their_own_slabs():
    """Two fields, each a slab at its own local z and with its own world2rf; the view with blending row [1, 0] sees
    field 0 and the one with [0, 1] field 1.  Each view's points lie on its field's slab at world z = c_k - world2rf_k.
    A world2rf sign flipped in the field-cube test puts field 1's slab outside its cube (no points)."""
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", G, n_init_frames=3)
    torch.manual_seed(1)
    lt.append_rf(2)
    lt = lt.to("cuda")
    assert lt.blending_weights.detach().cpu().tolist() == [[1.0, 0.0], [0.5, 0.5], [0.0, 1.0]]
    cs = [_slab(lt.tensorfs[0], 36), _slab(lt.tensorfs[1], 40)]
    w2 = [torch.tensor([0.0, 0.0, 0.0]), torch.tensor([0.3, -0.2, 1.5])]
    with torch.no_grad():
        for k in range(2):
            lt.world2rf[k].copy_(w2[k].cuda())
        for v, k in ((0, 0), (2, 1)):
            lt.r_c2w[v].copy_(torch.eye(3, 2).cuda())
            lt.t_c2w[v].copy_((torch.tensor([0.1, 0.0, cs[k] + 0.6]) - w2[k]).cuda())
    vs, cell = 1 / 256, 4.0 / (G - 1)
    for v, k in ((0, 0), (2, 1)):
        cloud = point_cloud(lt, 64, 48, view_ids=[v], voxel_size=vs, capacity=1 << 16, max_norm=1.0)
        xyz = cloud["xyz"].double().cpu()
        world_z = cs[k] - float(w2[k][2])
        assert len(xyz) > 500 and cloud["n_kept"] > 0.5 * 64 * 48, (v, len(xyz))
        step = float(lt.tensorfs[k].stepSize)
        assert float((xyz[:, 2] - world_z).abs().max()) <= cell + step + vs, (v, float(xyz[:, 2].min()), world_z)


# ---- 7. point_cloud arguments and invariants ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene2():
    return _scene("two_counts")


def test_view_ids_empty_and_duplicated(scene2):
    kw = dict(voxel_size=1 / 128, min_acc=0.05, capacity=1 << 16)
    empty = point_cloud(scene2, W, H, view_ids=[], **kw)
    assert empty["n_rays"] == 0 and empty["n_kept"] == 0 and len(empty["xyz"]) == 0 and len(empty["count"]) == 0
    one = point_cloud(scene2, W, H, view_ids=[0], **kw)
    two = point_cloud(scene2, W, H, view_ids=[0, 0], **kw)
    assert len(one["xyz"]) > 50 and two["n_rays"] == 2 * one["n_rays"] and two["n_kept"] == 2 * one["n_kept"]
    assert torch.equal(two["count"], 2 * one["count"])
    assert torch.equal(two["xyz"], one["xyz"]) and torch.equal(two["rgb"], one["rgb"])
    mc = point_cloud(scene2, W, H, view_ids=[0], min_count=3, **kw)
    keep = one["count"] >= 3
    assert torch.equal(mc["xyz"], one["xyz"][keep]) and torch.equal(mc["count"], one["count"][keep])


def test_test_ids_colours(scene2):
    _, frames, _ = _checked_cloud(scene2, 1 / 64, (0, 0, 0), 0.05, 1.0, test_ids=[0, 1])
    plain = []
    point_cloud(scene2, W, H, voxel_size=1 / 64, min_acc=0.05, _frames=plain)
    changed = [not torch.equal(a[2], b[2]) for a, b in zip(frames, plain) if a[0] in (0, 1)]
    assert any(changed)                                     # the held-out exposure is really applied


def test_weights_budget_chunks(scene2):
    S = max(rf.sample_table(False, -1, "cuda").numel() for rf in scene2.tensorfs)
    assert S == max(2 * (int(rf.nSamples) // 6) for rf in scene2.tensorfs)
    kw = dict(voxel_size=1 / 128, min_acc=0.05, capacity=1 << 16)
    ref = point_cloud(scene2, W, H, **kw)
    for budget, m in ((4 * S * 97, 97), (4 * S * 97 - 1, 96), (4 * S, 1)):
        frames = []
        c = point_cloud(scene2, W, H, weights_budget=budget, view_ids=[1], _frames=frames, **kw)
        assert {f[2].shape[0] for f in frames[:-1]} == {m} and len(frames) == -(-W * H // m)
    c = point_cloud(scene2, W, H, weights_budget=4 * S * 97, **kw)
    assert all(torch.equal(c[k], ref[k]) for k in ("xyz", "rgb", "count"))
    with pytest.raises(ValueError, match="weights_budget"):
        point_cloud(scene2, W, H, weights_budget=4 * S - 1, **kw)


def test_sizes_below_one_raise(scene2):
    for w, h in ((0, H), (W, 0), (-1, H), (W, -5), (0, 0)):
        with pytest.raises(ValueError, match="W and H"):
            point_cloud(scene2, w, h)


def test_capacity_boundary_through_point_cloud(scene2):
    """The smallest table that holds the scene's voxels returns the same cloud as a large one; half of it raises."""
    kw = dict(voxel_size=1 / 64, min_acc=0.05)
    big = point_cloud(scene2, W, H, capacity=1 << 20, **kw)
    P = len(big["count"])
    cap = 2
    while cap // 2 < P:
        cap *= 2
    fit = point_cloud(scene2, W, H, capacity=cap, **kw)
    assert all(torch.equal(fit[k], big[k]) for k in ("xyz", "rgb", "count"))
    with pytest.raises(RuntimeError, match="capacity"):
        point_cloud(scene2, W, H, capacity=cap // 2, **kw)
