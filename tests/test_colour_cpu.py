"""CPU-only: the frame-colour restatement (tests/colour_oracle.py) on pixel round trips and hand-built cases, the
LrfColourFrame mirror (lrf_sizeof 17; 16 stays 0), and lrf_frame_colours / lrf_colour_extract refusing bad
arguments with LRF_ERR_INVALID and a message before they touch a device (the non-NULL pointers below are never
dereferenced)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import colour_oracle as co
from localrf_b200 import _lib
from localrf_b200.ray_utils import get_ray_directions_360, get_ray_directions_lean

INVALID = -1
FAKE = 0x10000                       # never read
EYE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)


def _random_c2w(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
    return np.concatenate([R, rng.uniform(-2, 2, (3, 1))], 1).astype(np.float32)


@pytest.mark.parametrize("fov360, W, H, seed", [(False, 37, 23, 0), (False, 9, 31, 1), (True, 41, 19, 2),
                                                (True, 63, 33, 3)])
def test_pixel_round_trip(fov360, W, H, seed):
    """Every pixel's ray (ray_utils), a point at depth s along it, projected back: the same pixel and d_v = s up to
    rounding, apart from fov360 points flagged as near a pixel edge."""
    rng = np.random.default_rng(seed)
    c2w = _random_c2w(rng)
    jj, ii = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    ii, jj = ii.reshape(-1), jj.reshape(-1)
    intr = np.array([rng.uniform(0.6, 1.4) * W, rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H], np.float32)
    if fov360:
        d = get_ray_directions_360(ii, jj, W, H)
    else:
        d = get_ray_directions_lean(ii, jj, float(intr[0]), torch.from_numpy(intr[1:]))
    d = d.double().numpy()
    for s in (0.05, 1.0, 37.5):
        p = (d * s) @ c2w[:, :3].astype(np.float64).T + c2w[:, 3].astype(np.float64)
        i, j, dv, ok, flagged = co.project(p.astype(np.float32), W, H, fov360, intr, c2w)
        assert ok.all()
        good = ~flagged
        assert flagged.sum() <= 0.01 * len(p)
        assert np.array_equal(i[good], ii.numpy()[good]) and np.array_equal(j[good], jj.numpy()[good])
        assert np.allclose(dv, s, rtol=1e-4)


def test_points_behind_or_outside_the_pinhole_frame():
    intr = np.array([10, 5, 4], np.float32)
    p = np.array([[0, 0, 1], [0, 0, 0], [0.6, 0, -1], [0.49, 0.39, -1], [-0.51, 0, -1], [0, -0.41, -1],
                  [np.nan, 0, -1]], np.float32)
    i, j, dv, ok, _ = co.project(p, 10, 8, False, intr, EYE)
    assert ok.tolist() == [False, False, False, True, False, False, False]
    assert (i[3], j[3]) == (9, 0)


def test_fov360_poles_and_seam():
    p = np.array([[0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [-1, 0, 0]], np.float32)
    i, j, dv, ok, flagged = co.project(p, 8, 4, True, np.zeros(3, np.float32), EYE)
    assert ok.all() and j[0] == 3 and j[1] == 0 and np.array_equal(dv, np.ones(5, np.float32))
    assert 0 <= i.min() and i.max() < 8


def _one_pixel(img, acc=1.0, depth=2.0, normals=None, **kw):
    """One point 2 in front of an identity pinhole camera on a 1 x 1 frame."""
    sums = np.zeros((1, 5), np.uint64)
    args = dict(min_acc=0.5, depth_tol=0.02, min_cos=0.1) | kw
    co.frame_colours(sums, np.array([[0, 0, -2]], np.float32), normals, 1, 1, False,
                     np.array([1, 0.5, 0.5], np.float32), EYE, np.float32([depth]), np.float32([acc]),
                     np.asarray(img, np.float32).reshape(1, 1, 3), **args)
    return sums[0]


def test_depth_test_and_pixel_rules():
    assert _one_pixel([0.5, 0.25, 1.0]).tolist() == [1, 65536, 65536 * 2 ** 23, 65536 * 2 ** 22, 65536 * 2 ** 24]
    assert _one_pixel([2.0, -1.0, 0.0]).tolist() == [1, 65536, 65536 * 2 ** 24, 0, 0]      # clamped
    assert _one_pixel([np.nan, 0, 0]).tolist() == [0] * 5
    assert _one_pixel([0, np.inf, 0]).tolist() == [0] * 5
    assert _one_pixel([0.5] * 3, acc=0.5, depth=1.0)[0] == 1                         # s = 2, acc exactly min_acc
    assert _one_pixel([0.5] * 3, acc=0.4999, depth=0.9998)[0] == 0
    assert _one_pixel([0.5] * 3, depth=2.04)[0] == 1 and _one_pixel([0.5] * 3, depth=1.95)[0] == 0
    assert _one_pixel([0.5] * 3, acc=0.0, depth=0.0, min_acc=-1.0)[0] == 0
    assert _one_pixel([0.5] * 3, depth=np.inf)[0] == 0


def test_normal_weights():
    n = lambda v: np.array([v], np.float32)
    assert _one_pixel([1, 1, 1], normals=n([0, 0, 1]))[:2].tolist() == [1, 65536]
    assert _one_pixel([1, 1, 1], normals=n([0, 0, 2]))[:2].tolist() == [1, 65536]            # capped at 1
    assert _one_pixel([1, 1, 1], normals=n([0, 0, 0]))[0] == 0
    assert _one_pixel([1, 1, 1], normals=n([0, 0, -1]))[0] == 0
    w = np.float32(0.6)
    assert _one_pixel([1, 1, 1], normals=n([0.8, 0, 0.6]))[:2].tolist() == [1, int(w * np.float32(65536))]
    assert _one_pixel([1, 1, 1], normals=n([0.8, 0, 0.6]), min_cos=0.61)[0] == 0


def test_extract_means_and_rounding():
    sums = np.array([[0, 0, 0, 0, 0], [2, 3, 3 * 2 ** 24, 0, 3 * 2 ** 23], [1, 1, 2 ** 24 // 510, 0, 0],
                     [5, 0, 0, 0, 0], [2 ** 40, 65536, 0, 0, 0]], np.uint64)
    rgb, count = co.colour_extract(sums)
    assert count.tolist() == [0, 2, 1, 5, 2 ** 31 - 1]
    assert rgb.tolist() == [[0, 0, 0], [255, 0, 128], [0, 0, 0], [0, 0, 0], [0, 0, 0]]


def test_struct_mirror():
    L = _lib.lib()
    assert L.lrf_sizeof(17) == C.sizeof(_lib.LrfColourFrame) == 3 * 4 + 4 + 5 * 8 + 3 * 4 + 4
    assert L.lrf_sizeof(16) == 0 and L.lrf_sizeof(18) == 0


def _frame(**kw):
    f = _lib.LrfColourFrame(W=8, H=6, fov360=0, intrinsics=FAKE, cam2world=FAKE, depth=FAKE, acc=FAKE, image=FAKE,
                            min_acc=0.5, depth_tol=0.02, min_cos=0.1)
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def _err(rc, text):
    assert rc == INVALID, rc
    assert text in _lib.lib().lrf_last_error().decode()


@pytest.mark.parametrize("kw, text", [
    (dict(W=0), "W and H"), (dict(H=0), "W and H"), (dict(W=-3), "W and H"), (dict(W=1 << 16, H=1 << 15), "W and H"),
    (dict(intrinsics=None), "intrinsics"), (dict(intrinsics=None, fov360=1), "intrinsics"),
    (dict(cam2world=None), "cam2world"), (dict(depth=None), "depth"), (dict(acc=None), "acc"),
    (dict(image=None), "image"), (dict(min_acc=math.nan), "min_acc"),
    (dict(depth_tol=0.0), "depth_tol"), (dict(depth_tol=-0.1), "depth_tol"), (dict(depth_tol=math.inf), "depth_tol"),
    (dict(depth_tol=math.nan), "depth_tol"), (dict(min_cos=0.0), "min_cos"), (dict(min_cos=-0.5), "min_cos"),
    (dict(min_cos=1.0001), "min_cos"), (dict(min_cos=math.nan), "min_cos"),
])
def test_frame_refusals(kw, text):
    _err(_lib.lib().lrf_frame_colours(C.byref(_frame(**kw)), FAKE, None, 10, FAKE, None), text)


def test_frame_edges_accepted_by_the_checks_and_pointer_refusals():
    """The limits themselves pass the checks (n = 0 launches nothing, so no device is touched); NULL and misaligned
    pointers and out-of-range n are refused."""
    L = _lib.lib()
    for kw in (dict(W=1, H=1), dict(W=(1 << 31) - 1, H=1), dict(min_acc=-math.inf), dict(min_acc=math.inf),
               dict(min_cos=1.0), dict(min_cos=1e-30), dict(depth_tol=1e30)):
        assert L.lrf_frame_colours(C.byref(_frame(**kw)), FAKE, None, 0, FAKE, None) == 0, kw
    assert L.lrf_frame_colours(C.byref(_frame()), FAKE, FAKE, 0, FAKE, None) == 0
    _err(L.lrf_frame_colours(C.byref(_frame(W=1 << 16, H=1 << 15)), FAKE, None, 0, FAKE, None), "W and H")
    _err(L.lrf_frame_colours(None, FAKE, None, 10, FAKE, None), "frame")
    _err(L.lrf_frame_colours(C.byref(_frame()), None, None, 10, FAKE, None), "xyz")
    _err(L.lrf_frame_colours(C.byref(_frame()), FAKE, None, 10, None, None), "sums")
    _err(L.lrf_frame_colours(C.byref(_frame()), FAKE, None, 10, FAKE + 4, None), "8-byte")
    _err(L.lrf_frame_colours(C.byref(_frame()), FAKE, None, -1, FAKE, None), "n must")
    _err(L.lrf_frame_colours(C.byref(_frame()), FAKE, None, 1 << 31, FAKE, None), "n must")


def test_extract_refusals():
    L = _lib.lib()
    assert L.lrf_colour_extract(FAKE, 0, FAKE, FAKE, None) == 0
    assert L.lrf_colour_extract(FAKE, 0, FAKE + 1, FAKE + 3, None) == 0            # rgb / count need no alignment here
    _err(L.lrf_colour_extract(None, 10, FAKE, FAKE, None), "sums")
    _err(L.lrf_colour_extract(FAKE + 4, 10, FAKE, FAKE, None), "8-byte")
    _err(L.lrf_colour_extract(FAKE, 10, None, FAKE, None), "rgb / count")
    _err(L.lrf_colour_extract(FAKE, 10, FAKE, None, None), "rgb / count")
    _err(L.lrf_colour_extract(FAKE, -1, FAKE, FAKE, None), "n must")
    _err(L.lrf_colour_extract(FAKE, 1 << 31, FAKE, FAKE, None), "n must")


# ---- the exact extract, the zero-weight rule and the float64 reference ---------------------------------------------
def _fraction_rgb(S, Q):
    from fractions import Fraction
    return 0 if Q == 0 else min(math.floor(Fraction(255 * S, Q << 24) + Fraction(1, 2)), 255)


def _fp64_chain(S, Q):
    """The extract as fp64 operations each rounded (u64 -> double, the quotient, * 255, + 0.5), as it once was."""
    return np.floor(np.asarray(S, np.uint64).astype(np.float64) / (np.asarray(Q, np.uint64).astype(np.float64)
                                                                    * 16777216.0) * 255.0 + 0.5)


def _near_half_levels(rng, q_max, n):
    """n sums (Q, S) with Q in [q_max / 2, q_max] and S one unit off, or on, an exact half level of 255 S / (Q 2^24)."""
    Q = rng.integers(q_max // 2, q_max + 1, n, dtype=np.uint64)
    L = rng.integers(0, 255, n)
    off = rng.integers(-1, 2, n)
    S = [min(max(((2 * int(l) + 1) * (int(q) << 24)) // 510 + int(o), 0), int(q) << 24) for q, l, o in zip(Q, L, off)]
    return Q, np.array(S, np.uint64)


@pytest.mark.parametrize("log_q", [16, 22, 28, 30, 34])
def test_extract_is_exact_next_to_half_levels(log_q):
    """lrf_colour_extract's rule is floor(255 S / (Q 2^24) + 1/2) exactly: against Fraction on sums one unit from a
    half level.  The fp64 chain it replaces is off by a level in some of them once Q nears 2^30 (thousands of
    full-weight views of one point)."""
    rng = np.random.default_rng(log_q)
    Q, S = _near_half_levels(rng, 1 << log_q, 30000 if log_q == 30 else 3000)
    sums = np.zeros((len(Q), 5), np.uint64)
    sums[:, 0], sums[:, 1], sums[:, 2], sums[:, 3], sums[:, 4] = 7, Q, S, S[::-1] * 0, np.minimum(S, Q << 24)
    rgb, count = co.colour_extract(sums)
    want = np.array([_fraction_rgb(int(s), int(q)) for s, q in zip(S, Q)])
    assert np.array_equal(rgb[:, 0], want) and (count == 7).all()
    assert all(co.extract_exact(int(s), int(q)) == x for s, q, x in zip(S[:500], Q[:500], want[:500]))
    if log_q == 30:
        assert (_fp64_chain(S, Q) != want).sum() > 100


def test_extract_on_the_limits():
    """Q past 2^53, S up to 2^64 - 1, exact half levels (rounded up), counts saturated at 2^31 - 1, and hand-written S
    above Q 2^24 saturated at 255."""
    big = (1 << 64) - 1
    rows = [[1, 1 << 40, big, (1 << 63), 0], [1, (1 << 53) + 1, (1 << 63) + 12345, 1, 0],
            [2 ** 31 - 1, 255, 2 ** 23, 3 * 2 ** 23, 509 * 2 ** 23], [2 ** 31, 510, 2 ** 24, 0, 0],
            [big, 1, 1 << 25, 0, 0], [4, 0, 0, 0, 0], [1, 65536, 0, 1, 65536 * (2 ** 24 - 1)]]
    rgb, count = co.colour_extract(np.array(rows, np.uint64))
    for r, got in zip(rows, rgb.tolist()):
        assert got == [_fraction_rgb(s, r[1]) for s in r[2:]], (r, got)
    assert count.tolist() == [1, 1, 2 ** 31 - 1, 2 ** 31 - 1, 2 ** 31 - 1, 4, 1]
    assert rgb[2].tolist() == [1, 2, 255] and rgb[3].tolist() == [1, 0, 0] and rgb[4].tolist() == [255, 0, 0]


def test_a_view_of_zero_weight_adds_nothing():
    """With min_cos below 2^-16 a grazing normal passes the cosine test with q = floor(w 2^16) = 0: that view adds
    nothing, the count included, so count > 0 still means the point has a colour."""
    assert _one_pixel([0.9, 0.8, 0.7], normals=np.array([[1, 0, 1e-5]], np.float32), min_cos=1e-6).tolist() == [0] * 5
    sums = np.zeros((1, 5), np.uint64)
    for nz in (1e-5, 1.0):                             # the same point seen grazing, then frontally
        co.frame_colours(sums, np.array([[0, 0, -2]], np.float32), np.array([[1, 0, nz]], np.float32), 1, 1, False,
                         np.array([1, 0.5, 0.5], np.float32), EYE, np.float32([2]), np.float32([1]),
                         np.full((1, 1, 3), 0.5, np.float32), min_acc=0.5, depth_tol=0.02, min_cos=2.0 ** -20)
    assert sums[0].tolist() == [1, 65536] + [65536 * 2 ** 23] * 3           # n . (0, 0, 2) / 2 = 1


def _view64(W, H, fov360, intr, c2w, depth, acc, img):
    return dict(c2w=c2w, fov360=fov360, focal=intr[0], center=intr[1:], depth=np.asarray(depth).reshape(H, W),
                acc=np.asarray(acc).reshape(H, W), image=np.asarray(img).reshape(H, W, 3))


def _restated(xyz, normals, views, opts):
    sums = np.zeros((len(xyz), 5), np.uint64)
    flagged = np.zeros(len(xyz), bool)
    for view in views:
        flagged |= co.frame_colours(sums, xyz, normals, *view, **opts)
    rgb, count = co.colour_extract(sums)
    return rgb, count, flagged


def test_reference64_on_the_hand_built_cases():
    cases = [dict(img=[0.5, 0.25, 1.0]), dict(img=[2.0, -1.0, 0.0]), dict(img=[np.nan, 0, 0]), dict(img=[0, np.inf, 0]),
             dict(img=[0.5] * 3, acc=0.4999, depth=0.9998), dict(img=[0.5] * 3, depth=2.04),
             dict(img=[0.5] * 3, depth=1.95), dict(img=[0.5] * 3, acc=0.0, depth=0.0, min_acc=-1.0),
             dict(img=[0.5] * 3, depth=np.inf), dict(img=[1, 1, 1], normals=[0, 0, 2]),
             dict(img=[1, 1, 1], normals=[0, 0, -1]), dict(img=[0.2, 0.4, 0.6], normals=[0.8, 0, 0.6]),
             dict(img=[1, 1, 1], normals=[0.8, 0, 0.6], min_cos=0.61),
             dict(img=[0.9, 0.8, 0.7], normals=[1, 0, 1e-5], min_cos=1e-6)]
    for c in cases:
        opts = dict(min_acc=c.get("min_acc", 0.5), depth_tol=0.02, min_cos=c.get("min_cos", 0.1))
        nrm = None if "normals" not in c else np.array([c["normals"]], np.float32)
        view = (1, 1, False, np.array([1, 0.5, 0.5], np.float32), EYE, np.float32([c.get("depth", 2.0)]),
                np.float32([c.get("acc", 1.0)]), np.asarray(c["img"], np.float32).reshape(1, 1, 3))
        xyz = np.array([[0, 0, -2]], np.float32)
        rgb, count, _ = _restated(xyz, nrm, [view], opts)
        ref = co.frame_colours64(xyz, nrm, [_view64(*view)], **opts)
        assert ref["n_flagged"] == 0, c
        assert ref["count"].tolist() == count.tolist() and np.array_equal(ref["rgb"], rgb), c


def _random_views(rng, specs, P):
    """Cameras with depth and opacity maps and images, and points placed in their pixels at the pixel's depth +- 4 %
    (as test_gpu_colours builds them, without non-finite values)."""
    xyz, views = [], []
    for fov360, W, H in specs:
        c2w = _random_c2w(rng)
        R, t = c2w[:, :3].astype(np.float64), c2w[:, 3].astype(np.float64)
        intr = np.array([rng.uniform(0.5, 1.5) * W, rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H], np.float32)
        s = rng.uniform(0.5, 6, H * W).astype(np.float32)
        acc = rng.uniform(0.2, 1.2, H * W).astype(np.float32)
        depth = (s * acc).astype(np.float32)
        img = rng.uniform(-0.2, 1.2, (H, W, 3)).astype(np.float32)
        views.append((W, H, fov360, intr, c2w, depth, acc, img))
        n = P // len(specs)
        u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
        k = np.minimum(v.astype(np.int64), H - 1) * W + np.minimum(u.astype(np.int64), W - 1)
        r = s[k].astype(np.float64) * (1 + rng.uniform(-0.04, 0.04, n))
        if fov360:
            phi, theta = v * math.pi / H - math.pi / 2, u * 2 * math.pi / W + math.pi
            c = np.stack([np.cos(phi) * np.sin(theta), np.sin(phi), np.cos(phi) * np.cos(theta)], 1) * r[:, None]
        else:
            c = np.stack([(u - intr[1]) / intr[0], -(v - intr[2]) / intr[0], -np.ones(n)], 1) * r[:, None]
        xyz.append(c @ R.T + t)
    return np.concatenate(xyz).astype(np.float32), views


@pytest.mark.parametrize("fov360, normals", [(False, False), (False, True), (True, False), (True, True)])
def test_reference64_agrees_with_the_restatement(fov360, normals):
    """On random cameras, every point that neither flags equals in count and rgb, and few are flagged: under 0.1 % of
    the (point, view) pairs without normals; with them, q = floor(w 2^16) is within the weight's float32 error of the
    next integer in a few per cent of the counted pairs."""
    rng = np.random.default_rng(11 + 2 * fov360 + normals)
    P = 20000
    xyz, views = _random_views(rng, [(fov360, 53, 41), (fov360, 17, 96), (fov360, 64, 31)], P)
    nrm = None
    if normals:
        nrm = rng.standard_normal((len(xyz), 3)).astype(np.float32)
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    opts = dict(min_acc=0.5, depth_tol=0.02, min_cos=0.1)
    rgb, count, flagged = _restated(xyz, nrm, views, opts)
    ref = co.frame_colours64(xyz, nrm, [_view64(*v) for v in views], **opts)
    assert ref["n_flagged"] < (2e-2 if normals else 1e-3) * ref["n_pairs"], ref["n_flagged"]
    good = ~ref["flagged"] & ~flagged
    assert np.array_equal(ref["count"][good], count[good]) and np.array_equal(ref["rgb"][good], rgb[good])
    assert (count[good] > 0).sum() > 0.1 * len(xyz) and (count[good] >= 2).sum() > 10
