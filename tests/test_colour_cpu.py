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
