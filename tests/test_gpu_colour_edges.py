"""GPU: the frame colouring (lrf_frame_colours, lrf_colour_extract, export.frame_colours) across the cameras, frame
sizes, weights, sums and scenes its C ABI accepts.  The kernels equal their numpy restatement (tests/colour_oracle.py)
bit for bit, with canaries before and after every output; frame_colours equals the independent float64 reference
colour_oracle.frame_colours64 on every point none of whose views it flags.

Cases: pixel coordinates exactly on a pixel edge, the frame's edges, -0.0 and just below 0; negative focal and centres
far outside the frame; 1-pixel-wide and -high frames; fov360 points on the seam, at the poles, at a range that
underflows or overflows and at the camera centre; special acc, depth, depth_tol, min_acc, min_cos, normal, image and
camera values; grazing views whose weight rounds to 0; more than 2^24 points; one frame of 7.2 * 10^8 pixels, whose
image offsets pass 2^31; views on two streams into one sums; the extract on sums written word by word and on sums the
kernel adds to, up to 2^64 - 1; eight scenes end to end; chunked renders, mixed frame sizes, a repeated view, no
points and frames from a generator."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import colour_oracle as co
import localrf_b200 as L
from localrf_b200 import _lib
from localrf_b200.export import _chunk_rays, _render_view, frame_colours

pytestmark = pytest.mark.gpu

PAD = 64
CANARY = -0x5A5A5A5A5A5A5A5B
EYE = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)
OPTS = dict(min_acc=0.5, depth_tol=0.02, min_cos=0.1)


def _cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _frame(view, opts, keep):
    """LrfColourFrame of view = (W, H, fov360, intr, c2w, depth, acc, img) copied to the device (kept alive in keep)."""
    W, H, fov360, intr, c2w, depth, acc, img = view
    t = [_cuda(np.asarray(a, np.float32)) for a in (intr, c2w, depth, acc, img)]
    keep.append(t)
    return _lib.LrfColourFrame(W=W, H=H, fov360=int(fov360), intrinsics=t[0].data_ptr(), cam2world=t[1].data_ptr(),
                               depth=t[2].data_ptr(), acc=t[3].data_ptr(), image=t[4].data_ptr(), **opts)


def _padded_sums(P, preload=None):
    sums = torch.full((P + 2 * PAD, 5), CANARY, dtype=torch.int64, device="cuda")
    if preload is None:
        sums[PAD:PAD + P] = 0
    else:
        sums[PAD:PAD + P] = torch.from_numpy(np.asarray(preload, np.uint64).view(np.int64)).cuda()
    return sums


def _extract(sums, P, dirty=False):
    """lrf_colour_extract of sums[PAD:PAD + P] with canaries around rgb and count (and, with `dirty`, garbage inside)
    -> host (sums, rgb, count) after checking every canary."""
    lib = _lib.lib()
    rgb = torch.full((P + 2 * PAD, 3), 0xA5, dtype=torch.uint8, device="cuda")
    cnt = torch.full((P + 2 * PAD,), -7, dtype=torch.int32, device="cuda")
    if dirty:
        rgb[PAD:PAD + P] = torch.randint(0, 256, (P, 3), dtype=torch.uint8, device="cuda")
        cnt[PAD:PAD + P] = torch.randint(-2 ** 31, 2 ** 31 - 1, (P,), dtype=torch.int32, device="cuda")
    _lib.check(lib.lrf_colour_extract(sums[PAD:].data_ptr(), P, rgb[PAD:].data_ptr(), cnt[PAD:].data_ptr(), None))
    torch.cuda.synchronize()
    for a, fill in ((sums, CANARY), (rgb, 0xA5), (cnt, -7)):
        assert bool((a[:PAD] == fill).all()) and bool((a[PAD + P:] == fill).all()), "a canary was overwritten"
    return (sums[PAD:PAD + P].cpu().numpy().view(np.uint64), rgb[PAD:PAD + P].cpu().numpy(),
            cnt[PAD:PAD + P].cpu().numpy())


def _run(xyz, normals, views, preload=None, dirty=False):
    """Every (view, opts) of `views` launched in order into one zeroed (or preloaded) sums, then the extract."""
    lib = _lib.lib()
    P = len(xyz)
    sums = _padded_sums(P, preload)
    xd = _cuda(np.asarray(xyz, np.float32))
    nd = None if normals is None else _cuda(np.asarray(normals, np.float32))
    keep = []
    for view, opts in views:
        f = _frame(view, opts, keep)
        _lib.check(lib.lrf_frame_colours(C.byref(f), xd.data_ptr(), None if nd is None else nd.data_ptr(), P,
                                         sums[PAD:].data_ptr(), None))
    return _extract(sums, P, dirty)


def _restated(xyz, normals, views, preload=None):
    sums = np.zeros((len(xyz), 5), np.uint64) if preload is None else np.array(preload, np.uint64)
    flagged = np.zeros(len(xyz), bool)
    for view, opts in views:
        flagged |= co.frame_colours(sums, xyz, normals, *view, **opts)
    return sums, flagged


def _check_bits(xyz, normals, views, preload=None, all_points=False):
    """Kernels against the restatement: sums bit for bit (every point with all_points, else the unflagged ones), rgb
    and count as the restatement extracts them from the device's sums -> (sums, rgb, count)."""
    sums, rgb, cnt = _run(xyz, normals, views, preload)
    want, flagged = _restated(np.asarray(xyz, np.float32), normals, views, preload)
    ok = np.ones(len(xyz), bool) if all_points else ~flagged
    assert np.array_equal(sums[ok], want[ok]), (sums[ok], want[ok])
    w_rgb, w_cnt = co.colour_extract(sums)
    assert np.array_equal(rgb, w_rgb) and np.array_equal(cnt, w_cnt)
    return sums, rgb, cnt


def _view64(view):
    W, H, fov360, intr, c2w, depth, acc, img = view
    return dict(c2w=c2w, fov360=fov360, focal=intr[0], center=intr[1:], depth=np.asarray(depth).reshape(H, W),
                acc=np.asarray(acc).reshape(H, W), image=np.asarray(img).reshape(H, W, 3))


def _check_float64(xyz, normals, views, rgb, cnt):
    """Same opts in every view: the device's rgb and count equal frame_colours64 on the points it does not flag."""
    ref = co.frame_colours64(xyz, normals, [_view64(v) for v, _ in views], **views[0][1])
    ok = ~ref["flagged"]
    assert ok.mean() > 0.99, ok.mean()
    assert np.array_equal(ref["count"][ok], cnt[ok]) and np.array_equal(ref["rgb"][ok], rgb[ok])


# ---- 1. pixel edges, cameras and frame shapes ---------------------------------------------------------------------
def _pixel_image(W, H):
    """Every pixel its own colour, exact in float32."""
    k = np.arange(W * H, dtype=np.float64)
    return (np.stack([k % 251, (k // 251) % 241, (k // 60000) % 239], 1) / 256).astype(np.float32).reshape(H, W, 3)


@pytest.mark.parametrize("cx", [0.0, -0.0])
def test_pinhole_pixel_edges(cx):
    """Identity camera, f = 2, d_v = 1: u = 2 c_0 + cx exactly.  u on an integer belongs to that pixel; W - ulp to the
    last; W and anything below 0 to none; u = -0.0 (cx = -0.0) to pixel 0.  The same for v."""
    W, H = 7, 5
    below = lambda a: float(np.nextafter(np.float32(a), np.float32(0)))
    us = [0.0, 1.0, 3.0, 6.0, below(W), float(W), -2.0 ** -30, 2.5, 0.0]
    vs = [0.0, 4.0, 2.0, 1.0, 3.5, 0.5, 1.0, below(H), float(H)]
    xyz = np.array([[u / 2, -v / 2, -1.0] for u, v in zip(us, vs)], np.float32)
    xyz[0] = [-0.0, -0.25, -1.0]                       # c_0 = -0.0 (with c_1 < 0 and c_2 < 0 every term is -0.0)
    view = (W, H, False, np.array([2, cx, cx], np.float32), EYE, np.ones(W * H, np.float32),
            np.ones(W * H, np.float32), _pixel_image(W, H))
    i, j, _, ok, _ = co.project(xyz, W, H, False, view[3], EYE)
    assert ok.tolist() == [True, True, True, True, True, False, False, True, False]
    assert i[ok].tolist() == [0, 1, 3, 6, 6, 2] and j[ok].tolist() == [0, 4, 2, 1, 3, 4]
    sums, rgb, cnt = _check_bits(xyz, None, [(view, OPTS)], all_points=True)
    assert cnt.tolist() == [1, 1, 1, 1, 1, 0, 0, 1, 0]
    img = view[7].reshape(-1, 3)
    for p in np.nonzero(ok)[0]:
        assert rgb[p].tolist() == np.floor(img[j[p] * W + i[p]] * 255 + 0.5).astype(int).tolist()


def _placed(rng, view, n, spread=0.04):
    """n points in random pixels of view (W, H, fov360, intr, c2w, depth, acc, img) at the pixel's s = depth / acc
    times 1 +- spread."""
    W, H, fov360, intr, c2w, depth, acc, _ = view
    R, t = c2w[:, :3].astype(np.float64), c2w[:, 3].astype(np.float64)
    s = depth.astype(np.float64) / acc
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    k = np.minimum(v.astype(np.int64), H - 1) * W + np.minimum(u.astype(np.int64), W - 1)
    r = s[k] * (1 + rng.uniform(-spread, spread, n))
    if fov360:
        phi, theta = v * math.pi / H - math.pi / 2, u * 2 * math.pi / W + math.pi
        c = np.stack([np.cos(phi) * np.sin(theta), np.sin(phi), np.cos(phi) * np.cos(theta)], 1) * r[:, None]
    else:
        c = np.stack([(u - intr[1]) / intr[0], -(v - intr[2]) / intr[0], -np.ones(n)], 1) * r[:, None]
    return (c @ R.T + t).astype(np.float32)


def _random_view(rng, W, H, fov360, intr=None):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
    c2w = np.concatenate([R, rng.uniform(-2, 2, (3, 1))], 1).astype(np.float32)
    if intr is None:
        intr = [rng.uniform(0.5, 1.5) * W, rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H]
    s = rng.uniform(0.5, 6, H * W).astype(np.float32)
    acc = rng.uniform(0.3, 1.2, H * W).astype(np.float32)
    return (W, H, fov360, np.array(intr, np.float32), c2w, (s * acc).astype(np.float32), acc,
            rng.uniform(-0.1, 1.1, (H, W, 3)).astype(np.float32))


SHAPES = {   # W, H, fov360, intrinsics (None: random)
    "pin_1x1": (1, 1, False, None), "pin_1x13": (1, 13, False, None), "pin_13x1": (13, 1, False, None),
    "fov_1x1": (1, 1, True, None), "fov_1x9": (1, 9, True, None), "fov_9x1": (9, 1, True, None),
    "neg_focal": (29, 23, False, [-17.5, 14.0, 11.0]), "far_centre": (29, 23, False, [40.0, 1.0e5, -3.0e4]),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_cameras_and_frame_shapes(shape):
    """Random points at the rendered depth of random pixels, seen by that camera and two others of the same shape:
    bit for bit against the restatement and equal to the float64 reference."""
    W, H, fov360, intr = SHAPES[shape]
    rng = np.random.default_rng(list(SHAPES).index(shape))
    views = [_random_view(rng, W, H, fov360, intr) for _ in range(3)]
    xyz = np.concatenate([_placed(rng, v, 3000) for v in views])
    normals = rng.standard_normal(xyz.shape).astype(np.float32)
    for nrm in (None, normals):
        sums, rgb, cnt = _check_bits(xyz, nrm, [(v, OPTS) for v in views])
        # (10^5 pixels off axis, the float32 point's rounding moves its pixel by tens: few land where they were put)
        assert (cnt > 0).sum() > (0.01 if shape == "far_centre" else 0.15) * len(xyz), (cnt > 0).sum()
        if nrm is None and shape != "far_centre":    # (there the float64 reference rightly flags every point)
            _check_float64(xyz, None, [(v, OPTS) for v in views], rgb, cnt)


def test_fov360_seam_poles_and_range_limits():
    """Points exactly on the seam (c_0 = +-0, c_2 < 0: theta = +-pi, both column 0), at both poles (rows 0 and H - 1,
    column of atan2(0, 0) = 0), at a range whose squares underflow to 0 or overflow, and at the camera centre, with and
    without normals.  asinf and atan2f are exact at these arguments, so every point is compared bit for bit."""
    xyz = np.array([[0.0, 0.0, -1.0], [-0.0, -0.0, -1.0], [0.0, 0.3, -2.0], [-0.0, -0.3, -2.0], [0, 1, 0],
                    [0, -2, 0], [0, 0, 1], [1e-30, 0, -1e-30], [1e20, 0, 0], [0, 0, 0], [1, 0, 0], [-1, 0, 0]],
                   np.float32)                         # (c_0 = -0.0 needs every term of its sum -0.0: c_1, c_2 <= -0)
    big_tol = dict(min_acc=0.5, depth_tol=1e30, min_cos=0.1)
    for W, H in ((33, 17), (32, 16), (1, 1)):
        view = (W, H, True, np.zeros(3, np.float32), EYE, np.ones(W * H, np.float32), np.ones(W * H, np.float32),
                _pixel_image(W, H))
        i, j, _, ok, _ = co.project(xyz, W, H, True, view[3], EYE)
        assert ok.tolist() == [True] * 7 + [False, False, False, True, True]
        assert set(i[:4].tolist()) <= {0, W - 1} and (W != 32 or i[:4].tolist() == [0] * 4), i[:4]
        assert j[4] == H - 1 and j[5] == 0
        for nrm in (None, np.tile(np.float32([[0, 0, 1]]), (len(xyz), 1))):
            sums, rgb, cnt = _check_bits(xyz, nrm, [(view, big_tol)], all_points=True)
            assert cnt[7:10].tolist() == [0, 0, 0]
            if nrm is None:
                assert cnt[:7].tolist() == [1] * 7


# ---- 2. special values ----------------------------------------------------------------------------------------------
INF, NAN = math.inf, math.nan
SUB = float(np.float32(1.4e-45))
ONE_MINUS = float(np.nextafter(np.float32(1), np.float32(0)))
SPECIAL = {   # acc, depth, image, normal, opts overrides, nan camera -> expected count of the point (0, 0, -2)
    "acc_at_min": (0.5, 1.0, [0.5] * 3, None, {}, False, 1),
    "acc_subnormal": (SUB, 2 * SUB, [0.5] * 3, None, dict(min_acc=0.0), False, 1),
    "acc_minus_zero": (-0.0, 0.0, [0.5] * 3, None, dict(min_acc=-INF), False, 0),
    "acc_nan": (NAN, 1.0, [0.5] * 3, None, dict(min_acc=-INF), False, 0),
    "acc_negative": (-1.0, -2.0, [0.5] * 3, None, dict(min_acc=-INF), False, 0),
    "min_acc_inf": (1.0, 2.0, [0.5] * 3, None, dict(min_acc=INF), False, 0),
    "min_acc_minus_inf": (0.25, 0.5, [0.5] * 3, None, dict(min_acc=-INF), False, 1),
    "acc_inf": (INF, INF, [0.5] * 3, None, dict(min_acc=-INF), False, 0),
    "tol_overflows": (1.0, 1e10, [0.5] * 3, None, dict(depth_tol=3e38), False, 1),
    "tol_exact_edge": (1.0, 4.0, [0.5] * 3, None, dict(depth_tol=0.5), False, 1),     # |2 - 4| = 0.5 * 4 exactly
    "tol_subnormal_equal": (1.0, 2.0, [0.5] * 3, None, dict(depth_tol=SUB), False, 1),
    "tol_subnormal_ulp": (1.0, float(np.nextafter(np.float32(2), np.float32(3))), [0.5] * 3, None,
                          dict(depth_tol=SUB), False, 0),
    "cos1_unit": (1.0, 2.0, [0.5] * 3, [0, 0, 1], dict(min_cos=1.0), False, 1),
    "cos1_long": (1.0, 2.0, [0.5] * 3, [0, 0, 3], dict(min_cos=1.0), False, 1),
    "cos1_tilted": (1.0, 2.0, [0.5] * 3, [0.2, 0, 0.98], dict(min_cos=1.0), False, 0),
    "long_normal": (1.0, 2.0, [0.25, 0.5, 1.0], [0, 0, 5], {}, False, 1),
    "normal_inf": (1.0, 2.0, [0.5] * 3, [0, 0, INF], {}, False, 1),
    "normal_inf_nan": (1.0, 2.0, [0.5] * 3, [INF, 0, 1], {}, False, 0),
    "normal_nan": (1.0, 2.0, [0.5] * 3, [0, NAN, 1], {}, False, 0),
    "image_edges": (1.0, 2.0, [-0.0, 1.0, ONE_MINUS], None, {}, False, 1),
    "image_inf": (1.0, 2.0, [0.5, INF, 0.5], None, {}, False, 0),
    "image_minus_inf": (1.0, 2.0, [0.5, 0.5, -INF], None, {}, False, 0),
    "camera_nan": (1.0, 2.0, [0.5] * 3, None, {}, True, 0),
}


@pytest.mark.parametrize("case", list(SPECIAL))
def test_special_values(case):
    acc, depth, img, normal, over, nan_cam, want = SPECIAL[case]
    c2w = EYE.copy()
    if nan_cam:
        c2w[1, 2] = np.nan
    view = (1, 1, False, np.array([1, 0.5, 0.5], np.float32), c2w, np.float32([depth]), np.float32([acc]),
            np.asarray(img, np.float32).reshape(1, 1, 3))
    nrm = None if normal is None else np.array([normal], np.float32)
    sums, rgb, cnt = _check_bits(np.array([[0, 0, -2]], np.float32), nrm, [(view, OPTS | over)], all_points=True)
    assert cnt.tolist() == [want]
    if want:
        assert sums[0, 1] == 65536                     # w >= 1 or no normals: full weight, capped
    if case == "image_edges":
        assert sums[0, 2:].tolist() == [0, 65536 << 24, 65536 * (2 ** 24 - 1)] and rgb[0].tolist() == [0, 255, 255]


def test_grazing_views_add_nothing():
    """min_cos = 2^-20 lets a view with w = 10^-6 pass the cosine test, but its q = floor(w 2^16) is 0: it adds
    nothing, the count included.  Seen grazing by one camera and frontally by another, the point has count 1 and
    the frontal pixel's colour."""
    n = np.array([[1, 0, 1e-6]], np.float32)
    xyz = np.array([[0, 0, -2]], np.float32)
    opts = dict(min_acc=0.5, depth_tol=0.02, min_cos=2.0 ** -20)
    one = lambda c2w, c: (1, 1, False, np.array([1, 0.5, 0.5], np.float32), c2w, np.float32([2]), np.float32([1]),
                          np.full((1, 1, 3), c, np.float32))
    side = np.array([[0, 0, 1, 2], [0, 1, 0, 0], [-1, 0, 0, -2]], np.float32)      # at (2, 0, -2), looking along -x
    grazing, frontal = (one(EYE, 0.25), opts), (one(side, 0.75), opts)
    sums, rgb, cnt = _check_bits(xyz, n, [grazing])
    assert sums[0].tolist() == [0] * 5 and cnt.tolist() == [0] and rgb.tolist() == [[0, 0, 0]]
    for order in ([grazing, frontal], [frontal, grazing, grazing]):
        sums, rgb, cnt = _check_bits(xyz, n, order)
        assert cnt.tolist() == [1] and sums[0, 1] == 65536 and rgb.tolist() == [[191, 191, 191]]


# ---- 3. sizes past 32-bit and 24-bit limits -------------------------------------------------------------------------
def test_more_than_2_24_points():
    """2^24 + 5 points on a 1 x 1 frame: every seventh misses the depth test, the last five differ.  Checked on the
    device against the pattern, and the tail against the restatement; then the extract over n = 2^24 + 1 rows."""
    lib = _lib.lib()
    P = (1 << 24) + 5
    idx = torch.arange(P, device="cuda")
    z = torch.where(idx % 7 == 0, -2.5, -2.0).float()
    xyz = torch.stack([torch.zeros_like(z), torch.zeros_like(z), z], 1)
    xyz[-5:] = torch.tensor([[0, 0, -2.03], [0, 0, -1.97], [0, 0, -2.05], [1.2, 0, -2], [0, 0, 2]], device="cuda")
    view = (1, 1, False, np.array([1, 0.5, 0.5], np.float32), EYE, np.float32([2]), np.float32([1]),
            np.array([[[0.25, 0.5, 0.75]]], np.float32))
    keep = []
    f = _frame(view, OPTS, keep)
    sums = _padded_sums(P)
    _lib.check(lib.lrf_frame_colours(C.byref(f), xyz.data_ptr(), None, P, sums[PAD:].data_ptr(), None))
    torch.cuda.synchronize()
    body = sums[PAD:PAD + P]
    hit = (idx % 7 != 0)
    want = torch.stack([hit.long(), hit.long() * 65536, hit.long() * (65536 << 22), hit.long() * (65536 << 23),
                        hit.long() * (3 * (65536 << 22))], 1)
    assert torch.equal(body[:-5], want[:-5])
    tail = slice(P - 1000, P)
    w_tail, _ = _restated(xyz[tail].cpu().numpy(), None, [(view, OPTS)])
    assert np.array_equal(body[tail].cpu().numpy().view(np.uint64), w_tail)
    assert body[-5:, 0].tolist() == [1, 1, 0, 0, 0]
    assert bool((sums[:PAD] == CANARY).all()) and bool((sums[PAD + P:] == CANARY).all())
    # the extract over 2^24 + 1 rows written word by word: S <= Q 2^24, Q < 2^20, exact in int64 on the device
    n = (1 << 24) + 1
    q = (idx[:n] * 2654435761) % ((1 << 20) - 1)
    s = (idx[:n] * 40503) % (1 << 20) * q * 16
    rows = torch.stack([idx[:n], q, s, q << 24, q * 7], 1)
    sums2 = _padded_sums(n)
    sums2[PAD:PAD + n] = rows
    _, rgb, cnt = _extract(sums2, n, dirty=True)
    rgb, cnt = torch.from_numpy(rgb).cuda().long(), torch.from_numpy(cnt).cuda().long()
    den = torch.where(q == 0, 1, q << 25)
    exp = torch.where(q[:, None] == 0, 0, (rows[:, 2:] * 510 + (q[:, None] << 24)) // den[:, None])
    assert torch.equal(rgb, exp) and torch.equal(cnt, idx[:n])


def test_one_frame_past_2_31_image_floats():
    """A 40000 x 18000 frame (3 W H = 2.16 * 10^9 image floats): points in pixels whose image offset 3 k passes 2^31,
    in the last pixel and in low pixels.  depth and acc point into the image's own allocation (offsets 0 and W H);
    only the hit pixels are written, and the expected sums come from those values."""
    lib = _lib.lib()
    W, H = 40000, 18000
    n = W * H
    assert 3 * n > 2 ** 31
    img = torch.empty(3 * n, dtype=torch.float32, device="cuda")
    pix = [(1000, 0), (7, 2), (0, 17896), (39999, 17893), (12345, 17950), (39999, 17999), (20000, 17990)]
    assert [3 * (j * W + i) > 2 ** 31 for i, j in pix] == [False, False, True, False, True, True, True]
    rng = np.random.default_rng(5)
    vals = []
    for i, j in pix:
        k = j * W + i
        a = float(rng.choice([0.75, 1.0, 0.4]))                 # 0.4 < min_acc: that pixel does not count
        col = (rng.integers(0, 2 ** 24, 3) / 2 ** 24).astype(np.float32)
        img[k] = a                                              # depth = acc: s = 1 = d_v
        img[n + k] = a
        img[3 * k:3 * k + 3] = torch.from_numpy(col).cuda()
        vals.append((a, col))
    xyz = torch.tensor([[i + 0.5, -(j + 0.5), -1.0] for i, j in pix] + [[W + 0.5, -0.5, -1.0]], device="cuda")
    intr = torch.tensor([1.0, 0.0, 0.0], device="cuda")
    c2w = torch.from_numpy(EYE).cuda()
    f = _lib.LrfColourFrame(W=W, H=H, fov360=0, intrinsics=intr.data_ptr(), cam2world=c2w.data_ptr(),
                            depth=img.data_ptr(), acc=img.data_ptr() + 4 * n, image=img.data_ptr(), **OPTS)
    P = len(xyz)
    sums = _padded_sums(P)
    _lib.check(lib.lrf_frame_colours(C.byref(f), xyz.data_ptr(), None, P, sums[PAD:].data_ptr(), None))
    got, rgb, cnt = _extract(sums, P)
    for p, (a, col) in enumerate(vals):
        c24 = (col.astype(np.float64) * 2 ** 24).astype(np.int64)
        want = [1, 65536] + (65536 * c24).tolist() if a >= 0.5 else [0] * 5
        assert got[p].tolist() == want, (pix[p], got[p], want)
    assert got[-1].tolist() == [0] * 5
    del img
    torch.cuda.empty_cache()


def test_views_on_two_streams_into_one_sums():
    """Six views launched alternately on two side streams (each waiting for the zeroed sums), joined by events before
    the extract: the same bytes as one stream."""
    lib = _lib.lib()
    rng = np.random.default_rng(9)
    views = [_random_view(rng, 41, 29, bool(v % 2)) for v in range(6)]
    xyz = np.concatenate([_placed(rng, v, 20000) for v in views])
    P = len(xyz)
    want = _run(xyz, None, [(v, OPTS) for v in views])
    xd = _cuda(xyz)
    sums = _padded_sums(P)
    keep = []
    frames = [_frame(v, OPTS, keep) for v in views]
    ready = torch.cuda.Event()
    ready.record()
    side = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in side:
        s.wait_event(ready)
    for v, f in enumerate(frames):
        s = side[v % 2]
        _lib.check(lib.lrf_frame_colours(C.byref(f), xd.data_ptr(), None, P, sums[PAD:].data_ptr(), s.cuda_stream))
    for s in side:
        done = torch.cuda.Event()
        done.record(s)
        torch.cuda.current_stream().wait_event(done)
    got = _extract(sums, P)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert (want[2] > 0).sum() > 0.3 * P


# ---- 4. the extract ---------------------------------------------------------------------------------------------------
def _fraction_rgb(S, Q):
    from fractions import Fraction
    return 0 if Q == 0 else min(math.floor(Fraction(255 * S, Q << 24) + Fraction(1, 2)), 255)


def _near_half_levels(rng, q_max, n):
    Q = rng.integers(q_max // 2, q_max + 1, n, dtype=np.uint64)
    L_ = rng.integers(0, 255, n)
    off = rng.integers(-1, 2, n)
    S = [min(max(((2 * int(l) + 1) * (int(q) << 24)) // 510 + int(o), 0), int(q) << 24) for q, l, o in zip(Q, L_, off)]
    return Q, np.array(S, np.uint64)


def test_extract_on_sums_written_word_by_word():
    """Sums one unit from a half level for Q up to 2^30 (where an fp64 chain is off by a level in thousands), Q past
    2^53, S up to 2^64 - 1, counts at 2^31 - 1, 2^31 and 2^64 - 1, means exactly on a half level, Q = 0 with a count,
    into dirty rgb and count buffers: every byte the exact rule's."""
    rng = np.random.default_rng(17)
    rows = []
    for log_q in (16, 24, 28, 30):
        Q, S = _near_half_levels(rng, 1 << log_q, 30000 if log_q == 30 else 2000)
        rows += [[1, int(q), int(s), int(s2), int(s3)] for q, s, s2, s3 in zip(Q, S, S[::-1] % (Q << 24), S // 3)]
    big = (1 << 64) - 1
    rows += [[2 ** 31 - 1, 1 << 40, big, 1 << 63, 0], [2 ** 31, (1 << 53) + 1, (1 << 63) + 12345, 1, 0],
             [big, 255, 2 ** 23, 3 * 2 ** 23, 509 * 2 ** 23], [5, 510, 2 ** 24, 255 << 24, 0], [3, 0, 0, 0, 0],
             [7, 0, 5, 6, 7], [1, (1 << 54) + 3, big, big - (1 << 40), 1 << 60]]
    sums = np.array(rows, np.uint64)
    _, rgb, cnt = _extract(_padded_sums(len(rows), sums), len(rows), dirty=True)
    want = np.array([[_fraction_rgb(int(s), int(r[1])) for s in r[2:]] for r in rows])
    assert np.array_equal(rgb, want)
    assert np.array_equal(cnt, np.minimum(sums[:, 0], 2 ** 31 - 1).astype(np.int32))
    assert rgb[-5].tolist() == [1, 2, 255] and rgb[-4].tolist() == [1, 128, 0] and rgb[-3].tolist() == [0, 0, 0]


def test_extract_on_sums_the_kernel_adds_to():
    """Preloaded sums, then one full-weight white view (2^40 per colour word) added by the kernel: S reaching
    2^64 - 1, Q past 2^53, counts past 2^31, and rows on and next to a half level."""
    big = (1 << 64) - 1
    pre = [[2 ** 31 - 1, (1 << 40) + 5, big - (1 << 40), big - (1 << 40), 0],
           [2 ** 64 - 2, (1 << 53) + 7, 1 << 62, 0, (1 << 63)],
           [0, 65536, 0, 0, 0],           # Q ends at 2^17 and S at 2^40: a mean of exactly 1/2 -> 128
           [9, 0, 0, 0, 0]]
    xyz = np.tile(np.float32([[0, 0, -2]]), (4, 1))
    view = (1, 1, False, np.array([1, 0.5, 0.5], np.float32), EYE, np.float32([2]), np.float32([1]),
            np.ones((1, 1, 3), np.float32))
    sums, rgb, cnt = _check_bits(xyz, None, [(view, OPTS)], preload=np.array(pre, np.uint64), all_points=True)
    assert sums[0, 2] == big and sums[1, 0] == 2 ** 64 - 1
    want = [[_fraction_rgb(int(s), int(r[1])) for s in r[2:]] for r in sums.tolist()]
    assert rgb.tolist() == want
    assert rgb[2].tolist() == [128, 128, 128] and cnt.tolist() == [2 ** 31 - 1, 2 ** 31 - 1, 1, 10]


# ---- 5. end to end against the float64 reference --------------------------------------------------------------------
FW, FH = 56, 40


def _lt(kind):
    """Small scenes over the bench's field (poses jittered, density_shift 2 so views see surfaces), as the point-cloud
    edge tests build them; fov360 and intrinsics scenes on top."""
    import bench
    over = dict(fea_pe=2, view_pe=2) if kind == "pe" else {}
    torch.manual_seed(0)
    if kind == "fov360":
        aabb = 2 * torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
        lt = L.LocalTensorfs(camera_prior=None, fov=360, n_init_frames=3, n_overlap=30, WH=(96, 48),
                             n_iters_per_frame=600, n_iters_reg=100, lr_R_init=5e-3, lr_t_init=5e-4, lr_i_init=0,
                             lr_exposure_init=1e-3, rf_lr_init=2e-2, rf_lr_basis=1e-3, lr_decay_target_ratio=0.1,
                             N_voxel_list={}, update_AlphaMask_list=[], lr_upsample_reset=True, device="cpu",
                             aabb=aabb, gridSize=[48] * 3, **bench.field_kwargs(density_shift=2.0))
    else:
        lt = bench._scene(L.LocalTensorfs, "cpu", 48, n_init_frames=3, density_shift=2.0, **over)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(3):
            lt.r_c2w[i].add_(0.1 * torch.randn(3, 2, generator=g))
            lt.t_c2w[i].add_(0.1 * torch.randn(3, generator=g))
    if kind in ("two_counts", "zero_row"):
        torch.manual_seed(1)
        lt.append_rf(2)
    if kind == "two_counts":
        lt.tensorfs[1].upsample_volume_grid([80, 80, 80])
    lt = lt.to("cuda")
    if kind == "bf16":
        lt.set_grid_storage("bf16")
    elif kind == "alpha":
        with torch.no_grad():
            lt.tensorfs[0].density_line[1][:, :, :20] = -20.0
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
    elif kind == "intrinsics":
        with torch.no_grad():
            lt.center_rel.copy_(torch.tensor([0.43, 0.58], device="cuda"))
            lt.focal_offset.fill_(1.13)
    return lt


def _rendered(lt, v, w, h):
    """(depth [h, w], acc [h, w], dirs [h w, 3]) of view v's eval render at w x h, as frame_colours renders it; None
    when no field renders the view."""
    dev = torch.device("cuda")
    S, per_chunk = _chunk_rays(lt, 256 << 20, dev)
    n = w * h
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    weights = torch.empty(min(per_chunk, n) * S, dtype=torch.float32, device=dev)
    frame = tuple(torch.empty(shape, device=dev) for shape in ((n, 3), n, n, (n, 3)))
    plan = None
    with torch.no_grad():
        for lo, plan, _, _, _, dirs in _render_view(lt, v, w, h, False, min(per_chunk, n), ids, weights, dev,
                                                    frame[:3]):
            frame[3][lo:lo + len(dirs)] = dirs
    if plan is None:
        return None
    return tuple(frame[i].cpu().numpy() for i in (1, 2, 3))


def _scene_points(lt, renders, rng, per_view=1500):
    """Points at s (1 +- 3 %) along random rays with acc >= 0.1 of each rendered view."""
    pts = []
    for v, (depth, acc, dirs) in renders.items():
        M = lt.get_cam2world([v])[0].detach().double().cpu().numpy()
        good = np.nonzero((acc.reshape(-1) >= 0.1) & np.isfinite(depth.reshape(-1)))[0]
        assert len(good) > 100, len(good)
        r = rng.choice(good, per_view)
        s = depth.reshape(-1)[r].astype(np.float64) / acc.reshape(-1)[r] * (1 + rng.uniform(-0.03, 0.03, per_view))
        pts.append((dirs[r].astype(np.float64) * s[:, None]) @ M[:, :3].T + M[:, 3])
    return np.concatenate(pts).astype(np.float32)


def _checked_colours(lt, frames, xyz, normals=None, opts=None, max_flagged=1e-3, **kw):
    """frame_colours against frame_colours64 on the renders: few flagged pairs, and exact counts and rgb on every
    point with no flagged view -> (result, reference)."""
    opts = opts or dict(min_acc=0.1, depth_tol=0.02, min_cos=0.1)
    fc = frame_colours(lt, xyz, frames, normals=normals, **opts, **kw)
    views = []
    for v, img in frames:
        img = np.asarray(img.cpu() if torch.is_tensor(img) else img, np.float32)
        h, w = img.shape[:2]
        r = _rendered(lt, v, w, h)
        if r is None:
            continue
        M = lt.get_cam2world([v])[0].detach().cpu().numpy()
        views.append(dict(c2w=M, fov360=lt.fov == 360, focal=float(lt.focal(w).detach().cpu()),
                          center=lt.center(w, h).detach().cpu().numpy(), depth=r[0].reshape(h, w),
                          acc=r[1].reshape(h, w), image=img))
    nrm = None if normals is None else np.asarray(normals.cpu() if torch.is_tensor(normals) else normals)
    ref = co.frame_colours64(np.asarray(xyz.cpu() if torch.is_tensor(xyz) else xyz), nrm, views, **opts)
    assert ref["n_flagged"] < max_flagged * max(ref["n_pairs"], 1), (ref["n_flagged"], ref["n_pairs"])
    ok = ~ref["flagged"]
    cnt, rgb = fc["count"].cpu().numpy(), fc["rgb"].cpu().numpy()
    assert np.array_equal(cnt[ok], ref["count"][ok]) and np.array_equal(rgb[ok], ref["rgb"][ok])
    return fc, ref


def _images(rng, views, w, h):
    return [(v, rng.uniform(-0.05, 1.05, (h, w, 3)).astype(np.float32)) for v in views]


@pytest.mark.parametrize("kind", ["bench", "pe", "bf16", "alpha", "two_counts", "zero_row", "fov360", "intrinsics"])
def test_scene_against_float64(kind):
    lt = _lt(kind)
    rng = np.random.default_rng(21)
    w, h = (FW, FH) if kind != "fov360" else (64, 32)
    renders = {v: r for v in range(3) if (r := _rendered(lt, v, w, h)) is not None}
    assert sorted(renders) == ([0, 2] if kind == "zero_row" else [0, 1, 2])
    xyz = _scene_points(lt, renders, rng)
    frames = _images(rng, range(3), w, h)
    fc, ref = _checked_colours(lt, frames, xyz)
    assert fc["n_rays"] == len(renders) * w * h                # the all-zero blending row renders nothing
    assert (ref["count"] > 0).mean() > 0.3, np.bincount(ref["count"])
    if kind == "bench":                                         # with normals: the weight's rounding flags more pairs
        normals = rng.standard_normal(xyz.shape).astype(np.float32)
        fc, ref = _checked_colours(lt, frames, xyz, normals=normals, max_flagged=3e-2)
        assert (ref["count"] > 0).mean() > 0.1


@pytest.fixture(scope="module")
def bench_scene():
    lt = _lt("bench")
    rng = np.random.default_rng(33)
    renders = {v: _rendered(lt, v, FW, FH) for v in range(3)}
    return lt, _scene_points(lt, renders, rng), _images(rng, range(3), FW, FH)


def test_chunked_renders_give_the_same_bytes(bench_scene):
    lt, xyz, frames = bench_scene
    S, _ = _chunk_rays(lt, 256 << 20, torch.device("cuda"))
    want = frame_colours(lt, xyz, frames)
    got = frame_colours(lt, xyz, frames, weights_budget=97 * 4 * S)
    assert _chunk_rays(lt, 97 * 4 * S, torch.device("cuda"))[1] == 97
    assert torch.equal(got["rgb"], want["rgb"]) and torch.equal(got["count"], want["count"])
    assert got["n_rays"] == want["n_rays"] == 3 * FW * FH and int((want["count"] > 0).sum()) > 1000


def test_frames_of_three_sizes_in_one_call(bench_scene):
    lt, xyz, _ = bench_scene
    rng = np.random.default_rng(4)
    frames = [(0, rng.uniform(0, 1, (FH, FW, 3)).astype(np.float32)),
              (1, rng.uniform(0, 1, (23, 81, 3)).astype(np.float32)),
              (2, rng.uniform(0, 1, (61, 37, 3)).astype(np.float32))]
    fc, ref = _checked_colours(lt, frames, xyz)
    assert fc["n_rays"] == FW * FH + 81 * 23 + 37 * 61 and (ref["count"] > 0).sum() > 500


def test_a_repeated_view_doubles_the_count(bench_scene):
    lt, xyz, frames = bench_scene
    once = frame_colours(lt, xyz, frames[:1])
    twice = frame_colours(lt, xyz, frames[:1] * 2)
    assert torch.equal(twice["count"], 2 * once["count"]) and torch.equal(twice["rgb"], once["rgb"])
    assert twice["n_rays"] == 2 * once["n_rays"] and int((once["count"] > 0).sum()) > 300


def test_no_points_and_frames_from_a_generator(bench_scene):
    lt, xyz, frames = bench_scene
    empty = frame_colours(lt, np.zeros((0, 3), np.float32), frames)
    assert empty["rgb"].shape == (0, 3) and empty["count"].shape == (0,) and empty["n_rays"] == 0   # nothing renders
    want = frame_colours(lt, xyz, frames)
    got = frame_colours(lt, xyz, ((v, img) for v, img in frames))
    assert torch.equal(got["rgb"], want["rgb"]) and torch.equal(got["count"], want["count"])
