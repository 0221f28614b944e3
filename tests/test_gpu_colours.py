"""GPU: colours from the frames (lrf_frame_colours / lrf_colour_extract and localrf_b200.export.frame_colours).  The
kernels equal their numpy restatement (tests/colour_oracle.py) bit for bit, with canaries past every output; the
result does not depend on the frame order or the run; on an opaque analytic solid, meshed with export.mesh and
photographed with a known colour function of the world point, every coloured vertex carries that function's value
within the pixel and depth footprint, hidden vertices get no colour, and the same holds across the seam of two fields;
numpy, pinned and CUDA images give the same bytes, and malformed input raises before anything renders."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import colour_oracle as co
import localrf_b200 as L
from localrf_b200 import _lib
from localrf_b200.export import _chunk_rays, _render_view, frame_colours, mesh

pytestmark = pytest.mark.gpu

PAD = 64
CANARY = -0x5A5A5A5A5A5A5A5B


def _cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _look_at(eye, target):
    z = np.asarray(eye, np.float64) - np.asarray(target, np.float64)
    z /= np.linalg.norm(z)
    x = np.cross([0.0, 0.0, 1.0], z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1), np.asarray(eye, np.float64)


# ---- 1. kernels vs the restatement --------------------------------------------------------------------------------
def _kernel_views(rng, P):
    """Several cameras, each with a depth map s and an opacity map acc (depth = s acc), and P / 5 points per camera
    placed in random pixels at that pixel's s times 1 +- up to 4% (so about half pass the depth test there; other
    cameras see them at random); images with NaN, infinite and out-of-range values."""
    xyz, views = [], []
    specs = [(False, 53, 41), (False, 17, 96), (True, 64, 31), (True, 33, 17), (False, 1, 1)]
    for fov360, W, H in specs:
        R, t = _look_at(rng.uniform(-4, 4, 3), rng.uniform(-1, 1, 3))
        c2w = np.concatenate([R, t[:, None]], 1).astype(np.float32)
        intr = np.array([rng.uniform(0.5, 1.5) * W, rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H], np.float32)
        s = rng.uniform(0.5, 6, H * W).astype(np.float32)
        acc = rng.uniform(0.2, 1.2, H * W).astype(np.float32)
        acc[rng.random(H * W) < 0.05] = 0.0
        acc[rng.random(H * W) < 0.05] = 0.5
        acc[rng.random(H * W) < 0.02] = np.nan
        depth = (s * acc).astype(np.float32)
        depth[rng.random(H * W) < 0.02] = np.inf
        img = rng.uniform(-0.2, 1.2, (H, W, 3)).astype(np.float32)
        img.reshape(-1)[rng.random(H * W * 3) < 0.02] = np.nan
        img.reshape(-1)[rng.random(H * W * 3) < 0.01] = np.inf
        views.append((W, H, fov360, intr, c2w, depth, acc, img))
        n = P // len(specs) + (P % len(specs) if W == 1 else 0)
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


def _run_kernels(xyz, normals, views, order, opts):
    lib = _lib.lib()
    P = len(xyz)
    sums = torch.full((P + 2 * PAD, 5), CANARY, dtype=torch.int64, device="cuda")
    sums[PAD:PAD + P] = 0
    xd = _cuda(xyz)
    nd = None if normals is None else _cuda(normals)
    keep = []
    for v in order:
        W, H, fov360, intr, c2w, depth, acc, img = views[v]
        t = [_cuda(a) for a in (intr, c2w, depth, acc, img)]
        keep.append(t)
        f = _lib.LrfColourFrame(W=W, H=H, fov360=int(fov360), intrinsics=t[0].data_ptr(), cam2world=t[1].data_ptr(),
                                depth=t[2].data_ptr(), acc=t[3].data_ptr(), image=t[4].data_ptr(), **opts)
        _lib.check(lib.lrf_frame_colours(C.byref(f), xd.data_ptr(), None if nd is None else nd.data_ptr(), P,
                                         sums[PAD:].data_ptr(), None))
    rgb = torch.full((P + 2 * PAD, 3), 0xA5, dtype=torch.uint8, device="cuda")
    cnt = torch.full((P + 2 * PAD,), -7, dtype=torch.int32, device="cuda")
    _lib.check(lib.lrf_colour_extract(sums[PAD:].data_ptr(), P, rgb[PAD:].data_ptr(), cnt[PAD:].data_ptr(), None))
    torch.cuda.synchronize()
    for a, fill in ((sums, CANARY), (rgb, 0xA5), (cnt, -7)):
        assert bool((a[:PAD] == fill).all()) and bool((a[PAD + P:] == fill).all()), "a canary was overwritten"
    return (sums[PAD:PAD + P].cpu().numpy().view(np.uint64), rgb[PAD:PAD + P].cpu().numpy(),
            cnt[PAD:PAD + P].cpu().numpy())


@pytest.mark.parametrize("normals_kind", ["null", "random", "unit"])
def test_kernels_equal_the_restatement(normals_kind):
    rng = np.random.default_rng(7)
    P = 200_003
    xyz, views = _kernel_views(rng, P)
    normals = None
    if normals_kind != "null":
        normals = rng.standard_normal((P, 3)).astype(np.float32)
        if normals_kind == "unit":
            normals /= np.linalg.norm(normals, axis=1, keepdims=True)
        normals[rng.random(P) < 0.1] = 0.0
    opts = dict(min_acc=0.5, depth_tol=0.02, min_cos=0.1)
    want = np.zeros((P, 5), np.uint64)
    flagged = np.zeros(P, bool)
    for W, H, fov360, intr, c2w, depth, acc, img in views:
        flagged |= co.frame_colours(want, xyz, normals, W, H, fov360, intr, c2w, depth, acc, img, **opts)
    sums, rgb, cnt = _run_kernels(xyz, normals, views, range(len(views)), opts)
    ok = ~flagged
    assert flagged.sum() < 0.001 * P
    assert np.array_equal(sums[ok], want[ok])
    passed = (want[:, 0] > 0).sum()
    assert 0.05 * P < passed < 0.95 * P, passed
    assert (want[:, 0] >= 2).sum() > 100
    w_rgb, w_cnt = co.colour_extract(sums)
    assert np.array_equal(rgb, w_rgb) and np.array_equal(cnt, w_cnt)
    # frame order and a repeated run give the same bytes
    again = _run_kernels(xyz, normals, views, [4, 2, 0, 3, 1], opts)
    assert all(np.array_equal(a, b) for a, b in zip((sums, rgb, cnt), again))


def test_kernels_with_no_points():
    lib = _lib.lib()
    sums = torch.full((8, 5), CANARY, dtype=torch.int64, device="cuda")
    one = torch.zeros(3, dtype=torch.float32, device="cuda")
    f = _lib.LrfColourFrame(W=1, H=1, fov360=0, intrinsics=one.data_ptr(), cam2world=sums.data_ptr(),
                            depth=one.data_ptr(), acc=one.data_ptr(), image=one.data_ptr(), min_acc=0.5,
                            depth_tol=0.02, min_cos=0.1)
    _lib.check(lib.lrf_frame_colours(C.byref(f), one.data_ptr(), None, 0, sums.data_ptr(), None))
    _lib.check(lib.lrf_colour_extract(sums.data_ptr(), 0, one.data_ptr(), one.data_ptr(), None))
    torch.cuda.synchronize()
    assert bool((sums == CANARY).all()) and bool((one == 0).all())


# ---- 3-5. an opaque analytic solid photographed with a known colour function --------------------------------------
W0, H0 = 96, 72


def _paint(p):
    """f(p): a smooth colour of the world point, float64 [..., 3]; every channel's gradient is at most GRAD."""
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return np.stack([0.5 + 0.4 * np.sin(3 * x + 2 * y + 1), 0.5 + 0.4 * np.cos(2 * y - 3 * z),
                     0.5 + 0.4 * np.sin(2 * z + 2 * x + 2)], -1)


GRAD = 0.4 * math.sqrt(13)
BACKGROUND = np.array([0.1, 0.9, 0.3], np.float32)


def _solid(rf, centre, r, hh, S=1e4):
    """relu density S P(x, y) L(z) of an upright cylinder (component 0 of plane / line 0), P and L ramping from 0 to
    1 across one grid cell at the surface: opaque a fraction of a cell inside its level-0.005 surface."""
    G = rf.gridSize.tolist()[0]
    cell = 4.0 / (G - 1)
    c = torch.linspace(-2, 2, G, dtype=torch.float64)
    yy, xx = torch.meshgrid(c, c, indexing="ij")
    P = (0.5 + (r - torch.hypot(xx - centre[0], yy - centre[1])) / cell).clamp(0, 1)
    Lz = (0.5 + (hh - (c - centre[2]).abs()) / cell).clamp(0, 1)
    with torch.no_grad():
        for i in range(3):
            rf.density_plane[i].zero_()
            rf.density_line[i].zero_()
        rf.density_plane[0][0, 0] = P.float().cuda()
        rf.density_line[0][0, 0, :, 0] = (S * Lz).float().cuda()
    rf.fea2denseAct = "relu"
    return cell


def _scene(n_fields, target_local, r, hh, grid=160):
    """A LocalTensorfs whose every view looks at the cylinder from one half of the space around it (so its far side is
    hidden from all), and every field holding the same cylinder in world space."""
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", grid, n_init_frames=4)
    for _ in range(n_fields - 1):
        lt.append_rf(2)
    lt = lt.to("cuda")
    w = [lt.world2rf[k].detach().cpu().double().numpy() for k in range(n_fields)]
    if n_fields == 2:
        with torch.no_grad():
            lt.world2rf[1].copy_(lt.world2rf[0] - torch.tensor([0.8, 0.0, 0.0], device="cuda"))
            lt.blending_weights.fill_(0.5)
        w = [lt.world2rf[k].detach().cpu().double().numpy() for k in range(n_fields)]
    target = np.asarray(target_local, np.float64) - w[0]
    cell = 0.0
    for k in range(n_fields):
        cell = _solid(lt.tensorfs[k], tuple(target + w[k]), r, hh)
        lt.tensorfs[k].nSamples = 6 * 512          # eval samples about 0.004 apart around the solid: depth to 0.3%
    eyes = []
    n_views = len(lt.r_c2w)
    for v in range(n_views):
        a = math.radians(-70 + 140 * v / max(n_views - 1, 1))
        e = math.radians((35, -20, 10, 50, -5, 25)[v % 6])
        eye = target + 1.7 * np.array([math.cos(a) * math.cos(e), math.sin(a) * math.cos(e), math.sin(e)])
        R, t = _look_at(eye, target)
        with torch.no_grad():
            lt.r_c2w[v].copy_(torch.from_numpy(R[:, :2]).float())
            lt.t_c2w[v].copy_(torch.from_numpy(t).float())
        eyes.append(t)
    return lt, target, np.array(eyes), cell, w


def _photos(lt, W, H):
    """Per view, the photo: f of the world point each pixel's render back-projects to (s = depth / acc along its
    direction), BACKGROUND where acc < 0.5.  -> [(view, [H, W, 3] float32)]."""
    dev = torch.device("cuda")
    S, per_chunk = _chunk_rays(lt, 256 << 20, dev)
    n = W * H
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    weights = torch.empty(min(per_chunk, n) * S, dtype=torch.float32, device=dev)
    out = []
    with torch.no_grad():
        for v in range(len(lt.r_c2w)):
            frame = (torch.empty(n, 3, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev),
                     torch.empty(n, 3, device=dev))
            plan = None
            for lo, plan, _, _, _, dirs in _render_view(lt, v, W, H, False, min(per_chunk, n), ids, weights, dev,
                                                        frame[:3]):
                frame[3][lo:lo + len(dirs)] = dirs
            assert plan is not None
            c2w = plan.keep[0][0].double().cpu().numpy()
            depth, acc, dirs = (frame[i].double().cpu().numpy() for i in (1, 2, 3))
            with np.errstate(all="ignore"):
                p = (dirs * (depth / acc)[:, None]) @ c2w[:, :3].T + c2w[:, 3]
            img = np.where((acc >= 0.5)[:, None], _paint(p), BACKGROUND).astype(np.float32)
            assert (acc >= 0.5).mean() > 0.1
            out.append((v, img.reshape(H, W, 3)))
    return out


def _tolerance(lt, W, eyes, target, radius, depth_tol=0.02):
    """|f(vertex) - colour| bound: a counted pixel's point lies within s (depth_tol |d| + sqrt(2) / 2 / focal) of the
    vertex (|d| <= sqrt(1 + 2 (W / 2 focal)^2) for the frame's corner), s at most the farthest camera distance; plus
    the rounding of the 8-bit result."""
    focal = float(lt.focal(W).detach().cpu())
    s_max = float(np.linalg.norm(eyes - target, axis=1).max()) + radius
    d = math.sqrt(1 + 2 * (W / 2 / focal) ** 2)
    return GRAD * s_max * (depth_tol * d + math.sqrt(2) / 2 / focal) + 1 / 255


def _facing(xyz, normals, eyes):
    """[V, P] cosine between each vertex's normal and the direction to each camera.  (The tests pass the cylinder's
    radial directions: the surface of a disc sampled on the grid is a staircase, so the mesh normals of its side lean
    by up to 45 degrees from them.)"""
    to = eyes[:, None, :] - xyz[None]
    return np.einsum("vpa,pa->vp", to, normals) / np.linalg.norm(to, axis=-1)


@pytest.fixture(scope="module")
def solid():
    r, hh = 0.4, 0.35
    lt, target, eyes, cell, w = _scene(1, (0.0, 0.0, 0.0), r, hh)
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(v) for v in -w[0]))
    return lt, m, target, eyes, cell, (r, hh), _photos(lt, W0, H0)


def _check_known_answer(fc, m, tol, min_coloured):
    xyz = m["xyz"].double().cpu().numpy()
    cnt, rgb = fc["count"].cpu().numpy(), fc["rgb"].cpu().numpy().astype(np.float64) / 255
    seen = cnt > 0
    assert seen.mean() > min_coloured, seen.mean()
    err = np.abs(rgb[seen] - _paint(xyz[seen])).max()
    assert err <= tol, (err, tol)
    return seen


def test_known_answer_on_an_opaque_solid(solid):
    lt, m, target, eyes, cell, (r, hh), frames = solid
    assert len(m["faces"]) > 2000
    tol = _tolerance(lt, W0, eyes, target, math.hypot(r, hh))
    xyz = m["xyz"].double().cpu().numpy()
    loc = xyz - target
    nrm = np.concatenate([loc[:, :2], np.zeros((len(loc), 1))], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    side = np.abs(loc[:, 2]) < hh - 3 * cell
    hidden = (np.abs(loc[:, 2]) < hh / 2) & (_facing(xyz, nrm, eyes) < -0.3).all(0)    # the ray crosses >= 0.24
    visible = side & (_facing(xyz, nrm, eyes) > 0.7).any(0)
    assert hidden.sum() > 100 and visible.sum() > 100
    for normals in (None, m["normals"]):
        fc = frame_colours(lt, m["xyz"], frames, normals=normals)
        assert fc["n_rays"] == len(frames) * W0 * H0
        seen = _check_known_answer(fc, m, tol, 0.2)
        assert not seen[hidden].any()
        assert seen[visible].mean() > 0.7, seen[visible].mean()
        assert fc["rgb"].is_cuda and fc["count"].dtype == torch.int32 and fc["rgb"].dtype == torch.uint8
        assert (fc["rgb"][~torch.from_numpy(seen).cuda()] == 0).all()


def test_frame_order_and_repeated_runs(solid):
    lt, m, target, eyes, cell, _, frames = solid
    a = frame_colours(lt, m["xyz"], frames, normals=m["normals"])
    b = frame_colours(lt, m["xyz"], frames[::-1], normals=m["normals"])
    c = frame_colours(lt, m["xyz"], frames, normals=m["normals"])
    for k in ("rgb", "count"):
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k])


def test_image_forms_give_the_same_bytes(solid):
    lt, m, target, eyes, cell, _, frames = solid
    want = frame_colours(lt, m["xyz"], frames, normals=m["normals"])
    pinned = [(v, torch.from_numpy(img).pin_memory()) for v, img in frames]
    on_dev = [(v, torch.from_numpy(img).cuda()) for v, img in frames]
    strided = [(v, np.ascontiguousarray(img[:, :, ::-1])[:, :, ::-1]) for v, img in frames]   # negative strides
    xyz_host = m["xyz"].cpu().numpy()
    for fr, xyz in ((pinned, m["xyz"]), (on_dev, m["xyz"]), (strided, m["xyz"]), (frames, xyz_host)):
        got = frame_colours(lt, xyz, fr, normals=m["normals"])
        assert torch.equal(got["rgb"], want["rgb"]) and torch.equal(got["count"], want["count"])


def test_double_resolution_agrees_within_its_footprint(solid):
    lt, m, target, eyes, cell, (r, hh), _ = solid
    frames = _photos(lt, 2 * W0, 2 * H0)
    fc = frame_colours(lt, m["xyz"], frames, normals=m["normals"])
    assert fc["n_rays"] == len(frames) * 4 * W0 * H0
    _check_known_answer(fc, m, _tolerance(lt, 2 * W0, eyes, target, math.hypot(r, hh)), 0.2)


def test_two_fields_with_the_solid_across_their_seam():
    r, hh = 0.3, 0.3
    lt, target, eyes, cell, w = _scene(2, (0.4, 0.0, 0.0), r, hh)
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(v) for v in -w[0]))
    xyz = m["xyz"].double().cpu().numpy()
    owner = np.argmin(np.stack([np.abs(xyz + w[k]).max(1) for k in range(2)]), 0)
    fc = frame_colours(lt, m["xyz"], _photos(lt, W0, H0), normals=m["normals"])
    seen = _check_known_answer(fc, m, _tolerance(lt, W0, eyes, target, math.hypot(r, hh)), 0.2)
    for k in range(2):
        assert (seen & (owner == k)).sum() > 200, k


def test_malformed_input_raises_before_rendering(solid):
    lt, m, target, eyes, cell, _, frames = solid
    consumed = []

    def watched(fr):
        for x in fr:
            consumed.append(x[0])
            yield x

    xyz = m["xyz"]
    bad_calls = [dict(xyz=xyz[:, :2]), dict(xyz=xyz.double()), dict(xyz=xyz[None]), dict(normals=m["normals"][1:]),
                 dict(normals=m["normals"].half()), dict(min_acc=math.nan), dict(depth_tol=0.0),
                 dict(depth_tol=math.inf), dict(min_cos=0.0), dict(min_cos=1.5), dict(weights_budget=4)]
    for kw in bad_calls:
        args = dict(xyz=xyz, normals=m["normals"]) | kw
        with pytest.raises(ValueError):
            frame_colours(lt, args.pop("xyz"), watched(frames), **args)
        assert consumed == [], kw
    img = frames[0][1]
    bad_frames = [(len(lt.r_c2w), img), (-1, img), (0.5, img), (0, img[:, :, :2]), (0, img.astype(np.float64)),
                  (0, img[None]), (0, img[:0]), (0, torch.from_numpy(img)), (0, "image"),
                  (0, torch.from_numpy(img).cuda().half())]
    for fr in bad_frames:
        with pytest.raises((ValueError, TypeError)):
            frame_colours(lt, xyz, [fr])
