"""CPU-only: the C ABI of the training call's backward (lrf_exposure_clamp, lrf_backward_batch_scratch_bytes,
lrf_render_backward_batch) -- exports, the struct mirror, scratch sizes and every LRF_ERR_INVALID case, refused
before any device work (the fake pointers below are never dereferenced); and tests/camera_oracle.py against float64
torch autograd through the ops of the composed path."""
import ctypes as C

import numpy as np
import pytest
import torch

from localrf_b200 import _lib
from localrf_b200.ray_utils import get_ray_directions_lean, get_rays_lean
import camera_oracle

INVALID = -1
FAKE = 0x10000                       # 16-byte aligned, never read


def test_exports_and_struct_mirror():
    L = _lib.lib()
    for name in ("lrf_exposure_clamp", "lrf_backward_batch_scratch_bytes", "lrf_render_backward_batch"):
        assert hasattr(L, name) and name in _lib.EXPORTS
    assert L.lrf_sizeof(7) == C.sizeof(_lib.LrfCameraGrads) == 4 * 8
    assert L.lrf_version() == _lib.ABI_VERSION == 4


def test_scratch_bytes():
    L = _lib.lib()
    f = L.lrf_backward_batch_scratch_bytes
    for n, s, v in ((0, 344, 1), (-4, 344, 1), (16, 1, 1), (16, 344, 0), (16, 344, 3), (16, 344, -1)):
        assert f(n, s, v) == 0, (n, s, v)
    sizes = [f(n, 344, 4) for n in (4, 64, 1024, 4096)]
    assert all(a < b for a, b in zip(sizes, sizes[1:])) and sizes[0] > 0
    # at least the generated rays plus the field backward's own block
    assert f(4096, 344, 16) >= 4096 * 6 * 4 + L.lrf_backward_scratch_bytes(4096, 344)
    assert f(4096, 344, 16) % 16 == 0


def _fake_field():
    s = _lib.LrfField()
    s.grid[:] = [8, 8, 8]
    s.aabb[:] = [-1, -1, -1, 1, 1, 1]
    s.n_dcomp, s.n_acomp, s.app_dim, s.featureC = 8, 24, 27, 128
    for name in ("dplane", "dline", "aplane", "aline"):
        for i in range(3):
            getattr(s, name)[i] = FAKE
    for name in ("basis", "w1", "b1", "w2", "b2", "w3", "b3", "z_vals"):
        setattr(s, name, FAKE)
    s.n_samples = 64
    return s


def _fake_batch(n=64, views=4):
    b = _lib.LrfBatch()
    b.n_rays, b.ray_ids, b.W, b.H = n, FAKE, 32, 24
    b.intrinsics, b.cam2world, b.n_views, b.world2rf = FAKE, FAKE, views, FAKE
    return b


def _fake_grads():
    g = _lib.LrfGradients()
    for name in ("d_dplane", "d_dline", "d_aplane", "d_aline"):
        for i in range(3):
            getattr(g, name)[i] = FAKE
    for name in ("d_w1b", "d_b1", "d_w2", "d_b2", "d_w3", "d_b3"):
        setattr(g, name, FAKE)
    return g


def _call(field=None, batch=None, grads=None, scratch_bytes=None, **ptrs):
    L = _lib.lib()
    f, b, g = field or _fake_field(), batch or _fake_batch(), grads or _fake_grads()
    cg = _lib.LrfCameraGrads()
    need = L.lrf_backward_batch_scratch_bytes(max(b.n_rays, 1), f.n_samples, max(b.n_views, 1))
    p = dict(prep=FAKE, x=FAKE, g_rgb=FAKE, g_depth=FAKE, g_dirs=None, scratch=FAKE)
    p.update(ptrs)
    return L.lrf_render_backward_batch(C.byref(f), p["prep"], C.byref(b), p["x"], p["g_rgb"], p["g_depth"],
                                       p["g_dirs"], C.byref(g), C.byref(cg), p["scratch"],
                                       need if scratch_bytes is None else scratch_bytes, None)


def _err():
    return _lib.lib().lrf_last_error().decode()


@pytest.mark.parametrize("case", ["rays", "accumulate", "blend", "indivisible", "no_rays", "scratch_small",
                                  "scratch_null", "field_grad_null", "plane_grad_null", "rgb_linear_null",
                                  "grad_rgb_null", "grad_depth_null", "ray_ids_null", "cam2world_null"])
def test_invalid_before_device_work(case):
    b, g = _fake_batch(), _fake_grads()
    kw = {}
    if case == "rays":
        b.rays = FAKE
    elif case == "accumulate":
        b.accumulate = 1
    elif case == "blend":
        b.blend = FAKE
    elif case == "indivisible":
        b.n_rays = 63
    elif case == "no_rays":
        b.n_rays = 0
    elif case == "scratch_small":
        kw["scratch_bytes"] = _lib.lib().lrf_backward_batch_scratch_bytes(64, 64, 4) - 1
    elif case == "scratch_null":
        kw["scratch"] = None
    elif case == "field_grad_null":
        g.d_w2 = None
    elif case == "plane_grad_null":
        g.d_aline[2] = None
    elif case == "rgb_linear_null":
        kw["x"] = None
    elif case == "grad_rgb_null":
        kw["g_rgb"] = None
    elif case == "grad_depth_null":
        kw["g_depth"] = None
    elif case == "ray_ids_null":
        b.ray_ids = None
    elif case == "cam2world_null":
        b.cam2world = None
    assert _call(batch=b, grads=g, **kw) == INVALID, case
    assert _err()


def test_invalid_messages():
    b = _fake_batch()
    b.rays = FAKE
    assert _call(batch=b) == INVALID and "rays must be NULL" in _err()
    b = _fake_batch()
    b.blend = FAKE
    assert _call(batch=b) == INVALID and "blend" in _err()
    assert _call(scratch_bytes=16) == INVALID and "lrf_backward_batch_scratch_bytes" in _err()


def test_exposure_clamp_invalid():
    L = _lib.lib()
    assert L.lrf_exposure_clamp(FAKE, None, 10, 3, FAKE, None) == INVALID
    assert L.lrf_exposure_clamp(FAKE, None, 12, 0, FAKE, None) == INVALID
    assert L.lrf_exposure_clamp(None, None, 12, 3, FAKE, None) == INVALID
    assert L.lrf_exposure_clamp(FAKE, None, 12, 3, None, None) == INVALID


# ---- the float64 restatement against float64 torch autograd ---------------------------------------------------
def _case(seed, V=3, R=40, W=20, H=15):
    g = torch.Generator().manual_seed(seed)
    n = V * R
    ids = torch.randint(0, W * H, (n,), generator=g) + (torch.arange(n) // R) * W * H
    c2w = torch.randn(V, 3, 4, generator=g, dtype=torch.float64)
    intr = torch.tensor([17.5, 9.3, 7.1], dtype=torch.float64)
    E = torch.eye(3, dtype=torch.float64) + 0.3 * torch.randn(V, 3, 3, generator=g, dtype=torch.float64)
    x = torch.rand(n, 3, generator=g, dtype=torch.float64) * 1.6 - 0.3
    E[0] = torch.eye(3, dtype=torch.float64)            # view 0: identity, so E x hits 0 and 1 exactly
    x[:R:4, 0], x[1:R:4, 1], x[2:R:4, 2] = 0.0, 1.0, 1.0
    w2rf = torch.randn(3, generator=g, dtype=torch.float64)
    d_rays = torch.randn(n, 6, generator=g, dtype=torch.float64)
    g_rgb = torch.randn(n, 3, generator=g, dtype=torch.float64)
    g_dir = torch.randn(n, 3, generator=g, dtype=torch.float64)
    return ids, W, H, c2w, intr, E, x, w2rf, d_rays, g_rgb, g_dir


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("with_dirs", [True, False])
def test_camera_oracle_vs_autograd(seed, with_dirs):
    ids, W, H, c2w, intr, E, x, w2rf, d_rays, g_rgb, g_dir = _case(seed)
    V, n = c2w.shape[0], ids.shape[0]
    leaves = [t.clone().requires_grad_(True) for t in (c2w, intr, E, w2rf)]
    c2w_l, intr_l, E_l, w2_l = leaves
    i, j = ids % W, (ids // W) % H
    dirs = get_ray_directions_lean(i.double(), j.double(), intr_l[0:1], intr_l[1:3])
    cam2rf = c2w_l.clone()
    cam2rf[:, :3, 3] = cam2rf[:, :3, 3] + w2_l
    cam2rf = cam2rf.repeat_interleave(n // V, dim=0)
    rays_o, rays_d = get_rays_lean(dirs, cam2rf)
    rgb = torch.bmm(E_l.repeat_interleave(n // V, dim=0), x[..., None])[..., 0].clamp(0, 1)
    loss = (torch.cat([rays_o, rays_d], -1) * d_rays).sum() + (rgb * g_rgb).sum()
    if with_dirs:
        loss = loss + (dirs * g_dir).sum()
    grads = torch.autograd.grad(loss, leaves)
    ref = camera_oracle.camera_backward(d_rays.numpy(), x.numpy(), g_rgb.numpy(), ids.numpy(), W, H, c2w.numpy(),
                                        intr.numpy(), E.numpy(), g_dir.numpy() if with_dirs else None)
    # get_ray_directions_lean rounds the pixel centres through fp32 (`i.float() + 0.5`): 6e-8 relative in the
    # directions, hence in what multiplies them; everything else is float64
    for key, gt in zip(("d_cam2world", "d_intrinsics", "d_exposure", "d_world2rf"), grads):
        gt = gt.numpy()
        np.testing.assert_allclose(ref[key], gt, rtol=0, atol=1e-6 * np.abs(gt).max(), err_msg=key)
    # the bounds pass the gradient: view 0 has E x exactly 0 / 1 on a quarter of its channels
    y = x[: n // V]
    assert bool(((y == 0) | (y == 1)).any())


def test_camera_oracle_directions_match_ray_utils():
    ids, W, H, c2w, intr, *_ = _case(3)
    i, j = ids % W, (ids // W) % H
    want = get_ray_directions_lean(i.double(), j.double(), intr[0:1], intr[1:3]).numpy()
    np.testing.assert_allclose(camera_oracle.directions(ids.numpy(), W, H, intr.numpy()), want, rtol=0, atol=1e-6)
