"""float64 restatement of the camera side of the training call's backward (lrf_render_backward_batch, stages 1 and
3): from dL/d(rays) [n,6], the pre-exposure colour x [n,3] and the output gradients, the gradients of cam2world,
the intrinsics (focal, cx, cy), the exposure and world2rf, and d_dir = dL/d(camera-space directions).

Forward being differentiated (local_tensorfs.py:397-499, one field):
    dir  = ((i + .5 - cx) / f, -(j + .5 - cy) / f, -1)         (get_ray_directions_lean; fov 360: no intrinsics)
    rays = (t_v + world2rf, R_v dir)                              (get_rays_lean)
    rgb  = clamp(E_v x, 0, 1)                                     (bmm + clamp; both ends pass the gradient)
"""
import numpy as np


def directions(ray_ids, W, H, intr, fov360=False):
    ids = np.asarray(ray_ids, np.int64)
    i = (ids % W).astype(np.float64) + 0.5
    j = ((ids // W) % H).astype(np.float64) + 0.5
    if fov360:
        phi = j * np.pi / H - np.pi / 2
        theta = i * 2 * np.pi / W + np.pi
        return np.stack([np.cos(phi) * np.sin(theta), np.sin(phi), np.cos(phi) * np.cos(theta)], -1)
    f, cx, cy = (float(v) for v in intr)
    return np.stack([(i - cx) / f, -(j - cy) / f, -np.ones_like(i)], -1)


def camera_backward(d_rays, x, grad_rgb, ray_ids, W, H, cam2world, intr, exposure=None, grad_directions=None,
                    fov360=False):
    """-> dict d_cam2world [V,3,4], d_intrinsics [3], d_exposure [V,3,3], d_world2rf [3], d_dir [n,3] (float64)."""
    d_rays = np.asarray(d_rays, np.float64)
    x = np.asarray(x, np.float64)
    g = np.asarray(grad_rgb, np.float64)
    c2w = np.asarray(cam2world, np.float64)
    V, n = c2w.shape[0], d_rays.shape[0]
    view = np.arange(n) // (n // V)
    E = np.broadcast_to(np.eye(3), (V, 3, 3)) if exposure is None else np.asarray(exposure, np.float64)
    y = np.einsum("nab,nb->na", E[view], x)
    gp = g * ((y >= 0) & (y <= 1))                                    # clamp backward, bounds included
    dirs = directions(ray_ids, W, H, intr, fov360)
    d_o, d_d = d_rays[:, :3], d_rays[:, 3:]
    d_c2w = np.zeros((V, 3, 4))
    np.add.at(d_c2w[:, :, :3], view, d_d[:, :, None] * dirs[:, None, :])
    np.add.at(d_c2w[:, :, 3], view, d_o)
    d_exp = np.zeros((V, 3, 3))
    np.add.at(d_exp, view, gp[:, :, None] * x[:, None, :])
    d_dir = np.einsum("nab,na->nb", c2w[view, :, :3], d_d)
    if grad_directions is not None:
        d_dir = d_dir + np.asarray(grad_directions, np.float64)
    if fov360:
        d_intr = np.zeros(3)
    else:
        f = float(intr[0])
        d_intr = np.array([-(d_dir[:, 0] * dirs[:, 0] + d_dir[:, 1] * dirs[:, 1]).sum() / f,
                           -d_dir[:, 0].sum() / f, d_dir[:, 1].sum() / f])
    return dict(d_cam2world=d_c2w, d_intrinsics=d_intr, d_exposure=d_exp, d_world2rf=d_o.sum(0), d_dir=d_dir)
