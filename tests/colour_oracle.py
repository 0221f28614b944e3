"""numpy restatement of lrf_frame_colours and lrf_colour_extract (include/localrf_b200.h), written from the header's
formulas: float32 operations in the stated order (numpy rounds each one to nearest and never fuses them), integer sums
and fp64 means.

The pinhole pixel is exact.  The fov360 pixel goes through asinf and atan2f, which CUDA computes within a few ulps and
numpy's float64 correctly: the restatement takes the correctly rounded float32 angle, runs the rest of the float32
chain for the angle moved ULPS ulps down and up, and flags the point when the two pixels differ.  Every step after the
angle is monotone, so an unflagged point's pixel is the device's whatever the angle's last bits."""
import numpy as np

F = np.float32
PI = F(np.pi)
ULPS = 8


def _steps(a, k):
    for _ in range(abs(k)):
        a = np.nextafter(a, F(np.inf) if k > 0 else F(-np.inf))
    return a


def camera_coords(xyz, c2w):
    """c_b = (R_0b (p_0 - t_0) + R_1b (p_1 - t_1)) + R_2b (p_2 - t_2), float32 [P, 3]."""
    x = np.asarray(xyz, F)
    M = np.asarray(c2w, F).reshape(3, 4)
    e = [x[:, a] - M[a, 3] for a in range(3)]
    return np.stack([(M[0, b] * e[0] + M[1, b] * e[1]) + M[2, b] * e[2] for b in range(3)], 1)


def project(xyz, W, H, fov360, intr, c2w):
    """-> (i, j, d_v, ok, flagged): the pixel of each point (int64; valid where ok), its depth, whether it projects into
    the frame at all, and (fov360) whether the device's pixel may differ from i, j."""
    c = camera_coords(xyz, c2w)
    P = len(c)
    with np.errstate(all="ignore"):
        if not fov360:
            f, cx, cy = (F(v) for v in np.asarray(intr, F))
            dv = -c[:, 2]
            u = np.floor((c[:, 0] / dv) * f + cx)
            v = np.floor((-c[:, 1] / dv) * f + cy)
            ok = (c[:, 2] < 0) & (u >= 0) & (u.astype(np.float64) < W) & (v >= 0) & (v.astype(np.float64) < H)
            i = np.where(ok, u, 0).astype(np.int64)
            j = np.where(ok, v, 0).astype(np.int64)
            return i, j, dv, ok, np.zeros(P, bool)
        dv = np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2])
        ok = (dv > 0) & np.isfinite(dv)
        q = np.clip(c[:, 1] / dv, F(-1), F(1))
        phi = np.arcsin(q.astype(np.float64)).astype(F)
        theta = np.arctan2(c[:, 0].astype(np.float64), c[:, 2].astype(np.float64)).astype(F)

        def jj(ph):
            t = np.floor(((ph + PI / F(2)) * F(H)) / PI)
            return np.clip(np.where(ok, t, 0), 0, H - 1).astype(np.int64)

        def ii(th):
            t = np.floor(((th - PI) * F(W)) / (F(2) * PI))
            return np.mod(np.where(ok, t, 0).astype(np.int64), W)

        j, i = jj(phi), ii(theta)
        flagged = ok & ((jj(_steps(phi, -ULPS)) != jj(_steps(phi, ULPS))) |
                        (ii(_steps(theta, -ULPS)) != ii(_steps(theta, ULPS))))
        return i, j, dv, ok, flagged


def frame_colours(sums, xyz, normals, W, H, fov360, intr, c2w, depth, acc, image, min_acc, depth_tol, min_cos):
    """Adds one view to sums [P, 5] uint64 in place -> flagged [P] (fov360 points whose pixel may differ)."""
    x = np.asarray(xyz, F)
    M = np.asarray(c2w, F).reshape(3, 4)
    i, j, dv, ok, flagged = project(x, W, H, fov360, intr, M)
    k = np.where(ok, j * W + i, 0)
    a = np.asarray(acc, F).reshape(-1)[k]
    d = np.asarray(depth, F).reshape(-1)[k]
    img = np.asarray(image, F).reshape(-1, 3)[k]
    with np.errstate(all="ignore"):
        s = d / a
        keep = ok & (a >= F(min_acc)) & (a > 0) & np.isfinite(s) & (s > 0) & (np.abs(dv - s) <= F(depth_tol) * s)
        w = np.ones(len(x), F)
        if normals is not None:
            n = np.asarray(normals, F)
            t = [M[a_, 3] - x[:, a_] for a_ in range(3)]
            ln = np.sqrt((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2])
            w = ((n[:, 0] * t[0] + n[:, 1] * t[1]) + n[:, 2] * t[2]) / ln
            keep &= w >= F(min_cos)
        keep &= np.isfinite(img).all(1)
        q = (np.minimum(np.where(keep, w, 0), F(1)) * F(65536)).astype(np.uint64)
        c24 = (np.clip(np.where(keep[:, None], img, 0), F(0), F(1)) * F(16777216)).astype(np.uint64)
    add = np.concatenate([np.ones((len(x), 1), np.uint64), q[:, None], q[:, None] * c24], 1)
    sums[keep] += add[keep]
    return flagged


def colour_extract(sums):
    """-> (rgb [P, 3] uint8, count [P] int32)."""
    sums = np.asarray(sums, np.uint64)
    count = np.minimum(sums[:, 0], np.uint64(2 ** 31 - 1)).astype(np.int32)
    den = sums[:, 1].astype(np.float64) * 16777216.0
    with np.errstate(all="ignore"):
        c = np.floor(sums[:, 2:].astype(np.float64) / den[:, None] * 255.0 + 0.5)
    rgb = np.where(sums[:, 1:2] == 0, 0, c).astype(np.uint8)
    return rgb, count
