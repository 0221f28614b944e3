"""numpy restatement of lrf_frame_colours and lrf_colour_extract (include/localrf_b200.h), written from the header's
formulas: float32 operations in the stated order (numpy rounds each one to nearest and never fuses them), integer sums
and the extract's exact integer quotient.  frame_colours64 below is an independent float64 reference of the same
operation from the camera model of ray_utils.

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
        keep &= q > 0                                    # a view of weight 0 adds nothing, the count included
        c24 = (np.clip(np.where(keep[:, None], img, 0), F(0), F(1)) * F(16777216)).astype(np.uint64)
    add = np.concatenate([np.ones((len(x), 1), np.uint64), q[:, None], q[:, None] * c24], 1)
    sums[keep] += add[keep]
    return flagged


def extract_exact(S, Q):
    """floor(255 S / (Q 2^24) + 1/2) of Python integers (0 for Q = 0), saturated at 255: (510 S + Q 2^24) // (Q 2^25)."""
    return 0 if Q == 0 else min((510 * S + (Q << 24)) // (Q << 25), 255)


def colour_extract(sums):
    """-> (rgb [P, 3] uint8, count [P] int32), the means exact in Python integers."""
    sums = np.asarray(sums, np.uint64)
    count = np.minimum(sums[:, 0], np.uint64(2 ** 31 - 1)).astype(np.int32)
    Q = sums[:, 1:2].astype(object)
    num = sums[:, 2:].astype(object) * 510 + Q * (1 << 24)
    den = np.where(Q == 0, 1, Q * (1 << 25))
    rgb = np.where(Q == 0, 0, np.minimum(num // den, 255)).astype(np.uint8)
    return rgb, count


U32 = 2.0 ** -24                      # unit roundoff of float32


def _ulp32(a):
    a = np.abs(np.asarray(a, np.float64)).astype(F)
    return (np.nextafter(a, F(np.inf)) - a).astype(np.float64)


def frame_colours64(xyz, normals, views, min_acc, depth_tol, min_cos, slack=2.0):
    """An independent float64 reference of localrf_b200.export.frame_colours, from the camera model of ray_utils.

    views: one dict per view with c2w [3, 4] (LocalTensorfs.get_cam2world() of the view: o = c2w[:, 3], R =
    c2w[:, :3]), fov360, for pinhole focal and center [2] (lt.focal(w), lt.center(w, h)), depth and acc [h, w] (the
    device's float32 render) and image [h, w, 3].  A point's camera coordinates are c = R^T (p - o).
    - pinhole: get_ray_directions_lean gives pixel (i, j) the direction ((i + 0.5 - cx) / f, -(j + 0.5 - cy) / f, -1),
      so c lies on the ray of the continuous pixel u = cx + f c_0 / d, v = cy - f c_1 / d at planar depth d = -c_2
      (which is what the render's depth measures along a z = -1 direction).  Pixel centres sit at i + 0.5, so the point
      lands in (floor(u), floor(v)) when c_2 < 0 and that lies in [0, w) x [0, h).
    - fov360: get_ray_directions_360 gives (i, j) the unit direction at phi = (j + 0.5) pi / h - pi / 2, theta =
      (i + 0.5) 2 pi / w + pi, so with r = |c| (the depth: the directions are unit vectors), phi = asin(c_1 / r) and
      theta = atan2(c_0, c_2): u = (theta - pi) w / (2 pi) mod w, v = (phi + pi / 2) h / pi, and the pixel is
      (floor(u), min(floor(v), h - 1)) (v = h is the upper pole).
    The pixel counts when acc >= min_acc, acc > 0, s = depth / acc is finite and > 0 and |d - s| <= depth_tol s; with
    normals the weight is w = n . (o - p) / |o - p| and needs w >= min_cos; a pixel with a non-finite channel does not
    count.  It adds q = floor(min(w, 1) 2^16) (1 without normals) when q > 0, and q floor(clamp(channel, 0, 1) 2^24),
    into Python-integer sums; rgb = floor(255 sum q c24 / (sum q 2^24) + 1/2), exactly.

    A (point, view) pair is flagged when a decision lies within `slack` times a first-order bound of the float32
    chain's rounding error of its boundary.  The bound counts one unit roundoff U = 2^-24 per float32 operation on
    each term's magnitude: E_b = 3 U sum_a |R_ab| (|p_a| + |o_a|) on c_b; the quotient, product and sum on u, v; the
    range and the quotient c_1 / r (propagated through asin exactly, so the bound stays finite at the poles) and
    ULPS ulps of the float32 asinf and atan2f; s = depth / acc; the weight's nine operations (about 9 U of w, so
    with normals a few per cent of the counted pairs have w 2^16 that close to an integer and are flagged).  The decisions: u or v
    against an integer (the frame's edges, the fov360 seam and the row clamp at the poles included), c_2 against 0
    and r against 0, |d - s| against depth_tol s, acc against min_acc, w against min_cos, and w 2^16 against an
    integer.

    -> dict(rgb [P, 3] uint8, count [P] int64, flagged [P] bool (a view of the point is flagged), n_flagged (flagged
    pairs), n_pairs)."""
    x = np.asarray(xyz, F).astype(np.float64)
    nrm = None if normals is None else np.asarray(normals, F).astype(np.float64)
    P = len(x)
    cnt = np.zeros(P, np.int64)
    Q = np.zeros(P, object)
    S = np.zeros((P, 3), object)
    flagged = np.zeros(P, bool)
    n_flagged = 0
    sl = slack * U32
    for view in views:
        M = np.asarray(view["c2w"], F).astype(np.float64).reshape(3, 4)
        R, o = M[:, :3], M[:, 3]
        depth = np.asarray(view["depth"], F)
        acc_m = np.asarray(view["acc"], F)
        img = np.asarray(view["image"], F)
        h, w = img.shape[:2]
        with np.errstate(all="ignore"):
            c = (x - o) @ R
            E = 3 * sl * ((np.abs(x) + np.abs(o)) @ np.abs(R))
            if not view["fov360"]:
                f = float(np.float32(view["focal"]))
                cx, cy = (float(np.float32(a)) for a in view["center"])
                d = -c[:, 2]
                Ed = E[:, 2]
                xr, yr = c[:, 0] / d, -c[:, 1] / d
                u, v = cx + f * xr, cy + f * yr
                Eu = abs(f) * ((E[:, 0] + np.abs(xr) * Ed) / np.abs(d) + sl * np.abs(xr)) + sl * 2 * (np.abs(u) + abs(cx))
                Ev = abs(f) * ((E[:, 1] + np.abs(yr) * Ed) / np.abs(d) + sl * np.abs(yr)) + sl * 2 * (np.abs(v) + abs(cy))
                near = (u + Eu >= 0) & (u - Eu <= w) & (v + Ev >= 0) & (v - Ev <= h)
                amb = near & (c[:, 2] < Ed) & ((np.abs(c[:, 2]) <= Ed) | (np.floor(u - Eu) != np.floor(u + Eu)) |
                                               (np.floor(v - Ev) != np.floor(v + Ev)))
                ok = (c[:, 2] < 0) & (u >= 0) & (u < w) & (v >= 0) & (v < h)
                i, j = np.where(ok, np.floor(u), 0).astype(np.int64), np.where(ok, np.floor(v), 0).astype(np.int64)
            else:
                d = np.sqrt((c * c).sum(1))
                Ed = (np.abs(c) * E).sum(1) / d + 2 * sl * d
                y = np.clip(c[:, 1] / d, -1, 1)
                Ey = (E[:, 1] + np.abs(y) * Ed) / d + sl
                phi = np.arcsin(y)
                Ephi = (np.maximum(np.abs(np.arcsin(np.clip(y - Ey, -1, 1)) - phi),
                                   np.abs(np.arcsin(np.clip(y + Ey, -1, 1)) - phi)) + ULPS * _ulp32(phi)
                        + sl * np.abs(phi))
                rho2 = c[:, 0] ** 2 + c[:, 2] ** 2
                theta = np.arctan2(c[:, 0], c[:, 2])
                Eth = ((np.abs(c[:, 2]) * E[:, 0] + np.abs(c[:, 0]) * E[:, 2]) / rho2 + ULPS * _ulp32(theta)
                       + sl * np.abs(theta))
                Eth = np.where(np.sqrt(rho2) <= E[:, 0] + E[:, 2], np.inf, Eth)
                v = (phi + np.pi / 2) * h / np.pi
                u = (theta - np.pi) * w / (2 * np.pi)
                Ev = h / np.pi * (Ephi + 2 * sl * (np.abs(phi) + np.pi / 2))
                Eu = w / (2 * np.pi) * (Eth + 2 * sl * (np.abs(theta) + np.pi))
                row = lambda t: np.clip(np.floor(t), 0, h - 1)
                ok = (d > 0) & np.isfinite(d)
                amb = ok & (((np.floor(u + Eu) != np.floor(u - Eu)) & (w > 1)) | (row(v - Ev) != row(v + Ev)) |
                            (d <= Ed) | (d > 2.0 ** 60) | (d < 2.0 ** -60))
                i = np.mod(np.where(ok, np.floor(u), 0), w).astype(np.int64)
                j = np.where(ok, row(v), 0).astype(np.int64)
            k = j * w + i
            a = acc_m.reshape(-1)[k].astype(np.float64)
            s = depth.reshape(-1)[k].astype(np.float64) / a
            ok &= (a >= min_acc) & (a > 0) & np.isfinite(s) & (s > 0)
            amb |= ok & ((np.abs(a - min_acc) <= sl * abs(min_acc)) | (np.abs(s) >= 2.0 ** 127) | (np.abs(s) < 2.0 ** -125))
            gap = np.abs(d - s) - depth_tol * s
            Eg = Ed + sl * (3 * np.abs(s) + np.abs(d - s) + 2 * depth_tol * np.abs(s))
            amb |= ok & (np.abs(gap) <= Eg)
            ok &= gap <= 0
            wt = np.ones(P)
            if nrm is not None:
                t = o - x
                ln = np.sqrt((t * t).sum(1))
                wt = (nrm * t).sum(1) / ln
                Ew = sl * (4 * (np.abs(nrm) * np.abs(t)).sum(1) / ln + 4 * np.abs(wt))
                amb |= ok & (np.abs(wt - min_cos) <= Ew + sl * min_cos)
                ok &= wt >= min_cos
                w16 = wt * 65536
                amb |= ok & (wt <= 1 + Ew) & (np.abs(w16 - np.round(w16)) <= 65536 * Ew)
            pix = img.reshape(-1, 3)[k].astype(np.float64)
            ok &= np.isfinite(pix).all(1)
            q = np.floor(np.minimum(np.where(ok, wt, 0), 1) * 65536).astype(np.int64)
            ok &= q > 0
            c24 = np.floor(np.clip(np.where(ok[:, None], pix, 0), 0, 1) * 2.0 ** 24).astype(np.int64)
        flagged |= amb
        n_flagged += int(amb.sum())
        idx = np.nonzero(ok)[0]
        cnt[idx] += 1
        Q[idx] += q[idx].astype(object)
        S[idx] += q[idx, None].astype(object) * c24[idx].astype(object)
    rgb = np.zeros((P, 3), np.uint8)
    for p in np.nonzero(cnt)[0].tolist():
        for ch in range(3):
            rgb[p, ch] = extract_exact(int(S[p, ch]), int(Q[p]))
    return dict(rgb=rgb, count=cnt, flagged=flagged, n_flagged=n_flagged, n_pairs=P * len(views))
