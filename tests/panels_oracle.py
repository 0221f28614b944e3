"""numpy restatement of the test-frame comparison panels (renderer.py:79-124), from their formulas.

The flow rows and the statistics are float32 arithmetic as numpy performs it on the reference's float32 arrays, so
given the same predicted flows they are bit-exact.  The predicted flows themselves (get_pred_flow) are computed in
float64 here and rounded once: the reference's bmm order is not restated, so they agree to a few fp32 ulps.
"""
import math

import numpy as np

F32 = np.float32


def nearest_index(src, dst):
    """cv2.resize(..., INTER_NEAREST) source index of every destination index: min(floor(x * (1 / (dst / src))),
    src - 1), with the scale formed in double as OpenCV forms it."""
    inv = 1.0 / (dst / src)
    return np.array([min(math.floor(x * inv), src - 1) for x in range(dst)], dtype=np.int64)


def resize_nearest(a, W, H):
    """a [h0, w0, ...] -> [H, W, ...] with OpenCV's nearest rule."""
    return a[nearest_index(a.shape[0], H)][:, nearest_index(a.shape[1], W)]


def quantile_ranks(n, q=0.9):
    """-> (lo, hi, gamma): the ranks np.quantile(., q) interpolates between in n float32 values, and its weight.
    numpy 2.x keeps q, the virtual index (n - 1) * q, its floor and the weight in float32.  Above 2^24 the float32
    floor + 1 rounds to even, so hi is lo itself or two ranks up as often as the next rank."""
    vi = F32(n - 1) * F32(q)
    prev = np.floor(vi)
    nxt = prev + F32(1)
    lo, hi = int(prev), int(nxt)
    if vi >= F32(n - 1):
        lo = hi = n - 1
    return lo, min(hi, n - 1), F32(vi - prev)


def quantile(a, q=0.9):
    """np.quantile(a, q) (method "linear") for a float32 array, restated: the ranks of quantile_ranks, interpolated
    with _lerp's two branches."""
    a = np.asarray(a, dtype=F32).ravel()
    if np.isnan(a).any():
        return F32(np.nan)
    lo, hi, gamma = quantile_ranks(a.size, q)
    s = np.sort(a, kind="stable")
    A, B = s[lo], s[hi]
    with np.errstate(invalid="ignore", over="ignore"):
        d = F32(B - A)
        if gamma >= F32(0.5):
            return F32(B - F32(d * F32(F32(1) - gamma)))
        return F32(A + F32(d * gamma))


def hi_mode(W, H):
    """Where numpy's upper neighbour of the 0.9 quantile of a W x H frame's 2 W H values lies: 0 the lower rank
    itself, 1 the next rank, 2 two ranks up (lrf_panels.cu's hi_mode)."""
    lo, hi, _ = quantile_ranks(2 * W * H)
    return hi - lo


def neighbour_gt(W, H, inf_from, seed):
    """A ground-truth channel of W H values such that [zeros(W H); gt] sorted is finite below rank `inf_from` and
    +inf from it on (inf_from >= W H; None: no infinity): shuffled negatives and positives, then the infinities."""
    N = W * H
    k_inf = 0 if inf_from is None else 2 * N - inf_from
    g = np.random.default_rng(seed)
    finite = g.uniform(0.5, 2.0, N - k_inf) * np.where(g.random(N - k_inf) < 0.5, -1.0, 1.0)
    return g.permutation(np.concatenate([finite, np.full(k_inf, np.inf)])).astype(F32)


def lower_median(a):
    """torch.median of a flat array: the lower median sorted[(n - 1) // 2], NaN when the array holds a NaN."""
    a = np.asarray(a, dtype=F32).ravel()
    if np.isnan(a).any():
        return F32(np.nan)
    return np.sort(a)[(a.size - 1) // 2]


def cam2cam(cam2world, idx, offset):
    """get_cam2cams for one camera in float64: [3,4] = (Rk^T Rrel, Rk^T (trel - tk)), k = clamp(idx + offset)."""
    c = np.asarray(cam2world, dtype=np.float64)
    k = min(max(idx + offset, 0), len(c) - 1)
    Rk, tk, Rl, tl = c[k, :, :3], c[k, :, 3], c[idx, :, :3], c[idx, :, 3]
    return np.concatenate([Rk.T @ Rl, (Rk.T @ (tl - tk))[:, None]], 1)


def pred_flow(depth, directions, cam2world, idx, offset, focal, center, W, H):
    """get_pred_flow for the frame's W*H rays -> [H, W, 2] float32 (float64 arithmetic, one rounding)."""
    m = cam2cam(cam2world, idx, offset)
    pts = np.asarray(directions, np.float32).astype(np.float64) * np.asarray(depth, np.float32).astype(np.float64)[:, None]
    q = pts @ m[:, :3].T + m[:, 3]
    z = np.maximum(-q[:, 2], 1e-6)
    p = np.arange(W * H)
    u = q[:, 0] / z * float(focal) + float(center[0]) - 0.5 - (p % W)
    v = -q[:, 1] / z * float(focal) + float(center[1]) - 0.5 - (p // W)
    return np.stack([u, v], -1).astype(np.float32).reshape(H, W, 2)


def flow_panel(pred, flow, mask, W):
    """[3H, 2W] panel of one direction from the predicted flow [H,W,2] and the RESIZED ground truth flow [H,W,2] /
    mask [H,W] -> (panel, (q0, q1))."""
    cols, qs = [], []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for c in range(2):
            cmp = np.vstack([pred[..., c], flow[..., c]]).astype(F32)
            q = quantile(cmp)
            qs.append(q)
            cmp = cmp / q
            err = np.abs(pred[..., c] - flow[..., c]) * mask / F32(W)
            cols.append(np.vstack([cmp, err]))
        panel = np.hstack(cols)
    return np.clip(panel, F32(0), F32(1)), tuple(qs)


def normalise(v):
    """(v - t) / s with t the lower median and s the mean of |v - t| in float64, rounded once -> (vn, t, s)."""
    v = np.asarray(v, dtype=F32).ravel()
    t = lower_median(v)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        r = np.abs(v - t).astype(np.float64)
        s = F32(math.fsum(r.tolist()) / v.size) if np.isfinite(r).all() else F32(np.mean(r))
        return (v - t) / s, t, s


def depth_panel(depth, invdepth, W, H):
    """[3H, W] panel from the rendered depth [W*H] and the RESIZED inverse depth [H, W] -> (panel, (tx, sx, tg, sg))."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        x = F32(1) / np.maximum(np.asarray(depth, F32).ravel(), F32(1e-6))
        xn, tx, sx = normalise(x)
        gn, tg, sg = normalise(np.asarray(invdepth, F32).ravel())
        panel = np.vstack([(F32(0.5) * xn).reshape(H, W), (F32(0.5) * gn).reshape(H, W),
                           ((xn - gn) * (xn - gn)).reshape(H, W)])
    return np.clip(panel, F32(0), F32(1)), (tx, sx, tg, sg)


# ---- the fixture's cases (tests/golden/make_golden_panels.py): inputs regenerated from a seed, so the fixture only
# stores outputs and a checksum of the inputs --------------------------------------------------------------------
CASES = {
    # name: (seed, W, H, h0, w0, n_cams, idx, kind)
    "base_64x48": (1, 64, 48, 96, 128, 6, 3, "random"),
    "odd_37x23": (2, 37, 23, 61, 100, 5, 2, "random"),
    "up_64x48": (3, 64, 48, 15, 20, 4, 1, "random"),
    "idx_first": (4, 40, 30, 60, 80, 5, 0, "random"),
    "idx_last": (5, 40, 30, 60, 80, 5, 4, "random"),
    "zero_flow": (6, 32, 24, 48, 64, 1, 0, "zero_flow"),
    "tiny_depth": (7, 48, 32, 64, 96, 4, 2, "tiny_depth"),
    "zero_mask": (8, 40, 30, 60, 80, 4, 2, "zero_mask"),
    "big_480x270": (9, 480, 270, 540, 960, 8, 5, "random"),
}
FULL_OUTPUT_PIXELS = 64 * 48          # cases up to this size store whole panels; larger ones a fixed sample


def make_case(name):
    """-> dict of the case's inputs, float32 numpy (directions of a pinhole camera, as get_ray_directions_lean)."""
    return build_case(*CASES[name])


def build_case(seed, W, H, h0, w0, n_cams, idx, kind="random"):
    """The inputs of one frame of the given sizes and kind (see CASES), regenerated from `seed`."""
    g = np.random.default_rng(seed)
    rot = []
    for _ in range(n_cams):
        q, r = np.linalg.qr(np.eye(3) + 0.05 * g.standard_normal((3, 3)))
        rot.append(q * np.sign(np.diag(r))[None, :])
    t = np.stack([0.02 * g.standard_normal(3) + np.array([0.0, 0.0, -0.1 * i]) for i in range(n_cams)])
    cam2world = np.concatenate([np.stack(rot), t[..., None]], -1).astype(F32)
    focal, center = F32(0.9 * W), np.array([W / 2.0, H / 2.0], F32)
    p = np.arange(W * H)
    i, j = (p % W).astype(F32), (p // W).astype(F32)
    depth = (0.5 + 4.5 * g.random(W * H)).astype(F32)
    fwd_flow = (3 * g.standard_normal((h0, w0, 2))).astype(F32)
    bwd_flow = (3 * g.standard_normal((h0, w0, 2))).astype(F32)
    fwd_mask = (g.random((h0, w0)) > 0.2).astype(F32)
    bwd_mask = (g.random((h0, w0)) > 0.2).astype(F32)
    invdepth = (g.random((h0, w0)) + 0.1).astype(F32)
    if kind == "zero_flow":         # identity camera, unit depth, rays through the pixel centres: pred is exactly 0
        cam2world = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)[None].astype(F32)
        focal, center = F32(1.0), np.zeros(2, F32)
        depth = np.ones(W * H, F32)
        dirs = np.stack([i + F32(0.5), -(j + F32(0.5)), -np.ones_like(i)], -1).astype(F32)
        fwd_flow[:] = 0
        bwd_flow[...] = 0
        bwd_flow[: h0 // 8] = 2.0                    # 1/8 positive: q stays 0, those rows become inf -> 1
    else:
        dirs = np.stack([(i + F32(0.5) - center[0]) / focal, -(j + F32(0.5) - center[1]) / focal,
                         -np.ones_like(i)], -1).astype(F32)
    if kind == "tiny_depth":
        k = g.permutation(W * H)[:40]
        depth[k] = np.array([0.0, 1e-7, 1e-6, 5e-7], F32)[np.arange(40) % 4]
    if kind == "zero_mask":
        fwd_mask[:] = 0
        bwd_mask[:] = 0
    return dict(W=W, H=H, idx=idx, cam2world=cam2world, focal=focal, center=center, depth=depth, directions=dirs,
                fwd_flow=fwd_flow, fwd_mask=fwd_mask, bwd_flow=bwd_flow, bwd_mask=bwd_mask, invdepth=invdepth)


def input_digest(c):
    import hashlib
    h = hashlib.sha256()
    for k in ("cam2world", "focal", "center", "depth", "directions", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask",
              "invdepth"):
        h.update(np.ascontiguousarray(c[k]).tobytes())
    return h.hexdigest()


def sample_index(name, size, n=4096):
    """The fixed flat positions a large case's outputs are stored at."""
    return np.sort(np.random.default_rng(1000 + CASES[name][0]).choice(size, size=min(n, size), replace=False))


# ---- tolerances against the reference's block ----------------------------------------------------------------
EPS = float(np.finfo(np.float32).eps)


def ulps(a, b):
    """Distance in fp32 ulps between two finite float32 values of one sign."""
    a, b = np.float32(a), np.float32(b)
    return abs(int(a.view(np.int32)) - int(b.view(np.int32)))


def depth_bound(depth, invdepth, W, H, s_ulps=1):
    """Per-element bound [3H, W] on |panel - reference panel| for the depth panel when the two differ only in the
    MAD scales s, by at most s_ulps fp32 ulps each (the reference takes torch's fp32 mean, the kernel rounds an fp64
    mean once).  Then xn = (v - t) / s moves by at most (s_ulps + 1) eps |xn| (s, then one rounding of the
    quotient); the halved rows by (s_ulps + 2) eps |0.5 xn|; the squared row by 2 |df| dd + dd^2 + eps df^2 with
    dd = (s_ulps + 1) eps (|xn| + |gn|) + eps |df| bounding the change of df = xn - gn.  Clamping to [0, 1] does not
    increase a difference."""
    k = float(s_ulps)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        x = F32(1) / np.maximum(np.asarray(depth, F32).ravel(), F32(1e-6))
        xn, _, _ = normalise(x)
        gn, _, _ = normalise(np.asarray(invdepth, F32).ravel())
        xn, gn = xn.astype(np.float64), gn.astype(np.float64)
        df = xn - gn
        dd = (k + 1) * EPS * (np.abs(xn) + np.abs(gn)) + EPS * np.abs(df)
        rows = [(k + 2) * EPS * np.abs(0.5 * xn), (k + 2) * EPS * np.abs(0.5 * gn),
                2 * np.abs(df) * dd + dd * dd + EPS * df * df]
    return np.vstack([r.reshape(H, W) for r in rows]) + 1e-12


def within(a, b, bound):
    """|a - b| <= bound elementwise, NaN only where both are NaN, equal infinities."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    ok = ~np.isnan(a)
    with np.errstate(invalid="ignore"):
        d = np.where(a[ok] == b[ok], 0.0, np.abs(a[ok] - b[ok]))
    return bool(np.all(d <= np.broadcast_to(bound, a.shape)[ok]))


def flow_bound(ref, W, H):
    """Bound on |pred - reference pred|: 1e-5 max(1, |flow|), or 4 eps (W + H + |flow|) where that is larger --
    pts2px adds terms of the image's size (x / z * f and cx) before subtracting the pixel, so fp32 arithmetic in
    any order leaves absolute errors of a few eps (W + H) however small the flow is."""
    ref = np.abs(np.asarray(ref, np.float64))
    return np.maximum(1e-5 * np.maximum(1.0, ref), 4 * EPS * (W + H + ref))
