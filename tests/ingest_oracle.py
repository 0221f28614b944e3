"""Numpy restatement of the per-frame conversions of LocalRFDataset.read_meta (dataLoader/localrf_dataset.py:143-258)
that lrf_ingest_frame runs on the device, written as the kernels compute them, so each can be held bit for bit
against cv2 / numpy (tests/test_ingest_cpu.py).

    image      img[..., ::-1].astype(float32) / 255, then cv2.resize(fx = fy = 1 / k, INTER_AREA)
    flows      cv2.resize(encoded uint16, image size, INTER_AREA), then decode_flow and * float32(flow_scale)
    invdepth   astype(float32), then cv2.resize(image size, INTER_AREA)
    motion     cv2.resize(uint8, image size, INTER_AREA) > 0
    weight     cv2.Laplacian(cv2.cvtColor((img * 255).astype(uint8), RGB2GRAY), CV_32F).var(), times the mask

INTER_AREA as used here has three forms: the same size is a copy; an integer reduction by k = 2 or 4 is a block
sum in a fixed order (`reduce`) times float32(1 / k^2); an enlargement is separable linear
interpolation with the area rule's weights (`area_weights`), horizontal then vertical, in float32 without fused
multiply-adds, rounded to nearest even and saturated for integer outputs.
"""
import numpy as np

F32 = np.float32


def area_weights(dst, src):
    """Per output index: (source index, weight of the next source index) of cv2's INTER_AREA enlargement along one
    axis of `src` -> `dst` >= src samples.  scale is 1 / (dst / src) in double, as cv::resize forms it."""
    inv_scale = dst / src
    scale = 1.0 / inv_scale
    sx = np.floor(np.arange(dst) * scale).astype(np.int64)
    f = ((np.arange(dst) + 1) - (sx + 1) * inv_scale).astype(F32)
    f = np.where(f <= 0, F32(0), f - np.floor(f)).astype(F32)
    edge = sx >= src - 1
    return np.where(edge, src - 1, sx), np.where(edge, F32(0), f).astype(F32)


def enlarge(a, h, w):
    """a [hs][ws](...) uint16 or float32 -> [h][w](...) by the enlargement rule (h >= hs, w >= ws)."""
    hs, ws = a.shape[:2]
    x = a.astype(F32)
    sx, fx = area_weights(w, ws)
    sy, fy = area_weights(h, hs)
    ex = (slice(None),) + (None,) * (a.ndim - 2)
    x1 = np.minimum(sx + 1, ws - 1)
    hor = x[:, sx] * (F32(1) - fx)[ex] + x[:, x1] * fx[ex]     # two float32 products, one float32 sum
    y1 = np.minimum(sy + 1, hs - 1)
    ey = (slice(None), None) + (None,) * (a.ndim - 2)
    out = hor[sy] * (F32(1) - fy)[ey] + hor[y1] * fy[ey]
    if a.dtype == np.uint16:
        return np.clip(np.rint(out), 0, 65535).astype(np.uint16)
    return out.astype(F32)


def reduce(a, k):
    """a [k h][k w](...) float32 -> [h][w](...), k in {2, 4}, times float32(1 / k^2) after the block sum: for k = 2
    the four values in row-major order, ((a + b) + c) + d; for k = 4 each row's four values in order, then the four
    row sums in order.  (These are what cv2 computes for 3-channel float images; other factors it sums otherwise.)"""
    if k not in (2, 4):
        raise NotImplementedError(f"reduction by {k}")
    h, w = a.shape[0] // k, a.shape[1] // k
    assert a.shape[0] == k * h and a.shape[1] == k * w
    a = a.astype(F32)
    if k == 2:
        s = (((a[0::2, 0::2] + a[0::2, 1::2]) + a[1::2, 0::2]) + a[1::2, 1::2]).astype(F32)
    else:
        rows = [(((a[dy::4, 0::4] + a[dy::4, 1::4]) + a[dy::4, 2::4]) + a[dy::4, 3::4]).astype(F32)
                for dy in range(4)]
        s = (((rows[0] + rows[1]) + rows[2]) + rows[3]).astype(F32)
    return (s * F32(1.0 / (k * k))).astype(F32)


def resize(a, h, w):
    """INTER_AREA to [h][w] in one of its three supported forms; anything else raises NotImplementedError."""
    hs, ws = a.shape[:2]
    if (hs, ws) == (h, w):
        return a.copy()
    if hs % h == 0 and ws % w == 0 and hs // h == ws // w and a.dtype == np.float32:
        return reduce(a, hs // h)
    if h >= hs and w >= ws:
        return enlarge(a, h, w)
    raise NotImplementedError(f"{hs}x{ws} -> {h}x{w}")


def image(bgr, k=1):
    """uint8 BGR [h0][w0][3] -> float32 RGB [h0 / k][w0 / k][3]."""
    img = bgr[..., ::-1].astype(F32) / F32(255)
    return img if k == 1 else reduce(img, k)


def flow(encoded, h, w, flow_scale):
    """uint16 [hf][wf][3] (file channel order) -> flow float32 [h][w][2], mask float32 [h][w]."""
    e = resize(encoded, h, w)
    f = (e[..., :2].astype(F32) - F32(32768)) / F32(256)
    return (f * F32(flow_scale)).astype(F32), (e[..., 2] > 32768).astype(F32)


def invdepth(d, h, w):
    return resize(d.astype(F32), h, w)


def motion(m, h, w):
    """uint8 mask -> bool [h][w] (same size only)."""
    if m.shape[:2] != (h, w):
        raise NotImplementedError("motion masks are taken at the image size only")
    return m > 0


def gray(img):
    """float32 RGB -> cv2's 15-bit RGB2GRAY of (img * 255).astype(uint8), as int32."""
    u = (img * F32(255)).astype(np.uint8).astype(np.int32)
    return (9798 * u[..., 0] + 19235 * u[..., 1] + 3735 * u[..., 2] + (1 << 14)) >> 15


def laplacian(g):
    """4-neighbour Laplacian with reflect-101 borders, float32 (exact: integer values)."""
    p = np.pad(g, 1, mode="reflect")              # numpy's "reflect" is OpenCV's BORDER_REFLECT_101
    return (p[:-2, 1:-1] + p[2:, 1:-1] + p[1:-1, :-2] + p[1:-1, 2:] - 4 * p[1:-1, 1:-1]).astype(F32)


def pairwise_sum(a):
    """numpy's float32 pairwise summation of a contiguous array: leaves of at most 128 values summed with eight
    accumulators, longer runs split at half the length rounded down to a multiple of 8."""
    n = len(a)
    if n < 8:
        s = F32(-0.0)
        for v in a:
            s = F32(s + v)
        return s
    if n <= 128:
        r = [F32(v) for v in a[:8]]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = F32(r[j] + a[i + j])
            i += 8
        s = F32(F32(F32(r[0] + r[1]) + F32(r[2] + r[3])) + F32(F32(r[4] + r[5]) + F32(r[6] + r[7])))
        for v in a[i:]:
            s = F32(s + v)
        return s
    n2 = n // 2
    n2 -= n2 % 8
    return F32(pairwise_sum(a[:n2]) + pairwise_sum(a[n2:]))


def variance(x):
    """np.float32 .var() of a contiguous array, restated: mean = sum / n, then the sum of squared deviations / n."""
    x = np.ascontiguousarray(x, dtype=F32).reshape(-1)
    n = F32(x.size)
    mean = F32(pairwise_sum(x) / n)
    d = (x - mean).astype(F32)
    return F32(pairwise_sum((d * d).astype(F32)) / n)


def loss_weight(img, mask=None, numpy_var=False):
    """float32 [h][w]: the Laplacian variance of the frame, zero where a motion mask is off.  numpy_var takes the
    variance from numpy's own .var() (which `variance` restates in Python, too slowly for large frames)."""
    lap = laplacian(gray(img))
    v = lap.var() if numpy_var else variance(lap)
    w = np.full(img.shape[:2], v, F32)
    return w if mask is None else (w * mask).astype(F32)


def frame(bgr, k=1, depth=None, fwd=None, bwd=None, mask=None, numpy_var=False):
    """Every array read_meta builds for one frame, as a dict of float32 [n_px](w) arrays keyed as in a blob."""
    img = image(bgr, k)
    h, w = img.shape[:2]
    out = {"rgbs": img.reshape(-1, 3)}
    m = motion(mask, h, w) if mask is not None else None
    out["loss_weights"] = loss_weight(img, m, numpy_var).reshape(-1, 1)
    if depth is not None:
        out["invdepths"] = invdepth(depth, h, w).reshape(-1, 1)
    if fwd is not None:
        scale = h / fwd.shape[0]
        for key, e in (("fwd", fwd), ("bwd", bwd)):
            f, fm = flow(e, h, w, scale)
            out[f"{key}_flow"], out[f"{key}_mask"] = f.reshape(-1, 2), fm.reshape(-1, 1)
    return out


def tree_depth(n):
    """Halvings of numpy's recursion over n values until every node is a leaf (what lrf_ingest_frame sizes its slot
    tree by)."""
    sizes, depth = {n}, 0
    while any(s > 128 for s in sizes):
        nxt = set()
        for s in sizes:
            if s > 128:
                h = s // 2 - (s // 2) % 8
                nxt |= {h, s - h}
        sizes, depth = nxt, depth + 1
    return depth


def slot_tree_sum(a):
    """pairwise_sum as lrf_ingest_frame evaluates it: slot i of 2^D sums the leaf the bits of i select (or is empty
    below a leaf that ends higher up), then the slots are added back pairwise, an empty right slot passing the left
    one through.  Equal to pairwise_sum by construction; the CPU tests hold it to np.sum."""
    n, D = len(a), tree_depth(len(a))
    vals, full = [F32(0)] * (1 << D), [False] * (1 << D)
    for i in range(1 << D):
        off, ln, empty = 0, n, False
        for d in range(D - 1, -1, -1):
            if ln <= 128:
                empty = bool(i & ((2 << d) - 1))
                break
            h = ln // 2 - (ln // 2) % 8
            if (i >> d) & 1:
                off, ln = off + h, ln - h
            else:
                ln = h
        if not empty:
            vals[i], full[i] = pairwise_sum(a[off:off + ln]), True
    step = 1
    while step < (1 << D):
        for i in range(0, 1 << D, 2 * step):
            if full[i + step]:
                vals[i] = F32(vals[i] + vals[i + step])
        step *= 2
    return vals[0]


def write_golden_scene(z, scene, d):
    """Writes the files of `scene` stored in tests/golden/ingest.npz under directory d."""
    import os
    prefix = f"file:{scene}/"
    for key in z.files:
        if key.startswith(prefix):
            p = os.path.join(d, key[len(prefix):])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as fh:
                fh.write(z[key].tobytes())


def scene_frames(d, cfg):
    """frame -> the arrays of `frame` for every image of the scene at d, decoded with cv2 as read_meta decodes
    them (consecutive flow names, masks/<frame>.png else masks/all.png)."""
    import os
    import cv2
    names = sorted(os.listdir(os.path.join(d, "images")))
    k = 1 if cfg["downsampling"] == -1 else cfg["downsampling"]
    out = []
    for i, name in enumerate(names):
        base = os.path.splitext(name)[0]
        nxt = os.path.splitext(names[(i + 1) % len(names)])[0]
        mp = os.path.join(d, "masks", base + ".png")
        if not os.path.isfile(mp):
            mp = os.path.join(d, "masks", "all.png")
        m = cv2.imread(mp, cv2.IMREAD_UNCHANGED) if os.path.isfile(mp) else None
        if m is not None and m.ndim != 2:
            m = m[..., 0]
        depth = cv2.imread(os.path.join(d, "depth", base + ".png"), -1) if cfg["load_depth"] else None
        fwd = bwd = None
        if cfg["load_flow"]:
            fwd = cv2.imread(os.path.join(d, "flow_ds", f"fwd_{nxt}.png"), cv2.IMREAD_UNCHANGED)
            bwd = cv2.imread(os.path.join(d, "flow_ds", f"bwd_{base}.png"), cv2.IMREAD_UNCHANGED)
        out.append(frame(cv2.imread(os.path.join(d, "images", name)), k, depth, fwd, bwd, m))
    return out
