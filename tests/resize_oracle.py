"""numpy restatement of cv2.resize(src, (W, H)) -- INTER_LINEAR on a float32 [h0, w0, 3] image -- as OpenCV's portable
code computes it (IPP disabled, or a build without IPP).  lrf_resize_linear must equal it bit for bit.

Three forms:
  * the same size: a copy;
  * exactly 2x on both axes (w0 == 2 W and h0 == 2 H): OpenCV switches to INTER_AREA, whose 2x2 block sum is
    (((a + b) + c) + d) * 0.25 in row-major order;
  * anything else: separable linear.  Per output column, in double, scale_x = 1 / (W / w0) and
    fx = float((dx + 0.5) scale_x - 0.5), sx = floor(fx), fx -= sx in float; sx < 0 gives sx = 0, fx = 0; a column
    with sx + 1 >= w0 copies S[min(sx, w0 - 1)], the others are S[sx] (1 - fx) + S[sx + 1] fx.  Rows take fy the same
    way but are never reset: rows clamp(sy) and clamp(sy + 1) are blended with (1 - fy, fy) even when the clamp makes
    them one row.  Horizontal pass first, into float32 rows, then the vertical pass.
Every product and sum rounds once (float32 numpy arithmetic, no FMA).
"""
import numpy as np

F32 = np.float32


def _coeffs(dst, src):
    """-> (s, f): float32 blend weight f of index s + 1 for each of `dst` outputs over `src` inputs, before any
    border rule."""
    scale = 1.0 / (float(dst) / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(F32)).astype(F32)


def area2(a):
    """The exact 2x reduction of a [2H, 2W, 3] float32 image: row-major block sum times 0.25."""
    s = ((a[0::2, 0::2] + a[0::2, 1::2]) + a[1::2, 0::2]) + a[1::2, 1::2]
    return (s * F32(0.25)).astype(F32)


def linear(a, W, H):
    """The separable linear form (no 2x switch) of a [h0, w0, 3] float32 image to [H, W, 3]."""
    h0, w0 = a.shape[:2]
    sx, fx = _coeffs(W, w0)
    neg = sx < 0
    sx[neg], fx[neg] = 0, F32(0)
    copy = sx + 1 >= w0
    sx0 = np.minimum(sx, w0 - 1)
    sx1 = np.minimum(sx + 1, w0 - 1)
    ax = (F32(1) - fx).astype(F32)
    blend = a[:, sx0] * ax[None, :, None] + a[:, sx1] * fx[None, :, None]
    rows = np.where(copy[None, :, None], a[:, sx0], blend).astype(F32)      # [h0, W, 3]
    sy, fy = _coeffs(H, h0)
    sy0, sy1 = np.clip(sy, 0, h0 - 1), np.clip(sy + 1, 0, h0 - 1)
    ay = (F32(1) - fy).astype(F32)
    return (rows[sy0] * ay[:, None, None] + rows[sy1] * fy[:, None, None]).astype(F32)


def row_chunk(row, W, x0, x1):
    """Columns [x0, x1) of linear(a, W, 1) for a 1-row image a whose row is the torch float32 tensor `row` [w0, 3],
    on row's device: the same rule as _coeffs and linear (the index in float64, rounded to float32, then every
    product and sum of the blend a separate float32 operation).  For rows too long to restate on the host."""
    import torch
    w0 = row.shape[0]
    x = torch.arange(x0, x1, dtype=torch.float64, device=row.device)
    f = ((x + 0.5) * (1.0 / (float(W) / w0)) - 0.5).to(torch.float32)
    s = torch.floor(f)
    fx = f - s
    s = s.to(torch.int64)
    neg = s < 0
    s = torch.where(neg, 0, s)
    fx = torch.where(neg, 0, fx)
    copy = (s + 1 >= w0)[:, None]
    a0, a1 = row[s.clamp(max=w0 - 1)], row[(s + 1).clamp(max=w0 - 1)]
    h = torch.where(copy, a0, a0 * (1 - fx)[:, None] + a1 * fx[:, None])
    _, fy = _coeffs(1, 1)                                 # one row: weights (1, 0) on the row itself
    return h * float(F32(1) - fy[0]) + h * float(fy[0])


def resize(a, W, H):
    """cv2.resize(a, (W, H)) of a float32 [h0, w0, 3] image, as OpenCV computes it without IPP."""
    a = np.ascontiguousarray(a, dtype=F32)
    h0, w0 = a.shape[:2]
    if (w0, h0) == (W, H):
        return a.copy()
    if w0 == 2 * W and h0 == 2 * H:
        return area2(a)
    return linear(a, W, H)
