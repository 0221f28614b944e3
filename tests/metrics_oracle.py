"""numpy restatement of the test-frame metrics (renderer.py:162-163; rgb_ssim, utils/utils.py:232-287) and of the
8-bit frame conversions (renderer.py:127,176; visualize_depth, utils/utils.py:179-197), written from the formula.
TEST INFRASTRUCTURE: the tests of localrf_b200/metrics.py, lrf_frame_to_u8 and tools/metrics_time.py compare the
device kernels against it; nothing under localrf_b200/ imports it."""
import math

import numpy as np


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def mse(img, gt):
    """mean((gt - img)^2): fp32 differences and squares, summed in fp64."""
    d = _f32(gt) - _f32(img)
    return float(np.sum((d * d).astype(np.float64)) / d.size)


def kernel_taps(filter_size, filter_sigma):
    """The Gaussian taps as lrf_metrics.cu's gaussian_taps forms them: one libm exp per tap, a sequential sum,
    then one division per tap.  The reference's vectorised np.exp and pairwise np.sum may differ from these in
    the last bit of a tap."""
    hw = filter_size // 2
    shift = (2 * hw - filter_size + 1) / 2.0
    f = [math.exp(-0.5 * (x * x)) for x in (((k - hw) + shift) / filter_sigma for k in range(filter_size))]
    s = 0.0
    for v in f:
        s += v
    return np.array([v / s for v in f])


def ssim(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False,
         taps="reference"):
    """SSIM of two [H,W,3] float32 frames: the squares and the cross product are fp32 products, the separable
    "valid" Gaussian filter (first along H, then along W) and the map are fp64.  taps="reference" builds the
    filter as rgb_ssim does (utils/utils.py:251-255); taps="kernel" as the device kernel does (kernel_taps), with
    which the map is the kernel's operation for operation."""
    a, b = _f32(img0), _f32(img1)
    assert a.ndim == 3 and a.shape[-1] == 3 and a.shape == b.shape
    if taps == "kernel":
        f = kernel_taps(filter_size, filter_sigma)
    else:
        assert taps == "reference", taps
        hw = filter_size // 2
        shift = (2 * hw - filter_size + 1) / 2
        f = np.exp(-0.5 * ((np.arange(filter_size) - hw + shift) / filter_sigma) ** 2)
        f = f / np.sum(f)

    def filt(z):                       # taps summed from the window's last pixel to its first, as convolve2d does
        z = z.astype(np.float64)
        ho, wo = z.shape[0] - filter_size + 1, z.shape[1] - filter_size + 1
        v = sum(f[k] * z[k:k + ho] for k in reversed(range(filter_size)))
        return sum(f[k] * v[:, k:k + wo] for k in reversed(range(filter_size)))

    mu0, mu1 = filt(a), filt(b)
    mu00, mu11, mu01 = mu0 * mu0, mu1 * mu1, mu0 * mu1
    s00 = np.maximum(0.0, filt(a * a) - mu00)
    s11 = np.maximum(0.0, filt(b * b) - mu11)
    s01 = filt(a * b) - mu01
    s01 = np.sign(s01) * np.minimum(np.sqrt(s00 * s11), np.abs(s01))
    c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    m = (2 * mu01 + c1) * (2 * s01 + c2) / ((mu00 + mu11 + c1) * (s00 + s11 + c2))
    return m if return_map else float(np.mean(m))


INT_MIN = -2 ** 31


def rgb8(rgb):
    """[..., 3] float32 rgb -> the uint8 BGR bytes cv2.imwrite(255 * rgb[..., ::-1]) stores (renderer.py:176):
    255 * v in float32, then OpenCV's saturate_cast<uchar>(float) on x86-64 -- round half to even, and NaN or a
    rounded value outside int32 becomes INT_MIN, which saturates to 0."""
    with np.errstate(over="ignore", invalid="ignore"):
        v = (255 * _f32(rgb))[..., ::-1]              # float32: a Python-number factor keeps the array's dtype
        r = np.rint(v).astype(np.float64)
        ok = (r >= INT_MIN) & (r < 2.0 ** 31)           # False for NaN
    return np.clip(np.where(ok, r, INT_MIN), 0, 255).astype(np.uint8)


def depth8(depth, lo, hi, lut):
    """visualize_depth(depth, [lo, hi]) (utils/utils.py:179-197) with its colour map given as lut [256,3]:
    lut[(255 * clip((nan_to_num(d) - lo) / (hi - lo + 1e-8), 0, 1)).astype(uint8)].  lo and hi are Python
    numbers, as renderer.py:127 passes them, so the arithmetic is float32 with hi - lo + 1e-8 formed in double."""
    x = np.nan_to_num(_f32(depth))
    lo, hi = float(lo), float(hi)                      # a numpy float64 bound would promote the frame to float64
    with np.errstate(over="ignore", invalid="ignore"):
        x = (x - lo) / (hi - lo + 1e-8)
        idx = (255 * np.clip(x, 0, 1)).astype(np.uint8)
    return np.asarray(lut, np.uint8).reshape(256, 3)[idx]
