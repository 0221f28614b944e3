"""numpy restatement of the test-frame metrics (renderer.py:162-163; rgb_ssim, utils/utils.py:232-287), written
from the formula.  TEST INFRASTRUCTURE: the tests of localrf_b200/metrics.py and tools/metrics_time.py compare the
device kernel against it; nothing under localrf_b200/ imports it."""
import numpy as np


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def mse(img, gt):
    """mean((gt - img)^2): fp32 differences and squares, summed in fp64."""
    d = _f32(gt) - _f32(img)
    return float(np.sum((d * d).astype(np.float64)) / d.size)


def ssim(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False):
    """SSIM of two [H,W,3] float32 frames: the squares and the cross product are fp32 products, the separable
    "valid" Gaussian filter (first along H, then along W) and the map are fp64."""
    a, b = _f32(img0), _f32(img1)
    assert a.ndim == 3 and a.shape[-1] == 3 and a.shape == b.shape
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
