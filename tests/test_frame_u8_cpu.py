"""CPU-only: the numpy 8-bit frame conversions (tests/metrics_oracle.py rgb8 / depth8) against the reference's
renderer outputs stored in tests/golden/frame_u8.npz; the reference's depth byte chain passing every colour-map
byte through unchanged; the kernel-tap SSIM oracle against the reference's rgb_ssim; lrf_frame_to_u8's argument
checks without a device."""
import ctypes as C
import os

import numpy as np
import pytest

from localrf_b200 import _lib
import metrics_oracle as orc
from test_metrics_cpu import golden_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "frame_u8.npz"))


def test_rgb8_oracle_matches_opencv():
    g = golden()
    np.testing.assert_array_equal(orc.rgb8(g["rgb"]), g["rgb8"])
    # the golden holds the cases the conversion turns on: ties to even, saturation at both ends, NaN and -inf
    v = 255 * g["rgb"]
    assert (v == 0.5).any() and (v == 1.5).any() and (v == 254.5).any()
    assert np.isnan(v).any() and (v == -np.inf).any() and (v > 1e8).any() and (v < -1).any()


@pytest.mark.parametrize("i", range(6))
def test_depth8_oracle_matches_visualize_depth(i):
    g = golden()
    lo, hi = g["ranges"][i]
    d, want = g[f"depth.{i}"], g[f"depth8.{i}"]
    np.testing.assert_array_equal(orc.depth8(d, lo, hi, g["lut"]), want)
    assert np.isnan(d).any() and np.isposinf(d).any() and np.isneginf(d).any()
    if lo < hi:                                       # every index occurs, at its crossing from either side
        assert set(want[:, 0]) == set(range(256))


def test_depth8_golden_holds_the_double_denominator_cases():
    """Depths where (hi - lo + 1e-8) rounded to float32 once (the reference) and formed in float32 from float32
    bounds pick different indices."""
    g = golden()
    for i, bits, ref_idx, f32_idx in ((1, 1053806543, 129, 130), (2, 1077516697, 255, 254)):
        lo, hi = (float(v) for v in g["ranges"][i])
        d = g[f"depth.{i}"]
        at = np.flatnonzero(d.view(np.uint32) == bits)
        assert len(at) >= 1
        assert int(g[f"depth8.{i}"][at[0], 0]) == ref_idx
        x = (d[at[0]] - np.float32(lo)) / (np.float32(hi) - np.float32(lo) + np.float32(1e-8))
        assert int(np.float32(255) * np.float32(x)) == f32_idx


def test_depth_byte_chain_returns_every_lut_byte():
    """renderer.py:127,156: visualize_depth turns the colour-mapped bytes into a float tensor (PIL.Image.fromarray,
    torchvision ToTensor) and the renderer multiplies by 255 and truncates (.byte()).  Every byte survives, so
    comparing the device's depth8 with the colour map directly is comparing it with the renderer's frame."""
    import torch
    from PIL import Image
    import torchvision.transforms as T
    b = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, -1)
    t = T.ToTensor()(Image.fromarray(b))
    back = torch.permute(t * 255, [1, 2, 0]).byte().numpy()
    np.testing.assert_array_equal(back, b)


@pytest.mark.parametrize("name", [c[0] for c in golden_cases()])
def test_kernel_taps_oracle_is_within_rounding_of_reference(name):
    case, params = next((c, p) for n, c, p in golden_cases() if n == name)
    want = orc.ssim(case["gt"], case["img"], **params, taps="reference", return_map=True)
    got = orc.ssim(case["gt"], case["img"], **params, taps="kernel", return_map=True)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got, case["ssim_map"], rtol=0, atol=1e-12)
    ref = orc.ssim(case["gt"], case["img"], **params, taps="reference")
    assert abs(orc.kernel_taps(params["filter_size"], params["filter_sigma"]).sum() - 1) <= 4e-16
    assert abs(orc.ssim(case["gt"], case["img"], **params, taps="kernel") - ref) <= 1e-13


def _call(L, rgb=8, rgb_stride=3, depth=8, depth_stride=1, N=16, lut=8, rgb8=8, depth8=8):
    p = lambda v: C.c_void_p(v) if v else None
    return L.lrf_frame_to_u8(p(rgb), rgb_stride, p(depth), depth_stride, N, 0.0, 5.0, p(lut), p(rgb8), p(depth8),
                             None)


@pytest.mark.parametrize("kw, word", [
    (dict(N=-1), b"N < 0"),
    (dict(rgb=0), b"rgb8"), (dict(rgb_stride=2), b"rgb8"), (dict(rgb_stride=-3), b"rgb8"),
    (dict(depth=0), b"depth8"), (dict(lut=0), b"depth8"), (dict(depth_stride=0), b"depth8"),
    (dict(depth_stride=-1), b"depth8"),
    (dict(rgb=0, rgb8=0, depth=0), b"depth8"), (dict(depth=0, depth8=0, rgb_stride=1), b"rgb8"),
])
def test_frame_to_u8_validation_without_gpu(kw, word):
    L = _lib.lib()
    assert _call(L, **kw) == -1
    assert word in L.lrf_last_error()


def test_frame_to_u8_takes_double_bounds():
    """The bounds are doubles: a binding that passed floats would hand the kernel a different denominator."""
    L = _lib.lib()
    assert L.lrf_frame_to_u8.argtypes[5:7] == [C.c_double, C.c_double]
