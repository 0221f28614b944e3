"""CPU-only: tests/resize_oracle.py against cv2.resize(src, (W, H)) with OpenCV's IPP code disabled, bit for bit, over
every form of the INTER_LINEAR rule (the exact 2x switch to INTER_AREA, 2x on one axis, 4x, odd ratios, enlargements,
mixed, 1-pixel inputs and outputs, the same size).  With IPP active the differences from the default cv2.resize are
printed, not asserted: they depend on the code path IPP picks for the host CPU."""
import numpy as np
import pytest

import resize_oracle as ro

cv2 = pytest.importorskip("cv2")

# (w0, h0, W, H)
GRID = [
    (960, 540, 480, 270),          # exact 2x: INTER_AREA
    (64, 64, 32, 32),
    (2, 2, 1, 1),
    (64, 48, 32, 48),              # 2x on one axis only: linear
    (64, 48, 64, 24),
    (64, 64, 16, 16),              # 4x: linear, not area
    (1920, 1080, 480, 270),
    (963, 541, 481, 270),
    (1921, 1081, 960, 540),
    (77, 100, 50, 33),
    (64, 64, 130, 200),            # enlargements
    (17, 31, 40, 9),               # mixed up / down
    (8, 8, 4, 8),
    (5, 5, 1, 1),                  # 1-pixel outputs and inputs
    (1, 1, 7, 5),
    (1, 9, 4, 3),
    (9, 1, 3, 4),
    (7, 5, 1, 3),
    (40, 30, 40, 30),              # same size
    (3, 2, 3, 2),
]


@pytest.fixture
def ipp_off():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def frame(w0, h0, seed):
    return np.random.default_rng(seed).random((h0, w0, 3), dtype=np.float32)


@pytest.mark.parametrize("w0,h0,W,H", GRID)
def test_oracle_equals_cv2_without_ipp(ipp_off, w0, h0, W, H):
    for seed in range(2):
        a = frame(w0, h0, seed)
        if seed:
            a = (a * 4000 - 2000).astype(np.float32)              # wider exponents, negative values
        want = cv2.resize(a, (W, H))
        got = ro.resize(a, W, H)
        assert got.shape == want.shape == (H, W, 3) and got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (w0, h0, W, H, seed)


def test_ipp_difference_is_reported():
    """Prints, per shape, the largest difference between the default cv2.resize (IPP when the build has it) and
    OpenCV's portable code; nothing is asserted about it."""
    was = cv2.ipp.useIPP()
    try:
        cv2.ipp.setUseIPP(True)
        print(f"\nIPP in use: {cv2.ipp.useIPP()}, version: {cv2.ipp.getIppVersion()}")
        for w0, h0, W, H in GRID:
            a = frame(w0, h0, 0)
            d = np.abs(cv2.resize(a, (W, H)).astype(np.float64) - ro.resize(a, W, H))
            print(f"{w0}x{h0} -> {W}x{H}: max |default - portable| = {d.max():.3g}, values differing: "
                  f"{int(np.count_nonzero(d))} of {d.size}")
    finally:
        cv2.ipp.setUseIPP(was)

