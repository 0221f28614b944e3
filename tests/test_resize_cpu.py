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


SPECIAL = np.array([np.inf, -np.inf, np.nan, -0.0, 0.0, 1e-45, -1e-45, 1e-40, -3e-39, 3e38, -3e38, 1.0, -1.0],
                   np.float32)


def special_frame(w0, h0, seed):
    """Normal values with a third of them replaced by infinities, NaN, signed zeros, subnormals and +-3e38 (whose
    blends and block sums overflow)."""
    g = np.random.default_rng(seed)
    a = g.standard_normal((h0, w0, 3)).astype(np.float32)
    k = g.random(a.shape) < 0.3
    a[k] = g.choice(SPECIAL, int(k.sum()))
    return a


def same_bits(a, b):
    """Bitwise equality, NaN matching NaN whatever its sign and payload (which the hardware picks: x86 and the GPU
    make different default NaNs)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and \
        np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


# every form with special values: 2x (area), same size, linear down, up, mixed, 1-pixel rows and columns
SPECIAL_GRID = [(64, 64, 32, 32), (20, 20, 20, 20), (17, 13, 40, 9), (9, 7, 3, 2), (5, 5, 64, 64), (33, 17, 11, 50),
                (1, 9, 4, 3), (9, 1, 3, 4), (12, 12, 4, 3)]


@pytest.mark.parametrize("w0,h0,W,H", SPECIAL_GRID)
def test_oracle_equals_cv2_on_special_values(ipp_off, w0, h0, W, H):
    with np.errstate(invalid="ignore", over="ignore"):
        for seed in range(2):
            a = special_frame(w0, h0, seed)
            assert same_bits(ro.resize(a, W, H), cv2.resize(a, (W, H))), (w0, h0, W, H, seed)


@pytest.mark.parametrize("w0,W", [(20_000_001, 17_000_003), (3, 17_000_003)])
def test_oracle_equals_cv2_where_the_float_index_loses_precision(ipp_off, w0, W):
    """1-row frames whose float32 column index (x + 0.5) w0 / W - 0.5 cannot tell neighbouring columns apart: at
    20,000,001 -> 17,000,003 the index passes 2^24, where every float32 is an even integer and fx is 0; at
    3 -> 17,000,003 the step between columns, 1.8e-7, is below the index's ulp near 2."""
    a = np.random.default_rng(w0).random((1, w0, 3), dtype=np.float32)
    assert same_bits(ro.resize(a, W, 1), cv2.resize(a, (W, 1)))


@pytest.mark.parametrize("w0,W", [(2, 1001), (7, 3), (1001, 999), (3, 17_001), (1, 5), (5, 1)])
def test_row_chunk_equals_linear(w0, W):
    """The torch restatement the device checks of very long rows use, on the host, against linear() in chunks."""
    import torch
    with np.errstate(invalid="ignore", over="ignore"):
        a = special_frame(w0, 1, W)
        want = ro.linear(a, W, 1)[0]
        for x0, x1 in ((0, W), (0, W // 2), (W // 3, W)):
            got = ro.row_chunk(torch.from_numpy(a[0]), W, x0, x1).numpy()
            assert same_bits(got, want[x0:x1]), (w0, W, x0, x1)


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

