"""CPU: the numpy restatement of the test-frame comparison panels (panels_oracle.py) against the reference's block
(tests/golden/test_panels.npz), its quantile against np.quantile bit for bit, and the argument checks of
lrf_test_panels, which must fail before touching a device."""
import ctypes as C
import os

import numpy as np
import pytest

import panels_oracle as PO
from localrf_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "test_panels.npz")


def golden():
    return np.load(GOLDEN)


def bits_equal(a, b):
    """Bitwise equality with every NaN equal to every other."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both_nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(both_nan | (a.view(np.uint32) == b.view(np.uint32))))


def oracle_outputs(c, fwd_pred, bwd_pred):
    W, H = c["W"], c["H"]
    fwd, qf = PO.flow_panel(fwd_pred, PO.resize_nearest(c["fwd_flow"], W, H), PO.resize_nearest(c["fwd_mask"], W, H), W)
    bwd, qb = PO.flow_panel(bwd_pred, PO.resize_nearest(c["bwd_flow"], W, H), PO.resize_nearest(c["bwd_mask"], W, H), W)
    dep, ts = PO.depth_panel(c["depth"], PO.resize_nearest(c["invdepth"], W, H), W, H)
    return fwd, bwd, dep, np.array([*qf, *qb, *ts], np.float32)


def stored(g, name, key, full, W, H):
    if W * H > PO.FULL_OUTPUT_PIXELS:
        return full.reshape(-1)[PO.sample_index(name, full.size)], g[f"{name}.{key}"]
    return full, g[f"{name}.{key}"]


@pytest.mark.parametrize("name", list(PO.CASES))
def test_oracle_matches_reference_block(name):
    g = golden()
    c = PO.make_case(name)
    assert PO.input_digest(c) == str(g[f"{name}.digest"]), "the case generator no longer reproduces the fixture's inputs"
    W, H = c["W"], c["H"]
    preds = [PO.pred_flow(c["depth"], c["directions"], c["cam2world"], c["idx"], off, c["focal"], c["center"], W, H)
             for off in (1, -1)]
    for key, p in zip(("fwd_pred", "bwd_pred"), preds):
        mine, ref = stored(g, name, key, p, W, H)
        assert np.all(np.abs(mine - ref) <= PO.flow_bound(ref, W, H)), key
    if W * H > PO.FULL_OUTPUT_PIXELS:
        return                                     # the flow rows need the reference's whole predicted flows
    fwd, bwd, dep, stats = oracle_outputs(c, g[f"{name}.fwd_pred"], g[f"{name}.bwd_pred"])
    ref = g[f"{name}.stats"]
    # given the reference's predicted flows, the quantiles, medians and flow panels are bit-exact
    assert bits_equal(stats[[0, 1, 2, 3, 4, 6]], ref[[0, 1, 2, 3, 4, 6]])
    assert bits_equal(fwd, g[f"{name}.fwd_cmp"]) and bits_equal(bwd, g[f"{name}.bwd_cmp"])
    # the MAD scales: the reference's fp32 mean (torch's CPU summation) against the fp64 one, within a few ulps
    k = 0
    for i in (5, 7):
        assert bits_equal(stats[i], ref[i]) or PO.ulps(stats[i], ref[i]) <= 4, (stats[i], ref[i])
        k = max(k, 0 if bits_equal(stats[i], ref[i]) else PO.ulps(stats[i], ref[i]))
    # depth rows: within what those ulps on the MAD scales imply (panels_oracle.depth_bound states the reasoning)
    bound = PO.depth_bound(c["depth"], PO.resize_nearest(c["invdepth"], W, H), W, H, s_ulps=max(k, 1))
    assert PO.within(dep, g[f"{name}.depth_cmp"], bound)


def quantile_arrays(rng, count):
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, np.inf, -np.inf, 1.0, -1.0, 2.5], np.float32)
    for i in range(count):
        n = int(rng.choice([2, 3, 4, 5, 7, 10, 11, 100, 255, 256, 257, 1000, 4095, 65537, 100000])) if i % 10 else \
            int(rng.integers(2, 100001))
        kind = i % 6
        if kind == 0:
            a = rng.standard_normal(n)
        elif kind == 1:                                    # heavy ties
            a = rng.integers(-3, 4, n).astype(np.float64)
        elif kind == 2:                                    # special values mixed in
            a = rng.standard_normal(n)
            k = rng.integers(0, n, max(1, n // 7))
            a[k] = rng.choice(special, k.size)
        elif kind == 3:                                    # subnormals and signed zeros only
            a = rng.choice(special[:6], n)
        elif kind == 4:                                    # a NaN somewhere
            a = rng.standard_normal(n)
            a[rng.integers(0, n)] = np.nan
        else:                                              # infinities around the quantile
            a = rng.choice(np.array([np.inf, -np.inf, 0.0, 1.0], np.float32), n)
        yield a.astype(np.float32)


def test_quantile_restatement_equals_numpy():
    rng = np.random.default_rng(7)
    for a in quantile_arrays(rng, 3000):
        with np.errstate(invalid="ignore"):
            want = np.quantile(a, 0.9)
        assert want.dtype == np.float32                   # numpy 2.x keeps float32 input in float32
        assert bits_equal(PO.quantile(a), want), (a.size, want)


# (W, H, hi_mode): frames whose 2 W H values put numpy's float32 virtual index above 2^24
NEIGHBOUR_SIZES = [(4096, 2276, 0), (4096, 2304, 2), (4096, 2272, 1), (7680, 4320, 0)]
# the offset from the lower rank where the infinities of each of the four statistics' arrays begin (None: none);
# numpy's quantile is NaN exactly when its upper neighbour is an infinity (gamma is 0 at these sizes)
INF_OFFSETS = (1, 2, 3, None)


@pytest.mark.parametrize("W,H,mode", NEIGHBOUR_SIZES)
def test_quantile_restatement_at_the_neighbour_sizes(W, H, mode):
    """The restatement the device's neighbour tests rest on: at sizes where numpy's upper neighbour is the lower rank
    itself (0), the next rank (1) or two ranks up (2), its ranks, and its value on arrays whose first infinity sits
    just past the lower rank, equal np.quantile's."""
    assert PO.hi_mode(W, H) == mode
    lo, hi, gamma = PO.quantile_ranks(2 * W * H)
    assert gamma == 0 and lo > W * H
    for k, off in enumerate(INF_OFFSETS[:2] if mode != 2 else INF_OFFSETS[:3]):
        a = np.concatenate([np.zeros(W * H, np.float32), PO.neighbour_gt(W, H, lo + off, k)])
        with np.errstate(invalid="ignore"):
            want = np.quantile(a, 0.9)
        assert np.isnan(want) == (lo + off <= hi), (off, want)
        assert bits_equal(PO.quantile(a), want), (off, PO.quantile(a), want)


def test_lower_median_equals_sorted_rule():
    rng = np.random.default_rng(8)
    for n in (1, 2, 3, 4, 9, 10, 1001):
        a = rng.integers(-2, 3, n).astype(np.float32)
        assert PO.lower_median(a) == np.sort(a)[(n - 1) // 2]
    assert np.isnan(PO.lower_median(np.array([1.0, np.nan, 2.0], np.float32)))


def test_nearest_index_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    for (h0, w0) in ((96, 128), (61, 100), (15, 20), (1, 1), (7, 3), (540, 960)):
        src = np.arange(h0 * w0, dtype=np.float32).reshape(h0, w0)
        for (W, H) in ((64, 48), (37, 23), (480, 270), (1, 1), (3, 7), (2 * w0 + 1, 3 * h0)):
            want = cv2.resize(src, (W, H), interpolation=cv2.INTER_NEAREST).reshape(H, W)
            assert np.array_equal(PO.resize_nearest(src, W, H), want), (h0, w0, W, H)
    for (h0, w0), (H, W) in NEAREST_EXTREMES:
        src = np.arange(h0 * w0, dtype=np.float32).reshape(h0, w0)             # indices below 2^24: exact
        want = cv2.resize(src, (W, H), interpolation=cv2.INTER_NEAREST).reshape(H, W)
        assert np.array_equal(PO.resize_nearest(src, W, H), want), (h0, w0, W, H)


# ((h0, w0), (H, W)): a pixel to a 4096 x 2304 frame and back, neighbouring sizes, 3 <-> 7
NEAREST_EXTREMES = [((1, 1), (2304, 4096)), ((2304, 4096), (1, 1)), ((1000, 999), (999, 1000)),
                    ((999, 1000), (1000, 999)), ((3, 7), (7, 3)), ((7, 3), (3, 7)), ((3, 7), (2304, 4096)),
                    ((2304, 4096), (7, 3)), ((1, 4096), (2304, 1)), ((2304, 1), (1, 4096))]


# ---- the C ABI without a device ------------------------------------------------------------------------------
def test_struct_mirror_and_exports():
    L = _lib.lib()
    assert L.lrf_sizeof(10) == C.sizeof(_lib.LrfPanelFrame) == 4 * 4 + 2 * 8 + 15 * 8
    assert "lrf_test_panels" in _lib.EXPORTS and "lrf_test_panels_scratch_bytes" in _lib.EXPORTS
    assert "lrf_panels.cu" in _lib.SOURCES
    assert L.lrf_test_panels_scratch_bytes(0, 4) == 0 and L.lrf_test_panels_scratch_bytes(4, -1) == 0
    assert L.lrf_test_panels_scratch_bytes(46341, 23171) == 0                  # 2 W H >= 2^31
    assert L.lrf_test_panels_scratch_bytes(64, 48) > 10 * 64 * 48 * 4


def valid_frame():
    """A frame whose pointers are bogus but non-NULL: every call below must fail before dereferencing one."""
    f = _lib.LrfPanelFrame()
    f.W, f.H, f.h0, f.w0, f.n_cams, f.idx = 8, 4, 6, 5, 3, 1
    for name in ("depth", "directions", "cam2world", "intrinsics", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask",
                 "invdepth", "fwd_panel", "bwd_panel", "depth_panel"):
        setattr(f, name, 0x1000)
    return f


def call(f, scratch=0x2000, nbytes=None):
    L = _lib.lib()
    if nbytes is None:
        nbytes = L.lrf_test_panels_scratch_bytes(max(f.W, 1), max(f.H, 1))
    return L.lrf_test_panels(C.byref(f), scratch, nbytes, None)


@pytest.mark.parametrize("change", [
    ("W", 0), ("H", -2), ("h0", 0), ("w0", 0), ("n_cams", 0), ("idx", -1), ("idx", 3), ("depth", None),
    ("fwd_flow", None), ("bwd_mask", None), ("directions", None), ("cam2world", None), ("intrinsics", None),
    ("fwd_panel", None), ("bwd_panel", None), ("depth_panel", None)])
def test_invalid_arguments_without_device(change):
    f = valid_frame()
    setattr(f, *change)
    assert call(f) == -1
    assert _lib.lib().lrf_last_error()


def test_invalid_scratch_and_frame_without_device():
    L = _lib.lib()
    assert L.lrf_test_panels(None, 0x2000, 1 << 20, None) == -1
    f = valid_frame()
    assert call(f, scratch=None) == -1
    assert call(f, scratch=0x2004) == -1                                       # not 8-byte aligned
    assert call(f, nbytes=L.lrf_test_panels_scratch_bytes(8, 4) - 1) == -1
    f.W, f.H = 46341, 23171
    assert call(f, nbytes=1 << 40) == -1


def test_host_depth_is_refused_without_device():
    """test_panels takes the frame's device from depth: a host depth is refused before anything touches a device."""
    import torch
    from localrf_b200 import metrics
    c = PO.make_case("odd_37x23")
    with pytest.raises(ValueError, match="CUDA"):
        metrics.test_panels(torch.from_numpy(c["depth"]), torch.from_numpy(c["directions"]),
                            torch.from_numpy(c["cam2world"]), c["idx"], float(c["focal"]), c["center"], c["W"],
                            c["H"], fwd_flow=c["fwd_flow"], fwd_mask=c["fwd_mask"], bwd_flow=c["bwd_flow"],
                            bwd_mask=c["bwd_mask"], invdepth=c["invdepth"])
