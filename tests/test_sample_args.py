"""CPU-only: the LrfFrameStore / LrfRayGather mirrors, lrf_gather_rays refusing bad arguments with LRF_ERR_INVALID
and a message before it touches a device (the non-NULL pointers below are never dereferenced), and the host
restatement of LocalRFDataset.sample (tests/sample_oracle.py) reproducing every blob of the unmodified reference in
tests/golden/ray_sample.npz, bit for bit, when replayed over the stand-in dataset."""
import ctypes as C
import os

import numpy as np
import pytest

from localrf_b200 import _lib
import sample_oracle as so

INVALID = -1
FAKE = 0x10000                       # never read
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ray_sample.npz")
GROUPS = ("invdepth", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask")


def _args(flow=True, depth=True):
    s = _lib.LrfFrameStore()
    s.n_px, s.capacity = 1536, 4
    s.slot_frame = s.rgb = s.loss_weight = FAKE
    g = _lib.LrfRayGather()
    g.n_rays, g.n_views = 64, 16
    g.ids = g.idx = g.rgb = g.loss_weight = FAKE
    for name in GROUPS:
        on = depth if name == "invdepth" else flow
        setattr(s, name, FAKE if on else None)
        setattr(g, name, FAKE if on else None)
    return s, g


def _refused(s, g, text):
    L = _lib.lib()
    assert L.lrf_gather_rays(C.byref(s), C.byref(g), None) == INVALID
    assert text in L.lrf_last_error(), L.lrf_last_error()


def test_struct_mirrors():
    L = _lib.lib()
    assert L.lrf_sizeof(8) == C.sizeof(_lib.LrfFrameStore) == 2 * 8 + 8 * 8
    assert L.lrf_sizeof(9) == C.sizeof(_lib.LrfRayGather) == 2 * 8 + 9 * 8
    assert _lib.LrfFrameStore.bwd_mask.offset == 9 * 8 and _lib.LrfRayGather.bwd_mask.offset == 10 * 8
    assert "lrf_gather_rays" in _lib.EXPORTS and "lrf_data.cu" in _lib.SOURCES


def test_invalid():
    L = _lib.lib()
    s, g = _args()
    assert L.lrf_gather_rays(None, C.byref(g), None) == INVALID
    assert L.lrf_gather_rays(C.byref(s), None, None) == INVALID
    for name in ("slot_frame", "rgb", "loss_weight"):
        s, g = _args()
        setattr(s, name, None)
        _refused(s, g, b"of the store is NULL")
    for name in ("ids", "idx", "rgb", "loss_weight"):
        s, g = _args()
        setattr(g, name, None)
        _refused(s, g, b"of the gather is NULL")
    for n_rays, n_views in ((65, 16), (64, 0), (-16, 16)):
        s, g = _args()
        g.n_rays, g.n_views = n_rays, n_views
        _refused(s, g, b"multiple of n_views")
    for cap in (0, -3):
        s, g = _args()
        s.capacity = cap
        _refused(s, g, b"capacity must be >= 1")
    s, g = _args()
    s.n_px = 0
    _refused(s, g, b"n_px")
    for name in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"):
        s, g = _args()
        setattr(s, name, None)                        # a flow group that is only partly given
        _refused(s, g, b"partly given")
        s, g = _args()
        setattr(g, name, None)                        # an output of a group the store has
        _refused(s, g, b"flow outputs")
        s, g = _args(flow=False)
        setattr(g, name, FAKE)                        # an output of a group the store lacks
        _refused(s, g, b"flow outputs")
    s, g = _args(depth=False)
    g.invdepth = FAKE
    _refused(s, g, b"invdepth")
    s, g = _args()
    g.invdepth = None
    _refused(s, g, b"invdepth")


@pytest.mark.parametrize("case", ["flow_depth", "rgb_only"])
def test_oracle_reproduces_reference_blobs(case):
    z = np.load(GOLDEN)
    ds, ops, want = so.golden_case(z, case)
    got = list(so.replay(ds, ops, lambda *a: so.sample(ds, *a)))
    assert len(got) == len(want) == 28
    for i, (a, b) in enumerate(zip(got, want)):
        assert a["train_test_poses"] == b["train_test_poses"], i
        for k in so.BLOB_ARRAYS:
            if b[k] is None:
                assert a[k] is None, (i, k)
                continue
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (i, k)
            assert np.array_equal(a[k], b[k]), (i, k)
    # the script covers what it claims: both inclusion sets, counts <= 4 and > 4, both values of the coin
    assert {b["train_test_poses"] for b in want} == {False, True}
    assert any(b["rgbs"].shape[0] == 128 for b in want)
