"""CPU-only: lrf_supervision_losses and its backward refuse bad arguments with LRF_ERR_INVALID /
LRF_ERR_UNSUPPORTED and a message before they touch a device.  The non-NULL pointers below are never
dereferenced: each call fails its argument check first."""
import ctypes as C

import pytest

from localrf_b200 import _lib

INVALID, UNSUPPORTED = -1, -2
FAKE = 0x10000                       # 16-byte aligned, never read
FLOW_PTRS = ("view_ids", "depth_map", "directions", "ij", "cam2world", "focal", "center", "fwd_flow", "bwd_flow",
             "fwd_mask", "bwd_mask")


def _batch(N=64, V=4, n_cams=8, flow=1, depth=1):
    b = _lib.LrfLossBatch()
    b.n_rays, b.n_views, b.n_cams, b.starting_id = N, V, n_cams, 0
    b.use_flow, b.use_depth = flow, depth
    b.flow_weight, b.depth_weight = 1.0, 1.0
    for name, _ in _lib.LrfLossBatch._fields_:
        if name not in ("n_rays", "n_views", "n_cams", "starting_id", "use_flow", "use_depth", "flow_weight",
                        "depth_weight"):
            setattr(b, name, FAKE)
    return b


def _both(b, code, msg, scratch=FAKE, nbytes=1 << 30):
    L = _lib.lib()
    g = _lib.LrfLossGrads()
    for rc in (L.lrf_supervision_losses(C.byref(b), FAKE, scratch, nbytes, None),
               L.lrf_supervision_losses_backward(C.byref(b), FAKE, C.byref(g), scratch, nbytes, None)):
        assert rc == code, rc
        assert msg in L.lrf_last_error(), L.lrf_last_error()


def test_struct_mirrors():
    L = _lib.lib()
    assert L.lrf_sizeof(4) == C.sizeof(_lib.LrfLossBatch) == 4 * 8 + 4 * 4 + 15 * 8
    assert L.lrf_sizeof(5) == C.sizeof(_lib.LrfLossGrads) == 6 * 8


def test_scratch_bytes():
    L = _lib.lib()
    assert L.lrf_supervision_scratch_bytes(4096, 16, 20) > 8 * 4096
    for n, v, c in ((0, 1, 1), (10, 3, 1), (12, 0, 1), (12, 3, 0), (-4, 2, 1)):
        assert L.lrf_supervision_scratch_bytes(n, v, c) == 0


def test_sizes():
    _both(_batch(N=65, V=4), INVALID, b"multiple of n_views")
    _both(_batch(N=0, V=4), INVALID, b"multiple of n_views")
    _both(_batch(N=64, V=0), INVALID, b"multiple of n_views")
    _both(_batch(n_cams=0), INVALID, b"n_cams must be >= 1")
    _both(_batch(N=4097, V=1), UNSUPPORTED, b"4096 rays per view")
    _both(_batch(N=2 * 4097, V=2, flow=0, depth=0), UNSUPPORTED, b"4096 rays per view")


@pytest.mark.parametrize("name", ("rgb_map", "rgb_train", "loss_weights"))
def test_null_rgb_pointers(name):
    b = _batch(flow=0, depth=0)
    setattr(b, name, None)
    _both(b, INVALID, b"rgb_map / rgb_train / loss_weights is NULL")


@pytest.mark.parametrize("name", FLOW_PTRS)
def test_null_flow_pointers(name):
    b = _batch(depth=0)
    setattr(b, name, None)
    _both(b, INVALID, b"flow term is NULL")
    b.use_flow = 0                                 # a term that is off may leave its pointers NULL
    _both(b, INVALID, b"scratch is NULL", scratch=None)


@pytest.mark.parametrize("name", ("depth_map", "invdepths"))
def test_null_depth_pointers(name):
    b = _batch(flow=0)
    setattr(b, name, None)
    _both(b, INVALID, b"depth term is NULL")


def test_scratch():
    L = _lib.lib()
    b = _batch()
    need = L.lrf_supervision_scratch_bytes(64, 4, 8)
    _both(b, INVALID, b"scratch is NULL", scratch=None)
    _both(b, INVALID, b"8-byte aligned", scratch=FAKE + 4)
    _both(b, INVALID, b"smaller than lrf_supervision_scratch_bytes", nbytes=need - 1)


def test_null_outputs():
    L = _lib.lib()
    b = _batch()
    assert L.lrf_supervision_losses(C.byref(b), None, FAKE, 1 << 30, None) == INVALID
    assert b"losses is NULL" in L.lrf_last_error()
    assert L.lrf_supervision_losses_backward(C.byref(b), None, C.byref(_lib.LrfLossGrads()), FAKE, 1 << 30,
                                             None) == INVALID
    assert L.lrf_supervision_losses_backward(C.byref(b), FAKE, None, FAKE, 1 << 30, None) == INVALID
    assert b"grad_losses / grads is NULL" in L.lrf_last_error()
    assert L.lrf_supervision_losses(None, FAKE, FAKE, 1 << 30, None) == INVALID
