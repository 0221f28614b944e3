"""CPU-only: the LrfIngestFrame mirror, and lrf_ingest_frame refusing bad arguments (LRF_ERR_INVALID) and layouts it
does not convert (LRF_ERR_UNSUPPORTED) with a message before it touches a device (the non-NULL pointers below are
never dereferenced)."""
import ctypes as C

from localrf_b200 import _lib

INVALID, UNSUPPORTED = -1, -2
FAKE = 0x10000                       # never read
W, H = 40, 30


def _args(flow=True, depth=True, mask=True):
    s = _lib.LrfFrameStore()
    s.n_px, s.capacity = W * H, 4
    s.slot_frame = s.rgb = s.loss_weight = FAKE
    s.invdepth = FAKE if depth else None
    for name in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"):
        setattr(s, name, FAKE if flow else None)
    f = _lib.LrfIngestFrame()
    f.slot, f.w, f.h = 1, W, H
    f.image, f.w0, f.h0, f.image_stride = FAKE, W, H, 3 * W
    if depth:
        f.invdepth, f.wd, f.hd, f.invdepth_stride = FAKE, W, H, W
    if flow:
        f.fwd_flow = f.bwd_flow = FAKE
        f.wf, f.hf, f.flow_stride, f.flow_scale = W // 2, H // 2, 3 * (W // 2), 2.0
    if mask:
        f.mask, f.wm, f.hm, f.mask_stride = FAKE, W, H, W
    return s, f


def _call(s, f, scratch=FAKE, n=None):
    L = _lib.lib()
    n = L.lrf_ingest_scratch_bytes(W * H) if n is None else n
    return L.lrf_ingest_frame(C.byref(s) if s is not None else None, C.byref(f) if f is not None else None,
                              scratch, n, None)


def _refused(s, f, code, text, **kw):
    assert _call(s, f, **kw) == code
    msg = _lib.lib().lrf_last_error()
    assert text in msg, msg


def test_struct_mirror():
    L = _lib.lib()
    assert L.lrf_sizeof(11) == C.sizeof(_lib.LrfIngestFrame) == 128
    assert _lib.LrfIngestFrame.flow_scale.offset == 96 and _lib.LrfIngestFrame.mask_stride.offset == 120
    assert {"lrf_ingest_frame", "lrf_ingest_scratch_bytes"} <= set(_lib.EXPORTS) and "lrf_ingest.cu" in _lib.SOURCES


def test_invalid():
    s, f = _args()
    assert _call(None, f) == INVALID and _call(s, None) == INVALID
    for name in ("slot_frame", "rgb", "loss_weight"):
        s, f = _args()
        setattr(s, name, None)
        _refused(s, f, INVALID, b"of the store is NULL")
    s, f = _args()
    s.fwd_mask = None
    _refused(s, f, INVALID, b"partly given")
    for slot in (-1, 4):
        s, f = _args()
        f.slot = slot
        _refused(s, f, INVALID, b"slot must lie")
    for w, h in ((W + 1, H), (0, H), (W, -H)):
        s, f = _args()
        f.w, f.h = w, h
        _refused(s, f, INVALID, b"n_px")
    s, f = _args()
    f.image = None
    _refused(s, f, INVALID, b"image is NULL")
    s, f = _args()
    f.image_stride = 3 * W - 1
    _refused(s, f, INVALID, b"row stride")
    s, f = _args()
    f.w0 = 0
    _refused(s, f, INVALID, b"sizes must be >= 1")
    s, f = _args()
    f.invdepth = None                                   # the store has depth
    _refused(s, f, INVALID, b"invdepth must be set")
    s, f = _args(depth=False)
    f.invdepth, f.wd, f.hd, f.invdepth_stride = FAKE, W, H, W   # the store has none
    _refused(s, f, INVALID, b"invdepth must be set")
    for name in ("fwd_flow", "bwd_flow"):
        s, f = _args()
        setattr(f, name, None)
        _refused(s, f, INVALID, b"fwd_flow and bwd_flow")
    s, f = _args(flow=False)
    f.fwd_flow = FAKE
    _refused(s, f, INVALID, b"fwd_flow and bwd_flow")
    s, f = _args()
    f.flow_stride = 3 * f.wf - 3
    _refused(s, f, INVALID, b"row stride")
    s, f = _args()
    f.mask_stride = W - 1
    _refused(s, f, INVALID, b"row stride")
    s, f = _args()
    _refused(s, f, INVALID, b"scratch is NULL", scratch=None)
    _refused(s, f, INVALID, b"not 8-byte aligned", scratch=FAKE + 4)
    _refused(s, f, INVALID, b"smaller than", n=_lib.lib().lrf_ingest_scratch_bytes(W * H) - 8)


def test_unsupported():
    for w0, h0 in ((3 * W, 3 * H), (2 * W, 4 * H), (W // 2, H // 2), (W + 1, H)):
        s, f = _args()
        f.w0, f.h0, f.image_stride = w0, h0, 3 * w0
        _refused(s, f, UNSUPPORTED, b"the image must be")
    for wd, hd in ((3 * W, 3 * H), (W + 2, H)):
        s, f = _args()
        f.wd, f.hd, f.invdepth_stride = wd, hd, wd
        _refused(s, f, UNSUPPORTED, b"invdepth must be")
    for wf, hf in ((2 * W, 2 * H), (W + 1, H // 2)):
        s, f = _args()
        f.wf, f.hf, f.flow_stride = wf, hf, 3 * wf
        _refused(s, f, UNSUPPORTED, b"the flows must be")
    s, f = _args()
    f.wm, f.hm = W // 2, H // 2
    _refused(s, f, UNSUPPORTED, b"the mask must be")
    s, f = _args()
    s.n_px = 3000 * 3000
    f.w, f.h, f.w0, f.h0, f.image_stride = 3000, 3000, 3000, 3000, 9000
    f.wd, f.hd, f.invdepth_stride, f.wm, f.hm, f.mask_stride = 3000, 3000, 3000, 3000, 3000, 3000
    _refused(s, f, UNSUPPORTED, b"2^16 leaves")
