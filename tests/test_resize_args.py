"""CPU-only: lrf_resize_linear refusing bad arguments (LRF_ERR_INVALID) with a message before it touches a device (the
non-NULL pointers below are never dereferenced), and its binding."""
import ctypes as C

import pytest

from localrf_b200 import _lib

INVALID = -1
FAKE = 0x10000                       # never read
GOOD = dict(src=FAKE, w0=64, h0=48, src_stride=3 * 64, dst=FAKE, W=20, H=15, dst_stride=3 * 20)


def _call(**over):
    a = dict(GOOD, **over)
    return _lib.lib().lrf_resize_linear(a["src"], a["w0"], a["h0"], a["src_stride"], a["dst"], a["W"], a["H"],
                                        a["dst_stride"], None)


def test_symbol_and_prototype():
    L = _lib.lib()
    assert "lrf_resize_linear" in _lib.EXPORTS
    assert L.lrf_resize_linear.argtypes == [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                            C.c_int32, C.c_int64, C.c_void_p]


@pytest.mark.parametrize("over,text", [
    (dict(src=None), b"src / dst is NULL"),
    (dict(dst=None), b"src / dst is NULL"),
    (dict(w0=0), b">= 1"),
    (dict(h0=-1), b">= 1"),
    (dict(W=0), b">= 1"),
    (dict(H=0), b">= 1"),
    (dict(w0=65536, h0=32768, src_stride=3 * 65536), b"below 2^31"),
    (dict(W=32768, H=65536, dst_stride=3 * 32768), b"below 2^31"),
    (dict(src_stride=3 * 64 - 1), b"src_stride"),
    (dict(src_stride=0), b"src_stride"),
    (dict(dst_stride=3 * 20 - 1), b"dst_stride"),
])
def test_invalid(over, text):
    assert _call(**over) == INVALID
    msg = _lib.lib().lrf_last_error()
    assert text in msg, msg

