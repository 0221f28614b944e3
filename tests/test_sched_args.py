"""CPU-only: the schedule-time entry points (lrf_sched.cu through lrf_abi.cu) refuse bad arguments with
LRF_ERR_INVALID and a message before they touch a device.  The non-NULL pointers below are never dereferenced:
each call fails its argument check first."""
import ctypes as C

from localrf_b200 import _lib

INVALID = -1
FAKE = 0x10000                       # 16-byte aligned, never read


def _field():
    """a field that passes make_field's checks (sizes, aabb, aligned non-NULL grid pointers)"""
    f = _lib.LrfField()
    f.n_dcomp, f.n_acomp = 8, 24
    for a in range(3):
        f.grid[a] = 16
        f.aabb[a], f.aabb[3 + a] = -2.0, 2.0
    for i in range(3):
        f.dplane[i] = f.dline[i] = f.aplane[i] = f.aline[i] = FAKE
    return f


def _expect(rc, msg):
    L = _lib.lib()
    assert rc == INVALID, rc
    assert msg in L.lrf_last_error(), L.lrf_last_error()


def test_upsample_arguments():
    L = _lib.lib()
    _expect(L.lrf_upsample(FAKE, 8, 8, FAKE, 16, 16, 6, None), b"multiple of 4")       # C = 6
    _expect(L.lrf_upsample(FAKE, 8, 8, FAKE, 16, 16, 0, None), b"multiple of 4")
    for H, W, H2, W2 in ((0, 8, 16, 16), (8, 0, 16, 16), (8, 8, 0, 16), (8, 8, 16, 0), (-1, 8, 16, 16)):
        _expect(L.lrf_upsample(FAKE, H, W, FAKE, H2, W2, 8, None), b"bad upsample arguments")
    _expect(L.lrf_upsample(None, 8, 8, FAKE, 16, 16, 8, None), b"bad upsample arguments")
    _expect(L.lrf_upsample(FAKE + 4, 8, 8, FAKE, 16, 16, 8, None), b"16-byte aligned")
    _expect(L.lrf_upsample(FAKE, 8, 8, FAKE + 8, 16, 16, 8, None), b"16-byte aligned")


def test_tv_arguments():
    L = _lib.lib()
    for H, W, Cc in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (-3, 4, 4)):
        _expect(L.lrf_tv_sums(FAKE, H, W, Cc, FAKE, None), b"bad tv arguments")
        _expect(L.lrf_tv_sums_backward(FAKE, H, W, Cc, FAKE, 1.0, 1.0, FAKE, None), b"bad tv arguments")
    _expect(L.lrf_tv_sums(FAKE, 4, 4, 4, None, None), b"bad tv arguments")


def test_sample_ray_arguments():
    L = _lib.lib()
    aabb = (C.c_float * 6)(-1, -1, -1, 1, 1, 1)
    _expect(L.lrf_sample_ray(FAKE, None, -1, 8, aabb, 0.1, 10.0, 0.01, FAKE, FAKE, FAKE, None), b"sizes")
    _expect(L.lrf_sample_ray(FAKE, None, 4, 0, aabb, 0.1, 10.0, 0.01, FAKE, FAKE, FAKE, None), b"sizes")
    _expect(L.lrf_sample_ray(FAKE, None, 4, 8, aabb, 0.1, 10.0, 0.01, None, FAKE, FAKE, None), b"NULL")


def test_alpha_mask_build_arguments():
    L = _lib.lib()
    f = _field()
    for dims in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (4, 4, -1)):
        _expect(L.lrf_alpha_mask_build(C.byref(f), (C.c_int32 * 3)(*dims), 0.01, 1e-4, FAKE, FAKE, FAKE, None),
                b"lattice dims must be >= 1")
    ok = (C.c_int32 * 3)(4, 4, 4)
    _expect(L.lrf_alpha_mask_build(C.byref(f), ok, 0.01, 1e-4, FAKE, FAKE, None, None), b"kept is NULL")
    _expect(L.lrf_alpha_mask_build(C.byref(f), ok, 0.01, 1e-4, None, None, None, None), b"alpha_scratch is NULL")


def test_density_l1_backward_arguments():
    L = _lib.lib()
    f = _field()
    for i in range(3):
        for which in ("plane", "line"):
            planes = (C.c_void_p * 3)(FAKE, FAKE, FAKE)
            lines = (C.c_void_p * 3)(FAKE, FAKE, FAKE)
            (planes if which == "plane" else lines)[i] = None
            _expect(L.lrf_density_l1_backward(C.byref(f), FAKE, planes, lines, None), b"gradient buffer is NULL")
    _expect(L.lrf_density_l1_backward(C.byref(f), None, (C.c_void_p * 3)(FAKE, FAKE, FAKE),
                                      (C.c_void_p * 3)(FAKE, FAKE, FAKE), None), b"grad_out is NULL")
