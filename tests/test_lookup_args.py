"""CPU-only: the VM lookups, their backward and the stand-alone MLP refusing bad arguments (LRF_ERR_INVALID) with a
message before they touch a device (the fake pointers below are never dereferenced), and accepting M = 0 with NULL
data pointers without a device.  The alignment refusals guard the kernels' 16-byte accesses: the backward adds into
d_plane / d_line with float4 atomics, lrf_app_products stores `out` as float4 and lrf_mlp_forward stages `prepared`
with TMA bulk copies."""
import ctypes as C

import pytest

from localrf_b200 import _lib

OK, INVALID = 0, -1
FAKE = 0x10000                       # 16-byte aligned, never read
BACKWARD = ("lrf_density_feature_backward", "lrf_app_products_backward")
FORWARD = ("lrf_density_feature", "lrf_app_feature", "lrf_app_products")
GRAD_ALIGN = b"plane/line gradient buffers must be 16-byte aligned"


def _field():
    s = _lib.LrfField()
    s.grid[:] = [8, 9, 10]
    s.aabb[:] = [-1, -1, -1, 1, 1, 1]
    s.n_dcomp, s.n_acomp, s.app_dim, s.featureC = 8, 24, 27, 128
    for name in ("dplane", "dline", "aplane", "aline"):
        for i in range(3):
            getattr(s, name)[i] = FAKE
    s.basis = FAKE
    return s


def _grads(plane=(FAKE,) * 3, line=(FAKE,) * 3):
    return (C.c_void_p * 3)(*plane), (C.c_void_p * 3)(*line)


def _backward(name, M=64, xyz=FAKE, gout=FAKE, plane=(FAKE,) * 3, line=(FAKE,) * 3, d_xyz=FAKE):
    pp, lp = _grads(plane, line)
    return getattr(_lib.lib(), name)(C.byref(_field()), xyz, gout, M, pp, lp, d_xyz, None)


def _message():
    return _lib.lib().lrf_last_error()


@pytest.mark.parametrize("name", BACKWARD)
@pytest.mark.parametrize("which", ["plane", "line"])
@pytest.mark.parametrize("i", [0, 1, 2])
@pytest.mark.parametrize("off", [4, 8, 12])
def test_backward_refuses_misaligned_gradient_buffer(name, which, i, off):
    bufs = [FAKE] * 3
    bufs[i] = FAKE + off
    assert _backward(name, **{which: tuple(bufs)}) == INVALID
    assert GRAD_ALIGN in _message(), _message()


@pytest.mark.parametrize("name", BACKWARD)
def test_backward_refuses_misaligned_gradient_buffer_at_m0(name):
    """The buffers are checked before the early return of an empty batch."""
    assert _backward(name, M=0, xyz=None, gout=None, line=(FAKE, FAKE + 4, FAKE)) == INVALID
    assert GRAD_ALIGN in _message(), _message()


def test_density_l1_backward_null_gradient_buffer():
    """lrf_density_l1_backward shares the NULL check (not the 16-byte one: its adds are scalar)."""
    pp, lp = _grads(plane=(FAKE, None, FAKE))
    assert _lib.lib().lrf_density_l1_backward(C.byref(_field()), FAKE, pp, lp, None) == INVALID
    assert b"gradient buffer is NULL" in _message()


@pytest.mark.parametrize("name", BACKWARD)
def test_backward_null_gradient_buffer(name):
    assert _backward(name, plane=(FAKE, None, FAKE)) == INVALID
    assert b"gradient buffer is NULL" in _message()


@pytest.mark.parametrize("off", [4, 8, 12])
def test_app_products_refuses_misaligned_out(off):
    assert _lib.lib().lrf_app_products(C.byref(_field()), FAKE, 64, FAKE + off, None) == INVALID
    assert b"out must be 16-byte aligned" in _message(), _message()


@pytest.mark.parametrize("off", [4, 8, 12])
def test_mlp_forward_refuses_misaligned_prepared(off):
    assert _lib.lib().lrf_mlp_forward(FAKE + off, FAKE, FAKE, 64, FAKE, None) == INVALID
    assert b"prepared must be 16-byte aligned" in _message(), _message()


def test_mlp_forward_null_prepared():
    assert _lib.lib().lrf_mlp_forward(None, FAKE, FAKE, 64, FAKE, None) == INVALID
    assert b"prepared is NULL" in _message()


# ---- M = 0 and M < 0 -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BACKWARD)
def test_backward_m0_null_data_accepted(name):
    assert _backward(name, M=0, xyz=None, gout=None, d_xyz=None) == OK


@pytest.mark.parametrize("name", FORWARD)
def test_forward_m0_null_data_accepted(name):
    assert getattr(_lib.lib(), name)(C.byref(_field()), None, 0, None, None) == OK


def test_mlp_forward_m0_null_data_accepted():
    assert _lib.lib().lrf_mlp_forward(FAKE, None, None, 0, None, None) == OK


@pytest.mark.parametrize("M", [-1, -(1 << 40)])
@pytest.mark.parametrize("name", BACKWARD)
def test_backward_negative_m(name, M):
    assert _backward(name, M=M) == INVALID
    assert b"bad xyz/grad_out/M" in _message()


@pytest.mark.parametrize("M", [-1, -(1 << 40)])
@pytest.mark.parametrize("name", FORWARD)
def test_forward_negative_m(name, M):
    assert getattr(_lib.lib(), name)(C.byref(_field()), FAKE, M, FAKE, None) == INVALID
    assert b"bad xyz/out/M" in _message()


@pytest.mark.parametrize("M", [-1, -(1 << 40)])
def test_mlp_forward_negative_m(M):
    assert _lib.lib().lrf_mlp_forward(FAKE, FAKE, FAKE, M, FAKE, None) == INVALID
    assert b"bad feats/viewdirs/rgb/M" in _message()


@pytest.mark.parametrize("name", BACKWARD)
@pytest.mark.parametrize("null", ["xyz", "gout"])
def test_backward_null_data(name, null):
    assert _backward(name, **{null: None}) == INVALID
    assert b"bad xyz/grad_out/M" in _message()


@pytest.mark.parametrize("null", [0, 1, 2])
def test_mlp_forward_null_data(null):
    args = [FAKE, FAKE, FAKE]
    args[null] = None
    assert _lib.lib().lrf_mlp_forward(FAKE, args[0], args[1], 64, args[2], None) == INVALID
    assert b"bad feats/viewdirs/rgb/M" in _message()
