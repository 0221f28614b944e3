"""-m gpu: lrf_resize_linear across the sizes, strides and values its C ABI accepts, bit for bit against
tests/resize_oracle.py (which equals cv2.resize without IPP, tests/test_resize_cpu.py), through
metrics.resize_linear and through ctypes: every form at its borders up to 7680 x 4320, enlargements whose last columns
copy, 1-pixel rows and columns, special values, odd and long row strides with canaries in the gaps, pinned memory, a
non-default stream, rows whose float32 index loses precision, and rows of more than 2^31 floats (one thread's pixel
offset past 32 bits), where the card has the memory.  NaN matches NaN whatever its bits (test_resize_cpu.same_bits)."""
import numpy as np
import pytest
import torch

import resize_oracle as ro
from test_resize_cpu import same_bits, special_frame

pytestmark = pytest.mark.gpu
F32 = np.float32
CANARY = np.array([0xDEADBEEF], np.uint32).view(np.float32)[0]      # -6.3e18: no value of these tests


def frame(w0, h0, seed):
    a = np.random.default_rng(seed).random((h0, w0, 3), dtype=np.float32)
    return a if seed % 2 == 0 else (a * 4000 - 2000).astype(F32)


def host(t):
    return t.detach().cpu().numpy()


def abi(src, w0, h0, s_src, dst, W, H, s_dst, stream=None):
    """lrf_resize_linear on raw pointers (device or pinned host), on `stream` (a handle) or the legacy stream."""
    from localrf_b200 import _lib
    _lib.check(_lib.lib().lrf_resize_linear(src.data_ptr(), w0, h0, s_src, dst.data_ptr(), W, H, s_dst, stream))


def both_paths(a, W, H):
    """-> (metrics.resize_linear, ctypes on contiguous device buffers) of a [h0, w0, 3] numpy frame, on the host."""
    from localrf_b200.metrics import resize_linear
    h0, w0 = a.shape[:2]
    src = torch.from_numpy(a).cuda()
    got = host(resize_linear(src, W, H))
    dst = torch.empty(H, W, 3, device="cuda")
    abi(src, w0, h0, 3 * w0, dst, W, H, 3 * W)
    torch.cuda.synchronize()
    return got, host(dst)


FORMS = [
    (1, 1, 1, 1), (7, 5, 7, 5), (1920, 1080, 1920, 1080),                          # same size: a copy
    (2, 2, 1, 1), (6, 2, 3, 1), (2, 4096, 1, 2048), (3840, 2160, 1920, 1080),      # exact 2x: INTER_AREA
    (7680, 4320, 3840, 2160),
    (64, 48, 32, 48), (3840, 2160, 1920, 2160), (3840, 2160, 3840, 1080),          # 2x on one axis: linear
    (9, 9, 3, 3), (5760, 3240, 1920, 1080), (16, 12, 4, 3), (7680, 4320, 1920, 1080),   # 3x, 4x
    (1921, 1081, 960, 540), (1001, 999, 1000, 998), (999, 1000, 1000, 999), (7, 3, 3, 7),  # odd ratios
    (3, 2, 100, 7), (2, 2, 4096, 3), (10, 10, 37, 41), (480, 270, 1921, 1081),     # enlargements
    (1, 1, 4096, 1), (1, 1, 1, 4096), (1, 1, 4096, 4096), (4096, 1, 1, 1),         # 1-pixel sources and outputs
    (1, 4096, 1, 1), (4096, 4096, 1, 1), (1, 7, 5, 1), (7, 1, 1, 5), (2, 1, 4096, 1), (1, 2, 1, 4096),
]


@pytest.mark.parametrize("w0,h0,W,H", FORMS)
def test_every_form_at_its_borders(w0, h0, W, H):
    for seed in range(2):
        a = frame(w0, h0, seed)
        want = ro.resize(a, W, H)
        for got in both_paths(a, W, H):
            assert got.shape == (H, W, 3) and np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
                (w0, h0, W, H, seed)


@pytest.mark.parametrize("w0,W", [(3, 100), (2, 4096), (10, 37), (480, 1921), (1, 4096)])
def test_enlargements_copy_their_last_columns(w0, W):
    """The enlargements above reach the copy branch (sx + 1 >= w0) on their last columns, and blend before it when
    the source has two columns: a test of the form would otherwise not see that branch."""
    sx, _ = ro._coeffs(W, w0)
    copy = np.maximum(sx, 0) + 1 >= w0
    assert copy[-1] and (w0 == 1 or not copy[W // 2])


SPECIAL_FORMS = [(64, 64, 32, 32), (20, 20, 20, 20), (17, 13, 40, 9), (9, 7, 3, 2), (5, 5, 64, 64),
                 (33, 17, 11, 50), (1, 9, 4, 3), (9, 1, 3, 4), (12, 12, 4, 3), (1920, 1080, 960, 540),
                 (1921, 1081, 960, 540)]


@pytest.mark.parametrize("w0,h0,W,H", SPECIAL_FORMS)
def test_special_values(w0, h0, W, H):
    """+-inf, NaN, -0, subnormals and +-3e38, whose blends and block sums overflow (test_resize_cpu checks the
    restatement against cv2 on the same frames)."""
    with np.errstate(invalid="ignore", over="ignore"):
        for seed in range(2):
            a = special_frame(w0, h0, seed)
            want = ro.resize(a, W, H)
            for got in both_paths(a, W, H):
                assert same_bits(got, want), (w0, h0, W, H, seed)


def padded(a, stride, fill, tail, device="cuda", pin=False):
    """A [h, w, 3] frame in a flat float32 buffer, rows `stride` floats apart, `tail` floats after the last row's
    stride, every other float `fill`."""
    h, w = a.shape[:2]
    buf = torch.full((h * stride + tail,), float(fill), dtype=torch.float32)
    buf[:h * stride].view(h, stride)[:, :3 * w] = torch.from_numpy(np.ascontiguousarray(a).reshape(h, 3 * w))
    return buf.pin_memory() if pin else buf.to(device)


def unpad(buf, w, h, stride):
    """-> (the [h, w, 3] frame, the row gaps [h, stride - 3w], the tail) of a padded buffer, on the host."""
    b = host(buf)
    rows = b[:h * stride].reshape(h, stride)
    return rows[:, :3 * w].reshape(h, w, 3), rows[:, 3 * w:], b[h * stride:]


def untouched(x):
    return bool(np.all(x.view(np.uint32) == CANARY.view(np.uint32)))


@pytest.mark.parametrize("w0,h0,W,H", [(17, 13, 40, 9), (64, 64, 32, 32), (20, 20, 20, 20), (9, 1, 3, 4),
                                       (1, 9, 4, 3), (1921, 1081, 960, 540)])
@pytest.mark.parametrize("extra_src,extra_dst", [(1, 5), (7, 2), (5, 13), (1001, 3 * 997), (0, 11), (13, 0)])
def test_strides_leave_the_gaps_alone(w0, h0, W, H, extra_src, extra_dst):
    """Row strides of 3 w0 + k and 3 W + k floats, odd and not multiples of 3 or 4, or far longer than a row.  The
    source's gaps hold NaN, which would show in any output that read one; the destination's gaps and the floats after
    its last row hold a canary, which must come back unchanged."""
    a = frame(w0, h0, 1)
    want = ro.resize(a, W, H)
    s_src, s_dst = 3 * w0 + extra_src, 3 * W + extra_dst
    src = padded(a, s_src, np.nan, 5)
    dst = padded(np.zeros((H, W, 3), F32), s_dst, CANARY, 64)
    dst[:H * s_dst].view(H, s_dst)[:, :3 * W] = float(CANARY)
    abi(src, w0, h0, s_src, dst, W, H, s_dst)
    torch.cuda.synchronize()
    got, gaps, tail = unpad(dst, W, H, s_dst)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert untouched(gaps) and untouched(tail)


@pytest.mark.parametrize("w0,h0,W,H", [(1921, 1081, 960, 540), (3840, 2160, 1920, 1080), (5, 5, 64, 64)])
def test_pinned_memory_streams_and_repeats(w0, h0, W, H):
    """A pinned source and a pinned destination through the ABI, with strides; a non-blocking stream whose earlier
    work (a spin, then the copy that fills the source) the kernel must wait for; three calls give the same bits."""
    a = frame(w0, h0, 0)
    want = ro.resize(a, W, H)
    s_src, s_dst = 3 * w0 + 5, 3 * W + 7
    for pin_src, pin_dst in ((True, False), (False, True), (True, True)):
        src = padded(a, s_src, np.nan, 3, pin=pin_src)
        dst = padded(np.zeros((H, W, 3), F32), s_dst, CANARY, 16, pin=pin_dst)
        dst[:H * s_dst].view(H, s_dst)[:, :3 * W] = float(CANARY)
        abi(src, w0, h0, s_src, dst, W, H, s_dst)
        torch.cuda.synchronize()
        got, gaps, tail = unpad(dst, W, H, s_dst)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (pin_src, pin_dst)
        assert untouched(gaps) and untouched(tail)
    filled = padded(a, s_src, np.nan, 3)
    stream = torch.cuda.Stream()
    outs = []
    for _ in range(3):
        src = torch.full_like(filled, float("nan"))
        dst = torch.full(((H * s_dst) + 16,), float(CANARY), device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)                       # ~10 ms: the fill below lands well after the launch
            src.copy_(filled)
            abi(src, w0, h0, s_src, dst, W, H, s_dst, stream.cuda_stream)
        stream.synchronize()
        outs.append(unpad(dst, W, H, s_dst))
    for got, gaps, tail in outs:
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert untouched(tail)


@pytest.mark.parametrize("w0,W", [(20_000_001, 17_000_003), (3, 17_000_003)])
def test_rows_where_the_float_index_loses_precision(w0, W):
    """1-row frames whose float32 column index cannot tell neighbouring columns apart (test_resize_cpu checks the
    restatement against cv2 at these sizes)."""
    a = np.random.default_rng(w0).random((1, w0, 3), dtype=np.float32)
    want = ro.resize(a, W, 1)
    for got in both_paths(a, W, 1):
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---- rows of more than 2^31 floats -----------------------------------------------------------------------------
# 3 x passes 2^31 from x = 715,827,883: the output offset of every form, the source offset of the copy (w0 = W) and of
# the linear rule (w0 >= 715,827,883), and 3 (2 x + dx) of the exact 2x from W = 357,913,942.  One row each, checked
# in full on the device in chunks, plus the columns around 715,827,883 and the last ones by name.
EDGE = 715_827_883
BIG = {
    # name: (w0, h0, W, H)
    "linear_up": (2, 1, 716_000_000, 1),                  # output offsets; its last columns copy
    "copy": (716_000_000, 1, 716_000_000, 1),             # source and output offsets of the copy
    "linear_down": (716_000_000, 1, 537_000_001, 1),      # source offsets of the linear rule
    "area2": (716_000_000, 2, 358_000_000, 1),            # 3 (2 x + dx) of the 2x block sum
    "int_max": (2 ** 31 - 1, 1, 2 ** 30, 1),              # the float index of the last columns is 2^31: INT_MAX in int
}
CHUNK = 1 << 24


def need_bytes(w0, h0, W, H):
    """The source, the output and the chunked check's temporaries (about 120 bytes a column), with 1 GiB spare."""
    return 12 * (w0 * h0 + W * H) + 120 * CHUNK + (1 << 30)


def expected(name, src, w0, W, x0, x1):
    """Columns [x0, x1) of the one output row, on the device: the copy, the 2x block sum in row-major order, or
    resize_oracle.row_chunk's linear rule."""
    if name == "copy":
        return src[3 * x0:3 * x1].view(-1, 3)
    if name == "area2":
        r0, r1 = src[:3 * w0].view(-1, 3), src[3 * w0:].view(-1, 3)
        s = ((r0[2 * x0:2 * x1:2] + r0[2 * x0 + 1:2 * x1:2]) + r1[2 * x0:2 * x1:2]) + r1[2 * x0 + 1:2 * x1:2]
        return s * 0.25
    return ro.row_chunk(src.view(-1, 3), W, x0, x1)


@pytest.mark.parametrize("name", list(BIG))
def test_rows_past_2_31_floats(name):
    w0, h0, W, H = BIG[name]
    last = np.floor(F32((W - 1 + 0.5) * (1.0 / (W / w0)) - 0.5))        # the last column's source index
    assert max(w0, W) >= EDGE                                           # an offset passes 2^31
    if name in ("linear_up", "int_max"):
        assert last + 1 >= w0                                           # the last columns copy
    if name == "int_max":
        assert last == 2.0 ** 31                                        # past INT_MAX in the kernel's int
    torch.cuda.empty_cache()                                            # what earlier cases left cached
    free, total = torch.cuda.mem_get_info()
    need = need_bytes(w0, h0, W, H)
    if free < need:
        pytest.skip(f"{name} needs {need / 2 ** 30:.1f} GiB of device memory, {free / 2 ** 30:.1f} GiB is free")
    print(f"\n{name}: {w0}x{h0} -> {W}x{H}, {need / 2 ** 30:.1f} GiB needed, {free / 2 ** 30:.1f} GiB free of "
          f"{total / 2 ** 30:.1f}")
    g = torch.Generator(device="cuda").manual_seed(w0 + W)
    src = torch.rand(3 * w0 * h0, generator=g, device="cuda")
    dst = torch.full((3 * W + 64,), float(CANARY), device="cuda")
    abi(src, w0, h0, 3 * w0, dst, W, H, 3 * W)
    out = dst[:3 * W].view(W, 3)
    bad = []
    for x0 in range(0, W, CHUNK):
        x1 = min(W, x0 + CHUNK)
        if not torch.equal(out[x0:x1].view(torch.int32), expected(name, src, w0, W, x0, x1).view(torch.int32)):
            bad.append(x0)
    assert not bad, f"{name}: chunks of {CHUNK} columns from {bad[:8]} differ"
    for x0, x1 in ((EDGE - 3, EDGE + 3), (W - 3, W)):
        x0, x1 = max(0, min(x0, W)), min(x1, W)
        if x0 < x1:
            want, got = host(expected(name, src, w0, W, x0, x1)), host(out[x0:x1])
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, x0, x1, got, want)
    assert untouched(host(dst[3 * W:]))
