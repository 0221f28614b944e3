"""-m gpu: the two kernels that make a rendered test frame's outputs, at the shapes, strides and values their C ABI
accepts.

lrf_frame_to_u8 (8-bit BGR rgb and colour-mapped depth, renderer.py:127,176) is compared bit for bit with the
reference's outputs in tests/golden/frame_u8.npz and with tests/metrics_oracle.py (rgb8 / depth8): pixel counts
around the block size and past the grid-stride cap, strided and interleaved inputs, device and pinned outputs,
one output at a time, N = 0, and rgb outside the range where it equals OpenCV.

lrf_image_metrics (MSE and SSIM, renderer.py:162-163) is compared with metrics_oracle.ssim: every filter size,
shapes whose last tile has zero, one or a full set of output rows and columns, strided frames, integer frames,
constant and identical frames, non-finite pixels and a 1920x1080 frame.  With the kernel's own taps
(taps="kernel") the oracle does the kernel's fp64 arithmetic operation for operation, so the map is compared
bitwise; against the reference's taps it is within 1e-12."""
import os

import numpy as np
import pytest
import torch

import metrics_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xA5
RANGES = [(0, 5), (0.1, 0.7), (0.3, 2.9), (0.2, 1.9)]


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "frame_u8.npz"))


def frame_u8(rgb, rgb_stride, depth, depth_stride, n, lo, hi, lut, rgb8, depth8):
    """lrf_frame_to_u8 on the current stream; tensors (or None) are passed by data pointer."""
    from localrf_b200 import _lib
    from localrf_b200.tensorf import _ptr, _stream
    L = _lib.lib()
    rc = L.lrf_frame_to_u8(_ptr(rgb), rgb_stride, _ptr(depth), depth_stride, n, lo, hi, _ptr(lut), _ptr(rgb8),
                           _ptr(depth8), _stream(torch.device("cuda")))
    assert rc == 0, L.lrf_last_error()
    torch.cuda.synchronize()


def index_lut(seed):
    """A random colour map whose first channel is a permutation of 0..255: a byte names the index it came from."""
    rng = np.random.default_rng(seed)
    lut = rng.integers(0, 256, (256, 3), dtype=np.uint8)
    lut[:, 0] = rng.permutation(256)
    return lut


def assert_depth8_equal(got, want, depth, lut, what):
    bad = np.flatnonzero((got != want).any(-1))
    if len(bad):
        inv = np.argsort(lut[:, 0])
        rows = [f"d={depth[i]!r} (bits {int(np.float32(depth[i]).view(np.uint32))}) want index "
                f"{inv[want[i, 0]]} got {inv[got[i, 0]]}" for i in bad[:8]]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} depth8 pixels differ:\n" + "\n".join(rows))


def out_buffer(n, where):
    t = torch.full((n * 3 + 64,), SENTINEL, dtype=torch.uint8)   # 64 bytes past the frame must stay untouched
    return t.cuda() if where == "device" else t.pin_memory()


def test_golden_bitwise():
    g = golden()
    lut = g["lut"]
    lut_d = torch.from_numpy(lut).cuda()
    rgb = torch.from_numpy(g["rgb"]).cuda()
    n = len(g["rgb"])
    rgb8 = out_buffer(n, "device")
    frame_u8(rgb, 3, None, 1, n, 0.0, 5.0, None, rgb8, None)
    got = rgb8.cpu().numpy()
    np.testing.assert_array_equal(got[:3 * n].reshape(n, 3), g["rgb8"])
    assert (got[3 * n:] == SENTINEL).all()
    for i, (lo, hi) in enumerate(g["ranges"]):
        d = g[f"depth.{i}"]
        depth8 = out_buffer(len(d), "device")
        frame_u8(None, 3, torch.from_numpy(d).cuda(), 1, len(d), float(lo), float(hi), lut_d, None, depth8)
        got = depth8.cpu().numpy()
        assert (got[3 * len(d):] == SENTINEL).all()
        got = got[:3 * len(d)].reshape(-1, 3)
        assert_depth8_equal(got, g[f"depth8.{i}"], d, lut, f"golden range ({lo}, {hi})")
        np.testing.assert_array_equal(got, orc.depth8(d, lo, hi, lut))


def crossing_depths(lo, hi):
    """The float32 depths on either side of every index boundary of (lo, hi)."""
    den = hi - lo + 1e-8
    c = np.array([lo + k / 255 * den for k in range(1, 256)], np.float32)
    return np.concatenate([c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))])


def frame_values(n, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(n, 3, generator=g) * 1.2 - 0.1
    ties = torch.tensor([(k + 0.5) / 255 for k in range(256)], dtype=torch.float32)
    m = min(n * 3, len(ties))
    rgb.view(-1)[:m] = ties[:m]
    a, b = min(lo, hi), max(lo, hi)
    depth = torch.rand(n, generator=g) * (b - a + 1.0) + (a - 0.5)
    c = torch.from_numpy(crossing_depths(lo, hi))
    c = c[torch.randperm(len(c), generator=g)][:n]
    depth[torch.randperm(n, generator=g)[:len(c)]] = c
    if n >= 16:
        depth[:4] = torch.tensor([float("nan"), float("inf"), -float("inf"), -float("nan")])
        rgb[n - 1] = torch.tensor([float("nan"), -float("inf"), 1.5])
    return rgb, depth


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("rgb_stride, depth_stride", [(3, 1), (4, 4), (7, 1), (7, 4)])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 540673, 1920 * 1080])
def test_sizes_strides_and_output_memory(n, rgb_stride, depth_stride, where):
    """540673 pixels is one more than 132 SMs x 16 blocks x 256 threads: the grid-stride loop takes a second
    pass.  Stride 4 / 4 is the interleaved [N,4] pix layout (rgb in columns 0-2, depth in column 3); the other
    layouts fill the columns the kernel must not read with NaN."""
    ri = [1, 255, 256, 257, 540673, 1920 * 1080].index(n) + [3, 4, 7].index(rgb_stride)
    lo, hi = RANGES[ri % len(RANGES)]
    rgb, depth = frame_values(n, lo, hi, seed=n + rgb_stride + depth_stride)
    lut = index_lut(n)
    if (rgb_stride, depth_stride) == (4, 4):
        pix = torch.cat([rgb, depth[:, None]], 1).cuda()
        rgb_in, depth_in = pix, pix[:, 3:]
    else:
        rgb_in = torch.full((n, rgb_stride), float("nan"))
        rgb_in[:, :3] = rgb
        depth_in = torch.full((n, depth_stride), float("nan"))
        depth_in[:, 0] = depth
        rgb_in, depth_in = rgb_in.cuda(), depth_in.cuda()
    rgb8, depth8 = out_buffer(n, where), out_buffer(n, where)
    frame_u8(rgb_in, rgb_stride, depth_in, depth_stride, n, lo, hi, torch.from_numpy(lut).cuda(), rgb8, depth8)
    r8, d8 = rgb8.cpu().numpy(), depth8.cpu().numpy()
    assert (r8[3 * n:] == SENTINEL).all() and (d8[3 * n:] == SENTINEL).all()
    np.testing.assert_array_equal(r8[:3 * n].reshape(n, 3), orc.rgb8(rgb.numpy()))
    assert_depth8_equal(d8[:3 * n].reshape(n, 3), orc.depth8(depth.numpy(), lo, hi, lut), depth.numpy(),
                        lut, f"range ({lo}, {hi})")


@pytest.mark.parametrize("which", ["rgb8", "depth8"])
def test_one_output_leaves_the_other_untouched(which):
    n, (lo, hi) = 70001, RANGES[2]
    rgb, depth = frame_values(n, lo, hi, seed=4)
    lut = index_lut(4)
    rgb8, depth8 = out_buffer(n, "device"), out_buffer(n, "device")
    only_rgb = which == "rgb8"
    frame_u8(rgb.cuda(), 3, depth.cuda(), 1, n, lo, hi, torch.from_numpy(lut).cuda(),
             rgb8 if only_rgb else None, None if only_rgb else depth8)
    r8, d8 = rgb8.cpu().numpy(), depth8.cpu().numpy()
    if only_rgb:
        assert (d8 == SENTINEL).all() and (r8[3 * n:] == SENTINEL).all()
        np.testing.assert_array_equal(r8[:3 * n].reshape(n, 3), orc.rgb8(rgb.numpy()))
    else:
        assert (r8 == SENTINEL).all() and (d8[3 * n:] == SENTINEL).all()
        assert_depth8_equal(d8[:3 * n].reshape(n, 3), orc.depth8(depth.numpy(), lo, hi, lut), depth.numpy(), lut,
                            "depth8 only")


def test_zero_pixels_writes_nothing():
    rgb8, depth8 = out_buffer(4, "device"), out_buffer(4, "pinned")
    lut = torch.from_numpy(index_lut(0)).cuda()
    x = torch.zeros(12, device="cuda")
    frame_u8(x, 3, x, 1, 0, 0.0, 5.0, lut, rgb8, depth8)
    assert (rgb8.cpu() == SENTINEL).all() and (depth8 == SENTINEL).all()


def test_out_of_range_rgb_follows_the_documented_rule():
    """|255 v| < 2^31, NaN and -inf: OpenCV's x86-64 conversion (the oracle).  255 v >= 2^31 and +inf: 255 (OpenCV
    gives 0 there); 255 v <= -2^31: 0 (as OpenCV)."""
    edge = np.float32(2.0 ** 31 / 255)
    below = np.nextafter(edge, np.float32(0))                             # the largest v with 255 v < 2^31
    while np.float32(255) * below >= np.float32(2.0 ** 31):
        below = np.nextafter(below, np.float32(0))
    v = np.array([below, edge, -below, -edge, 1e20, -1e20, np.inf, -np.inf, np.nan, 3e9 / 255, 2.2e9 / 255,
                  2e9 / 255], np.float32)
    rgb = np.stack([v, v[::-1], np.roll(v, 5)], -1)
    rgb8 = out_buffer(len(rgb), "device")
    frame_u8(torch.from_numpy(rgb).cuda(), 3, None, 1, len(rgb), 0.0, 5.0, None, rgb8, None)
    got = rgb8.cpu().numpy()[:3 * len(rgb)].reshape(-1, 3)
    with np.errstate(over="ignore"):
        s = np.float32(255) * rgb[..., ::-1]
    high = s >= np.float32(2.0 ** 31)
    want = orc.rgb8(rgb)
    assert high.sum() >= 3 * 4 and (want[high] == 0).all()               # where OpenCV writes 0 ...
    want[high] = 255                                                      # ... the kernel saturates
    np.testing.assert_array_equal(got, want)
    assert (got[s < 0] == 0).all() and (got[np.isnan(s)] == 0).all()


# ---- lrf_image_metrics --------------------------------------------------------------------------------------

def strided(a, stride):
    """[H,W,3] float32 -> a CUDA [H,W,3] view whose pixels are `stride` floats apart (the rest NaN)."""
    H, W, _ = a.shape
    buf = torch.full((H, W, stride), float("nan"), device="cuda")
    buf[..., :3] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return buf[..., :3]


def device_metrics(img, gt, fs, sigma, max_val=1.0, strides=(3, 3)):
    from localrf_b200 import metrics
    a, b = strided(img, strides[0]), strided(gt, strides[1])
    H, W = img.shape[:2]
    out_map = torch.empty(2, dtype=torch.float64, device="cuda")
    out = torch.empty(2, dtype=torch.float64, device="cuda")
    m = torch.full((H - fs + 1, W - fs + 1, 3), -7.0, dtype=torch.float64, device="cuda")
    kw = dict(max_val=max_val, filter_size=fs, filter_sigma=sigma)
    metrics._enqueue(a, b, out_map, m, **kw)
    metrics._enqueue(a, b, out, None, **kw)
    out_map, out = out_map.cpu().numpy(), out.cpu().numpy()
    assert out_map.tobytes() == out.tobytes(), (out_map, out)            # same with and without the map
    return out, m.cpu().numpy()


def check_metrics(img, gt, fs, sigma, max_val=1.0, strides=(3, 3), what=""):
    out, m = device_metrics(img, gt, fs, sigma, max_val, strides)
    kw = dict(max_val=max_val, filter_size=fs, filter_sigma=sigma, return_map=True)
    with np.errstate(invalid="ignore", over="ignore"):                  # non-finite pixels
        want_k = orc.ssim(img, gt, taps="kernel", **kw)
        want_r = orc.ssim(img, gt, taps="reference", **kw)
        mse = orc.mse(img, gt)
    assert m.shape == want_k.shape
    np.testing.assert_array_equal(m, want_k, err_msg=what)               # bitwise (NaN where the oracle has NaN)
    fin = np.isfinite(want_r)
    assert (np.isfinite(m) == fin).all() and (np.isnan(m) == np.isnan(want_r)).all(), what
    np.testing.assert_allclose(m[fin], want_r[fin], rtol=0, atol=1e-12, err_msg=what)
    mean = float(np.mean(want_k))
    assert (np.isnan(out[1]) and np.isnan(mean)) or abs(out[1] - mean) <= 1e-12, (what, out[1], mean)
    assert (np.isnan(out[0]) and np.isnan(mse)) or abs(out[0] - mse) <= 1e-12 * mse, (what, out[0], mse)
    return out, m


STRIDES = [(3, 3), (4, 3), (3, 7), (8, 5)]


@pytest.mark.parametrize("fs", range(1, 17))
def test_ssim_every_filter_size_and_edge_tile(fs):
    """H in {fs, fs+1, 16+fs-1, 16+fs, 33} and W in {fs, 32+fs-1, 32+fs, 65}: the last 16 x 32 tile holds zero,
    one or a full set of output rows and columns.  Frames are uniform noise, a smooth image with noise, or
    integers with max_val 255; each shape runs with each sigma."""
    rng = np.random.default_rng(100 + fs)
    i = 0
    for H in (fs, fs + 1, 16 + fs - 1, 16 + fs, 33):
        for W in (fs, 32 + fs - 1, 32 + fs, 65):
            if H < fs:
                continue
            for sigma in (0.5, 1.5, 4.0):
                kind = i % 3
                if kind == 0:
                    a, b, mv = rng.random((H, W, 3), np.float32), rng.random((H, W, 3), np.float32), 1.0
                elif kind == 1:
                    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
                    a = np.stack([0.5 + 0.4 * np.sin(3 * xx + c) * np.cos(2 * yy - c) for c in range(3)], -1)
                    b = np.clip(a + 0.05 * rng.standard_normal(a.shape), 0, 1)
                    a, b, mv = a.astype(np.float32), b.astype(np.float32), 1.0
                else:
                    a = rng.integers(0, 256, (H, W, 3)).astype(np.float32)
                    b = np.clip(a + rng.integers(-20, 21, a.shape), 0, 255).astype(np.float32)
                    mv = 255.0
                check_metrics(a, b, fs, sigma, mv, STRIDES[i % 4], f"H={H} W={W} fs={fs} sigma={sigma}")
                i += 1


@pytest.mark.parametrize("fs", [1, 2, 8, 11, 16])
def test_ssim_constant_and_identical_frames(fs):
    H, W = 16 + fs, 32 + fs
    a = np.full((H, W, 3), 0.3, np.float32)
    b = np.full((H, W, 3), 0.7, np.float32)
    check_metrics(a, b, fs, 1.5, what="constant")
    check_metrics(255 * a, 255 * a, fs, 1.5, 255.0, (4, 3), "constant identical")
    c = np.random.default_rng(fs).random((H, W, 3), np.float32)
    out, m = check_metrics(c, c.copy(), fs, 1.5, strides=(3, 7), what="identical")
    assert (m == 1.0).all() and out[0] == 0.0 and out[1] == 1.0


@pytest.mark.parametrize("fs", [1, 4, 11, 16])
def test_ssim_non_finite_pixels(fs):
    """NaN and +-inf pixels in either frame: every window that holds one is NaN in the reference's map; the rest
    of the map is finite and matches."""
    rng = np.random.default_rng(fs)
    H, W = 40, 70
    a, b = rng.random((H, W, 3), np.float32), rng.random((H, W, 3), np.float32)
    for frame, val, (r, c, ch) in ((a, np.nan, (3, 5, 0)), (b, np.inf, (20, 40, 1)), (a, -np.inf, (35, 66, 2)),
                                   (b, -np.inf, (12, 12, 0)), (a, np.inf, (12, 12, 0))):
        frame[r, c, ch] = val
    out, m = check_metrics(a, b, fs, 1.5, strides=(4, 3), what="non-finite")
    assert np.isnan(out[0]) and np.isnan(out[1])
    assert np.isfinite(m).any() and not np.isfinite(m).all()


def test_ssim_1920x1080():
    """4080 tile CTAs: the final kernel sums four partials per thread."""
    rng = np.random.default_rng(1080)
    H, W = 1080, 1920
    yy, xx = np.meshgrid(np.linspace(0, 1, H, dtype=np.float32), np.linspace(0, 1, W, dtype=np.float32),
                         indexing="ij")
    a = np.stack([0.5 + 0.4 * np.sin(9 * xx + c) * np.cos(5 * yy - c) for c in range(3)], -1).astype(np.float32)
    b = np.clip(a + rng.normal(0, 0.03, a.shape).astype(np.float32), 0, 1).astype(np.float32)
    check_metrics(b, a, 11, 1.5, strides=(4, 3), what="1920x1080")
