"""CPU-only: tests/ingest_oracle.py, the numpy restatement of what lrf_ingest_frame computes, held bit for bit
against cv2 and numpy on seeded synthetic frames -- the conversions of LocalRFDataset.read_meta
(dataLoader/localrf_dataset.py:143-258) as the reference writes them."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
import ingest_oracle as io  # noqa: E402


def bits_equal(a, b):
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def ref_image(bgr, k):
    img = bgr[..., ::-1].astype(np.float32) / 255
    if k != 1:
        img = cv2.resize(img, None, fx=1 / k, fy=1 / k, interpolation=cv2.INTER_AREA)
    return img


def ref_flow(e, h, w, scale):
    """resize and decode_flow (utils/utils.py:67-71) of the reference, restated with its own numpy calls."""
    e = cv2.resize(e, (w, h), interpolation=cv2.INTER_AREA)
    f = e[..., :2].astype(np.float32)
    f -= 2 ** 15
    f /= 2 ** 8
    return f * scale, (e[..., 2] > 2 ** 15).astype(np.float32)


@pytest.mark.parametrize("h,w,k", [(31, 17, 1), (1, 1, 1), (2, 3, 1), (27, 45, 2), (270, 480, 2), (13, 9, 4),
                                   (135, 240, 4), (1, 1, 2), (1, 1, 4)])
def test_image_and_loss_weight(h, w, k):
    rng = np.random.default_rng(h * 1000 + w * 10 + k)
    bgr = rng.integers(0, 256, (k * h, k * w, 3), dtype=np.uint8)
    bgr[0, 0] = 255
    img = ref_image(bgr, k)
    assert bits_equal(io.image(bgr, k), img)
    lap = cv2.Laplacian(cv2.cvtColor((img * 255).astype(np.uint8), cv2.COLOR_RGB2GRAY), cv2.CV_32F)
    assert bits_equal(io.laplacian(io.gray(img)), lap)                   # reflect-101 corners included
    assert bits_equal(io.loss_weight(img), np.ones_like(img[..., 0]) * lap.var())
    mask = rng.integers(0, 3, (h, w), dtype=np.uint8) * 120
    want = np.ones_like(img[..., 0]) * lap.var() * (cv2.resize(mask, (w, h), interpolation=cv2.INTER_AREA) > 0)
    assert bits_equal(io.loss_weight(img, io.motion(mask, h, w)), want)


def test_gray_is_the_15_bit_conversion():
    rgb = np.stack(np.meshgrid(np.arange(256), np.arange(256), indexing="ij"), -1).reshape(-1, 2)
    for b in (0, 1, 77, 128, 254, 255):
        u = np.concatenate([rgb, np.full((len(rgb), 1), b)], 1).astype(np.uint8).reshape(256, 256, 3)
        img = (u.astype(np.float32) / 255)
        assert np.array_equal(io.gray(img), cv2.cvtColor((img * 255).astype(np.uint8), cv2.COLOR_RGB2GRAY))


@pytest.mark.parametrize("hs,ws,h,w", [(15, 20, 30, 40), (135, 240, 270, 480), (13, 17, 41, 37), (20, 20, 20, 20),
                                       (11, 9, 11, 31), (1, 1, 5, 3), (7, 5, 8, 6)])
def test_flow(hs, ws, h, w):
    rng = np.random.default_rng(hs * 100 + ws)
    e = rng.integers(0, 65536, (hs, ws, 3), dtype=np.uint16)
    e[0, 0], e[0, -1], e[-1, 0] = 65535, 0, 32768                         # saturating and boundary codes
    e[-1, -1] = (32768, 32769, 32769)
    scale = h / hs
    f, m = io.flow(e, h, w, scale)
    rf, rm = ref_flow(e, h, w, scale)
    assert bits_equal(f, rf) and bits_equal(m, rm)
    assert bits_equal(io.resize(e, h, w), cv2.resize(e, (w, h), interpolation=cv2.INTER_AREA))


@pytest.mark.parametrize("hs,ws,h,w", [(30, 40, 30, 40), (60, 80, 30, 40), (120, 160, 30, 40), (15, 20, 30, 40),
                                       (13, 17, 41, 37)])
def test_invdepth(hs, ws, h, w):
    d = np.random.default_rng(hs + ws).integers(0, 65536, (hs, ws), dtype=np.uint16)
    d[0, 0] = 65535
    want = cv2.resize(d.astype(np.float32), (w, h), interpolation=cv2.INTER_AREA)
    assert bits_equal(io.invdepth(d, h, w), want)


def test_unsupported_ratios():
    with pytest.raises(NotImplementedError):
        io.resize(np.zeros((30, 40), np.float32), 20, 20)                # neither a reduction nor an enlargement
    with pytest.raises(NotImplementedError):
        io.reduce(np.zeros((30, 30), np.float32), 3)
    with pytest.raises(NotImplementedError):
        io.motion(np.zeros((30, 40), np.uint8), 15, 20)


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 127, 128, 129, 136, 143, 144, 1000, 8191, 8192, 8193, 100003,
                               960 * 540, 480 * 270])
def test_variance_summation_order(n):
    rng = np.random.default_rng(n)
    x = rng.integers(-1020, 1021, n).astype(np.float32) * np.float32(rng.random() + 0.5)
    assert bits_equal(io.pairwise_sum(x), np.sum(x))
    assert bits_equal(io.variance(x), x.var())
    assert bits_equal(io.slot_tree_sum(x), np.sum(x))
    d = (x - np.float32(x.mean())).astype(np.float32)
    assert bits_equal(io.slot_tree_sum(d * d), np.sum(d * d))


def test_tree_depth_matches_the_library():
    from localrf_b200 import _lib
    L = _lib.lib()
    for n in (1, 128, 129, 5000, 518400, 2073600):
        D = io.tree_depth(n)
        assert L.lrf_ingest_scratch_bytes(n) == (16 + 4 * n + 5 * (1 << D) + n + 7) // 8 * 8
    assert L.lrf_ingest_scratch_bytes(0) == 0 and L.lrf_ingest_scratch_bytes(9_000_000) == 0


def test_golden_scenes():
    """The restatement, fed the files of tests/golden/ingest.npz, reproduces every array the unmodified reference's
    read_meta built from them."""
    import json
    import os
    import tempfile
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ingest.npz"))
    for case, scene in zip(z["cases"], z["scenes"]):
        cfg = json.loads(str(z[f"{case}.config"]))
        with tempfile.TemporaryDirectory() as d:
            io.write_golden_scene(z, str(scene), d)
            frames = io.scene_frames(d, cfg)
        for key in ("rgbs", "loss_weights", "invdepths", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"):
            name = f"{case}.frames.{key}"
            if name not in z:
                assert key not in ("rgbs", "loss_weights")
                continue
            for f, fr in enumerate(frames):
                assert bits_equal(fr[key], z[name][f]), (case, key, f)
