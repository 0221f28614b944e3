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


# (hs, ws, h, w) enlargements: by 2 and by 3 (every area weight is 0: the source pixel is repeated), odd ratios, one
# axis only, a 1 x 1 source, by 5 / 4 and 3 / 2 (weights .25, .5, .75: exact .5 ties for uint16), and the ratios
# 6 -> 8, 9 -> 12, 10 -> 14 and 14 -> 16 on each axis and 720 x 405 -> 960 x 540, where some area weight is exactly 0
# in double arithmetic (a fused multiply-add would leave about 1e-16 in its place).
ENLARGEMENTS = [(15, 20, 30, 40), (10, 10, 30, 30), (13, 17, 41, 37), (11, 9, 11, 31), (1, 1, 5, 3), (7, 5, 8, 6),
                (12, 16, 15, 20), (10, 14, 15, 21), (6, 6, 8, 8), (9, 6, 12, 8), (10, 9, 14, 12), (14, 10, 16, 14),
                (6, 14, 8, 16), (405, 720, 540, 960)]


def extreme_planes(hs, ws, seed):
    """uint16 [hs][ws] planes of zeros next to 65535: alternating columns, alternating rows (each in both phases)
    and a seeded mixture -- where a weight that should be exactly 0 or 1 shows in the result."""
    cols, rows = np.zeros((hs, ws), np.uint16), np.zeros((hs, ws), np.uint16)
    cols[:, 1::2] = rows[1::2] = 65535
    mix = (np.random.default_rng(seed).integers(0, 2, (hs, ws)) * 65535).astype(np.uint16)
    return {"cols": cols, "cols'": 65535 - cols, "rows": rows, "rows'": 65535 - rows, "mix": mix}


def flow_planes(hs, ws, seed):
    """uint16 [hs][ws][3] encoded flows: random codes with the saturating and mask-boundary codes in the corners,
    the zero / 65535 planes, and codes around 32768 whose neighbours differ by 1, 2, 3 and 6, so that the weights of
    an enlargement by 5 / 4 (.25, .5, .75) land on exact .5 ties next to even and to odd codes, and on the mask's
    32768 / 32769 threshold."""
    rng = np.random.default_rng(seed)
    e = rng.integers(0, 65536, (hs, ws, 3), dtype=np.uint16)
    e[0, 0], e[0, -1], e[-1, 0] = 65535, 0, 32768
    e[-1, -1] = (32768, 32769, 32769)
    x = extreme_planes(hs, ws, seed)
    near = rng.choice(np.array([32762, 32764, 32765, 32767, 32768, 32769, 32770, 32771, 32773, 32776], np.uint16),
                      (hs, ws, 3))
    near[0, 0], near[0, -1] = (0, 65535, 32768), (65535, 0, 32769)
    return {"random": e, "extreme": np.stack([x["cols"], x["rows'"], x["mix"]], -1), "near": near}


@pytest.mark.parametrize("hs,ws,h,w", ENLARGEMENTS + [(135, 240, 270, 480), (20, 20, 20, 20)])
def test_flow(hs, ws, h, w):
    scale = h / hs
    for name, e in flow_planes(hs, ws, hs * 100 + ws).items():
        f, m = io.flow(e, h, w, scale)
        rf, rm = ref_flow(e, h, w, scale)
        assert bits_equal(f, rf) and bits_equal(m, rm), name
        assert bits_equal(io.resize(e, h, w), cv2.resize(e, (w, h), interpolation=cv2.INTER_AREA)), name


def test_flow_planes_hold_ties_and_threshold_codes():
    """What flow_planes promises, so that the rounding and the mask threshold are really exercised: at 12 x 16 ->
    15 x 20 the "near" plane's blends land on exact .5 ties below even and below odd codes, some of them between
    32768 and 32769 in the mask's channel, which also resizes to 32768 and to 32769 themselves."""
    e = flow_planes(12, 16, 7)["near"]
    sx, fx = io.area_weights(20, 16)
    sy, fy = io.area_weights(15, 12)
    assert {0.25, 0.5, 0.75} <= set(fx.tolist()) and {0.25, 0.5, 0.75} <= set(fy.tolist())
    x = e.astype(np.float64)
    hor = x[:, sx] * (1 - fx)[None, :, None] + x[:, np.minimum(sx + 1, 15)] * fx[None, :, None]
    out = hor[sy] * (1 - fy)[:, None, None] + hor[np.minimum(sy + 1, 11)] * fy[:, None, None]   # exact in double
    ties = out[out % 1 == 0.5]
    assert (np.floor(ties) % 2 == 0).sum() > 10 and (np.floor(ties) % 2 == 1).sum() > 10
    assert (out[..., 2] == 32768.5).any()
    third = io.resize(e, 15, 20)[..., 2]
    assert (third == 32768).sum() > 10 and (third == 32769).sum() > 10


@pytest.mark.parametrize("hs,ws,h,w", ENLARGEMENTS + [(30, 40, 30, 40), (60, 80, 30, 40), (120, 160, 30, 40),
                                                      (24, 32, 6, 8)])
def test_invdepth(hs, ws, h, w):
    d = np.random.default_rng(hs + ws).integers(0, 65536, (hs, ws), dtype=np.uint16)
    d[0, 0] = 65535
    for name, d in dict(extreme_planes(hs, ws, hs + ws), random=d).items():
        want = cv2.resize(d.astype(np.float32), (w, h), interpolation=cv2.INTER_AREA)
        assert bits_equal(io.invdepth(d, h, w), want), name


def test_exact_zero_weight_at_6_to_8():
    """The case a fused multiply-add gets wrong: output 3 of 6 -> 8 has weight 4 - 3 * (8 / 6) = 0 exactly when the
    product rounds first, so a zero sample next to 65535 stays 0.0 (fused, it would be 65535 * 2.2e-16)."""
    s, f = io.area_weights(8, 6)
    assert s[3] == 2 and f[3] == 0
    d = np.zeros((6, 6), np.uint16)
    d[:, 3] = 65535
    got = io.invdepth(d, 8, 8)
    assert bits_equal(got, cv2.resize(d.astype(np.float32), (8, 8), interpolation=cv2.INTER_AREA))
    assert np.all(got[:, 3].view(np.uint32) == 0)


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


def test_scratch_bytes_boundary():
    """The deepest tree the library builds has 16 levels: 2^16 leaves of 128 values is the largest frame it takes,
    one more pixel is refused; 3840 x 2160 needs all 16.  The split at half the length rounded down to a multiple of
    8 leaves the right half up to 7 longer, so some smaller frames need a 17th level too: the library refuses
    exactly those the recursion says it must."""
    from localrf_b200 import _lib
    L = _lib.lib()
    top = 128 << 16
    assert io.tree_depth(top) == 16 and io.tree_depth(top + 1) == 17 and io.tree_depth(3840 * 2160) == 16
    assert L.lrf_ingest_scratch_bytes(top) == (16 + 4 * top + 5 * (1 << 16) + top + 7) // 8 * 8
    for n in (top + 1, top + 8, 2 * top, 1 << 40):
        assert io.tree_depth(n) > 16 and L.lrf_ingest_scratch_bytes(n) == 0, n
    assert io.tree_depth(7864328) == 16 and io.tree_depth(7864329) == 17       # the smallest frame refused
    for n in list(range(top - 70, top)) + [3840 * 2160, 3840 * 2160 + 1, 4096 * 2048 - 1, 2896 * 2896, 7864328,
                                           7864329]:
        D = io.tree_depth(n)
        want = (16 + 4 * n + 5 * (1 << D) + n + 7) // 8 * 8 if D <= 16 else 0
        assert L.lrf_ingest_scratch_bytes(n) == want, (n, D)


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
