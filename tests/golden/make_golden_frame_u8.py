"""Generate tests/golden/frame_u8.npz: the 8-bit frame outputs of the UNMODIFIED reference's renderer
(renderer.py:127,156,176) at the values where the conversions round or truncate.

Run in the build container only (needs the reference, see oracle/ref_loader.py):

    python tests/golden/make_golden_frame_u8.py

depth: visualize_depth(depth, [lo, hi], cmap) (utils/utils.py:179-197) with the bounds as Python numbers, as
renderer.py:127 passes [0, 5], then renderer.py:156's byte chain (`* 255`, `.byte()`).  The colour map is a
user LUT whose first channel is the LUT index, so a stored byte names the index the reference picked.  Values:
for every index k, the float32 neighbours of the depth where 255 * x crosses k, NaN, +-inf, +-float32 max, the
bounds themselves, depths beyond them and uniform ones.  Entries: `ranges` [R,2], `depth.{i}` float32 [M],
`depth8.{i}` uint8 [M,3].

rgb: cv2.imencode('.png', 255 * rgb[..., ::-1]) (what cv2.imwrite stores, renderer.py:176), decoded.  Values:
k/255 and its float32 neighbours, every float32 v with 255 * v exactly k + 0.5 (ties to even), negatives,
values above 1, NaN and -inf -- all with |255 v| < 2^31, where OpenCV's conversion does not depend on the
platform.  Entries: `rgb` float32 [N,3], `rgb8` uint8 [N,3] BGR.

Recorded environment: the `meta` entry.
"""
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
import utils.utils as ref_utils  # noqa: E402  (the reference's module, top-level name after load_reference)

META = (f"torch {torch.__version__} cpu; numpy {np.__version__}; opencv {cv2.__version__} x86-64; "
        "reference facebookresearch/localrf @ 3905e39")
# renderer.py:127 passes [0, 5]; the others make hi - lo + 1e-8 round differently in float32 and in double, and
# cover equal and inverted bounds
RANGES = [(0, 5), (0.1, 0.7), (0.3, 2.9), (0.2, 1.9), (1.1, 1.1), (2.0, 1.0)]


def index_lut():
    k = np.arange(256)
    return np.stack([k, (7 * k + 3) % 256, 255 - k], -1).astype(np.uint8)


def neighbours(v, n):
    """float32 v and its n float32 neighbours on each side."""
    out, lo, hi = [np.float32(v)], np.float32(v), np.float32(v)
    for _ in range(n):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return out


def depth_values(lo, hi, rng):
    den = hi - lo + 1e-8
    vals = []
    for k in range(1, 256):
        vals += neighbours(lo + k / 255 * den, 2)
    big = np.finfo(np.float32).max
    a, b = min(lo, hi), max(lo, hi)
    vals += [np.nan, -np.nan, np.inf, -np.inf, big, -big, 0.0, -0.0, lo, hi, a - 1, b + 1, a - 1e-3, b + 1e-3]
    vals += list(rng.uniform(a - 0.5, b + 0.5, 256))
    vals += list(np.array(KNOWN.get((lo, hi), []), np.uint32).view(np.float32))
    return np.array(vals, np.float32)


# depths (float32 bit patterns) where a float32 denominator picks another index than the reference
KNOWN = {(0.1, 0.7): [1053806543], (0.3, 2.9): [1077516697]}


def rgb_values(rng):
    vals = []
    for k in range(256):
        vals += neighbours(k / 255, 2)
        for v in neighbours((k + 0.5) / 255, 4):         # every float32 whose 255 * v is exactly k + 0.5
            if np.float32(255) * v == np.float32(k + 0.5):
                vals.append(v)
    vals += [-0.0, -1e-3, -0.5 / 255, -1.0, -100.0, 1.001, 1.5, 2.0, 100.0, 1e6, 8e6, np.nan, -np.nan, -np.inf]
    vals += list(rng.uniform(-0.1, 1.1, 300))
    v = np.array(vals, np.float32)
    v = np.concatenate([v, np.zeros((-len(v)) % 3, np.float32)])
    return v.reshape(-1, 3)


def main():
    rng = np.random.default_rng(23)
    lut = index_lut()
    out = {"lut": lut, "ranges": np.array(RANGES, np.float64)}
    for i, (lo, hi) in enumerate(RANGES):
        d = depth_values(lo, hi, rng)
        vis, _ = ref_utils.visualize_depth(d.reshape(1, -1), [lo, hi], lut[:, None, :])
        out[f"depth.{i}"] = d
        out[f"depth8.{i}"] = torch.permute(vis * 255, [1, 2, 0]).byte().numpy().reshape(-1, 3)   # renderer.py:156
    rgb = rgb_values(rng)
    ok, buf = cv2.imencode(".png", 255 * rgb[None][..., ::-1])                                   # renderer.py:176
    assert ok
    out["rgb"] = rgb
    out["rgb8"] = cv2.imdecode(buf, cv2.IMREAD_UNCHANGED).reshape(-1, 3)
    path = os.path.join(HERE, "frame_u8.npz")
    np.savez_compressed(path, meta=np.array(META), **out)
    print(f"frame_u8: {os.path.getsize(path) / 1e3:.1f} kB, {len(rgb)} rgb pixels, "
          f"{sum(len(out[f'depth.{i}']) for i in range(len(RANGES)))} depths")


if __name__ == "__main__":
    main()
