"""Generate tests/golden/ingest.npz: the per-frame arrays the UNMODIFIED reference's LocalRFDataset.read_meta
(dataLoader/localrf_dataset.py:143-258) builds from two tiny synthetic scenes, with the scenes' files themselves.

Run in the build container only (needs the reference, cv2 and joblib, see oracle/ref_loader.py):

    python tests/golden/make_golden_ingest.py

Scene "half": 7 frames, 40 x 30 jpg images, 16-bit inverse-depth PNGs at the image size, flows written with the
reference's encode_flow at 20 x 15 (as scripts/run_flow.py writes them, --scale 0.5), motion masks for frames 1
and 4 only.  Scene "down2": 80 x 60 jpg images loaded with downsampling = 2, depth at 80 x 60 (a 2x reduction),
flows at 20 x 15 (a 2x enlargement), masks/all.png at 40 x 30 for every frame.  Cases: "half" with flow and depth,
"half_rgb" with neither, "down2" with both; frames_chunk = 4, n_init_frames = 3, test frames every 3.  The files
are stored byte for byte (key "file:<scene>/<path>") so a test rebuilds the exact scene.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
import cv2  # noqa: E402
import utils.utils as ref_utils  # noqa: E402  (the reference's module, top-level name after load_reference)
from dataLoader.localrf_dataset import LocalRFDataset  # noqa: E402

META = "reference facebookresearch/localrf @ 3905e39, LocalRFDataset.read_meta; synthetic 7-frame scenes"
N_FRAMES = 7
KEYS = (("all_rgbs", "rgbs", 3), ("all_loss_weights", "loss_weights", 1), ("all_invdepths", "invdepths", 1),
        ("all_fwd_flow", "fwd_flow", 2), ("all_fwd_mask", "fwd_mask", 1), ("all_bwd_flow", "bwd_flow", 2),
        ("all_bwd_mask", "bwd_mask", 1))
CASES = {"half": ("half", -1, True), "half_rgb": ("half", -1, False), "down2": ("down2", 2, True)}


def smooth(rng, h, w, c):
    """Smooth noise (so the jpgs stay small) with some sharp pixels (so the Laplacian varies)."""
    base = rng.random((h // 5 + 2, w // 5 + 2, c)) * 255
    img = cv2.resize(base, (w, h), interpolation=cv2.INTER_CUBIC)
    img += rng.normal(0, 12, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8).reshape(h, w, c)


def write_scene(d, name):
    rng = np.random.default_rng(0 if name == "half" else 1)
    W, H = (40, 30) if name == "half" else (80, 60)
    for sub in ("images", "depth", "masks", "flow_ds"):
        os.makedirs(os.path.join(d, sub))
    for i in range(N_FRAMES):
        f = f"{i:05d}"
        cv2.imwrite(os.path.join(d, "images", f + ".jpg"), smooth(rng, H, W, 3), [cv2.IMWRITE_JPEG_QUALITY, 90])
        cv2.imwrite(os.path.join(d, "depth", f + ".png"), rng.integers(0, 65536, (H, W), dtype=np.uint16))
        for kind in ("fwd", "bwd"):
            flow = rng.normal(0.0, 3.0, (15, 20, 2)).astype(np.float32)
            flow[0, :3] = 200.0                           # out of the encodable range: the mask drops them
            mask = rng.random((15, 20)) > 0.2
            cv2.imwrite(os.path.join(d, "flow_ds", f"{kind}_{f}.png"), ref_utils.encode_flow(flow, mask))
        if name == "half" and i in (1, 4):
            m = (rng.random((30, 40)) > 0.3).astype(np.uint8) * 255
            cv2.imwrite(os.path.join(d, "masks", f + ".png"), m)
    if name == "down2":
        m = np.full((30, 40), 255, np.uint8)
        m[:6, :9] = 0
        cv2.imwrite(os.path.join(d, "masks", "all.png"), m)


def run_case(d, case):
    _, ds_factor, load = CASES[case]
    ds = LocalRFDataset(d, split="train", downsampling=ds_factor, load_depth=load, load_flow=load, frames_chunk=4,
                        n_init_frames=3, test_frame_every=3)
    while ds.has_left_frames():
        ds.activate_frames(1)
    n_px = ds.n_px_per_frame
    out = {}
    for attr, key, w in KEYS:
        a = getattr(ds, attr)
        if a is not None:
            assert a.dtype == np.float32, (attr, a.dtype)
            out[f"{case}.frames.{key}"] = a.reshape(N_FRAMES, n_px, w)
    out[f"{case}.test_mask"] = ds.test_mask
    out[f"{case}.config"] = np.array(json.dumps({"downsampling": ds_factor, "load_depth": load, "load_flow": load,
                                                 "frames_chunk": 4, "n_init_frames": 3, "test_frame_every": 3,
                                                 "img_wh": list(ds.img_wh)}))
    return out


def main():
    out = {}
    with tempfile.TemporaryDirectory() as root:
        for scene in ("half", "down2"):
            d = os.path.join(root, scene)
            write_scene(d, scene)
            for dirpath, _, files in os.walk(d):
                for fn in files:
                    p = os.path.join(dirpath, fn)
                    out[f"file:{scene}/{os.path.relpath(p, d)}"] = np.frombuffer(open(p, "rb").read(), np.uint8)
        for case, (scene, _, _) in CASES.items():
            out.update(run_case(os.path.join(root, scene), case))
    path = os.path.join(HERE, "ingest.npz")
    np.savez_compressed(path, meta=np.array(META), cases=np.array(list(CASES)),
                        scenes=np.array([CASES[c][0] for c in CASES]), **out)
    print(f"ingest: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
