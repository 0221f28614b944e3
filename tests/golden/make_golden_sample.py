"""Generate tests/golden/ray_sample.npz: training-ray blobs of the UNMODIFIED reference's LocalRFDataset.sample
(dataLoader/localrf_dataset.py:273-315) over a tiny synthetic scene, loaded by its own read_meta.

Run in the build container only (needs the reference, cv2 and joblib, see oracle/ref_loader.py):

    python tests/golden/make_golden_sample.py

The scene: 14 frames of 48 x 32 (images, 16-bit inverse-depth PNGs, masks/all.png, flow_ds/fwd_* / bwd_* written
with the reference's encode_flow), test frames every 4.  Case "flow_depth" loads depth and flow, case "rgb_only"
neither; both use frames_chunk = 6 and n_init_frames = 5, so frames arrive in several chunks and both inclusion
sets are non-empty.  Each case stores every frame's arrays as the dataset loaded them, its op script (seeds,
activate / deactivate, and samples for all four (is_refining, optimize_poses) pairs with inclusion counts both
<= 4 and > 4) and every blob.
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

META = "reference facebookresearch/localrf @ 3905e39, LocalRFDataset.sample; synthetic 14 x 48 x 32 scene"
W, H, N_FRAMES = 48, 32, 14
KEYS = (("all_rgbs", "rgbs", 3), ("all_loss_weights", "loss_weights", 1), ("all_invdepths", "invdepths", 1),
        ("all_fwd_flow", "fwd_flow", 2), ("all_fwd_mask", "fwd_mask", 1), ("all_bwd_flow", "bwd_flow", 2),
        ("all_bwd_mask", "bwd_mask", 1))

S = lambda bs, ref, opt, v=16: ["sample", bs, ref, opt, v]   # noqa: E731
QUAD = lambda bs, v=16: [S(bs, False, True, v), S(bs, True, True, v), S(bs, False, False, v), S(bs, True, False, v)]  # noqa: E731
OPS = ([["seed", 7]] + QUAD(64)                        # [0,5): 3 train frames (<= 4), 2 test frames
       + [["activate", 3]] + QUAD(64) + QUAD(40, 8)     # [0,8): 6 train frames, second chunk loaded
       + [["deactivate", 3]] + QUAD(64)                 # [3,8): 4 train frames, 1 test frame
       + [["seed", 11], ["activate", 4]] + QUAD(96)     # [3,12): 7 train frames, third chunk
       + [["deactivate", 6], ["activate", 2]] + QUAD(128, 16) + QUAD(48, 6))   # [6,14)


def write_scene(d):
    rng = np.random.default_rng(0)
    for sub in ("images", "depth", "masks", "flow_ds"):
        os.makedirs(os.path.join(d, sub))
    for i in range(N_FRAMES):
        name = f"{i:05d}"
        cv2.imwrite(os.path.join(d, "images", name + ".png"), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        cv2.imwrite(os.path.join(d, "depth", name + ".png"), rng.integers(0, 65536, (H, W), dtype=np.uint16))
        for kind in ("fwd", "bwd"):
            flow = rng.normal(0.0, 4.0, (H, W, 2)).astype(np.float32)
            flow[0, :4] = 200.0                           # out of the encodable range: the mask drops them
            mask = rng.random((H, W)) > 0.2
            cv2.imwrite(os.path.join(d, "flow_ds", f"{kind}_{name}.png"), ref_utils.encode_flow(flow, mask))
    motion = np.full((H, W), 255, np.uint8)
    motion[:5, :7] = 0
    cv2.imwrite(os.path.join(d, "masks", "all.png"), motion)


def run_case(d, name, load):
    import random
    ds = LocalRFDataset(d, split="train", load_depth=load, load_flow=load, frames_chunk=6, n_init_frames=5,
                        test_frame_every=4)
    n_px = ds.n_px_per_frame
    frames = {key: np.zeros((N_FRAMES, n_px, w), np.float32) for _, key, w in KEYS}
    seen = set()
    out, n = {}, 0

    def record():
        b0 = ds.active_frames_bounds[0]
        for f in range(b0, ds.loaded_frames):
            if f not in seen:
                seen.add(f)
                for attr, key, w in KEYS:
                    a = getattr(ds, attr)
                    if a is not None:
                        assert a.dtype == np.float32, (attr, a.dtype)
                        frames[key][f] = a[(f - b0) * n_px:(f - b0 + 1) * n_px].reshape(n_px, w)

    record()
    for op in OPS:
        if op[0] == "seed":
            random.seed(op[1])
            np.random.seed(op[1])
        elif op[0] == "activate":
            ds.activate_frames(op[1])
        elif op[0] == "deactivate":
            ds.deactivate_frames(op[1])
        else:
            blob = ds.sample(*op[1:])
            for k, v in blob.items():
                if v is not None:
                    out[f"{name}.{n}.{k}"] = np.asarray(v)
            n += 1
        record()
    assert len(seen) == N_FRAMES
    for _, key, _ in KEYS:
        if load or key in ("rgbs", "loss_weights"):
            out[f"{name}.frames.{key}"] = frames[key]
    out[f"{name}.test_mask"] = ds.test_mask
    out[f"{name}.config"] = np.array(json.dumps({"load_depth": load, "load_flow": load, "frames_chunk": 6,
                                                 "n_init_frames": 5, "n_samples": n, "ops": OPS}))
    print(name, n, "samples")
    return out


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        write_scene(d)
        out.update(run_case(d, "flow_depth", True))
        out.update(run_case(d, "rgb_only", False))
    path = os.path.join(HERE, "ray_sample.npz")
    np.savez_compressed(path, meta=np.array(META), names=np.array(["flow_depth", "rgb_only"]), **out)
    print(f"ray_sample: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
