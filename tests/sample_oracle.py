"""Host restatement of the training-ray sampler (LocalRFDataset.sample, dataLoader/localrf_dataset.py:273-315) and
a stand-in dataset that replays the reference's frame bookkeeping over stored frames.

`sample(ds, ...)` draws from the global `random` / `np.random` in the reference's order and gathers with numpy;
`FrameDataset` keeps `all_*` arrays the way the reference does -- chunked loading appended to the arrays,
`deactivate_frames` slicing the leading frames off -- so `sample` and localrf_b200.DeviceRaySampler read the same
state a real LocalRFDataset would have.  `replay` runs a golden op script against either.
"""
import json
import random

import numpy as np

QUANTITIES = (("all_rgbs", "rgbs", 3), ("all_loss_weights", "loss_weights", 1), ("all_invdepths", "invdepths", 1),
              ("all_fwd_flow", "fwd_flow", 2), ("all_fwd_mask", "fwd_mask", 1), ("all_bwd_flow", "bwd_flow", 2),
              ("all_bwd_mask", "bwd_mask", 1))
BLOB_ARRAYS = tuple(k for _, k, _ in QUANTITIES) + ("idx", "view_ids")


class FrameDataset:
    """`frames[key]` [n_frames, n_px, w] (key as in a blob), loaded `frames_chunk` at a time, as read_meta does."""

    def __init__(self, frames, test_mask, load_depth, load_flow, frames_chunk, n_init_frames):
        self.frames = frames
        self.n_px_per_frame = int(frames["rgbs"].shape[1])
        self.num_images = int(frames["rgbs"].shape[0])
        self.test_mask = np.asarray(test_mask)
        self.load_depth, self.load_flow = bool(load_depth), bool(load_flow)
        self.frames_chunk = max(frames_chunk, n_init_frames)
        for attr, _, _ in QUANTITIES:
            setattr(self, attr, None)
        self.active_frames_bounds = [0, 0]
        self.loaded_frames = 0
        self.activate_frames(n_init_frames)

    def _has(self, key):
        return key in ("rgbs", "loss_weights") or (key == "invdepths" and self.load_depth) or \
            (key not in ("rgbs", "loss_weights", "invdepths") and self.load_flow)

    def activate_frames(self, n_frames=1):
        b = self.active_frames_bounds
        b[1] = min(b[1] + n_frames, self.num_images)
        if b[1] > self.loaded_frames:
            n = min(self.frames_chunk, self.num_images - self.loaded_frames)
            lo = self.loaded_frames
            self.loaded_frames += n
            for attr, key, w in QUANTITIES:
                if self._has(key):
                    new = self.frames[key][lo:lo + n].reshape(-1, w)
                    old = getattr(self, attr)
                    setattr(self, attr, new if old is None else np.concatenate([old, new], 0))

    def deactivate_frames(self, first_frame):
        n = first_frame - self.active_frames_bounds[0]
        self.active_frames_bounds[0] = first_frame
        for attr, key, _ in QUANTITIES:
            if self._has(key):
                setattr(self, attr, getattr(self, attr)[n * self.n_px_per_frame:])


def sample(ds, batch_size, is_refining, optimize_poses, n_views=16):
    """The reference's blob from `ds`: the same four draws (a coin for the test-pose set when optimising poses, the
    views, the forced newest views when not refining, the pixels), then rows (frame - b0) * n_px + pixel."""
    b0, b1 = ds.active_frames_bounds
    tm = ds.test_mask[b0:b1]
    use_test = bool(optimize_poses) and tm.mean() > random.uniform(0, 1)
    pool = np.arange(b0, b1, dtype=np.int64)[tm == (1 if use_test else 0)]
    raw = np.random.randint(0, int(pool.shape[0]), n_views, dtype=np.int64)
    k = pool.shape[0]
    if not is_refining and k > 4:
        raw[0:6] = [k - 1, k - 1, k - 2, k - 2, k - 3, k - 4]
    view_ids = pool[raw]
    px = np.random.randint(0, ds.n_px_per_frame, batch_size, dtype=np.int64)
    idx = (px.reshape(n_views, -1) + view_ids[:, None] * ds.n_px_per_frame).reshape(-1)
    rows = idx - b0 * ds.n_px_per_frame
    blob = {key: (getattr(ds, attr)[rows] if ds._has(key) else None) for attr, key, _ in QUANTITIES}
    blob.update(idx=idx, view_ids=view_ids, train_test_poses=use_test)
    return blob


def replay(ds, ops, sample_fn):
    """Runs a golden op script: ["seed", s] seeds random and np.random; ["activate", n]; ["deactivate", first];
    ["sample", batch_size, is_refining, optimize_poses, n_views] -> sample_fn(...).  Yields each sample's blob."""
    for op in ops:
        if op[0] == "seed":
            random.seed(op[1])
            np.random.seed(op[1])
        elif op[0] == "activate":
            ds.activate_frames(op[1])
        elif op[0] == "deactivate":
            ds.deactivate_frames(op[1])
        else:
            yield sample_fn(*op[1:])


def golden_case(z, name):
    """(FrameDataset, ops, list of blobs) of one case of tests/golden/ray_sample.npz."""
    cfg = json.loads(str(z[f"{name}.config"]))
    frames = {key: z[f"{name}.frames.{key}"] for _, key, _ in QUANTITIES if f"{name}.frames.{key}" in z}
    ds = FrameDataset(frames, z[f"{name}.test_mask"], cfg["load_depth"], cfg["load_flow"], cfg["frames_chunk"],
                      cfg["n_init_frames"])
    blobs = []
    for i in range(cfg["n_samples"]):
        b = {k: z[f"{name}.{i}.{k}"] if f"{name}.{i}.{k}" in z else None for k in BLOB_ARRAYS}
        b["train_test_poses"] = bool(z[f"{name}.{i}.train_test_poses"])
        blobs.append(b)
    return ds, cfg["ops"], blobs
