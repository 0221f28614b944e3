"""Training rays from device-resident frames: LocalRFDataset.sample (dataLoader/localrf_dataset.py:273-315) and the
uploads of train.py:352-356, with the supervision gather as one kernel (lrf_gather_rays).

    sampler = DeviceRaySampler(train_dataset, device)      # once, after the dataset is built
    blob = sampler.sample(batch_size, is_refining, optimize_poses, n_views=16)

The host draws the view and pixel ids with the reference's own RNG calls, so a seeded run consumes `random` and
`np.random` draw for draw like the reference and every blob is bit-identical to what LocalRFDataset.sample returns.
The active frames live in device memory; a call uploads its V + N ids (one pinned, non-blocking copy) and gathers
rgb, loss weight, inverse depth, flows and flow masks on the device.  There is no CPU fallback.
"""
import ctypes as C
import random

import numpy as np
import torch

from . import _lib
from .tensorf import _ptr, _stream

# (dataset attribute, blob key, values per pixel); the order is the layout of a frame's staging buffer
_QUANTITIES = (("all_rgbs", "rgbs", 3), ("all_loss_weights", "loss_weights", 1), ("all_invdepths", "invdepths", 1),
               ("all_fwd_flow", "fwd_flow", 2), ("all_fwd_mask", "fwd_mask", 1), ("all_bwd_flow", "bwd_flow", 2),
               ("all_bwd_mask", "bwd_mask", 1))
_STORE_FIELDS = {"rgbs": "rgb", "loss_weights": "loss_weight", "invdepths": "invdepth", "fwd_flow": "fwd_flow",
                 "fwd_mask": "fwd_mask", "bwd_flow": "bwd_flow", "bwd_mask": "bwd_mask"}


class DeviceRaySampler:
    """LocalRFDataset.sample with the active frames resident on `device`.

    Reads only the dataset's state -- active_frames_bounds, test_mask, n_px_per_frame, load_depth, load_flow and
    the all_* arrays -- and never calls its sample().  On each call the resident frames follow active_frames_bounds:
    new frames are uploaded (each through a fresh pinned buffer of torch's caching host allocator, which is not
    reused before its copy has finished), frames below the first active one are forgotten.  Frame f lives in slot
    f % capacity of a ring of frame slots.  The ring grows, to max(span, 2 * capacity) slots with a device copy of
    the resident frames, only when the active span exceeds it; it never shrinks.  `capacity` sets the initial
    number of slots (at least the active span); pass train.py's n_max_frames to allocate once.

    Memory: 4 * (3 + 1 + 1 + 2 + 1 + 2 + 1) = 44 bytes per pixel with depth and flow on -- 22.8 MB per 960x540
    frame, 28.2 MB per 800x800 frame, 2.3-2.8 GB for 100 slots.  The reference holds the same data on the host.
    """

    def __init__(self, dataset, device, capacity=None):
        self.ds = dataset
        self.dev = torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("localrf_b200.DeviceRaySampler keeps the frames on a CUDA device (there is no CPU "
                               "fallback)")
        self.n_px = int(dataset.n_px_per_frame)
        self.quantities = [(attr, key, w) for attr, key, w in _QUANTITIES
                           if key in ("rgbs", "loss_weights") or (key == "invdepths" and dataset.load_depth)
                           or (key not in ("rgbs", "loss_weights", "invdepths") and dataset.load_flow)]
        self.floats_per_px = sum(w for _, _, w in self.quantities)
        b0, b1 = dataset.active_frames_bounds
        self.capacity = 0
        self.resident = (b0, b0)                       # frames [r0, r1) are on the device
        self.store = {}
        self._grow(max(b1 - b0, int(capacity or 0), 1))

    def _grow(self, capacity):
        """Reallocates the ring with `capacity` slots and copies the resident frames into their new slots."""
        old, old_cap = self.store, self.capacity
        with torch.cuda.device(self.dev):
            store = {key: torch.empty((capacity, self.n_px, w) if w > 1 else (capacity, self.n_px),
                                      dtype=torch.float32, device=self.dev) for _, key, w in self.quantities}
            store["slot_frame"] = torch.full((capacity,), -1, dtype=torch.int64, device=self.dev)
            for f in range(*self.resident):
                for _, key, _ in self.quantities:
                    store[key][f % capacity].copy_(old[key][f % old_cap])
                store["slot_frame"][f % capacity].fill_(f)
        self.store, self.capacity = store, capacity
        s = _lib.LrfFrameStore()
        s.n_px, s.capacity = self.n_px, capacity
        for key, t in store.items():
            setattr(s, _STORE_FIELDS.get(key, key), _ptr(t).value)
        self._cstore = s

    def _upload(self, f, b0):
        """Enqueues frame f (rows (f - b0) * n_px of the dataset's arrays) into its slot."""
        stage = torch.empty(self.n_px * self.floats_per_px, dtype=torch.float32, pin_memory=True)
        host = stage.numpy()
        rows = slice((f - b0) * self.n_px, (f - b0 + 1) * self.n_px)
        off, parts = 0, []
        for attr, key, w in self.quantities:
            n = self.n_px * w
            host[off:off + n] = getattr(self.ds, attr)[rows].reshape(-1)
            parts.append((key, off, n))
            off += n
        slot = f % self.capacity
        for key, o, n in parts:
            dst = self.store[key][slot]
            dst.copy_(stage[o:o + n].view(dst.shape), non_blocking=True)
        self.store["slot_frame"][slot].fill_(f)

    def _sync_frames(self):
        b0, b1 = (int(b) for b in self.ds.active_frames_bounds)
        r0, r1 = self.resident
        r0, r1 = max(r0, b0), min(max(r1, b0), b1)   # forget frames below b0 (bookkeeping only)
        if r1 <= r0:
            r0 = r1 = b0
        self.resident = (r0, r1)
        if b1 - b0 > self.capacity:
            self._grow(max(b1 - b0, 2 * self.capacity))
        with torch.cuda.device(self.dev):
            for f in range(r1, b1):
                self._upload(f, b0)
        self.resident = (r0, b1) if b1 > r1 else (r0, r1)

    def sample(self, batch_size, is_refining, optimize_poses, n_views=16):
        """-> the blob of LocalRFDataset.sample with device tensors: rgbs [N,3], loss_weights [N,1], invdepths
        [N,1] (or None), fwd_flow [N,2], fwd_mask [N,1], bwd_flow [N,2], bwd_mask [N,1] (or None), fp32, each
        contiguous and carved from one allocation; idx int64 [N]; view_ids int64 [V]; train_test_poses as the
        reference computes it; and view_ids_host, the numpy array the reference returns as view_ids (pass it to
        LocalTensorfs.forward, which reads the view ids on the host).

        Raises ValueError where the reference does: an empty inclusion set, or batch_size % n_views != 0.  The
        second check runs before any draw; the reference raises it only after drawing the views and pixels."""
        if n_views < 1 or batch_size % n_views != 0:
            raise ValueError(f"batch_size {batch_size} does not split into {n_views} views of equal size")
        ds = self.ds
        b0, b1 = (int(b) for b in ds.active_frames_bounds)
        active_test_mask = ds.test_mask[b0:b1]
        with np.errstate(invalid="ignore", divide="ignore"):
            test_ratio = active_test_mask.mean() if len(active_test_mask) else np.float64(np.nan)
        train_test_poses = test_ratio > random.uniform(0, 1) if optimize_poses else False
        inclusion_mask = active_test_mask if train_test_poses else 1 - active_test_mask
        frames = np.arange(b0, b1, dtype=np.int64)[inclusion_mask == 1]
        n_incl = len(frames)
        if n_incl == 0:
            raise ValueError("no frame of the active range is in the inclusion set (high <= 0)")
        raw = np.random.randint(0, n_incl, n_views, dtype=np.int64)
        if not is_refining and n_incl > 4:             # the newest views, as the reference forces them
            raw[:2] = n_incl - 1
            raw[2:4] = n_incl - 2
            raw[4] = n_incl - 3
            raw[5] = n_incl - 4
        view_ids = frames[raw]
        px = np.random.randint(0, self.n_px, batch_size, dtype=np.int64)

        self._sync_frames()
        N, V, dev = batch_size, n_views, self.dev
        ids_host = torch.empty(V + N, dtype=torch.int64, pin_memory=True)
        h = ids_host.numpy()
        h[:V] = view_ids
        h[V:] = px
        with torch.cuda.device(dev):
            ids = torch.empty(V + N, dtype=torch.int64, device=dev)
            ids.copy_(ids_host, non_blocking=True)
            idx = torch.empty(N, dtype=torch.int64, device=dev)
            out = torch.empty(N * self.floats_per_px, dtype=torch.float32, device=dev)
            g = _lib.LrfRayGather()
            g.n_rays, g.n_views, g.ids, g.idx = N, V, _ptr(ids).value, _ptr(idx).value
            blob = {"rgbs": None, "loss_weights": None, "invdepths": None, "fwd_flow": None, "fwd_mask": None,
                    "bwd_flow": None, "bwd_mask": None}
            off = 0
            for _, key, w in self.quantities:
                blob[key] = out[off:off + N * w].view(N, w)
                setattr(g, _STORE_FIELDS[key], _ptr(blob[key]).value)
                off += N * w
            _lib.check(_lib.lib().lrf_gather_rays(C.byref(self._cstore), C.byref(g), _stream(dev)))
        blob.update(idx=idx, view_ids=ids[:V], train_test_poses=train_test_poses, view_ids_host=view_ids)
        return blob
