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
    the all_* arrays -- and never calls its sample().  A train-split DeviceFrameDataset has no all_* arrays: it
    converts each new frame into its slot on the device (lrf_ingest_frame), with the same result.  On each call the resident frames follow active_frames_bounds:
    new frames are uploaded (each through a fresh pinned buffer of torch's caching host allocator, which is not
    reused before its copy has finished), frames below the first active one are forgotten.  Frame f lives in slot
    f % capacity of a ring of frame slots.  The ring grows, to max(span, 2 * capacity) slots with a device copy of
    the resident frames, only when the active span exceeds it; it never shrinks.  `capacity` sets the initial
    number of slots (at least the active span); pass train.py's n_max_frames to allocate once.

    Memory: 4 * (3 + 1 + 1 + 2 + 1 + 2 + 1) = 44 bytes per pixel with depth and flow on -- 22.8 MB per 960x540
    frame, 28.2 MB per 800x800 frame, 2.3-2.8 GB for 100 slots.  The reference holds the same data on the host.
    The test split (DeviceFrameDataset(split="test"), which this sampler refuses with ValueError, as the reference
    never samples it) holds every test frame the same way without the loss weight: 40 bytes per pixel.
    """

    def __init__(self, dataset, device, capacity=None):
        if isinstance(dataset, DeviceFrameDataset) and dataset.split != "train":
            raise ValueError(f"DeviceRaySampler draws from the train split, not the {dataset.split} split (the "
                             "reference never samples the test split)")
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
        """Enqueues frame f (rows (f - b0) * n_px of the dataset's arrays) into its slot; a DeviceFrameDataset
        converts the frame's raw pixels into the slot instead."""
        slot = f % self.capacity
        if isinstance(self.ds, DeviceFrameDataset):
            self.ds.ingest_frame(f, self._cstore, slot, self.dev)
            self.store["slot_frame"][slot].fill_(f)
            return
        stage = torch.empty(self.n_px * self.floats_per_px, dtype=torch.float32, pin_memory=True)
        host = stage.numpy()
        rows = slice((f - b0) * self.n_px, (f - b0 + 1) * self.n_px)
        off, parts = 0, []
        for attr, key, w in self.quantities:
            n = self.n_px * w
            host[off:off + n] = getattr(self.ds, attr)[rows].reshape(-1)
            parts.append((key, off, n))
            off += n
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


class DeviceFrameDataset:
    """LocalRFDataset (dataLoader/localrf_dataset.py), train or test split, with its frames converted on the device.

    Same constructor and the same state train.py reads -- img_wh, num_images, active_frames_bounds, test_mask,
    n_px_per_frame, load_depth / load_flow, activate_frames, deactivate_frames, has_left_frames, get_frame_fbase,
    all_fbases, all_image_paths, and with preprocessed poses transforms, first_pose, rel_poses, pose_scale.  Frames are
    read `frames_chunk` at a time from the same files, with the same fallbacks (masks/all.png, the frame_step flow
    names) and joblib threads, as read_meta reads them; but only the decoded 8-bit image, 16-bit inverse depth,
    16-bit encoded flows and 8-bit motion mask are kept, in pinned host memory, until a DeviceRaySampler places the
    frame in its ring: then they are uploaded (with flow and depth 8 bytes per output pixel when the flows are at
    half size, 17 when they are at the image size, against the 44 bytes per pixel of float32 the reference builds
    and keeps) and lrf_ingest_frame writes the slot, bit-identical to the
    arrays read_meta builds.  The host keeps no float copy of any frame, and a frame's raw bytes are dropped once its
    upload is enqueued.  There is no `sample`: draw batches with DeviceRaySampler(dataset, device).

    split="test" is the reference's test split: the frames with index % test_frame_every == 0, all read and
    converted at construction on `device` (the current CUDA device by default; the train split's frames go to its
    sampler's device instead) into the stacked float32 CUDA tensors the reference builds with np.stack: all_rgbs
    [N,h,w,3], all_invdepths [N,h,w] (load_depth), all_fwd_flow / all_bwd_flow [N,h,w,2] and all_fwd_mask /
    all_bwd_mask [N,h,w] (load_flow), None where the reference's are; all_loss_weights is None, as there.  Each
    frame's decoded planes go through lrf_ingest_frame exactly as a train frame's do, so its arrays are
    bit-identical to read_meta's, and are dropped once its upload is enqueued; the loss weight, which the reference
    computes and discards, is written to one shared scratch plane that is freed with the ingest scratch after
    construction.  img_wh, n_px_per_frame, num_images, all_fbases, get_frame_fbase and test_mask (over every frame,
    as in the reference) are there; active_frames_bounds = [0, min(n_init_frames, N)], loaded_frames = N and
    has_left_frames() keep the reference's values.  A DeviceRaySampler refuses this split.  Device memory: 4 * (3 +
    1 + 2 + 1 + 2 + 1) = 40 bytes per pixel and test frame with flow and depth (12 with neither), 20.7 MB per
    960x540 frame, 2.07 GB for 100 such frames; during construction 4 bytes per pixel more, once, plus
    lrf_ingest_scratch_bytes.  The host keeps no float copy (the reference keeps the same 40 B/px in numpy arrays).

    Supported layouts (anything else raises NotImplementedError; such datasets keep using LocalRFDataset): the
    image at its size or reduced by downsampling = 2 or 4 when both sides divide; inverse depth at the image size, a
    reduction of it by 2 or 4, or smaller; flows at the image size or smaller on both axes (scripts/run_flow.py
    writes them at half size), both flows of one frame the same size; motion masks at the image size.
    """

    def __init__(self, datadir, split="train", frames_chunk=20, downsampling=-1, load_depth=False, load_flow=False,
                 with_preprocessed_poses=False, n_init_frames=7, subsequence=[0, -1], test_frame_every=10,
                 frame_step=1, device=None):
        import json
        import os
        if split not in ("train", "test"):
            raise ValueError(f"DeviceFrameDataset is the train or the test split, got split={split!r}")
        self.root_dir, self.split = datadir, split
        self.frames_chunk = max(frames_chunk, n_init_frames)
        self.downsampling = downsampling
        self.load_depth, self.load_flow = load_depth, load_flow
        self.frame_step = frame_step
        if with_preprocessed_poses:
            with open(os.path.join(datadir, "transforms.json"), "r") as fh:
                self.transforms = json.load(fh)
            by_name = {os.path.basename(m["file_path"]): m["transform_matrix"] for m in self.transforms["frames"]}
            paths = sorted(by_name)
            poses = [np.array(by_name[p], dtype=np.float32) for p in paths]
            self.first_pose = np.array(by_name[paths[0]], dtype=np.float32)
            rel = np.stack([np.eye(4, dtype=np.float32)] +
                           [np.linalg.inv(poses[i - 1]) @ poses[i] for i in range(1, len(poses))], axis=0)
            self.pose_scale = 2e-2 / np.median(np.linalg.norm(rel[:, :3, 3], axis=-1))
            rel[:, :3, 3] *= self.pose_scale
            self.rel_poses = rel[::frame_step]
        else:
            paths = sorted(os.listdir(os.path.join(datadir, "images")))
        if subsequence != [0, -1]:
            paths = paths[subsequence[0]:subsequence[1]]
        self.image_paths = self.all_image_paths = paths[::frame_step]
        test = []
        for i, p in enumerate(self.image_paths):
            fbase = os.path.splitext(p)[0]
            index = int(fbase) if fbase.isnumeric() else i
            test.append(1 if test_frame_every > 0 and index % test_frame_every == 0 else 0)
        self.test_mask = np.array(test)
        if split == "test":
            self.image_paths = [p for p, t in zip(self.image_paths, test) if t]
            self.frames_chunk = len(self.image_paths)
            dev = torch.device("cuda" if device is None else device)
            if dev.type != "cuda" or not torch.cuda.is_available():
                raise RuntimeError("DeviceFrameDataset keeps the test split on a CUDA device (there is no CPU "
                                   "fallback)")
            self.device = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
            self.all_rgbs = self.all_invdepths = self.all_loss_weights = None
            self.all_fwd_flow = self.all_fwd_mask = self.all_bwd_flow = self.all_bwd_mask = None
        self.num_images = len(self.image_paths)
        self.all_fbases = {os.path.splitext(p)[0]: i for i, p in enumerate(self.image_paths)}
        self.white_bg = False
        self.near_far = [0.1, 1e3]
        self.scene_bbox = 2 * torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
        self._raw = {}                                 # frame -> its decoded planes (pinned), until ingested
        self._scratch = {}                             # device -> scratch of lrf_ingest_frame
        self.active_frames_bounds = [0, 0]
        self.loaded_frames = 0
        self.activate_frames(n_init_frames)

    def activate_frames(self, n_frames=1):
        b = self.active_frames_bounds
        b[1] = min(b[1] + n_frames, self.num_images)
        if b[1] > self.loaded_frames:
            self._read_chunk()

    def has_left_frames(self):
        return self.active_frames_bounds[1] < self.num_images

    def deactivate_frames(self, first_frame):
        self.active_frames_bounds[0] = first_frame
        for f in [f for f in self._raw if f < first_frame]:
            del self._raw[f]

    def get_frame_fbase(self, view_id):
        return list(self.all_fbases.keys())[view_id]

    def _paths(self, i):
        import os
        name = self.image_paths[i]
        base = os.path.splitext(name)[0]
        mask = os.path.join(self.root_dir, "masks", f"{base}.png")
        if not os.path.isfile(mask):
            mask = os.path.join(self.root_dir, "masks/all.png")
        out = {"image": os.path.join(self.root_dir, "images", name), "mask": mask,
               "invdepth": os.path.join(self.root_dir, "depth", f"{base}.png")}
        g = self.all_image_paths.index(name)
        nxt = os.path.splitext(self.all_image_paths[g + 1 if g + 1 < len(self.all_image_paths) else 0])[0]
        step = f"step{self.frame_step}_" if self.frame_step != 1 else ""
        out["fwd_flow"] = os.path.join(self.root_dir, "flow_ds", f"fwd_{step}{nxt}.png")
        out["bwd_flow"] = os.path.join(self.root_dir, "flow_ds", f"bwd_{step}{base}.png")
        return out

    def _read(self, i):
        """The decoded planes of frame i, each in a pinned buffer: image uint8 [h0][w0][3] BGR, invdepth uint16,
        flows uint16 [hf][wf][3] as stored, mask uint8 (or None)."""
        import os
        import cv2
        p = self._paths(i)
        planes = {"image": cv2.imread(p["image"])}
        if self.load_depth:
            d = cv2.imread(p["invdepth"], -1)
            if d.ndim != 2 or d.dtype not in (np.uint8, np.uint16):
                raise NotImplementedError(f"{p['invdepth']}: inverse depth must be an 8- or 16-bit single-channel "
                                          "image")
            planes["invdepth"] = d.astype(np.uint16)
        if self.load_flow:
            for key in ("fwd_flow", "bwd_flow"):
                e = cv2.imread(p[key], cv2.IMREAD_UNCHANGED)
                if e.ndim != 3 or e.shape[2] != 3 or e.dtype != np.uint16:
                    raise NotImplementedError(f"{p[key]}: encoded flow must be a 16-bit 3-channel image")
                planes[key] = e
        if os.path.isfile(p["mask"]):
            m = cv2.imread(p["mask"], cv2.IMREAD_UNCHANGED)
            if m.ndim != 2:
                m = m[..., 0]
            planes["mask"] = m if m.dtype == np.uint8 else (m > 0).astype(np.uint8)
        pinned = {}
        for key, a in planes.items():
            t = torch.empty(a.shape, dtype=torch.uint8 if a.dtype == np.uint8 else torch.int16, pin_memory=True)
            t.numpy().view(a.dtype)[...] = a
            pinned[key] = t
        return pinned

    def _layout(self, raw):
        """-> (w, h) of the frame after downsampling; raises NotImplementedError for an unsupported layout."""
        h0, w0 = raw["image"].shape[:2]
        k = 1 if self.downsampling == -1 else self.downsampling
        if k not in (1, 2, 4) or w0 % k or h0 % k:
            raise NotImplementedError(f"downsampling={self.downsampling} of a {w0}x{h0} image: only 2 and 4 of "
                                      "sides they divide are converted on the device")
        return w0 // int(k), h0 // int(k)

    def _read_chunk(self):
        from joblib import Parallel, delayed
        n = min(self.frames_chunk, self.num_images - self.loaded_frames)
        lo = self.loaded_frames
        frames = Parallel(n_jobs=-1, backend="threading")(delayed(self._read)(i) for i in range(lo, lo + n))
        self.loaded_frames += n
        w, h = self._layout(frames[0])
        for raw in frames:
            if self._layout(raw) != (w, h):
                raise NotImplementedError("frames of one dataset must share their size")
        self.img_wh = [w, h]
        self.n_px_per_frame = w * h
        for i, raw in enumerate(frames):
            self._raw[lo + i] = raw
        if self.split == "test":
            self._ingest_test_split(lo, n)

    def _ingest_test_split(self, lo, n):
        """Converts frames [lo, lo + n) -- the whole test split, read at once -- into the stacked all_* tensors: each
        through lrf_ingest_frame into a one-slot store whose pointers are the frame's rows."""
        dev = self.device
        w, h = self.img_wh
        with torch.cuda.device(dev):
            new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
            self.all_rgbs = new(n, h, w, 3)
            if self.load_depth:
                self.all_invdepths = new(n, h, w)
            if self.load_flow:
                self.all_fwd_flow, self.all_fwd_mask = new(n, h, w, 2), new(n, h, w)
                self.all_bwd_flow, self.all_bwd_mask = new(n, h, w, 2), new(n, h, w)
            weight = new(w * h)                        # the loss weight, computed and discarded as in the reference
            slot_frame = torch.full((1,), -1, dtype=torch.int64, device=dev)
            for k in range(n):
                s = _lib.LrfFrameStore()
                s.n_px, s.capacity = w * h, 1
                s.slot_frame, s.loss_weight = _ptr(slot_frame).value, _ptr(weight).value
                for field, attr in (("rgb", "all_rgbs"), ("invdepth", "all_invdepths"), ("fwd_flow", "all_fwd_flow"),
                                    ("fwd_mask", "all_fwd_mask"), ("bwd_flow", "all_bwd_flow"),
                                    ("bwd_mask", "all_bwd_mask")):
                    t = getattr(self, attr)
                    setattr(s, field, _ptr(t[k]).value if t is not None else None)
                self.ingest_frame(lo + k, s, 0, dev)
            self._scratch.pop(dev, None)   # freed blocks are reused on this stream only, after the queued launches

    def ingest_frame(self, f, store, slot, device):
        """Uploads frame f's raw planes and enqueues lrf_ingest_frame into `slot` of `store` (an LrfFrameStore) on
        the current stream of `device`; drops the host planes (torch's caching host allocator keeps a pinned block
        from reuse until its copy has finished)."""
        raw = self._raw.pop(f, None)
        if raw is None:
            raise RuntimeError(f"frame {f} is not loaded or was already placed in a ring (a DeviceFrameDataset "
                               "hands each frame to one DeviceRaySampler)")
        dev = torch.device(device)
        w, h = self.img_wh
        fr = _lib.LrfIngestFrame()
        fr.slot, fr.w, fr.h = slot, w, h
        with torch.cuda.device(dev):
            up = {k: t.to(dev, non_blocking=True) for k, t in raw.items()}
            img = up["image"]
            fr.image, fr.h0, fr.w0, fr.image_stride = _ptr(img).value, img.shape[0], img.shape[1], img.shape[1] * 3
            if "invdepth" in up:
                d = up["invdepth"]
                fr.invdepth, fr.hd, fr.wd, fr.invdepth_stride = _ptr(d).value, d.shape[0], d.shape[1], d.shape[1]
            if "fwd_flow" in up:
                a, b = up["fwd_flow"], up["bwd_flow"]
                if a.shape != b.shape:
                    raise NotImplementedError(f"frame {f}: the forward and backward flows differ in size")
                fr.fwd_flow, fr.bwd_flow = _ptr(a).value, _ptr(b).value
                fr.hf, fr.wf, fr.flow_stride = a.shape[0], a.shape[1], a.shape[1] * 3
                fr.flow_scale = float(np.float32(h / a.shape[0]))
            if "mask" in up:
                m = up["mask"]
                fr.mask, fr.hm, fr.wm, fr.mask_stride = _ptr(m).value, m.shape[0], m.shape[1], m.shape[1]
            L = _lib.lib()
            n = L.lrf_ingest_scratch_bytes(w * h)
            s = self._scratch.get(dev)
            if s is None or s.numel() < n:
                s = self._scratch[dev] = torch.empty(max(n, 8), dtype=torch.uint8, device=dev)
            _lib.check(L.lrf_ingest_frame(C.byref(store), C.byref(fr), C.c_void_p(_ptr(s).value), s.numel(),
                                          _stream(dev)))
