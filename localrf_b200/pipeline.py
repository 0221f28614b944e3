"""Frame-render pipeline around the fused kernel (SURVEY.md 8f rank 4; replaces the per-frame host work of
renderer.py:58-77,126-178).

The reference renders a frame, synchronises, pulls rgb / depth to the host as fp32 (`.cpu()`), converts
them with numpy / cv2 / matplotlib and only then starts the next frame.  Here a frame is

    one fused launch per active field  ->  one post-processing kernel (8-bit BGR + colour-mapped depth)

whose outputs are written by the GPU straight into pinned host buffers (zero-copy, 6 bytes per pixel instead
of 16), with a CUDA event per frame.  `submit()` never blocks; `fetch()` returns the OLDEST finished frame,
so encoding / writing frame i on the host overlaps the rendering of frames i+1..i+depth-1.  A frame submitted
with its ground truth (`gt=`) is also scored on the device (MSE and SSIM, renderer.py:162-163; metrics.py) into a
pinned double[2] of its slot, and one submitted with `panels=` gets the flow and depth comparison panels of
renderer.py:79-124 (metrics.test_panels) in pinned buffers of its slot.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, metrics
from .tensorf import _ptr, _stream


def jet_lut():
    """cv2.COLORMAP_JET as a [256,3] uint8 BGR table (what visualize_depth applies, utils/utils.py:195)."""
    import cv2
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_JET)[:, 0, :].copy()


class FramePipeline:
    def __init__(self, local_tensorfs, W, H, depth_minmax=(0.0, 5.0), n_buffers=3, lut=None, keep_float=False):
        self.lt, self.W, self.H = local_tensorfs, int(W), int(H)
        self.dev = local_tensorfs.blending_weights.device
        if self.dev.type != "cuda":
            raise RuntimeError("FramePipeline needs the scene model on a CUDA device")
        self.n = self.W * self.H
        self.minmax = (float(depth_minmax[0]), float(depth_minmax[1]))
        lut = jet_lut() if lut is None else np.ascontiguousarray(lut, np.uint8).reshape(256, 3)
        self.lut = torch.from_numpy(lut).to(self.dev)
        self.ids = torch.arange(self.n, dtype=torch.int64, device=self.dev)
        self.keep_float = keep_float
        self.slots = []
        for _ in range(int(n_buffers)):
            s = {"rgb8": torch.empty(self.n, 3, dtype=torch.uint8).pin_memory(),
                 "depth8": torch.empty(self.n, 3, dtype=torch.uint8).pin_memory(),
                 "metrics": torch.zeros(2, dtype=torch.float64).pin_memory(),
                 "event": torch.cuda.Event(), "busy": False, "tag": None, "has_gt": False}
            if keep_float:
                s["rgb"] = torch.empty(self.n, 3).pin_memory()
                s["depth"] = torch.empty(self.n).pin_memory()
            self.slots.append(s)
        self.head = self.tail = 0                       # ring: tail = oldest in flight, head = next to fill

    def in_flight(self):
        return sum(s["busy"] for s in self.slots)

    def _stage_gt(self, s, gt):
        """gt as a frame the metrics kernel can read: CUDA and pinned tensors as they are, anything else copied
        into the slot's pinned staging buffer (free: the slot's previous frame has been fetched)."""
        if isinstance(gt, torch.Tensor) and (gt.is_cuda or gt.is_pinned()):
            return gt
        if "gt" not in s:
            s["gt"] = torch.empty(self.n, 3).pin_memory()
        s["gt"].copy_(torch.as_tensor(gt, dtype=torch.float32).reshape(self.n, 3))
        return s["gt"]

    def _stage_panel_gt(self, s, name, x):
        """A host ground-truth array staged for the panel kernels through the slot's buffers for it (both free: the
        slot's previous frame has been fetched): a host copy into a pinned buffer, then an asynchronous copy to a
        device buffer on the current stream.  Unlike a pageable upload neither waits for the device, so submit()
        stays non-blocking."""
        bufs = s.setdefault("panel_gt", {})
        shape = tuple(x.shape)
        if name not in bufs or tuple(bufs[name][0].shape) != shape:
            bufs[name] = (torch.empty(shape, dtype=torch.float32).pin_memory(),
                          torch.empty(shape, dtype=torch.float32, device=self.dev))
        host, dev = bufs[name]
        host.copy_(torch.from_numpy(np.ascontiguousarray(x)))
        dev.copy_(host, non_blocking=True)
        return dev

    def _panel_buffers(self, s, flow, depth):
        """The slot's pinned panel outputs (allocated on first use) -> dict for metrics._enqueue_panels."""
        H, W = self.H, self.W
        want = {"fwd_panel": (3 * H, 2 * W), "bwd_panel": (3 * H, 2 * W)} if flow else {}
        if depth:
            want["depth_panel"] = (3 * H, W)
        for name, shape in want.items():
            if name not in s:
                s[name] = torch.empty(*shape).pin_memory()
        return {name: s[name] for name in want}

    @torch.no_grad()
    def submit(self, view_ids, gt=None, tag=None, panels=None, **forward_kw):
        """Enqueues one frame (all W*H rays of `view_ids`; kwargs as LocalTensorfs.forward: cam2world,
        world2rf, blending_weights, test_id, floater_thresh ...).  With `gt` ([H,W,3] float32: a CUDA tensor, a
        pinned tensor, or anything torch.as_tensor takes), the frame's MSE and SSIM against it are computed on
        the device as well (metrics.image_metrics).  With `panels` = dict(idx=, fwd_flow=, fwd_mask=, bwd_flow=,
        bwd_mask=, invdepth=, and optionally cam2world=, focal=, center=), the frame's flow and depth comparison
        panels are computed as metrics.test_panels computes them; cam2world defaults to the model's
        get_cam2world(), focal and center to focal(W) and center(W, H).  Raises if every buffer is in flight."""
        s = self.slots[self.head]
        if s["busy"]:
            raise RuntimeError("all frame buffers are in flight: fetch() before submitting more")
        g = None if gt is None else self._stage_gt(s, gt)
        out = (s["rgb"], s["depth"]) if self.keep_float else None
        rgb, depth, directions, _ = self.lt(self.ids, view_ids, self.W, self.H, is_train=False, out=out,
                                            **forward_kw)
        hold_panels, s["panels"] = None, None
        with torch.cuda.device(self.dev):
            st = _stream(self.dev)
            _lib.check(_lib.lib().lrf_frame_to_u8(_ptr(rgb), 3, _ptr(depth), 1, self.n, self.minmax[0],
                                                  self.minmax[1], _ptr(self.lut), _ptr(s["rgb8"]),
                                                  _ptr(s["depth8"]), st))
            if g is not None:
                metrics._enqueue(rgb, g, s["metrics"], W=self.W)
            if panels is not None:
                hold_panels = self._enqueue_panels(s, depth, directions, dict(panels))
            s["event"].record(torch.cuda.current_stream(self.dev))
        s["busy"], s["tag"], s["has_gt"] = True, tag, g is not None
        s["hold"] = (rgb, depth, g, hold_panels)        # keep device outputs alive until the event has passed
        self.head = (self.head + 1) % len(self.slots)

    def _enqueue_panels(self, s, depth, directions, p):
        idx = p.pop("idx")
        cam2world = p.pop("cam2world", None)
        focal, center = p.pop("focal", None), p.pop("center", None)
        if cam2world is None:
            cam2world = self.lt.get_cam2world()
        if focal is None:
            focal = self.lt.focal(self.W)
        if center is None:
            center = self.lt.center(self.W, self.H)
        gts = {k: p.pop(k, None) for k in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask", "invdepth")}
        if p:
            raise TypeError(f"unknown panels entries: {sorted(p)}")
        dev, depth, directions, cam2world, staged = metrics._panel_inputs(
            depth, directions, cam2world, self.W, self.H, stage=lambda name, x: self._stage_panel_gt(s, name, x),
            dev=self.dev, **gts)
        flow, dep = staged[0] is not None, staged[4] is not None
        outs = self._panel_buffers(s, flow, dep)
        s["panels"] = (flow, dep)
        if not (flow or dep):
            return None
        intr = metrics._intrinsics(focal, center, dev) if flow else None
        scratch = metrics._enqueue_panels(depth, directions, cam2world, idx, intr, self.W, self.H, staged, outs, dev)
        return (scratch, staged, directions, cam2world, intr)

    def fetch(self):
        """Blocks until the oldest submitted frame is complete -> dict(tag, rgb8 [H,W,3] uint8 BGR,
        depth8 [H,W,3] uint8 BGR, rgb [H,W,3] / depth [H,W] float32 when keep_float, mse / ssim floats
        when the frame was submitted with gt, and fwd_flow_cmp / bwd_flow_cmp [3H,2W] and depth_cmp [3H,W] float32
        when it was submitted with panels: None for a branch whose ground truth was not given).  The arrays are
        views of the pinned buffer: valid until `len(buffers)` more frames have been submitted."""
        s = self.slots[self.tail]
        if not s["busy"]:
            return None
        s["event"].synchronize()
        s["busy"] = False
        s.pop("hold", None)
        self.tail = (self.tail + 1) % len(self.slots)
        out = {"tag": s["tag"], "rgb8": s["rgb8"].numpy().reshape(self.H, self.W, 3),
               "depth8": s["depth8"].numpy().reshape(self.H, self.W, 3)}
        if self.keep_float:
            out["rgb"] = s["rgb"].numpy().reshape(self.H, self.W, 3)
            out["depth"] = s["depth"].numpy().reshape(self.H, self.W)
        if s["has_gt"]:
            out["mse"], out["ssim"] = (float(v) for v in s["metrics"].numpy())
        if s.get("panels") is not None:
            flow, dep = s["panels"]
            out["fwd_flow_cmp"] = s["fwd_panel"].numpy() if flow else None
            out["bwd_flow_cmp"] = s["bwd_panel"].numpy() if flow else None
            out["depth_cmp"] = s["depth_panel"].numpy() if dep else None
        return out

    def render(self, frames, **forward_kw):
        """Generator over `frames` (iterable of view-id tensors, or (view_ids, extra kwargs) pairs): keeps
        the ring full and yields finished frames in order."""
        for f in frames:
            view, extra = (f if isinstance(f, tuple) else (f, {}))
            if self.in_flight() == len(self.slots):
                yield self.fetch()
            self.submit(view, **{**forward_kw, **extra})
        while self.in_flight():
            yield self.fetch()
