"""Time bringing frames into training: LocalRFDataset.read_meta's per-frame conversions on the host plus
DeviceRaySampler's float32 upload ("host" arm) against DeviceFrameDataset + lrf_ingest_frame ("device" arm).

    python tools/ingest_time.py [--frames 100] [--chunk 20]

A synthetic scene of `--frames` 960x540 frames is written to a temporary directory as read_meta expects it: jpg
images, 16-bit inverse-depth PNGs at the image size, flows at half size (480x270, as scripts/run_flow.py writes
them).  The host arm restates read_meta with its cv2 / numpy calls (float conversion, INTER_AREA resizes,
decode_flow, Laplacian variance, concatenate_append onto the arrays of every loaded frame) and feeds a
DeviceRaySampler, which copies 44 B/px of float32 per new frame.  The device arm reads the same files with the same
joblib threads, keeps only the decoded planes (17 B/px) in pinned memory and converts them on the device.

The arms alternate chunk by chunk in one process.  Per chunk: the stall, host time from activate_frames until a
device synchronise after the sampler has placed the chunk's frames; the CUDA-event time of that placement (uploads
and, for the device arm, the kernels); host memory the dataset holds afterwards; bytes uploaded per frame.  One
JSON line per arm and chunk, then one summary line per arm, each with the GPU's name and power limit.
"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

W, H = 960, 540


def write_scene(d, n):
    import cv2
    rng = np.random.default_rng(0)
    for sub in ("images", "depth", "flow_ds"):
        os.makedirs(os.path.join(d, sub))
    base = cv2.resize(rng.random((H // 8, W // 8, 3)).astype(np.float32) * 255, (W, H))
    for i in range(n):
        f = f"{i:05d}"
        img = np.clip(base + rng.normal(0, 20, base.shape), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(d, "images", f + ".jpg"), img)
        cv2.imwrite(os.path.join(d, "depth", f + ".png"), rng.integers(0, 65536, (H, W), dtype=np.uint16))
        for kind in ("fwd", "bwd"):
            e = rng.integers(30000, 35000, (H // 2, W // 2, 3), dtype=np.uint16)
            cv2.imwrite(os.path.join(d, "flow_ds", f"{kind}_{f}.png"), e)


class HostFrames:
    """The train split of LocalRFDataset as the reference loads it (flow and depth on, no masks, downsampling -1):
    read_meta's per-frame steps and concatenate_append, restated with the same cv2 / numpy calls."""

    def __init__(self, d, n, chunk):
        self.d, self.names = d, sorted(os.listdir(os.path.join(d, "images")))
        self.num_images, self.frames_chunk = n, chunk
        self.load_depth = self.load_flow = True
        self.test_mask = np.zeros(n, dtype=np.int64)
        self.all_rgbs = self.all_loss_weights = self.all_invdepths = None
        self.all_fwd_flow = self.all_fwd_mask = self.all_bwd_flow = self.all_bwd_mask = None
        self.active_frames_bounds, self.loaded_frames = [0, 0], 0
        self.activate_frames(chunk)

    def _read(self, i):
        import cv2
        base = os.path.splitext(self.names[i])[0]
        nxt = os.path.splitext(self.names[(i + 1) % len(self.names)])[0]
        img = cv2.imread(os.path.join(self.d, "images", self.names[i]))[..., ::-1]
        img = img.astype(np.float32) / 255
        size = tuple(img.shape[1::-1])
        dep = cv2.resize(cv2.imread(os.path.join(self.d, "depth", base + ".png"), -1).astype(np.float32), size,
                         interpolation=cv2.INTER_AREA)
        out = {"img": img, "invdepth": dep}
        for kind, name in (("fwd", nxt), ("bwd", base)):
            e = cv2.imread(os.path.join(self.d, "flow_ds", f"{kind}_{name}.png"), cv2.IMREAD_UNCHANGED)
            scale = img.shape[0] / e.shape[0]
            e = cv2.resize(e, size, interpolation=cv2.INTER_AREA)
            f = e[..., :2].astype(np.float32)
            f -= 2 ** 15
            f /= 2 ** 8
            out[kind + "_flow"], out[kind + "_mask"] = f * scale, (e[..., 2] > 2 ** 15).astype(np.float32)
        return out

    def activate_frames(self, n=1):
        import cv2
        from joblib import Parallel, delayed
        b = self.active_frames_bounds
        b[1] = min(b[1] + n, self.num_images)
        if b[1] <= self.loaded_frames:
            return
        k = min(self.frames_chunk, self.num_images - self.loaded_frames)
        data = Parallel(n_jobs=-1, backend="threading")(
            delayed(self._read)(i) for i in range(self.loaded_frames, self.loaded_frames + k))
        self.loaded_frames += k
        lw = [np.ones_like(x["img"][..., 0]) * cv2.Laplacian(
            cv2.cvtColor((x["img"] * 255).astype(np.uint8), cv2.COLOR_RGB2GRAY), cv2.CV_32F).var() for x in data]
        self.img_wh = list(data[0]["img"].shape[1::-1])
        self.n_px_per_frame = self.img_wh[0] * self.img_wh[1]

        def append(old, new, dim):
            new = np.concatenate(new, 0).reshape(-1, dim)
            return new if old is None else np.concatenate([old, new], 0)
        self.all_rgbs = append(self.all_rgbs, [x["img"] for x in data], 3)
        self.all_invdepths = append(self.all_invdepths, [x["invdepth"] for x in data], 1)
        for key, dim in (("fwd_flow", 2), ("fwd_mask", 1), ("bwd_flow", 2), ("bwd_mask", 1)):
            setattr(self, "all_" + key, append(getattr(self, "all_" + key), [x[key] for x in data], dim))
        self.all_loss_weights = append(self.all_loss_weights, lw, 1)

    def host_bytes(self):
        return sum(getattr(self, a).nbytes for a in ("all_rgbs", "all_loss_weights", "all_invdepths", "all_fwd_flow",
                                                     "all_fwd_mask", "all_bwd_flow", "all_bwd_mask"))


def device_host_bytes(ds):
    return sum(t.numel() * t.element_size() for raw in ds._raw.values() for t in raw.values())


def main():
    from loss_time import gpu_identity
    from localrf_b200 import DeviceFrameDataset, DeviceRaySampler
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--chunk", type=int, default=20)
    a = ap.parse_args()
    gpu, power_w = gpu_identity()
    dev = torch.device("cuda")
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        write_scene(d, a.frames)
        print(f"# scene of {a.frames} {W}x{H} frames written in {time.perf_counter() - t0:.1f} s", file=sys.stderr)
        arms = {}
        stats = {"host": [], "device": []}
        for chunk in range(a.frames // a.chunk):
            for name in ("host", "device"):
                random.seed(chunk)
                np.random.seed(chunk)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if name not in arms:
                    ds = HostFrames(d, a.frames, a.chunk) if name == "host" else \
                        DeviceFrameDataset(d, load_depth=True, load_flow=True, frames_chunk=a.chunk,
                                           n_init_frames=a.chunk, test_frame_every=0)
                    arms[name] = (ds, DeviceRaySampler(ds, dev, capacity=a.frames))
                else:
                    arms[name][0].activate_frames(a.chunk)
                ds, sampler = arms[name]
                t_read = time.perf_counter()
                held_before = device_host_bytes(ds) if name == "device" else None
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                sampler._sync_frames()                       # what the next sample() does first
                e1.record()
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                n_px = ds.n_px_per_frame
                up = 4 * sampler.floats_per_px * n_px if name == "host" else held_before // a.chunk
                row = {"arm": name, "chunk": chunk, "active_frames": ds.active_frames_bounds[1],
                       "stall_ms": round(1e3 * (t1 - t0), 2), "read_ms": round(1e3 * (t_read - t0), 2),
                       "place_event_ms": round(e0.elapsed_time(e1), 3),
                       "host_bytes_held": ds.host_bytes() if name == "host" else device_host_bytes(ds),
                       "upload_bytes_per_px": round(up / n_px, 2), "gpu": gpu, "power_limit_w": power_w}
                stats[name].append(row)
                print(json.dumps(row), flush=True)
        for name, rows in stats.items():
            print(json.dumps({"arm": name, "summary": True, "frames": a.frames, "chunk": a.chunk, "w": W, "h": H,
                              "median_stall_ms": float(np.median([r["stall_ms"] for r in rows])),
                              "last_stall_ms": rows[-1]["stall_ms"],
                              "median_place_event_ms": float(np.median([r["place_event_ms"] for r in rows])),
                              "host_bytes_held_at_end": rows[-1]["host_bytes_held"],
                              "upload_bytes_per_px": rows[-1]["upload_bytes_per_px"], "gpu": gpu,
                              "power_limit_w": power_w}), flush=True)


if __name__ == "__main__":
    main()
