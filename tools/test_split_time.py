"""Time the test split: LocalRFDataset's test split as the reference builds it on the host ("host" arm) against
DeviceFrameDataset(split="test") ("device" arm), and renderer.render's ground-truth resize (cv2.resize) against
lrf_resize_linear.

    python tools/test_split_time.py [--frames 100] [--reps 3]

A synthetic scene is written to a temporary directory with only the files the test split reads: `--frames` test
frames of 960x540 (named 0, 10, 20, ... so that every one has index % 10 == 0), jpg images, 16-bit inverse-depth
PNGs at the image size and flows at half size.  Three measurements, the arms alternated in one process:

  construction   host time from the constructor to a device synchronise (the stall), host memory the dataset holds
                 afterwards (its float arrays, or the decoded planes it still keeps), device memory it holds.  The host
                 arm restates the reference's test split with read_meta's cv2 / numpy calls (tools/ingest_time.py's
                 HostFrames._read) and np.stack, and computes and drops the loss weights as the reference does.
  held-out frame FramePipeline at 480x270 with gt= and panels= over every test frame of a cfg5 scene (300^3, 64
                 cameras; frame k uses camera k % 64): host time and CUDA-event time per frame, ground truth as
                 cv2.resize of the host arrays plus the numpy panel inputs against resize_linear and the device split.
  resize alone   lrf_resize_linear by CUDA events over back-to-back launches at 960x540 -> 480x270,
                 1920x1080 -> 960x540 and 963x541 -> 481x270, beside cv2.resize's host time with IPP as the build
                 has it (the reference's path).
One JSON line per measurement, each with the GPU's name and power limit.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

W0, H0 = 960, 540
TEST_EVERY = 10


def write_scene(d, n):
    import cv2
    rng = np.random.default_rng(0)
    for sub in ("images", "depth", "flow_ds"):
        os.makedirs(os.path.join(d, sub))
    base = cv2.resize(rng.random((H0 // 8, W0 // 8, 3)).astype(np.float32) * 255, (W0, H0))
    for i in range(n):
        f = f"{TEST_EVERY * i:05d}"
        img = np.clip(base + rng.normal(0, 20, base.shape), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(d, "images", f + ".jpg"), img)
        cv2.imwrite(os.path.join(d, "depth", f + ".png"), rng.integers(0, 65536, (H0, W0), dtype=np.uint16))
        for kind in ("fwd", "bwd"):
            e = rng.integers(30000, 35000, (H0 // 2, W0 // 2, 3), dtype=np.uint16)
            cv2.imwrite(os.path.join(d, "flow_ds", f"{kind}_{f}.png"), e)


def host_test_split(d):
    """The reference's test split (flow and depth on, no masks): every frame read at once, read_meta's conversions,
    the loss weights computed and dropped, np.stack of the rest."""
    import cv2
    from joblib import Parallel, delayed
    from ingest_time import HostFrames
    hf = HostFrames.__new__(HostFrames)
    hf.d, hf.names = d, sorted(os.listdir(os.path.join(d, "images")))
    data = Parallel(n_jobs=-1, backend="threading")(delayed(hf._read)(i) for i in range(len(hf.names)))
    for x in data:                                      # the loss weights: computed, then dropped
        np.ones_like(x["img"][..., 0]) * cv2.Laplacian(
            cv2.cvtColor((x["img"] * 255).astype(np.uint8), cv2.COLOR_RGB2GRAY), cv2.CV_32F).var()
    out = {"all_rgbs": np.stack([x["img"] for x in data], 0),
           "all_invdepths": np.stack([x["invdepth"] for x in data], 0)}
    for key in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"):
        out["all_" + key] = np.stack([x[key] for x in data], 0)
    return out


def timed(fn, events, busy=False):
    """-> (host seconds, CUDA-event ms / events) of fn(); busy: the GPU first sleeps, so that back-to-back launches
    queue up behind it and the events time the kernels rather than the host's enqueueing."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if busy:
        torch.cuda._sleep(200_000_000)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, e0.elapsed_time(e1) / events


def main():
    import cv2
    import bench
    import localrf_b200 as L
    from loss_time import gpu_identity
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    gpu, power_w = gpu_identity()
    ident = {"gpu": gpu, "power_limit_w": power_w}
    dev = torch.device("cuda")
    torch.set_grad_enabled(False)
    L.lib()
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        write_scene(d, a.frames)
        print(f"# scene of {a.frames} {W0}x{H0} test frames written in {time.perf_counter() - t0:.1f} s",
              file=sys.stderr)

        # construction, alternated
        keep = {}
        for rep in range(a.reps):
            for arm in ("host", "device"):
                keep.pop(arm, None)
                torch.cuda.synchronize()
                mem0 = torch.cuda.memory_allocated(dev)
                t0 = time.perf_counter()
                if arm == "host":
                    ds = host_test_split(d)
                else:
                    ds = L.DeviceFrameDataset(d, split="test", load_depth=True, load_flow=True,
                                              test_frame_every=TEST_EVERY, device=dev)
                torch.cuda.synchronize()
                stall = time.perf_counter() - t0
                if arm == "host":
                    host_bytes = sum(v.nbytes for v in ds.values())
                else:
                    host_bytes = sum(v.nbytes for v in vars(ds).values() if isinstance(v, np.ndarray)) + \
                        sum(t.numel() * t.element_size() for raw in ds._raw.values() for t in raw.values())
                keep[arm] = ds
                print(json.dumps({"measure": "construction", "arm": arm, "rep": rep, "frames": a.frames,
                                  "w": W0, "h": H0, "stall_ms": round(1e3 * stall, 1), "host_bytes_held": host_bytes,
                                  "device_bytes_held": torch.cuda.memory_allocated(dev) - mem0, **ident}),
                      flush=True)
        host, dsd = keep["host"], keep["device"]

        # held-out frames in FramePipeline at 480x270, alternated
        W, H = W0 // 2, H0 // 2
        lt = bench.Workload("cfg5", 300).build(L.LocalTensorfs, quiet=True).to(dev)
        n_cams = len(lt.r_c2w)
        names = ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask")

        def frames(arm):
            for k in range(a.frames):
                if arm == "host":
                    gt = cv2.resize(host["all_rgbs"][k], (W, H))
                    p = {n: host["all_" + n][k] for n in names}
                    p["invdepth"] = host["all_invdepths"][k]
                else:
                    gt = L.metrics.resize_linear(dsd.all_rgbs[k], W, H)
                    p = {n: getattr(dsd, "all_" + n)[k] for n in names}
                    p["invdepth"] = dsd.all_invdepths[k]
                idx = k % n_cams
                yield torch.tensor([idx], device=dev), {"gt": gt, "panels": dict(idx=idx, **p), "test_id": True}

        def run(arm):
            pipe = L.FramePipeline(lt, W, H, n_buffers=3)
            for _ in pipe.render(frames(arm)):
                pass

        for arm in ("host", "device"):
            run(arm)                                          # warm-up: allocations, staging buffers
        for rep in range(a.reps):
            for arm in ("host", "device"):
                t, ev = timed(lambda: run(arm), a.frames)
                print(json.dumps({"measure": "held_out_frame", "arm": arm, "rep": rep, "w": W, "h": H,
                                  "frames": a.frames, "host_ms_per_frame": round(1e3 * t / a.frames, 3),
                                  "event_ms_per_frame": round(ev, 3), **ident}), flush=True)

        # lrf_resize_linear alone against cv2.resize on the host (IPP as the build has it)
        rng = np.random.default_rng(1)
        n_launch = 200
        for (w0, h0), (w, h) in (((960, 540), (480, 270)), ((1920, 1080), (960, 540)), ((963, 541), (481, 270))):
            src = rng.random((h0, w0, 3), dtype=np.float32)
            src_d = torch.from_numpy(src).to(dev)
            out = torch.empty(h, w, 3, device=dev)
            for _ in range(10):
                L.metrics.resize_linear(src_d, w, h, out=out)
            _, ev = timed(lambda: [L.metrics.resize_linear(src_d, w, h, out=out) for _ in range(n_launch)], n_launch, busy=True)
            ts = []
            for _ in range(50):
                t0 = time.perf_counter()
                cv2.resize(src, (w, h))
                ts.append(time.perf_counter() - t0)
            print(json.dumps({"measure": "resize", "src": f"{w0}x{h0}", "dst": f"{w}x{h}",
                              "kernel_us": round(1e3 * ev, 2), "launches": n_launch,
                              "cv2_host_us_median": round(1e6 * float(np.median(ts)), 1),
                              "cv2_ipp": bool(cv2.ipp.useIPP()), **ident}), flush=True)


if __name__ == "__main__":
    main()
