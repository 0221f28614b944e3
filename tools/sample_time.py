"""Time the first line of a training iteration, train.py:351-356: LocalRFDataset.sample's numpy gather plus the
uploads train.py makes ("host" arm) against localrf_b200.DeviceRaySampler.sample ("device" arm).

    python tools/sample_time.py [--iters 30] [--rounds 3]

The host arm is the reference's path: the sampler restated in tests/sample_oracle.py over host arrays of every
active frame, then the pageable `.to(device)` copies of view_ids, rgbs, loss_weights and idx (train.py:352-356) and
the pinned, non-blocking copies of the flows, flow masks and inverse depths that INTEGRATION.md's supervision-losses
block makes.  The device arm keeps the frames resident and makes one pinned ids upload and one lrf_gather_rays.

Rows, each the median of `--rounds` alternated rounds of `--iters` calls, with host wall time (the host waits for
the device only at the end of the window), CUDA-event time and the kernels and copies of one call (torch.profiler,
in a separate run):
  * "sample": the call alone, 100 active 800x800 frames with flow and depth, 16 views x 256 rays;
  * "iteration": a whole training step at the tools/train_forward_time.py workload (a 300^3 field, 100 frames,
    16 views x 256 rays, 800x800): the sample, the training call of LocalTensorfs.forward, supervision_losses with
    the flow and depth terms, get_reg_loss and optimizer_step.
Every line carries the GPU's name and power limit, read in the same call.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_FRAMES, V, R = 100, 16, 256


def dataset(W, H):
    import numpy as np
    import sample_oracle as so
    frames = {}
    for i, (_, key, w) in enumerate(so.QUANTITIES):
        pool = np.random.default_rng(i).random((4, W * H, w), dtype=np.float32)
        frames[key] = np.stack([pool[f % 4] + np.float32(f) for f in range(N_FRAMES)])
    test_mask = np.array([1 if f % 10 == 0 else 0 for f in range(N_FRAMES)])
    return so.FrameDataset(frames, test_mask, True, True, N_FRAMES, N_FRAMES)


def host_sample(ds, is_refining, dev):
    import sample_oracle as so
    blob = so.sample(ds, V * R, is_refining, True, V)
    out = {k: torch.from_numpy(blob[k]).to(dev) for k in ("view_ids", "rgbs", "loss_weights", "idx")}
    for k in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask", "invdepths"):
        out[k] = torch.from_numpy(blob[k]).pin_memory().to(dev, non_blocking=True)
    out["view_ids_host"] = blob["view_ids"]
    return out


def iteration(lt, W, H, get_blob):
    from localrf_b200 import supervision_losses
    blob = get_blob()
    rgb, depth, dirs, ij = lt(blob["idx"], blob["view_ids_host"], W, H, is_train=True)
    cr = lt.center_rel
    loss, flow, dloss = supervision_losses(
        rgb, blob["rgbs"], blob["loss_weights"], view_ids=blob["view_ids"], depth_map=depth, directions=dirs, ij=ij,
        cam2world=lt.get_cam2world(starting_id=0), starting_id=0, focal=lt.focal(W),
        center=torch.stack([cr[0] * W, cr[1] * H]), fwd_flow=blob["fwd_flow"], fwd_mask=blob["fwd_mask"],
        bwd_flow=blob["bwd_flow"], bwd_mask=blob["bwd_mask"], flow_weight=1.0 / ((W + H) / 2),
        invdepths=blob["invdepths"], depth_weight=0.1)
    tv, l1 = lt.get_reg_loss(None, 0, 0, 8e-5)
    lt.optimizer_step(loss + flow + dloss + l1, optimize_poses=True)


def device_ops(fn):
    """(kernels, copies) of one call of fn, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    copies = sum(1 for e in ev if "memcpy" in e.name.lower())
    return len(ev) - copies, copies


def main():
    import bench
    import localrf_b200 as L
    from loss_time import gpu_identity
    from train_forward_time import window
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_time.py measures on a CUDA device; none is available")
    gpu, power_w = gpu_identity()
    dev = torch.device("cuda")
    W, H = bench.IMG_W, bench.IMG_H
    ds = dataset(W, H)
    sampler = L.DeviceRaySampler(ds, dev)
    lt = bench._scene(L.LocalTensorfs, "cpu", 300, n_init_frames=N_FRAMES).to(dev)
    lt.is_refining = True
    arms = {"host": lambda: host_sample(ds, True, dev), "device": lambda: sampler.sample(V * R, True, True, V)}
    jobs = []
    for kind in ("sample", "iteration"):
        for name, get_blob in arms.items():
            fn = get_blob if kind == "sample" else (lambda g=get_blob: iteration(lt, W, H, g))
            jobs.append((kind, name, fn))
    for _, _, fn in jobs:                                  # warm-up: frame upload, module loads, allocator, memos
        for _ in range(3):
            fn()
    for kind in ("sample", "iteration"):
        mine = [j for j in jobs if j[0] == kind]
        times = {name: [] for _, name, _ in mine}
        for _ in range(args.rounds):                       # the two arms alternate
            for _, name, fn in mine:
                times[name].append(window(fn, args.iters))
        for _, name, fn in mine:
            kernels, copies = device_ops(fn)
            row = {"what": kind, "arm": name, "frames": N_FRAMES, "W": W, "H": H, "views": V, "rays": V * R,
                   "flow_depth": True, "field": "300^3" if kind == "iteration" else None,
                   "host_ms": round(statistics.median(t[0] for t in times[name]), 3),
                   "cuda_event_ms": round(statistics.median(t[1] for t in times[name]), 3),
                   "kernel_launches": kernels, "copies": copies, "gpu": gpu, "power_limit_w": power_w}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
