"""Time the training call of LocalTensorfs.forward, forward + backward: the _TrainRenderFn node (one lrf_render, one
lrf_exposure_clamp; lrf_render_backward_batch) against the composed path `lt._forward_autograd` (torch ops for ray
generation, cam2rf, exposure and clamp around the field's _RenderFn).

    python tools/train_forward_time.py [--iters 30] [--rounds 3]

Workload: a 300^3 field, 100 frames of which 16 are live (view ids 84..97 plus the last view twice, train.py's
forced duplicates), 16 views x 256 rays.  The two paths alternate `--rounds` times in one process; each line reports
the median round: host wall time per iteration (the host waits for the device only at the end of the window),
CUDA-event time per iteration, and kernel launches of one iteration (torch.profiler, in a separate run).  The
"iteration" rows time the whole step: the call, supervision_losses (rgb term), get_reg_loss and optimizer_step.
Every line carries the GPU's name and power limit, read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def scene():
    import bench
    import localrf_b200 as L
    lt = bench._scene(L.LocalTensorfs, "cpu", 300, n_init_frames=100).to("cuda")
    lt.is_refining = True
    gen = torch.Generator().manual_seed(0)
    views = list(range(84, 98)) + [99, 99]
    px = torch.randint(0, bench.IMG_W * bench.IMG_H, (16, 256), generator=gen)
    ids = (px + torch.tensor(views)[:, None] * bench.IMG_W * bench.IMG_H).reshape(-1).cuda()
    return lt, ids, views, bench.IMG_W, bench.IMG_H


def call_node(lt, ids, views, W, H):
    return lt(ids, views, W, H, is_train=True)


def call_composed(lt, ids, views, W, H):
    # what _forward_general hands the composed path in training: the newest field, no blend
    return lt._forward_autograd(ids, views, views, W, H, True, True, None, lt.world2rf, None,
                                [len(lt.tensorfs) - 1], 16384, False, 0)


def fwd_bwd(call, lt, ids, views, W, H, c):
    rgb, depth, dirs, ij = call(lt, ids, views, W, H)
    ((rgb * c).sum() + depth.sum()).backward()


def iteration(call, lt, ids, views, W, H, target):
    from localrf_b200 import supervision_losses
    rgb, depth, dirs, ij = call(lt, ids, views, W, H)
    loss = supervision_losses(rgb, target, torch.ones(rgb.shape[0], device="cuda"),
                              view_ids=torch.tensor(views, device="cuda"))[0]
    tv, l1 = lt.get_reg_loss(None, 0, 0, 8e-5)
    lt.optimizer_step(loss + l1, optimize_poses=True)


def window(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    host = (time.perf_counter() - t0) / iters
    torch.cuda.synchronize()
    return host * 1e3, a.elapsed_time(b) / iters


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    from loss_time import gpu_identity
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_forward_time.py measures on a CUDA device; none is available")
    gpu, power_w = gpu_identity()
    lt, ids, views, W, H = scene()
    c = torch.randn(ids.shape[0], 3, device="cuda")
    target = torch.rand(ids.shape[0], 3, device="cuda")
    jobs = []
    for kind in ("forward_backward", "iteration"):
        for name, call in (("node", call_node), ("composed", call_composed)):
            if kind == "forward_backward":
                fn = (lambda call=call: fwd_bwd(call, lt, ids, views, W, H, c))
            else:
                fn = (lambda call=call: iteration(call, lt, ids, views, W, H, target))
            jobs.append((kind, name, fn))
    for _, _, fn in jobs:                                  # warm-up: module loads, allocator, memos
        for _ in range(3):
            fn()
    for kind in ("forward_backward", "iteration"):
        mine = [j for j in jobs if j[0] == kind]
        times = {name: [] for _, name, _ in mine}
        for _ in range(args.rounds):                       # the two paths alternate
            for _, name, fn in mine:
                times[name].append(window(fn, args.iters))
        for _, name, fn in mine:
            row = {"what": kind, "path": name, "field": "300^3", "frames": 100, "live_frames": 16,
                   "rays": int(ids.shape[0]),
                   "host_ms_per_iter": round(statistics.median(t[0] for t in times[name]), 3),
                   "cuda_event_ms_per_iter": round(statistics.median(t[1] for t in times[name]), 3),
                   "kernel_launches": launches(fn), "gpu": gpu, "power_limit_w": power_w}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
