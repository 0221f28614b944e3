"""Time the Adam steps of one training iteration: the per-optimiser torch loop (`for o in opts: o.step()`, as the
reference's LocalTensorfs.optimizer_step calls it) against localrf_b200.adam_step (one lrf_adam_step launch).

    python tools/optim_time.py [--iters 50] [--rounds 3] [--grids 64 300 640] [--frames 5 16 100]

The optimisers are the scene model's: the field's (19 tensors in two groups), one Adam each for every live frame's
rotation, translation and exposure, and the intrinsics'.  Sixteen frames have gradients (the sampled views), or every
frame ("pose_grads": "all", the flow term on).  The two paths alternate, `--rounds` times each, in one process; each
line reports the median round.  Per workload and path: host wall time per step (the host waits for the device only
at the end of the window, so this is the rate the host can issue steps), CUDA-event time per step, kernel launches
of one step (torch.profiler, in a separate run), and for the field the bytes counted from shapes (28 B per element
for one fused pass: read p, g, m, v, write p, m, v) with the rate they imply over the step's CUDA-event time and its
share of the data-sheet 3.35 TB/s.  Every line carries the GPU's name and power limit, read in the same call.
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

HBM_BYTES_PER_S = 3.35e12


def field_tensors(G, gen):
    """The 19 tensors of a TensorVMSplit at G^3 (8 / 24 components per plane), channel-last like the model's."""
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    r = lambda *s: 0.1 * torch.randn(*s, device="cuda", generator=gen)
    grids = [cl(r(1, c, G, G)) for c in (8,) * 3 + (24,) * 3] + [cl(r(1, c, G, 1)) for c in (8,) * 3 + (24,) * 3]
    mlp = [r(27, 72), r(128, 27), r(128), r(128, 128), r(128), r(3, 131), r(3)]
    return [torch.nn.Parameter(t) for t in grids], [torch.nn.Parameter(t) for t in mlp]


def workload(G, n_frames, pose_grads):
    gen = torch.Generator(device="cuda").manual_seed(0)
    grids, mlp = field_tensors(G, gen)
    opts = [torch.optim.Adam([{"params": grids, "lr": 2e-2}, {"params": mlp, "lr": 1e-3}], betas=(0.9, 0.99))]
    with_grad = grids + mlp
    n_grad = n_frames if pose_grads == "all" else min(16, n_frames)
    for i in range(n_frames):
        ps = [torch.nn.Parameter(t.cuda()) for t in (torch.eye(3, 2), torch.zeros(3), torch.eye(3))]
        opts += [torch.optim.Adam([p], betas=(0.9, 0.99), lr=lr) for p, lr in zip(ps, (5e-3, 5e-4, 1e-3))]
        if i < n_grad:
            with_grad += ps
    intr = [torch.nn.Parameter(torch.ones(1, device="cuda")), torch.nn.Parameter(torch.full((2,), 0.5, device="cuda"))]
    opts.append(torch.optim.Adam(intr, betas=(0.9, 0.99), lr=1e-3))
    with_grad += intr
    for p in with_grad:
        p.grad = 1e-3 * torch.randn(p.shape, device="cuda", generator=gen).contiguous(
            memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
    field_elems = sum(p.numel() for p in grids + mlp)
    return opts, field_elems, sum(p.numel() for p in with_grad)


def step_torch(opts):
    for o in opts:
        o.step()


def step_fused(opts):
    from localrf_b200 import adam_step
    adam_step(opts)


def window(fn, opts, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        fn(opts)
    b.record()
    host = (time.perf_counter() - t0) / iters
    torch.cuda.synchronize()
    return host * 1e6, a.elapsed_time(b) / iters * 1e3


def launches(fn, opts):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn(opts)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    from loss_time import gpu_identity
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--grids", type=int, nargs="+", default=[64, 300, 640])
    ap.add_argument("--frames", type=int, nargs="+", default=[5, 16, 100])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_time.py measures on a CUDA device; none is available")
    gpu, power_w = gpu_identity()
    paths = (("torch_loop", step_torch), ("adam_step", step_fused))
    for G in args.grids:
        for n_frames in args.frames:
            for pose_grads in ("16", "all"):
                if pose_grads == "all" and n_frames <= 16:
                    continue                                  # the same workload as "16"
                opts, field_elems, grad_elems = workload(G, n_frames, pose_grads)
                for _, fn in paths:                           # warm-up: state creation, module loads
                    for _ in range(3):
                        fn(opts)
                times = {name: [] for name, _ in paths}
                for _ in range(args.rounds):                  # the two paths alternate
                    for name, fn in paths:
                        times[name].append(window(fn, opts, args.iters))
                for name, fn in paths:
                    host = statistics.median(t[0] for t in times[name])
                    dev = statistics.median(t[1] for t in times[name])
                    row = {"path": name, "grid": G, "live_frames": n_frames, "pose_grads": pose_grads,
                           "host_us_per_step": round(host, 1), "cuda_event_us_per_step": round(dev, 1),
                           "kernel_launches": launches(fn, opts), "field_elements": field_elems,
                           "elements_with_grad": grad_elems, "gpu": gpu, "power_limit_w": power_w}
                    if name == "adam_step":
                        nbytes = 28 * grad_elems
                        row.update(bytes_counted=nbytes, achieved_gb_per_s=round(nbytes / (dev * 1e-6) / 1e9, 1),
                                   share_of_3_35_tb_per_s=round(nbytes / (dev * 1e-6) / HBM_BYTES_PER_S, 3))
                    print(json.dumps(row), flush=True)
                del opts
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
