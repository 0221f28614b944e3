"""Time the supervision losses of a training step (train.py:369-423): the block as torch ops vs
localrf_b200.supervision_losses, forward + backward, at the training shape (16 views x 256 rays).

    python tools/loss_time.py [--iters 200] [--cams 16 100]

For each camera count prints one JSON line per implementation, with the GPU's name and power limit: host wall time per iteration (the host waits for
the device only at the end of the timed loop, so this is the rate the host can issue iterations), CUDA-event time
per iteration, and the kernel launches of one iteration counted with torch.profiler.  With --chain the cameras
are built from per-frame r_c2w / t_c2w leaves each iteration, as LocalTensorfs.get_cam2world builds them, and the
backward runs through that chain (the same for both implementations); without it cam2world is one leaf.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def batch(n_cams, chain, V=16, R=256, W=960, H=540):
    from localrf_b200.utils import sixD_to_mtx
    g = torch.Generator().manual_seed(0)
    N = V * R
    dev = "cuda"
    r = [(torch.eye(3, 2) + 0.02 * torch.randn(3, 2, generator=g)).to(dev).requires_grad_() for _ in range(n_cams)]
    t = [(0.02 * torch.randn(3, generator=g) + torch.tensor([0, 0, -0.1 * i])).to(dev).requires_grad_()
         for i in range(n_cams)]
    fixed = {
        "rgb_train": torch.rand(N, 3, generator=g), "loss_weights": 0.2 + torch.rand(N, 1, generator=g),
        "view_ids": torch.randint(0, n_cams, (V,), generator=g),
        "directions": torch.cat([torch.rand(N, 2, generator=g) - 0.5, -torch.ones(N, 1)], 1),
        "ij": torch.stack([torch.randint(0, W, (N,), generator=g), torch.randint(0, H, (N,), generator=g)], 1),
        "fwd_flow": 3 * torch.randn(N, 2, generator=g), "bwd_flow": 3 * torch.randn(N, 2, generator=g),
        "fwd_mask": (torch.rand(N, generator=g) > 0.2).float(), "bwd_mask": (torch.rand(N, generator=g) > 0.2).float(),
        "invdepths": torch.rand(N, generator=g) + 0.1,
    }
    fixed = {k: v.to(dev) for k, v in fixed.items()}
    rgb_map = torch.rand(N, 3, generator=g).to(dev).requires_grad_()
    depth_map = (0.5 + 4.5 * torch.rand(N, generator=g)).to(dev).requires_grad_()
    focal = torch.tensor([500.0], device=dev, requires_grad=True)
    center = torch.tensor([W / 2, H / 2], device=dev)

    leaf = torch.cat([sixD_to_mtx(torch.stack(r)), torch.stack(t)[..., None]], -1).detach().requires_grad_()

    def kwargs():
        cam2world = torch.cat([sixD_to_mtx(torch.stack(r)), torch.stack(t)[..., None]], -1) if chain else leaf
        return dict(fixed, rgb_map=rgb_map, depth_map=depth_map, cam2world=cam2world, focal=focal, center=center,
                    starting_id=0, flow_weight=1.0 / ((W + H) / 2), depth_weight=0.1)
    return kwargs


def step_torch(kwargs):
    from losses_oracle import torch_block
    sum(torch_block(kwargs())).backward()


def step_kernel(kwargs):
    from localrf_b200 import supervision_losses
    kw = kwargs()
    args = {k: v for k, v in kw.items() if k not in ("rgb_map", "rgb_train", "loss_weights")}
    sum(supervision_losses(kw["rgb_map"], kw["rgb_train"], kw["loss_weights"], **args)).backward()


def launches(fn, kwargs):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn(kwargs)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def measure(fn, kwargs, iters):
    for _ in range(10):
        fn(kwargs)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        fn(kwargs)
    b.record()
    host = (time.perf_counter() - t0) / iters
    torch.cuda.synchronize()
    return host * 1e6, a.elapsed_time(b) / iters * 1e3


def gpu_identity():
    """(name, power limit in W) of the current device, read through NVML (nvidia-smi if pynvml is missing)."""
    name = torch.cuda.get_device_name()
    idx = torch.cuda.current_device()
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        return name, pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(idx), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20)
        return name, float(out.stdout.strip().splitlines()[0])
    except Exception:
        return name, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--cams", type=int, nargs="+", default=[16, 100])
    ap.add_argument("--chain", action="store_true")
    args = ap.parse_args()
    gpu, power_w = gpu_identity()
    for n_cams in args.cams:
        kwargs = batch(n_cams, args.chain)
        for name, fn in (("torch", step_torch), ("kernel", step_kernel)):
            host_us, dev_us = measure(fn, kwargs, args.iters)
            print(json.dumps({"impl": name, "views": 16, "rays_per_view": 256, "n_cams": n_cams, "chain": args.chain,
                              "host_us_per_iter": round(host_us, 1), "cuda_event_us_per_iter": round(dev_us, 1),
                              "kernel_launches": launches(fn, kwargs), "gpu": gpu,
                              "power_limit_w": power_w}), flush=True)


if __name__ == "__main__":
    main()
