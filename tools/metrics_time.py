"""Test-frame metrics timing: lrf_image_metrics (CUDA events), metrics.rgb_ssim on numpy frames (host clock, upload
and sync included), the oracle's and -- when a staged copy is present (oracle/_ref) -- the reference's host
rgb_ssim, and FramePipeline over 32 cfg2 800x800 frames with and without gt."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bench  # noqa: E402
import localrf_b200 as L  # noqa: E402
import metrics_oracle as orc  # noqa: E402  (the tests' numpy restatement)
from localrf_b200 import metrics  # noqa: E402

torch.set_grad_enabled(False)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def median_host(fn, n):
    ts = []
    for _ in range(n):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    return sorted(ts)[n // 2]


def reference_rgb_ssim():
    ref = os.path.join(ROOT, "oracle", "_ref", "localTensoRF")
    if not os.path.isfile(os.path.join(ref, "utils", "utils.py")):
        return None
    from oracle import ref_loader
    for name, attrs in (("matplotlib", dict(use=lambda *a, **k: None)), ("matplotlib.pyplot", {}),
                        ("matplotlib.cm", {}), ("plyfile", {}), ("skimage", {}), ("skimage.measure", {})):
        ref_loader._stub(name, **attrs)
    sys.path.insert(0, ref)
    sys.modules.pop("utils", None)
    import utils.utils as U
    return U.rgb_ssim


def main():
    print(f"card: {card()}")
    dev = torch.device("cuda")
    ref_ssim = reference_rgb_ssim()
    g = torch.Generator(device="cuda").manual_seed(0)
    n_launch = 200
    for H, W in ((400, 400), (540, 960), (800, 800)):
        img = torch.rand(H, W, 3, device=dev, generator=g)
        gt = (img + 0.05 * torch.randn(H, W, 3, device=dev, generator=g)).clamp(0, 1)
        out = torch.empty(2, dtype=torch.float64, device=dev)
        for _ in range(20):
            metrics._enqueue(img, gt, out)
        torch.cuda.synchronize()
        # keep the GPU busy while the host enqueues, so the events time the kernels and not the launch overhead
        torch.cuda._sleep(100_000_000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n_launch):
            metrics._enqueue(img, gt, out)
        b.record()
        torch.cuda.synchronize()
        t_kernel = a.elapsed_time(b) / n_launch * 1e3
        a_np, b_np = gt.cpu().numpy(), img.cpu().numpy()
        t_host = median_host(lambda: metrics.rgb_ssim(a_np, b_np, 1), 20)
        t_orc = median_host(lambda: orc.ssim(a_np, b_np, 1.0), 3)
        line = (f"{W}x{H}: image_metrics {t_kernel:.1f} us per call (CUDA events, {n_launch} back-to-back calls); "
                f"rgb_ssim on numpy (upload + sync) {t_host * 1e3:.2f} ms; oracle (numpy, CPU) {t_orc * 1e3:.0f} ms")
        if ref_ssim is not None:
            line += f"; reference rgb_ssim (CPU) {median_host(lambda: ref_ssim(a_np, b_np, 1), 3) * 1e3:.0f} ms"
        print(line)

    lt = bench.build_scene(dev)                                  # cfg2: 300^3, one 800x800 frame
    W = H = 800
    view = torch.tensor([0], device=dev)
    with torch.no_grad():
        rgb, _, _, _ = lt(torch.arange(W * H, device=dev), view, W, H, is_train=False)
    gt_dev = (rgb.reshape(H, W, 3) + 0.03 * torch.randn(H, W, 3, device=dev, generator=g)).clamp(0, 1)
    gt_np = gt_dev.cpu().numpy()
    for label, gt in (("no gt", None), ("CUDA gt", gt_dev), ("numpy gt", gt_np)):
        pipe = L.FramePipeline(lt, W, H, n_buffers=3)
        frames = [(view, {} if gt is None else {"gt": gt})] * 32
        for _ in pipe.render(frames[:4]):
            pass
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = list(pipe.render(frames))
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        extra = "" if gt is None else f", ssim {got[-1]['ssim']:.6f}, mse {got[-1]['mse']:.3e}"
        print(f"FramePipeline, 32 cfg2 800x800 frames, {label}: {t * 1e3:.1f} ms ({t / 32 * 1e3:.2f} ms per frame{extra})")


if __name__ == "__main__":
    main()
