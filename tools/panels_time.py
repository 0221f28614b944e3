"""Test-frame comparison panels timing (renderer.py:79-124): the reference's block -- its torch calls on the device,
the two .cpu() reads of the predicted flows, cv2.resize and np.quantile on the host, compute_depth_loss after an
upload -- against metrics.test_panels (host time per call with a synchronisation, and CUDA-event time of
back-to-back calls) and against FramePipeline frames with and without panels=.  Sizes: 480x270 frames from 960x540
data and 960x540 frames from 1920x1080 data.  The reference arm needs a staged copy (oracle/_ref)."""
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


def reference_utils():
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
    return U


def reference_block(U, depth_map, directions, ij, cam2world, idx, focal, center, W, H, gt):
    """renderer.py:79-124 with the reference's functions; the inline numpy / cv2 lines restated."""
    import cv2
    view_ids = torch.tensor([idx], device=depth_map.device)
    fwd_c2c, bwd_c2c = U.get_fwd_bwd_cam2cams(cam2world, view_ids)
    pts = directions[None] * depth_map[None, ..., None]
    out = []
    for c2c, fl, mk in ((fwd_c2c, gt["fwd_flow"], gt["fwd_mask"]), (bwd_c2c, gt["bwd_flow"], gt["bwd_mask"])):
        pred = U.get_pred_flow(pts, ij, c2c, focal, center).cpu().numpy().reshape(H, W, 2)
        flow = cv2.resize(fl, (W, H), interpolation=cv2.INTER_NEAREST)
        mask = cv2.resize(mk, (W, H), interpolation=cv2.INTER_NEAREST)
        cols = []
        for c in range(2):
            cmp = np.vstack([pred[..., c], flow[..., c]])
            cmp /= np.quantile(cmp, 0.9)
            cols.append(np.vstack([cmp, np.abs(pred[..., c] - flow[..., c]) * mask / W]))
        out.append(torch.from_numpy(np.hstack(cols)).clamp(0, 1))
    inv = torch.from_numpy(cv2.resize(gt["invdepth"], (W, H), interpolation=cv2.INTER_NEAREST)).to(depth_map.device)
    xn, gn, d = U.compute_depth_loss(1 / depth_map[None].clamp(1e-6), inv.view(1, -1))
    out.append(torch.vstack([0.5 * xn[0].reshape(H, W), 0.5 * gn[0].reshape(H, W), d[0].reshape(H, W)]).clamp(0, 1))
    torch.cuda.synchronize()
    return out


def ground_truth(rng, h0, w0):
    return dict(fwd_flow=(3 * rng.standard_normal((h0, w0, 2))).astype(np.float32),
                fwd_mask=(rng.random((h0, w0)) > 0.2).astype(np.float32),
                bwd_flow=(3 * rng.standard_normal((h0, w0, 2))).astype(np.float32),
                bwd_mask=(rng.random((h0, w0)) > 0.2).astype(np.float32),
                invdepth=(rng.random((h0, w0)) + 0.1).astype(np.float32))


def main():
    print(f"card: {card()}")
    dev = torch.device("cuda")
    U = reference_utils()
    rng = np.random.default_rng(0)
    lt = bench.build_scene(dev)                                  # cfg2: 300^3
    cam2world = lt.get_cam2world()
    n_launch = 50
    for (W, H), (w0, h0) in (((480, 270), (960, 540)), ((960, 540), (1920, 1080))):
        gt = ground_truth(rng, h0, w0)
        gt_dev = {k: torch.from_numpy(v).to(dev) for k, v in gt.items()}
        view = torch.tensor([0], device=dev)
        ids = torch.arange(W * H, device=dev)
        _, depth, dirs, ij = lt(ids, view, W, H, is_train=False)
        focal, center = lt.focal(W), lt.center(W, H)
        args = (depth, dirs, cam2world, 0, focal, center, W, H)
        for _ in range(5):
            L.metrics.test_panels(*args, **gt_dev)
        torch.cuda.synchronize()
        t_dev_in = median_host(lambda: (L.metrics.test_panels(*args, **gt_dev), torch.cuda.synchronize()), 20)
        t_np_in = median_host(lambda: (L.metrics.test_panels(*args, **gt), torch.cuda.synchronize()), 20)
        torch.cuda._sleep(200_000_000)                          # keep the GPU busy while the host enqueues
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n_launch):
            L.metrics.test_panels(*args, **gt_dev)
        b.record()
        torch.cuda.synchronize()
        t_ev = a.elapsed_time(b) / n_launch
        line = (f"{W}x{H} from {w0}x{h0}: test_panels {t_ev * 1e3:.0f} us per frame (CUDA events, {n_launch} "
                f"back-to-back calls); host per call with sync: {t_dev_in * 1e3:.2f} ms (device ground truth), "
                f"{t_np_in * 1e3:.2f} ms (numpy ground truth, uploads included)")
        if U is not None:
            ref_args = (U, depth, dirs, ij, cam2world, 0, focal, center, W, H, gt)
            reference_block(*ref_args)
            t_ref = median_host(lambda: reference_block(*ref_args), 5)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            reference_block(*ref_args)
            b.record()
            torch.cuda.synchronize()
            line += f"; reference block {t_ref * 1e3:.1f} ms host ({a.elapsed_time(b):.1f} ms between CUDA events)"
        print(line)

        for label, panels in (("without panels", None), ("with panels (numpy gt)", dict(idx=0, **gt)),
                              ("with panels (device gt)", dict(idx=0, **gt_dev))):
            pipe = L.FramePipeline(lt, W, H, n_buffers=3)
            frames = [(view, {} if panels is None else {"panels": panels})] * 16
            for _ in pipe.render(frames[:4]):
                pass
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            list(pipe.render(frames))
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            print(f"  FramePipeline, 16 cfg2 {W}x{H} frames, {label}: {t / 16 * 1e3:.2f} ms per frame")


if __name__ == "__main__":
    main()
