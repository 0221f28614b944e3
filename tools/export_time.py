"""Time the point-cloud export (localrf_b200.export.point_cloud) on a cfg5-like scene: 8 fields at 640^3 (bench.py's
cfg5 slice: 64 frames along -z, the reference's cross-fade rows), extended to 100 frames, rendered at 480x270 and
960x540.

    python tools/export_time.py [--frames 100] [--grid 640] [--min-acc 0.5]

The fields are freshly initialised; at bench.py's density_shift of -5 they are nearly transparent and no ray keeps a
point, so every field's density_shift is raised to 2 (bench.py's distB): the rays turn opaque near the camera, and
the point kernel and the merge get about one point per ray.  The table has 2^26 slots (2^25 voxels).

Per size, one JSON line:
  - per-frame CUDA-event time of the render with weights (lrf_render + lrf_ray_opacity per field) and of the point
    kernel (lrf_frame_points), from a pass that replays point_cloud's chunk loop with events around each part;
  - host time of the whole export (point_cloud, which ends in its one host read), median of 3;
  - rays, points kept, voxels written, peak device memory of the export;
  - the same integer merge as torch ops (keys and fixed-point sums from the exporter's per-frame outputs,
    torch.unique + index_add_ on int64), CUDA-event time, and whether its voxel count agrees.
Every line carries the GPU's name and power limit, read in the same call.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def scene(n_frames, grid):
    import bench
    import localrf_b200 as L
    lt = bench.Workload("cfg5", grid=grid).build(L.LocalTensorfs, quiet=True)
    for f in range(len(lt.r_c2w), n_frames):
        lt.append_frame()
        with torch.no_grad():
            lt.t_c2w[-1].copy_(torch.tensor([0.0, 0.0, -0.05 * f]))
    for rf in lt.tensorfs:
        rf.density_shift = 2.0
    return lt.to("cuda")


def split_times(lt, W, H, views, voxel_size, capacity, min_acc):
    """Median per-frame CUDA-event ms of (render + weights, point kernel), replaying point_cloud's loop."""
    from localrf_b200 import _lib
    from localrf_b200.tensorf import _stream
    dev = torch.device("cuda")
    n = W * H
    S = max(rf.sample_table(False, -1, dev).numel() for rf in lt.tensorfs)
    per_chunk = min((256 << 20) // (4 * S), n)
    store = torch.zeros(8 * capacity + 4, dtype=torch.int64, device=dev)
    t = _lib.LrfVoxelTable(capacity=capacity, voxel_size=voxel_size, keys=store.data_ptr(),
                           sums=store.data_ptr() + 8 * capacity, stats=store.data_ptr() + 64 * capacity)
    w2rf = torch.stack([w.detach() for w in lt.world2rf]).contiguous()
    rows = lt.blending_weights.detach().float().contiguous()
    ids = torch.arange(n, device=dev)
    weights = torch.empty(per_chunk * S, device=dev)
    lib = _lib.lib()
    render, points = [], []
    with torch.no_grad():
        for v in views:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            frames = []
            for lo in range(0, n, per_chunk):
                m = min(per_chunk, n - lo)
                plan = lt._eval_plan(v, m, W, H, False, dev)
                acc = torch.empty(m, device=dev)
                outs = lt._run_weights(plan, ids.data_ptr() + 8 * lo, lt._alloc_outputs(m, dev, None, None), weights,
                                       acc)
                frames.append((m, plan, outs, acc))
            ev[1].record()
            for m, plan, (rgb, depth, dirs, _), acc in frames:
                f = _lib.LrfPointFrame(n_rays=m, rgb=rgb.data_ptr(), depth=depth.data_ptr(), acc=acc.data_ptr(),
                                       directions=dirs.data_ptr(), cam2world=plan.keep[0].data_ptr(),
                                       world2rf=w2rf.data_ptr(), blend=rows[v].data_ptr(), n_fields=len(lt.tensorfs),
                                       min_acc=min_acc, max_norm=1.0)
                _lib.check(lib.lrf_frame_points(C.byref(f), C.byref(t), _stream(dev)))
            ev[2].record()
            torch.cuda.synchronize()
            render.append(ev[0].elapsed_time(ev[1]))
            points.append(ev[1].elapsed_time(ev[2]))
    return statistics.median(render), statistics.median(points)


def torch_merge(lt, frames, voxel_size, min_acc):
    """The export's merge as torch ops on the exporter's per-frame outputs -> voxel count (min_count 1)."""
    w2rf = torch.stack([w.detach() for w in lt.world2rf])
    rows = lt.blending_weights.detach().float()
    keys, sums = [], []
    for v, _, rgb, depth, acc, dirs in frames:
        c2w = lt.get_cam2world([v])[0].detach()
        s = depth / acc
        c = dirs * s[:, None]
        p = torch.stack([((c2w[a, 0] * c[:, 0] + c2w[a, 1] * c[:, 1]) + c2w[a, 2] * c[:, 2]) + c2w[a, 3]
                         for a in range(3)], 1)
        inside = torch.zeros_like(acc, dtype=torch.bool)
        for k in torch.nonzero(rows[v] > 0)[:, 0].tolist():
            inside |= ((p + w2rf[k]).abs() <= 1.0).all(1)
        q = p / voxel_size
        kf = torch.floor(q)
        keep = (acc >= min_acc) & (acc > 0) & torch.isfinite(depth) & inside & ((kf >= -2 ** 20) & (kf < 2 ** 20)).all(1)
        ki = kf[keep].long() + 2 ** 20
        keys.append((ki[:, 0] << 42) | (ki[:, 1] << 21) | ki[:, 2])
        fu = ((q - kf)[keep] * 2.0 ** 32).long().clamp(max=2 ** 32 - 1)
        cu = (rgb[keep].clamp(0, 1) * 2.0 ** 24).long()
        sums.append(torch.cat([torch.ones_like(fu[:, :1]), fu, cu], 1))
    uk, inv = torch.unique(torch.cat(keys), return_inverse=True)
    acc_sums = torch.zeros(len(uk), 7, dtype=torch.int64, device=uk.device).index_add_(0, inv, torch.cat(sums))
    return int(acc_sums.shape[0])


def main():
    from loss_time import gpu_identity
    from localrf_b200.export import point_cloud
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--grid", type=int, default=640)
    ap.add_argument("--min-acc", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("export_time.py measures on a CUDA device; none is available")
    gpu, power_w = gpu_identity()
    lt = scene(args.frames, args.grid)
    views = list(range(args.frames))
    vs, cap, kw = 1 / 256, 1 << 26, dict(min_acc=args.min_acc)
    for W, H in ((480, 270), (960, 540)):
        point_cloud(lt, W, H, view_ids=views[:2], voxel_size=vs, capacity=cap, **kw)          # warm-up
        render_ms, points_ms = split_times(lt, W, H, views, vs, cap, args.min_acc)
        host = []
        for _ in range(3):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            cloud = point_cloud(lt, W, H, view_ids=views, voxel_size=vs, capacity=cap, **kw)
            host.append(time.perf_counter() - t0)
            peak = torch.cuda.max_memory_allocated() - base
        frames = []
        point_cloud(lt, W, H, view_ids=views, voxel_size=vs, capacity=cap, _frames=frames, **kw)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        n_torch = torch_merge(lt, frames, vs, args.min_acc)
        b.record()
        torch.cuda.synchronize()
        del frames
        row = {"what": "point_cloud export", "fields": len(lt.tensorfs), "grid": f"{args.grid}^3",
               "frames": args.frames, "W": W, "H": H, "voxel_size": vs, "capacity": cap, "min_acc": args.min_acc,
               "render_weights_ms_per_frame": round(render_ms, 3), "point_kernel_ms_per_frame": round(points_ms, 3),
               "export_host_s": round(statistics.median(host), 3), "rays": cloud["n_rays"],
               "points_kept": cloud["n_kept"], "voxels": int(cloud["xyz"].shape[0]),
               "peak_device_mib": round(peak / 2 ** 20, 1), "torch_merge_ms": round(a.elapsed_time(b), 1),
               "torch_merge_voxels_equal": n_torch == int(cloud["xyz"].shape[0]), "gpu": gpu,
               "power_limit_w": power_w}
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
