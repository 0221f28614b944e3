"""Render-launch time against the rows the launch shades: cfg2 and distB 4096-ray batches and 1024-ray cfg2 batches,
CUDA events around each launch with the L2 flushed before it, as bench.py times a step.  Each batch is timed on its
own with its shaded-row count (the render kernel's appearance-sample counter), and a least-squares line
time = fixed + per_row * rows over all of them gives the marginal cost of a 128-row MLP tile per SM.

usage: python tools/render_consumer_time.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import localrf_b200 as L  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_batches(name, n_rays, reps, batches, flush):
    dev = torch.device("cuda", 0)
    wl = bench.Workload(name, None)
    lt = wl.build(L.LocalTensorfs, quiet=True).to(dev)
    kw = wl.call_kwargs(lt, dev)
    ids_host, views_host = wl.batches()
    stats = torch.zeros(2, dtype=torch.int64, device=dev)
    out = []
    for bi in batches:
        ids = ids_host[bi][:n_rays].to(dev)
        view = views_host[bi].to(dev)
        for _ in range(3):
            lt(ids, view, bench.IMG_W, bench.IMG_H, **kw)
        stats.zero_()
        lt(ids, view, bench.IMG_W, bench.IMG_H, stats=stats, **kw)
        torch.cuda.synchronize()
        rows = int(stats[1])
        ms = []
        for _ in range(reps):
            flush.zero_(); flush.zero_()
            a, c = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            lt(ids, view, bench.IMG_W, bench.IMG_H, **kw)
            c.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(c))
        out.append({"workload": name, "rays": n_rays, "batch": int(bi), "rows": rows, "ms": float(np.median(ms))})
    del lt
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_consumer_time.py needs a CUDA device")
    torch.set_grad_enabled(False)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    batches = list(range(0, 156, 13))
    pts = (time_batches("cfg2", 4096, args.reps, batches, flush) + time_batches("distB", 4096, args.reps, batches, flush)
           + time_batches("cfg2", 1024, args.reps, batches, flush))
    rows = np.array([p["rows"] for p in pts], float)
    ms = np.array([p["ms"] for p in pts], float)
    per_row, fixed = np.polyfit(rows, ms, 1)
    groups = {}
    for p in pts:
        groups.setdefault(f'{p["workload"]} x{p["rays"]}', []).append(p)
    summary = {k: {"launches": len(v), "median_ms": float(np.median([p["ms"] for p in v])),
                   "median_rows": float(np.median([p["rows"] for p in v])),
                   "tiles_per_sm": float(np.median([p["rows"] for p in v])) / 128 / n_sms} for k, v in groups.items()}
    print(json.dumps({"card": card(), "n_sms": n_sms, "by_batch_kind": summary,
                      "fit": {"fixed_ms": float(fixed), "ms_per_row": float(per_row),
                              "us_per_tile_per_sm": float(per_row * 128 * n_sms * 1e3)},
                      "points": pts}, indent=1))


if __name__ == "__main__":
    main()
