"""Times colouring a mesh from the frames (localrf_b200.export.frame_colours) on the mesh_time.py scene: two 640^3
fields, meshed at voxel 1/128 and 1/256, with frames of 960x540 and 1920x1080.

Per frame, between CUDA events: the view's render with weights and opacity (the same calls frame_colours makes), and
the colour kernel (lrf_frame_colours) over every vertex, with normals and the default options, and without normals
under options that colour every vertex projecting into the frame (the random fields' fog does not match the mesh's
depth, and their cube-boundary mesh faces away from the cameras inside it); then frame_colours end to end over all
views with host images.  The card's name and power limit are read in the same run.

    python tools/colour_time.py
"""
import ctypes as C
import math
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import localrf_b200 as L  # noqa: E402
from localrf_b200 import _lib, export  # noqa: E402
from localrf_b200.tensorf import _stream  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def per_frame(lt, m, W, H, reps, opts, normals=True):
    """Mean CUDA-event ms of the render and of the colour kernel for one view, over `reps` passes of every view, and
    the vertices that view coloured on average."""
    dev = torch.device("cuda")
    lib = _lib.lib()
    S, per_chunk = export._chunk_rays(lt, 256 << 20, dev)
    n = W * H
    chunk = min(per_chunk, n)
    ids = torch.arange(n, dtype=torch.int64, device=dev)
    weights = torch.empty(chunk * S, dtype=torch.float32, device=dev)
    frame = (torch.empty(n, 3, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev))
    image = torch.rand(H, W, 3, device=dev)
    P = len(m["xyz"])
    sums = torch.zeros(P, 5, dtype=torch.int64, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    render = colour = 0.0
    count = 0
    with torch.no_grad():
        stream = _stream(dev)
        for rep in range(reps + 1):
            for v in range(len(lt.r_c2w)):
                ev[0].record()
                plan = None
                for _, plan, *_ in export._render_view(lt, v, W, H, False, chunk, ids, weights, dev, frame):
                    pass
                ev[1].record()
                f = _lib.LrfColourFrame(W=W, H=H, fov360=0, intrinsics=plan.keep[1].data_ptr(),
                                        cam2world=plan.keep[0].data_ptr(), depth=frame[1].data_ptr(),
                                        acc=frame[2].data_ptr(), image=image.data_ptr(), **opts)
                nrm = m["normals"].data_ptr() if normals else None
                _lib.check(lib.lrf_frame_colours(C.byref(f), m["xyz"].data_ptr(), nrm, P, sums.data_ptr(), stream))
                ev[2].record()
                torch.cuda.synchronize()
                if rep > 0:                                   # pass 0 warms up plans, modules and the allocator
                    render += ev[0].elapsed_time(ev[1])
                    colour += ev[1].elapsed_time(ev[2])
                    count += 1
    return render / count, colour / count, int(sums[:, 0].sum()) / ((reps + 1) * len(lt.r_c2w))


def main():
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", 640, n_init_frames=2, density_shift=2.0)
    lt.append_rf(2)
    lt = lt.to("cuda")
    with torch.no_grad():
        lt.world2rf[1].add_(torch.tensor([-0.5, 0.0, 0.0], device="cuda"))
    print(f"card: {card()}")
    rng = np.random.default_rng(0)
    for voxel in (1 / 128, 1 / 256):
        m = export.mesh(lt, voxel_size=voxel)
        print(f"voxel 1/{round(1 / voxel)}: {len(m['xyz'])} vertices")
        for W, H in ((960, 540), (1920, 1080)):
            render, colour, kept = per_frame(lt, m, W, H, 2, dict(min_acc=0.5, depth_tol=0.02, min_cos=0.1))
            _, every, kept_all = per_frame(lt, m, W, H, 2, dict(min_acc=-math.inf, depth_tol=1e30, min_cos=1.0),
                                          normals=False)
            frames = [(v, rng.random((H, W, 3), dtype=np.float32)) for v in range(len(lt.r_c2w))]
            export.frame_colours(lt, m["xyz"], frames[:1], normals=m["normals"])          # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fc = export.frame_colours(lt, m["xyz"], frames, normals=m["normals"])
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
            seen = int((fc["count"] > 0).sum())
            print(f"  {W}x{H}: render + weights {render:.2f} ms per frame; colour kernel {colour:.3f} ms per frame "
                  f"({kept:.0f} vertices coloured per frame), {every:.3f} ms without normals and with every "
                  f"projected vertex coloured ({kept_all:.0f}); frame_colours over {len(frames)} host frames "
                  f"{total * 1e3:.1f} ms, {seen} vertices coloured")


if __name__ == "__main__":
    main()
