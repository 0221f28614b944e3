"""Times floater removal (localrf_b200.export.keep_components) on the meshes of tools/mesh_time.py -- two random-init
640^3 fields meshed at voxel 1/128 and 1/256 -- and on a synthetic worst case for union-find: one path of 2^22
vertices whose edges are listed in descending order, so each union hooks the path's old root under the next vertex.

Prints CUDA-event time of lrf_mesh_components and lrf_components_select (median of 5 after a warm-up), keep_components
end to end (host clock around a synchronised call), and, as context, scipy.sparse.csgraph.connected_components on the
host copy of the faces, with the card's name and power limit read in the same run.

    python tools/components_time.py
"""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.sparse import coo_matrix  # noqa: E402
from scipy.sparse.csgraph import connected_components  # noqa: E402

import bench  # noqa: E402
import localrf_b200 as L  # noqa: E402
from localrf_b200 import _lib, export  # noqa: E402

REPS = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def event_ms(fn):
    """Median CUDA-event time of fn() over REPS calls, after one warm-up call."""
    fn()
    ts = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def host_ms(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def measure(name, m):
    lib = _lib.lib()
    faces, V = m["faces"], m["xyz"].shape[0]
    T = faces.shape[0]
    label = torch.empty(V, dtype=torch.int32, device="cuda")
    size = torch.empty(V, dtype=torch.int64, device="cuda")
    tail = torch.zeros(5, dtype=torch.int64, device="cuda")
    nb = lib.lrf_components_select_scratch_bytes(V)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = [torch.empty(V, dtype=torch.int32, device="cuda") for _ in range(2)] + \
        [torch.empty(V, dtype=torch.int64, device="cuda")]

    def link():
        _lib.check(lib.lrf_mesh_components(faces.data_ptr(), T, V, label.data_ptr(), size.data_ptr(),
                                           tail.data_ptr() + 32, None))

    def sel():
        _lib.check(lib.lrf_components_select(label.data_ptr(), size.data_ptr(), V, 1, 0, out[0].data_ptr(),
                                             out[1].data_ptr(), out[2].data_ptr(), tail.data_ptr(), scratch.data_ptr(),
                                             nb, None))

    t_link, t_sel = event_ms(link), event_ms(sel)
    t_all = host_ms(lambda: export.keep_components(m, keep=1))
    clean = export.keep_components(m, keep=1)
    f = faces.cpu().numpy().astype(np.int64)
    t0 = time.perf_counter()
    g = coo_matrix((np.ones(2 * T, np.int8), (np.concatenate([f[:, 0], f[:, 0]]), np.concatenate([f[:, 1], f[:, 2]]))),
                   shape=(V, V))
    n_comp, _ = connected_components(g, directed=False)
    t_scipy = (time.perf_counter() - t0) * 1e3
    print(f"{name}: {V / 1e6:.2f} M vertices, {T / 1e6:.2f} M triangles, {n_comp} component{'s' * (n_comp != 1)} "
          f"(the largest {int(clean['sizes'][0])} triangles): lrf_mesh_components {t_link:.2f} ms, lrf_components_select (keep=1) "
          f"{t_sel:.2f} ms, keep_components end to end {t_all:.2f} ms; scipy connected_components on the host copy "
          f"{t_scipy:.0f} ms")


def main():
    print(f"card: {card()}")
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", 640, n_init_frames=2, density_shift=2.0)
    lt.append_rf(2)
    lt = lt.to("cuda")
    with torch.no_grad():
        lt.world2rf[1].add_(torch.tensor([-0.5, 0.0, 0.0], device="cuda"))
    for voxel in (1 / 128, 1 / 256):
        measure(f"mesh at voxel 1/{round(1 / voxel)}", export.mesh(lt, voxel_size=voxel))
    del lt
    V = 1 << 22
    i = torch.arange(V - 1, 0, -1, dtype=torch.int32, device="cuda")            # edges (i - 1, i), i descending
    path = dict(xyz=torch.zeros(V, 3, device="cuda"), faces=torch.stack([i - 1, i, i], 1).contiguous())
    measure("path of 2^22 vertices, edges in descending order", path)


if __name__ == "__main__":
    main()
