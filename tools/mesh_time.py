"""Times the mesh export (localrf_b200.export.mesh) on a cfg5-like scene: two 640^3 fields, at voxel 1/128 and 1/256.

Prints CUDA-event time per stage (lattice, cells, extract, normals + colours), lattice points per second, and the
vertex and triangle counts at a few levels, with the card's name and power limit read in the same run.

    python tools/mesh_time.py
"""
import ctypes as C
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
import localrf_b200 as L  # noqa: E402
from localrf_b200 import _lib, export  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def stage_times(lt, voxel, level):
    """The export's stages one by one, each between CUDA events (the same calls export.mesh makes)."""
    lib = _lib.lib()
    n = len(lt.tensorfs)
    w2rf = torch.stack([w.detach().float().reshape(3) for w in lt.world2rf]).contiguous()
    fields = (_lib.LrfField * n)(*[rf._field() for rf in lt.tensorfs])
    steps = (C.c_float * n)(*[float(rf.stepSize) for rf in lt.tensorfs])
    s = _lib.LrfMeshScene(n_fields=n, fields=fields, step_size=steps, world2rf=w2rf.data_ptr(), voxel_size=voxel,
                          max_norm=1.0, level=level)
    brick = 64
    bricks = export._mesh_bricks(w2rf.tolist(), voxel, (0.0, 0.0, 0.0), 1.0, brick)
    cap, max_tri = 1 << 24, 1 << 25
    words = cap + (3 * cap + 1) // 2 + max_tri + (3 * max_tri + 1) // 2
    store = torch.zeros(words + 4, dtype=torch.int64, device="cuda")
    b = store.data_ptr()
    tk = b + 8 * cap + 8 * ((3 * cap + 1) // 2)
    t = _lib.LrfMeshTable(capacity=cap, max_triangles=max_tri, keys=b, verts=b + 8 * cap, tri_keys=tk,
                          tri_slots=tk + 8 * max_tri, stats=b + 8 * words)
    values = torch.empty((brick + 1) ** 3, device="cuda")
    dims = (C.c_int32 * 3)(brick + 1, brick + 1, brick + 1)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    lat = cel = 0.0
    for lo in bricks:
        lo = (C.c_int32 * 3)(*lo)
        ev[0].record()
        _lib.check(lib.lrf_mesh_lattice(C.byref(s), lo, dims, values.data_ptr(), None))
        ev[1].record()
        _lib.check(lib.lrf_mesh_cells(C.byref(s), lo, dims, values.data_ptr(), C.byref(t), None))
        ev[2].record()
        torch.cuda.synchronize()
        lat += ev[0].elapsed_time(ev[1])
        cel += ev[1].elapsed_time(ev[2])
    nb = lib.lrf_mesh_extract_scratch_bytes(cap, max_tri)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    xyz = torch.empty(cap // 2, 3, device="cuda")
    faces = torch.empty(max_tri, 3, dtype=torch.int32, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    ev[0].record()
    _lib.check(lib.lrf_mesh_extract(C.byref(t), xyz.data_ptr(), faces.data_ptr(), counts.data_ptr(),
                                    scratch.data_ptr(), nb, None))
    ev[1].record()
    torch.cuda.synchronize()
    ext = ev[0].elapsed_time(ev[1])
    return lat, cel, ext, len(bricks) * (brick + 1) ** 3, counts.tolist()


def main():
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", 640, n_init_frames=2, density_shift=2.0)
    lt.append_rf(2)
    lt = lt.to("cuda")
    with torch.no_grad():
        lt.world2rf[1].add_(torch.tensor([-0.5, 0.0, 0.0], device="cuda"))
    print(f"card: {card()}")
    for voxel in (1 / 128, 1 / 256):
        export.mesh(lt, voxel_size=voxel)                     # warm-up: library load, allocator
        lat, cel, ext, pts, (nv, nt) = stage_times(lt, voxel, 0.005)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = export.mesh(lt, voxel_size=voxel)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        print(f"voxel 1/{round(1 / voxel)}: lattice {lat:.1f} ms ({pts / lat / 1e6:.2f} G points/s), cells {cel:.1f} ms, "
              f"extract {ext:.1f} ms, mesh() end to end {total * 1e3:.1f} ms; {nv} vertices, {nt} triangles")
        for level in (0.001, 0.005, 0.05, 0.5):
            m = export.mesh(lt, voxel_size=voxel, level=level)
            print(f"  level {level}: {len(m['xyz'])} vertices, {len(m['faces'])} triangles")


if __name__ == "__main__":
    main()
