"""numpy restatement of the point-cloud export's kernels (include/localrf_b200.h: lrf_ray_opacity, lrf_frame_points,
lrf_voxel_extract): float32 operations in the kernels' order (numpy rounds every float32 operation once and never
fuses), np.cumsum in float64 for the sequential opacity sum, and Python integers for the voxel table."""
import math

import numpy as np

f32 = np.float32
KEY_BITS = 21
KEY_LIM = 1 << 20


def ray_opacity(weights, b, acc=None):
    """acc_k = (float) sum_s (double) w[r][s] in sample order; b * acc_k, added to `acc` when given.  weights [n, S]
    float32, b a float32 scalar or [n]."""
    acc_k = np.cumsum(np.asarray(weights, np.float64), axis=1)[:, -1].astype(f32)
    a = (np.asarray(b, f32) * acc_k).astype(f32)
    return a if acc is None else (np.asarray(acc, f32) + a).astype(f32)


def new_table():
    """{key: [count, sum f_x, sum f_y, sum f_z, sum r, sum g, sum b]} and the stats (points merged, out of range)."""
    return {"voxels": {}, "kept": 0, "out_of_range": 0}


def ray_points(rgb, depth, acc, dirs, c2w, world2rf, blend, min_acc, max_norm, voxel_size, origin):
    """Per ray: (keep, out_of_range, key int64, fraction sums uint64 [n,3], colour sums uint64 [n,3])."""
    rgb, depth, acc, dirs = (np.asarray(a, f32) for a in (rgb, depth, acc, dirs))
    M = np.asarray(c2w, f32).reshape(3, 4)
    w2 = np.asarray(world2rf, f32).reshape(-1, 3)
    vs = f32(voxel_size)
    org = np.asarray(origin, f32)
    with np.errstate(all="ignore"):
        keep = (acc >= f32(min_acc)) & (acc > 0) & np.isfinite(depth)
        s = depth / acc
        c = dirs * s[:, None]
        p = np.stack([((M[a, 0] * c[:, 0] + M[a, 1] * c[:, 1]) + M[a, 2] * c[:, 2]) + M[a, 3] for a in range(3)], 1)
        inside = np.zeros(len(acc), bool)
        for k in range(w2.shape[0]):
            if blend is not None and not (f32(blend[k]) > 0):
                continue
            inside |= np.all(np.abs(p + w2[k]) <= f32(max_norm), axis=1)
        keep &= inside
        q = (p - org) / vs
        k = np.floor(q)
        in_range = np.all((k >= -KEY_LIM) & (k < KEY_LIM), axis=1)
        out = keep & ~in_range
        keep &= in_range
        fr = q - k
        fu = np.zeros(fr.shape, np.uint64)
        fu[keep] = np.minimum((fr[keep] * f32(2.0 ** 32)).astype(np.uint64), np.uint64(2 ** 32 - 1))
        cu = (np.fmin(np.fmax(rgb, f32(0)), f32(1)) * f32(2.0 ** 24))
        cu = np.where(keep[:, None], cu, 0).astype(np.uint64)
        ki = np.where(keep[:, None], k, 0).astype(np.int64) + KEY_LIM
    key = (ki[:, 0] << 2 * KEY_BITS) | (ki[:, 1] << KEY_BITS) | ki[:, 2]
    return keep, out, key, fu, cu


def frame_points(table, rgb, depth, acc, dirs, c2w, world2rf, blend, min_acc, max_norm, voxel_size, origin):
    """Adds one view's kept rays to `table` (new_table())."""
    keep, out, key, fu, cu = ray_points(rgb, depth, acc, dirs, c2w, world2rf, blend, min_acc, max_norm, voxel_size,
                                        origin)
    table["kept"] += int(keep.sum())
    table["out_of_range"] += int(out.sum())
    if not keep.any():
        return table
    uk, inv = np.unique(key[keep], return_inverse=True)
    sums = np.zeros((len(uk), 7), np.uint64)
    np.add.at(sums[:, 0], inv, np.uint64(1))
    np.add.at(sums, (inv, slice(1, 4)), fu[keep])
    np.add.at(sums, (inv, slice(4, 7)), cu[keep])
    vox = table["voxels"]
    for kk, row in zip(uk.tolist(), sums.tolist()):
        cur = vox.setdefault(int(kk), [0] * 7)
        for j in range(7):
            cur[j] += int(row[j])
    return table


def extract(table, min_count, voxel_size, origin):
    """-> (xyz [P,3] float32, rgb [P,3] uint8, count [P] int32) in ascending key order, fp64 rounded once."""
    vs = float(f32(voxel_size))
    org = [float(f32(o)) for o in origin]
    keys = sorted(k for k, v in table["voxels"].items() if v[0] >= min_count)
    xyz = np.zeros((len(keys), 3), f32)
    rgb = np.zeros((len(keys), 3), np.uint8)
    count = np.zeros(len(keys), np.int32)
    for i, key in enumerate(keys):
        v = table["voxels"][key]
        cnt = float(v[0])
        fden, cden = cnt * 4294967296.0, cnt * 16777216.0
        for a in range(3):
            k = ((key >> (KEY_BITS * (2 - a))) & ((1 << KEY_BITS) - 1)) - KEY_LIM
            xyz[i, a] = f32(org[a] + (float(k) + float(v[1 + a]) / fden) * vs)
            rgb[i, a] = math.floor(float(v[4 + a]) / cden * 255.0 + 0.5)
        count[i] = min(v[0], 2 ** 31 - 1)
    return xyz, rgb, count


def read_ply(data):
    """(xyz, rgb) of a binary little-endian PLY with one vertex element of float x, y, z, uchar red, green, blue."""
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0", lines[:2]
    n = int(lines[2].split()[2])
    assert lines[2].startswith("element vertex ")
    props = [tuple(l.split()[1:]) for l in lines[3:-1]]
    assert props == [("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"), ("uchar", "green"),
                     ("uchar", "blue")], props
    body = np.frombuffer(data[end:], dtype=[("xyz", "<f4", 3), ("rgb", "u1", 3)])
    assert len(body) == n
    return body["xyz"].copy(), body["rgb"].copy()
