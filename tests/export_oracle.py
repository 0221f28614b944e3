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


def mix64(x):
    """splitmix64's finaliser of uint64 keys (numpy array or int), the probe start of lrf_frame_points."""
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return x ^ (x >> np.uint64(31))


def pack_key(k):
    """voxel index [.., 3] (each in [-2^20, 2^20)) -> the table's 63-bit key."""
    k = np.asarray(k, np.int64) + KEY_LIM
    return (k[..., 0] << 2 * KEY_BITS) | (k[..., 1] << KEY_BITS) | k[..., 2]


def probe_table(keys, capacity):
    """The occupied slots of an insert-only linear-probing table of `capacity` (a power of two) slots after the
    distinct `keys` are inserted, each probing from mix64(key) & (capacity - 1) upwards and wrapping to 0.  The set of
    occupied slots does not depend on the insertion order, so a concurrent insert ends with the same set."""
    mask = capacity - 1
    taken = set()
    for h in (mix64(np.asarray(sorted(set(int(k) for k in keys)), np.uint64)) & np.uint64(mask)).tolist():
        slot = int(h)
        while slot in taken:
            slot = (slot + 1) & mask
        taken.add(slot)
    return taken


U32 = 2.0 ** -24                      # unit roundoff of float32


def point_cloud64(frames, cam2world, world2rf, blend_rows, min_acc, max_norm, voxel_size, origin, min_count=1,
                  slack=2.0):
    """An independent float64 reference of localrf_b200.export.point_cloud from the rendered chunks.

    frames: (view, rgb [m,3], depth [m], acc [m], dirs [m,3]) per chunk; cam2world [V,3,4] the views' camera-to-world
    matrices (LocalTensorfs.get_cam2world()), used as o = c2w[:, 3], R = c2w[:, :3]; world2rf [F,3]; blend_rows [V,F].
    A ray's point is o + (dirs @ R^T) depth / acc in float64; it is kept when acc >= min_acc, acc > 0, depth is finite
    and max_a |p_a + world2rf_k_a| <= max_norm for a field with blend > 0, and lands in voxel floor((p - origin) /
    voxel_size).  (voxel_size and origin are the float32 values the table holds.)

    Each ray also gets a bound on the float32 pipeline's error in p (`slack` times the unit roundoff of each of its
    operations); a ray is ambiguous when a decision lies within that bound of its boundary: acc against min_acc, |p_a +
    world2rf_k_a| against max_norm, or q_a = (p_a - origin_a) / voxel_size against an integer.

    -> dict(voxels {key: [count, sum p (3), sum clamp(rgb) (3), largest error bound of a float32 point's position in
    its voxel: q_a's bound times voxel_size]} of the voxels with at least min_count points, ambiguous {(chunk index,
    ray)}, ambiguous_keys {keys of the 27 voxels around each ambiguous ray}, kept, n_rays)."""
    vs = float(f32(voxel_size))
    org = np.array([float(f32(o)) for o in origin])
    w2 = np.asarray(world2rf, np.float64).reshape(-1, 3)
    voxels, ambiguous, amb_keys = {}, set(), set()
    kept = n_rays = 0
    for ci, (v, rgb, depth, acc, dirs) in enumerate(frames):
        rgb, depth, acc, dirs = (np.asarray(a, np.float64) for a in (rgb, depth, acc, dirs))
        M = np.asarray(cam2world[v], np.float64)
        o, R = M[:, 3], M[:, :3]
        n_rays += len(acc)
        with np.errstate(all="ignore"):
            s = depth / acc
            c = dirs * s[:, None]
            p = o + (dirs @ R.T) * s[:, None]
            # float32: s, c (2 roundings), three products and three sums per axis, then q (two more)
            err = slack * U32 * (2 * np.abs(c) @ np.abs(R).T * 3 + np.abs(o) + np.abs(p))
            keep = (acc >= min_acc) & (acc > 0) & np.isfinite(depth)
            amb = np.abs(acc - min_acc) <= slack * U32 * abs(min_acc)
            inside = np.zeros(len(acc), bool)
            for k in range(w2.shape[0]):
                if not blend_rows[v][k] > 0:
                    continue
                d = np.abs(p + w2[k])
                e = err + slack * U32 * (np.abs(w2[k]) + d)
                inside |= np.all(d <= max_norm, axis=1)
                amb |= np.any(np.abs(d - max_norm) <= e, axis=1)
            keep &= inside
            q = (p - org) / vs
            eq = (err + slack * U32 * np.abs(p - org)) / vs + slack * U32 * np.abs(q)
            kf = np.floor(q)
            keep &= np.all((kf >= -KEY_LIM) & (kf < KEY_LIM), axis=1)
            amb |= np.any(np.abs(q - np.round(q)) <= eq, axis=1)
            cl = np.clip(np.nan_to_num(rgb, nan=0.0), 0.0, 1.0)
        amb &= np.isfinite(p).all(1) & (acc > 0) & np.isfinite(depth)
        for r in np.nonzero(amb)[0].tolist():
            ambiguous.add((ci, r))
            base = np.floor(q[r])
            for dk in np.ndindex(3, 3, 3):
                kk = base + np.array(dk) - 1
                if np.all(np.abs(kk + 0.5) < KEY_LIM):
                    amb_keys.add(int(pack_key(kk.astype(np.int64))))
        idx = np.nonzero(keep)[0]
        kept += len(idx)
        keys = pack_key(kf[idx].astype(np.int64))
        for r, key in zip(idx.tolist(), keys.tolist()):
            cur = voxels.setdefault(key, [0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
            cur[0] += 1
            for a in range(3):
                cur[1 + a] += p[r, a]
                cur[4 + a] += cl[r, a]
            cur[7] = max(cur[7], float(eq[r].max()) * vs)
    voxels = {k: v for k, v in voxels.items() if v[0] >= min_count}
    return dict(voxels=voxels, ambiguous=ambiguous, ambiguous_keys=amb_keys, kept=kept, n_rays=n_rays)


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
