"""numpy / scipy restatement of the connected-components entries (include/localrf_b200.h: lrf_mesh_components,
lrf_point_components, lrf_components_select): scipy.sparse.csgraph.connected_components, its labels renamed to the
lowest index of each component, the cells' fp32 keys in numpy float32 (one rounding per operation, no fusion), and
the ranking, selection and stable compaction as numpy sorts."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

f32 = np.float32
KEY_BITS = 21
KEY_LIM = 1 << 20


def lowest_labels(n, a, b):
    """Labels of the graph on n nodes with edges (a[i], b[i]): each node's label is the lowest node of its component."""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    if n == 0:
        return np.zeros(0, np.int32)
    g = coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    low = np.full(comp.max() + 1, n, np.int64)
    np.minimum.at(low, comp, np.arange(n))
    return low[comp].astype(np.int32)


def mesh_components(faces, n_vertices):
    """-> label [V] int32, size [V] int64 (triangles at each root, 0 elsewhere), triangles with an index outside
    [0, V)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ok = np.all((f >= 0) & (f < n_vertices), axis=1)
    g = f[ok]
    label = lowest_labels(n_vertices, np.concatenate([g[:, 0], g[:, 0]]), np.concatenate([g[:, 1], g[:, 2]]))
    size = np.bincount(label[g[:, 0]], minlength=n_vertices).astype(np.int64)
    return label, size, int((~ok).sum())


def cells(xyz, origin, cell_size):
    """Per point: (in range, cell index [n, 3] int64, key uint64): k_a = floor((x_a - origin_a) / cell_size) in
    float32, in range when every k_a lies in [-2^20, 2^20)."""
    x = np.asarray(xyz, f32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        k = np.floor((x - np.asarray(origin, f32)) / f32(cell_size))
        ok = np.all((k >= -KEY_LIM) & (k < KEY_LIM), axis=1)
    ki = np.where(ok[:, None], k, 0).astype(np.int64)
    return ok, ki, cell_keys(ki)


def cell_keys(k):
    """The keys of cells k [m, 3] (each k_a in [-2^20, 2^20)), as cell_key packs them."""
    u = (np.asarray(k, np.int64).reshape(-1, 3) + KEY_LIM).astype(np.uint64)
    return (u[:, 0] << np.uint64(2 * KEY_BITS)) | (u[:, 1] << np.uint64(KEY_BITS)) | u[:, 2]


def probe_start(key):
    """splitmix64's finaliser in uint64 arithmetic (wrapping products): the probe start of each key, as lrf_table.cuh's
    probe_start."""
    x = np.asarray(key, np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xbf58476d1ce4e5b9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94d049bb133111eb)
        return x ^ (x >> np.uint64(31))


def colliding_cells(capacity, slot, lo, hi):
    """The cells k with lo <= k < hi (per axis) whose probe starts at `slot` of a table of `capacity`, in
    lexicographic order, int64 [m, 3]."""
    axes = [np.arange(a, b, dtype=np.int64) for a, b in zip(lo, hi)]
    k = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    return k[(probe_start(cell_keys(k)) & np.uint64(capacity - 1)) == np.uint64(slot)]


def table_ok(keys, first, xyz, origin, cell_size, capacity):
    """Checks the cell table keys / first [capacity] that lrf_point_components left for xyz: the tags are exactly the
    keys of the in-range cells plus one, each once; first[slot] is the lowest point of the slot's cell, and
    0x7fffffff at an empty slot; each key sits on its probe path, every slot from probe_start(key) & (capacity - 1) up
    to its own (wrapping past the last) occupied.  -> True, or AssertionError naming what is wrong."""
    tags = np.asarray(keys).view(np.uint64).reshape(-1)
    first = np.asarray(first, np.int64).reshape(-1)
    assert len(tags) == len(first) == capacity, "the table is not `capacity` slots"
    ok, _, key = cells(xyz, origin, cell_size)
    idx = np.nonzero(ok)[0]
    uniq, inv = np.unique(key[idx], return_inverse=True)
    low = np.full(len(uniq), len(ok), np.int64)
    np.minimum.at(low, inv, idx)
    occ = tags != 0
    slots = np.nonzero(occ)[0]
    held = tags[slots] - np.uint64(1)
    order = np.argsort(held)
    assert np.array_equal(held[order], uniq), "the table's keys are not the cells' keys, each once"
    assert np.array_equal(first[slots[order]], low), "first[slot] is not the lowest point of the slot's cell"
    assert (first[~occ] == 0x7fffffff).all(), "an empty slot's first is not 0x7fffffff"
    if len(slots) == 0:
        return True
    assert not occ.all(), "no empty slot"
    e0 = int(np.nonzero(~occ)[0][0])
    j = np.arange(capacity)
    rot = np.roll(occ, -(e0 + 1))                        # position j is slot (e0 + 1 + j) mod capacity
    last_empty = np.maximum.accumulate(np.where(rot, -1, j))
    run = j - last_empty - 1                             # occupied slots just before position j (itself excluded)
    pos = (slots - e0 - 1) % capacity
    start = (probe_start(held) & np.uint64(capacity - 1)).astype(np.int64)
    dist = (slots - start) % capacity
    bad = dist > run[pos]
    assert not bad.any(), f"key {int(held[bad][0])} at slot {int(slots[bad][0])} is off its probe path"
    return True


def point_components(xyz, origin, cell_size):
    """-> label [n] int32, size [n] int64 (points at each root), cells used, points not finite or out of range."""
    ok, ki, key = cells(xyz, origin, cell_size)
    n = len(key)
    idx = np.nonzero(ok)[0]
    uniq, inv = np.unique(key[idx], return_inverse=True)
    rep = np.full(len(uniq), n, np.int64)
    np.minimum.at(rep, inv, idx)                                  # each cell's lowest point
    a, b = [idx], [rep[inv]]
    ucell = ki[idx][np.unique(inv, return_index=True)[1]]          # cell index of each unique key, in key order
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                if (dx, dy, dz) <= (0, 0, 0):
                    continue
                m = ucell + np.array([dx, dy, dz])
                inr = np.all((m >= -KEY_LIM) & (m < KEY_LIM), axis=1)
                mk = cell_keys(np.where(inr[:, None], m, 0))
                pos = np.searchsorted(uniq, mk)
                hit = inr & (pos < len(uniq))
                hit[hit] = uniq[pos[hit]] == mk[hit]
                a.append(rep[hit])
                b.append(rep[pos[hit]])
    label = lowest_labels(n, np.concatenate(a), np.concatenate(b))
    size = np.bincount(label, minlength=n).astype(np.int64)
    return label, size, len(uniq), int((~ok).sum())


def select(label, size, keep=0, min_size=0):
    """lrf_components_select -> dict(new_index [n] int32, rank [n_rows] int32, sizes [K] int64, counts [4])."""
    label, size = np.asarray(label, np.int64), np.asarray(size, np.int64)
    n = len(label)
    roots = np.nonzero(label == np.arange(n))[0]
    s = np.clip(size[roots], 0, 2 ** 31 - 1)                     # negative sizes rank (and sum) as 0
    order = np.lexsort((roots, -s))                              # size descending, then label ascending
    sizes = s[order]
    i = np.arange(len(order))
    kept_comp = (sizes >= min_size) & ((keep == 0) | (i < keep))
    comp_rank = np.full(n, -1, np.int64)
    comp_rank[roots[order][kept_comp]] = i[kept_comp]
    vr = np.full(n, -1, np.int64)
    good = (label >= 0) & (label < n)
    vr[good] = comp_rank[label[good]]
    kept = vr >= 0
    new_index = np.where(kept, np.cumsum(kept) - 1, -1).astype(np.int32)
    counts = [int(kept.sum()), int(kept_comp.sum()), len(order), int(sizes[kept_comp].sum())]
    return dict(new_index=new_index, rank=vr[kept].astype(np.int32), sizes=sizes.astype(np.int64), counts=counts)


def keep_mesh(xyz, faces, new_index, extra=()):
    """The kept rows of xyz (and of each array of `extra`) and the kept triangles renumbered, in their original order."""
    rows = new_index >= 0
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    tri = f[new_index[f[:, 0]] >= 0] if len(f) else f
    return np.asarray(xyz)[rows], new_index[tri].astype(np.int32), [np.asarray(e)[rows] for e in extra]
