"""GPU: the connected components of exported geometry (lrf_mesh_components / lrf_point_components /
lrf_components_select and localrf_b200.export.keep_components) against the scipy restatement of
tests/components_oracle.py bit for bit: labels, sizes, the ranking and selection, new_index and the compacted
outputs, with canary words after every output buffer."""
import ctypes as C

import numpy as np
import pytest
import torch

import components_oracle as co
from gpu_helpers import components_boxes, components_scene
from localrf_b200 import _lib
from localrf_b200.export import keep_components, mesh, point_cloud, write_ply

pytestmark = pytest.mark.gpu
PAD = 16
CANARY = -123456789


def _buf(n, dtype):
    return torch.full((n + PAD,), CANARY, dtype=dtype, device="cuda")


def _intact(t, n):
    assert (t[n:] == CANARY).all(), "a canary word past the written rows changed"


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype).contiguous()


def mesh_cc(faces, V):
    """lrf_mesh_components -> (label, size, stats[0]) as numpy, canaries checked."""
    f = _dev(np.asarray(faces, np.int64).reshape(-1, 3), torch.int32)
    T = f.shape[0]
    label, size, stats = _buf(V, torch.int32), _buf(V, torch.int64), _buf(1, torch.int64)
    _lib.check(_lib.lib().lrf_mesh_components(f.data_ptr() if T else None, T, V, label.data_ptr(), size.data_ptr(),
                                              stats.data_ptr(), None))
    torch.cuda.synchronize()
    for t, n in ((label, V), (size, V), (stats, 1)):
        _intact(t, n)
    return label[:V].cpu().numpy(), size[:V].cpu().numpy(), int(stats[0])


def point_cc(xyz, origin, cell, capacity):
    """lrf_point_components -> (label, size, stats[0], stats[1]) as numpy, canaries checked."""
    x = _dev(np.asarray(xyz, np.float32).reshape(-1, 3), torch.float32)
    n = x.shape[0]
    keys, first = _buf(capacity, torch.int64), _buf(capacity, torch.int32)
    label, size, stats = _buf(n, torch.int32), _buf(n, torch.int64), _buf(2, torch.int64)
    _lib.check(_lib.lib().lrf_point_components(x.data_ptr() if n else None, n, (C.c_float * 3)(*origin), cell,
                                               keys.data_ptr(), first.data_ptr(), capacity, label.data_ptr(),
                                               size.data_ptr(), stats.data_ptr(), None))
    torch.cuda.synchronize()
    for t, m in ((keys, capacity), (first, capacity), (label, n), (size, n), (stats, 2)):
        _intact(t, m)
    return label[:n].cpu().numpy(), size[:n].cpu().numpy(), int(stats[0]), int(stats[1])


def select(label, size, keep=0, min_size=0):
    """lrf_components_select on numpy label / size -> the oracle's dict layout, canaries checked."""
    n = len(label)
    lib = _lib.lib()
    lb, sz = _dev(label, torch.int32), _dev(size, torch.int64)
    nb = lib.lrf_components_select_scratch_bytes(n) if n else 0
    assert nb > 0 or n == 0
    scratch = torch.full((max(nb, 1),), 0x5A, dtype=torch.uint8, device="cuda")
    new_index, rank, sizes, counts = _buf(n, torch.int32), _buf(n, torch.int32), _buf(n, torch.int64), \
        _buf(4, torch.int64)
    _lib.check(lib.lrf_components_select(lb.data_ptr() if n else None, sz.data_ptr() if n else None, n, keep, min_size,
                                         new_index.data_ptr(), rank.data_ptr(), sizes.data_ptr(), counts.data_ptr(),
                                         scratch.data_ptr() if n else None, nb, None))
    torch.cuda.synchronize()
    c = counts[:4].cpu().tolist()
    for t, m in ((new_index, n), (counts, 4)):
        _intact(t, m)
    assert (rank[c[0]:n] == CANARY).all() and (sizes[c[2]:n] == CANARY).all()
    return dict(new_index=new_index[:n].cpu().numpy(), rank=rank[:c[0]].cpu().numpy(),
                sizes=sizes[:c[2]].cpu().numpy(), counts=c)


def same_selection(got, want):
    assert got["counts"] == want["counts"]
    for k in ("new_index", "rank", "sizes"):
        assert np.array_equal(got[k], want[k]), k


def check_mesh(faces, V, selections=((0, 0), (1, 0), (3, 2), (0, 5))):
    label, size, bad = mesh_cc(faces, V)
    wl, ws, wb = co.mesh_components(faces, V)
    assert np.array_equal(label, wl) and np.array_equal(size, ws) and bad == wb
    for keep, min_size in selections:
        same_selection(select(label, size, keep, min_size), co.select(wl, ws, keep, min_size))
    return label, size


def soup(rng, n_comp, V, extra_tris=2.0, isolated=0.05):
    """A triangle soup of n_comp planted components over V vertices with shuffled ids (about `isolated` of the vertices
    in no triangle), in shuffled triangle order: each component a random tree of triangles plus extra triangles inside
    it."""
    perm = rng.permutation(V)
    used = perm[:int(V * (1 - isolated))]
    cuts = np.sort(rng.choice(np.arange(1, len(used)), n_comp - 1, replace=False))
    tris = []
    for part in np.split(used, cuts):
        if len(part) == 1:
            tris.append([part[0]] * 3)
            continue
        k = np.arange(1, len(part))
        parent = part[(rng.random(len(k)) * k).astype(np.int64)]
        tris.append(np.stack([part[k], parent, part[rng.integers(0, len(part), len(k))]], 1))
        m = int(extra_tris * len(part))
        tris.append(part[rng.integers(0, len(part), (m, 3))])
    f = np.concatenate([np.asarray(t).reshape(-1, 3) for t in tris])
    return f[rng.permutation(len(f))].astype(np.int32)


@pytest.mark.parametrize("seed, n_comp, V", [(0, 5, 1000), (1, 300, 20000), (2, 5000, 200000), (3, 2, 3)])
def test_random_soups_with_planted_components(seed, n_comp, V):
    rng = np.random.default_rng(seed)
    f = soup(rng, n_comp, V)
    label, _ = check_mesh(f, V)
    assert len(np.unique(label[np.unique(f)])) == n_comp


@pytest.mark.parametrize("seed", range(2))
def test_triangle_order_and_index_rotation_change_nothing(seed):
    rng = np.random.default_rng(10 + seed)
    V = 50000
    f = soup(rng, 700, V)
    base = mesh_cc(f, V)
    sel = select(base[0], base[1], 0, 3)
    g = f[rng.permutation(len(f))]
    r = rng.integers(0, 3, len(g))
    g = np.stack([g[np.arange(len(g)), (r + j) % 3] for j in range(3)], 1)
    for faces in (g, f[::-1], np.roll(f, 1, axis=1)):
        other = mesh_cc(faces, V)
        assert all(np.array_equal(a, b) for a, b in zip(base, other))
        same_selection(select(other[0], other[1], 0, 3), sel)


@pytest.mark.parametrize("order", ["ascending", "descending", "random"])
def test_long_path(order):
    """A path of 2^20 vertices, edge i joining i and i + 1 (a degenerate triangle), in the given order."""
    V = 1 << 20
    i = np.arange(V - 1)
    f = np.stack([i, i + 1, i + 1], 1)
    if order == "descending":
        f = f[::-1]
    elif order == "random":
        f = f[np.random.default_rng(5).permutation(len(f))]
    label, size, bad = mesh_cc(f, V)
    assert bad == 0 and (label == 0).all() and size[0] == V - 1 and (size[1:] == 0).all()
    s = select(label, size, keep=1)
    assert s["counts"] == [V, 1, 1, V - 1] and np.array_equal(s["new_index"], np.arange(V))


def test_star_spanning_tree_singletons_and_empty():
    rng = np.random.default_rng(7)
    V = 100000
    leaves = rng.permutation(np.arange(1, V))
    check_mesh(np.stack([leaves, np.full(V - 1, 0), leaves], 1), V)                         # star at 0
    check_mesh(np.stack([leaves, np.full(V - 1, V // 2), leaves], 1), V)                    # star at a middle vertex
    parent = (rng.random(V - 1) * np.arange(1, V)).astype(np.int64)
    p = rng.permutation(V)
    label, size = check_mesh(np.stack([p[1:], p[parent], p[1:]], 1)[rng.permutation(V - 1)], V)   # one component
    assert (label == 0).all()
    label, size = check_mesh(np.zeros((0, 3), np.int32), 1000)                              # all singletons
    assert np.array_equal(label, np.arange(1000)) and (size == 0).all()
    s = select(label, size)
    assert s["counts"] == [1000, 1000, 1000, 0] and np.array_equal(s["sizes"], np.zeros(1000))
    check_mesh(np.zeros((0, 3), np.int32), 0)                                               # V = 0, T = 0
    assert mesh_cc([[0, 1, 2], [3, 3, 3]], 0)[2] == 2                                       # V = 0, T > 0
    assert select(np.zeros(0, np.int32), np.zeros(0, np.int64), 2, 1)["counts"] == [0, 0, 0, 0]
    check_mesh([[5, 5, 5], [1, 1, 2], [2, 3, 3], [7, 7, 7], [7, 7, 7]], 9)                  # degenerate triangles


def test_out_of_range_faces_are_counted_and_skipped():
    rng = np.random.default_rng(8)
    V = 5000
    f = soup(rng, 40, V).astype(np.int64)
    bad = rng.random(len(f)) < 0.1
    f[bad, rng.integers(0, 3, bad.sum())] = rng.choice([-1, V, V + 1000, -(1 << 31), (1 << 31) - 1], bad.sum())
    label, size = check_mesh(f.astype(np.int32), V)
    assert mesh_cc(f.astype(np.int32), V)[2] == int(bad.sum())


def test_synthetic_grid_mesh_of_4m_triangles():
    """A 1480 x 1480 vertex grid, two triangles per quad, with every 16th row of quads removed (93 strips), against
    the oracle."""
    n = 1480
    y, x = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing="ij")
    keep = (y % 16) != 15
    v = (y * n + x)[keep]
    f = np.concatenate([np.stack([v, v + 1, v + n + 1], 1), np.stack([v, v + n + 1, v + n], 1)]).astype(np.int32)
    assert len(f) > 4_000_000
    label, size = check_mesh(f, n * n, selections=((0, 0), (1, 0), (10, 1)))
    assert len(np.unique(label)) == 93


# ---- point clouds ----------------------------------------------------------------------------------------------------
def check_points(xyz, origin, cell, capacity, selections=((0, 0), (1, 0), (0, 3))):
    label, size, cells, out = point_cc(xyz, origin, cell, capacity)
    wl, ws, wc, wo = co.point_components(xyz, origin, cell)
    assert np.array_equal(label, wl) and np.array_equal(size, ws) and (cells, out) == (wc, wo)
    for keep, min_size in selections:
        same_selection(select(label, size, keep, min_size), co.select(wl, ws, keep, min_size))
    return label, size


@pytest.mark.parametrize("seed", range(3))
def test_random_clouds(seed):
    rng = np.random.default_rng(20 + seed)
    centres = rng.uniform(-1, 1, (60, 3))
    pts = np.concatenate([c + rng.normal(0, rng.uniform(0.005, 0.05), (rng.integers(1, 2000), 3)) for c in centres])
    pts = pts.astype(np.float32)[rng.permutation(len(pts))]
    label, _ = check_points(pts, (0.01, -0.02, 0.003), 1 / 64, 1 << 17)
    assert len(np.unique(label)) > 10


def test_cell_boundaries_non_finite_points_and_out_of_range_cells():
    h = np.float32(0.25)
    k = np.arange(-6, 7, dtype=np.float32)
    grid = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3) * h           # exactly on cell corners
    sparse = grid[np.all(np.abs(grid / h) % 3 == 0, axis=1)]                               # cells two apart
    lim = np.float32(h * (1 << 20))
    odd = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [lim, 0, 0], [-lim, 0, 0],
                    [np.nextafter(lim, np.float32(0)), 0, 0], [0, -lim - h, 0]], np.float32)
    for pts in (grid, sparse, np.concatenate([sparse, odd, sparse[:5]])):
        check_points(pts, (0.0, 0.0, 0.0), float(h), 1 << 14)
    label, size, cells, out = point_cc(odd, (0.0, 0.0, 0.0), float(h), 16)
    assert out == 5 and cells == 2 and np.array_equal(label, np.arange(7))
    assert check_points(np.zeros((0, 3), np.float32), (0.0, 0.0, 0.0), 1.0, 2)[0].shape == (0,)


def test_point_table_overflow_raises_and_names_capacity():
    pts = np.random.default_rng(3).uniform(-1, 1, (5000, 3)).astype(np.float32)
    label, size, cells, out = point_cc(pts, (0.0, 0.0, 0.0), 1 / 64, 64)
    assert cells > 32
    cloud = dict(xyz=torch.from_numpy(pts).cuda(), rgb=torch.zeros(5000, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError, match="capacity"):
        keep_components(cloud, cell_size=1 / 64, capacity=64)
    assert len(keep_components(cloud, cell_size=1 / 64)["xyz"]) == 5000


# ---- through export ------------------------------------------------------------------------------------------------
def test_mesh_floater_is_removed_whole(tmp_path):
    lt = components_scene(grid=128)
    components_boxes(lt.tensorfs[0], [(-0.6, 0.2, -0.5, 0.5), (0.5, 0.7, 0.3, 0.5)], 0.4)   # the scene, and a floater
    w = lt.world2rf[0].detach().cpu().double().numpy()
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(-x) for x in w))
    before = {k: v.clone() for k, v in m.items()}
    xyz, f = m["xyz"].cpu().numpy(), m["faces"].cpu().numpy()
    floater = (xyz[f[:, 0]].astype(np.float64) + w)[:, 0] > 0.35
    assert 100 < floater.sum() < 0.2 * len(f)
    clean = keep_components(m, keep=1)
    assert all(torch.equal(m[k], before[k]) for k in m)                             # the input is untouched
    label, size, _ = co.mesh_components(f, len(xyz))
    want = co.select(label, size, keep=1)
    assert want["counts"][1:3] == [1, 2] and want["sizes"].tolist() == [int((~floater).sum()), int(floater.sum())]
    kx, kf, (kn, kc) = co.keep_mesh(xyz, f, want["new_index"], (m["normals"].cpu().numpy(), m["rgb"].cpu().numpy()))
    assert set(clean) == {"xyz", "normals", "rgb", "faces", "component", "sizes"}
    assert np.array_equal(clean["xyz"].cpu().numpy(), kx) and np.array_equal(clean["faces"].cpu().numpy(), kf)
    assert np.array_equal(clean["normals"].cpu().numpy(), kn) and np.array_equal(clean["rgb"].cpu().numpy(), kc)
    assert np.array_equal(clean["sizes"].cpu().numpy(), want["sizes"]) and (clean["component"] == 0).all()
    assert len(kf) == int((~floater).sum())                                         # exactly the floater's triangles
    assert np.array_equal(kx[kf].view(np.uint32), xyz[f[~floater]].view(np.uint32))   # each triangle's corners
    path = tmp_path / "clean.ply"
    write_ply(path, clean["xyz"], clean["rgb"], faces=clean["faces"], normals=clean["normals"])
    head = path.read_bytes().split(b"end_header\n")[0].decode()
    assert f"element vertex {len(kx)}\n" in head and f"element face {len(kf)}\n" in head
    everything = keep_components(m)
    assert all(torch.equal(everything[k], m[k]) for k in m) and everything["sizes"].tolist() == want["sizes"].tolist()
    with pytest.raises(ValueError, match="outside"):
        keep_components(dict(m, faces=torch.where(m["faces"] == 0, len(xyz), m["faces"])), keep=1)
    with pytest.raises(ValueError, match="cell_size"):
        keep_components(m, cell_size=0.1)


def test_point_cloud_components_equal_the_restatement():
    lt = components_scene(n_init_frames=3)
    vs = 1 / 128
    cloud = point_cloud(lt, 64, 48, voxel_size=vs, min_acc=0.05, capacity=1 << 16)
    xyz = cloud["xyz"].cpu().numpy()
    assert len(xyz) > 100
    label, size, _, _ = co.point_components(xyz, (0, 0, 0), vs)
    for keep, min_size in ((0, 0), (1, 0), (0, 5), (4, 2)):
        clean = keep_components(cloud, keep=keep, min_size=min_size, cell_size=vs)
        want = co.select(label, size, keep, min_size)
        rows = want["new_index"] >= 0
        assert set(clean) == set(cloud) | {"component", "sizes"}
        for k in ("xyz", "rgb", "count"):
            assert np.array_equal(clean[k].cpu().numpy(), cloud[k].cpu().numpy()[rows]), k
        assert np.array_equal(clean["component"].cpu().numpy(), want["rank"])
        assert np.array_equal(clean["sizes"].cpu().numpy(), want["sizes"])
        assert all(clean[k] == cloud[k] for k in ("n_rays", "n_kept", "n_out_of_range"))
    with pytest.raises(ValueError, match="cell_size"):
        keep_components(cloud)
    with pytest.raises(ValueError, match="one row per vertex"):
        keep_components(dict(cloud, rgb=cloud["rgb"][1:]), cell_size=vs)
