"""-m gpu: the point-cloud export (localrf_b200.export, include/localrf_b200.h lrf_ray_opacity / lrf_frame_points /
lrf_voxel_extract).  The kernels equal their numpy restatement (tests/export_oracle.py) bit for bit on random and
adversarial rays, with canaries around every output; the export is repeatable across runs, view orders and chunkings;
on a small two-field scene the exporter's renders equal LocalTensorfs.forward, its opacity matches the field's own
weights, and its cloud equals the oracle's and a torch-op merge; a thin opaque slab exports onto its plane; and a table
too small for the cloud raises."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import export_oracle as eo
import localrf_b200 as L
from localrf_b200 import _lib
from localrf_b200.export import _voxel_table, point_cloud

pytestmark = pytest.mark.gpu

PAD = 64
CANARY_F = -12345.5


def _padded(n, cols, dtype, fill):
    shape = (n + 2 * PAD,) + ((cols,) if cols else ())
    return torch.full(shape, fill, dtype=dtype, device="cuda")


def _extract(t, store, min_count):
    """lrf_voxel_extract into canary-padded outputs -> (xyz, rgb, count, stats) on the host; every row outside the
    written ones keeps its canary."""
    lib = _lib.lib()
    cap = t.capacity
    nb = lib.lrf_voxel_extract_scratch_bytes(cap)
    assert nb > 0
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    xyz = _padded(cap, 3, torch.float32, CANARY_F)
    rgb = _padded(cap, 3, torch.uint8, 0xA5)
    cnt = _padded(cap, 0, torch.int32, -7)
    _lib.check(lib.lrf_voxel_extract(C.byref(t), min_count, xyz[PAD:].data_ptr(), rgb[PAD:].data_ptr(),
                                     cnt[PAD:].data_ptr(), store.data_ptr() + 8 * (8 * cap + 3), scratch.data_ptr(),
                                     nb, None))
    torch.cuda.synchronize()
    stats = store[8 * cap:].tolist()
    P = stats[3]
    for a, fill in ((xyz, CANARY_F), (rgb, 0xA5), (cnt, -7)):
        assert bool((a[:PAD] == fill).all()) and bool((a[PAD + P:] == fill).all()), "a canary was overwritten"
    return (xyz[PAD:PAD + P].cpu().numpy(), rgb[PAD:PAD + P].cpu().numpy(), cnt[PAD:PAD + P].cpu().numpy(), stats)


def _frame_points(t, rgb, depth, acc, dirs, c2w, w2rf, blend, min_acc, max_norm):
    cuda = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).cuda()
    keep = [cuda(a) for a in (rgb, depth, acc, dirs, c2w, w2rf)] + ([cuda(blend)] if blend is not None else [None])
    f = _lib.LrfPointFrame(n_rays=len(acc), rgb=keep[0].data_ptr(), depth=keep[1].data_ptr(), acc=keep[2].data_ptr(),
                           directions=keep[3].data_ptr(), cam2world=keep[4].data_ptr(), world2rf=keep[5].data_ptr(),
                           blend=None if keep[6] is None else keep[6].data_ptr(), n_fields=len(w2rf), min_acc=min_acc,
                           max_norm=max_norm)
    _lib.check(_lib.lib().lrf_frame_points(C.byref(f), C.byref(t), None))
    torch.cuda.synchronize()


# ---- 1. kernels vs the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,S,V,F", [(1, 1, 1, 1), (1000, 33, 4, 2), (1 << 18, 344, 2, 3)])
def test_ray_opacity_vs_oracle(n, S, V, F):
    g = torch.Generator().manual_seed(n + S)
    blend = torch.rand(V, F, generator=g)
    blend[0, 0] = 0.0
    acc = _padded(n, 0, torch.float32, CANARY_F)
    want = None
    lib = _lib.lib()
    for k in range(F):
        w = torch.rand(n, S, generator=g) ** 8
        w[torch.rand(n, S, generator=g) < 0.3] = 0.0
        w[:, 0] *= 1e-30
        wd, bd = w.cuda(), blend.cuda()
        _lib.check(lib.lrf_ray_opacity(wd.data_ptr(), n, S, V, bd.data_ptr() + 4 * k, F, int(k > 0),
                                       acc[PAD:].data_ptr(), None))
        b = blend[:, k].numpy().repeat(n // V)
        want = eo.ray_opacity(w.numpy(), b, want)
    torch.cuda.synchronize()
    assert bool((acc[:PAD] == CANARY_F).all()) and bool((acc[PAD + n:] == CANARY_F).all())
    assert np.array_equal(acc[PAD:PAD + n].cpu().numpy(), want)


def _random_rays(n, seed, n_fields):
    rng = np.random.default_rng(seed)
    dirs = np.concatenate([rng.uniform(-0.8, 0.8, (n, 2)), -np.ones((n, 1))], 1).astype(np.float32)
    depth = rng.uniform(0.05, 1.5, n).astype(np.float32)
    acc = rng.uniform(0, 1, n).astype(np.float32)
    rgb = rng.uniform(-0.1, 1.1, (n, 3)).astype(np.float32)
    m = max(n // 50, 1)
    idx = rng.choice(n, size=min(6 * m, n), replace=False)
    if n >= 6:
        depth[idx[:m]] = np.nan
        depth[idx[m:2 * m]] = np.inf
        acc[idx[2 * m:3 * m]] = 0.5                                  # exactly min_acc
        acc[idx[3 * m:4 * m]] = 0.0
        rgb[idx[4 * m:5 * m], 0] = np.nan
        depth[idx[5 * m:6 * m]] = 0.0
    a = rng.standard_normal(3) * 0.3
    R = _rot(a)
    c2w = np.concatenate([R, rng.uniform(-0.5, 0.5, (3, 1))], 1).astype(np.float32)
    w2rf = rng.uniform(-0.6, 0.6, (n_fields, 3)).astype(np.float32)
    blend = rng.uniform(0, 1, n_fields).astype(np.float32)
    if n_fields > 1:
        blend[-1] = 0.0
    return rgb, depth, acc, dirs, c2w, w2rf, blend


def _rot(a):
    cx, sx, cy, sy, cz, sz = math.cos(a[0]), math.sin(a[0]), math.cos(a[1]), math.sin(a[1]), math.cos(a[2]), math.sin(a[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


CASES = {   # (rays per frame, frames, fields, voxel_size, origin, max_norm, capacity, min_count)
    "one_ray": (1, 1, 1, 1 / 256, (0, 0, 0), 100.0, 2, 1),
    "small_2fields": (5000, 2, 2, 1 / 64, (0.3, -0.2, 0.1), 1.0, 1 << 14, 1),
    "coarse_min_count": (20000, 3, 3, 1 / 16, (-0.05, 0.0, 0.02), 0.8, 1 << 13, 3),
    "fine_1e6": (1 << 20, 1, 2, 1 / 512, (0, 0, 0), 1.0, 1 << 22, 1),
    "out_of_range": (20000, 1, 1, 1e-6, (0, 0, 0), 1.0, 1 << 16, 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_frame_points_and_extract_vs_oracle(case):
    n, frames, F, vs, origin, max_norm, cap, mc = CASES[case]
    t, store = _voxel_table(cap, vs, origin, "cuda")
    table = eo.new_table()
    for fr in range(frames):
        rgb, depth, acc, dirs, c2w, w2rf, blend = _random_rays(n, 10 * fr + F, F)
        if n == 1:
            acc[:], depth[:] = 1.0, 0.5
        _frame_points(t, rgb, depth, acc, dirs, c2w, w2rf, blend if fr % 2 == 0 else None, 0.5, max_norm)
        eo.frame_points(table, rgb, depth, acc, dirs, c2w, w2rf, blend if fr % 2 == 0 else None, 0.5, max_norm, vs,
                        origin)
    xyz, rgb8, count, stats = _extract(t, store, mc)
    assert stats[0] == table["kept"] and stats[1] == table["out_of_range"]
    assert stats[2] == len(table["voxels"]) <= cap // 2
    want = eo.extract(table, mc, vs, origin)
    assert len(xyz) == len(want[0])
    assert np.array_equal(xyz.view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(rgb8, want[1]) and np.array_equal(count, want[2])
    assert table["kept"] > 0 and (table["out_of_range"] > 0) == (case == "out_of_range")


# ---- a small two-field scene -------------------------------------------------------------------------------------
W, H = 48, 40


def _scene(grid=64, density_shift=2.0):
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", grid, n_init_frames=3, density_shift=density_shift)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(3):
            lt.r_c2w[i].add_(0.05 * torch.randn(3, 2, generator=g))
            lt.t_c2w[i].add_(0.1 * torch.randn(3, generator=g))
            lt.exposure[i].add_(0.05 * torch.randn(3, 3, generator=g))
    torch.manual_seed(1)
    lt.append_rf(2)                                 # blending rows [1, 0], [0.5, 0.5], [0, 1]
    lt = lt.to("cuda")
    assert lt.blending_weights.detach().cpu().tolist() == [[1.0, 0.0], [0.5, 0.5], [0.0, 1.0]]
    return lt


@pytest.fixture(scope="module")
def scene():
    return _scene()


def _bytes(cloud):
    return b"".join(cloud[k].cpu().numpy().tobytes() for k in ("xyz", "rgb", "count"))


def test_repeatable_across_runs_orders_and_chunks(scene):
    kw = dict(voxel_size=1 / 128, min_acc=0.05, capacity=1 << 16)
    a = point_cloud(scene, W, H, **kw)
    b = point_cloud(scene, W, H, **kw)
    c = point_cloud(scene, W, H, view_ids=[2, 0, 1], **kw)
    S = max(rf.sample_table(False, -1, "cuda").numel() for rf in scene.tensorfs)       # the eval table's length
    d = point_cloud(scene, W, H, weights_budget=4 * S * 97, **kw)            # chunks of 97 rays
    assert a["n_kept"] > 100 and len(a["xyz"]) > 50
    assert _bytes(a) == _bytes(b) == _bytes(c) == _bytes(d)
    assert a["n_rays"] == 3 * W * H and a["n_kept"] == c["n_kept"] == d["n_kept"]


def test_scene_renders_opacity_and_cloud_in_eval_table_chunks(scene):
    """The weights budget is counted in eval-table samples (2 (nSamples // 6) per ray): 4 S 500 bytes renders every
    view in chunks of exactly 500 rays."""
    lt = scene
    frames = []
    vs, origin, min_acc, max_norm = 1 / 128, (0.01, -0.02, 0.0), 0.05, 0.9
    S = max(rf.sample_table(False, -1, "cuda").numel() for rf in lt.tensorfs)
    assert S == max(2 * (int(rf.nSamples) // 6) for rf in lt.tensorfs)
    cloud = point_cloud(lt, W, H, test_ids=[1], voxel_size=vs, origin=origin, min_acc=min_acc, max_norm=max_norm,
                        capacity=1 << 16, weights_budget=4 * S * 500, _frames=frames)         # chunks of 500 rays
    assert [(v, lo, f[0].shape[0]) for v, lo, *f in frames] == \
        [(v, lo, min(500, W * H - lo)) for v in range(3) for lo in range(0, W * H, 500)]
    table = eo.new_table()
    w2rf = torch.stack([w.detach() for w in lt.world2rf]).cpu().numpy()
    bw = lt.blending_weights.detach().cpu().numpy()
    merged = {"keys": [], "fu": [], "cu": []}
    with torch.no_grad():
        for v, lo, rgb, depth, acc, dirs in frames:
            m = rgb.shape[0]
            ids = torch.arange(lo, lo + m, device="cuda")
            r_rgb, r_depth, r_dirs, _ = lt(ids, [v], W, H, is_train=False, test_id=v == 1)
            assert torch.equal(rgb, r_rgb) and torch.equal(depth, r_depth) and torch.equal(dirs, r_dirs)
            c2w = lt.get_cam2world([v])[0].detach()
            ref = torch.zeros(m, dtype=torch.float64, device="cuda")
            for k, rf in enumerate(lt.tensorfs):
                if bw[v, k] == 0:
                    continue
                rays = torch.cat([(c2w[:, 3] + lt.world2rf[k].detach()).expand(m, 3), dirs @ c2w[:, :3].T], 1)
                rf(rays.contiguous(), is_train=False, white_bg=True, return_weights=True)
                ref += float(bw[v, k]) * rf.last_weights.double().sum(1)
            assert float((acc.double() - ref).abs().max()) <= 1e-6
            args = [a.cpu().numpy() for a in (rgb, depth, acc, dirs)] + [c2w.cpu().numpy(), w2rf, bw[v]]
            eo.frame_points(table, *args, min_acc, max_norm, vs, origin)
            keep, _, key, fu, cu = eo.ray_points(*args, min_acc, max_norm, vs, origin)
            merged["keys"].append(key[keep]); merged["fu"].append(fu[keep]); merged["cu"].append(cu[keep])
    want = eo.extract(table, 1, vs, origin)
    got = [cloud[k].cpu().numpy() for k in ("xyz", "rgb", "count")]
    assert cloud["n_kept"] == table["kept"] > 100 and cloud["n_out_of_range"] == 0
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])

    # the same integer merge as torch ops: torch.unique + index_add_ on int64, means in float64 tensor ops
    keys = torch.from_numpy(np.concatenate(merged["keys"]))
    sums = torch.from_numpy(np.concatenate([np.ones((len(keys), 1), np.int64)] +
                                           [np.concatenate(merged[c]).astype(np.int64) for c in ("fu", "cu")], 1))
    uk, inv = torch.unique(keys, return_inverse=True)
    acc_sums = torch.zeros(len(uk), 7, dtype=torch.int64).index_add_(0, inv, sums)
    cnt = acc_sums[:, 0].double()
    kk = torch.stack([((uk >> (21 * (2 - a))) & ((1 << 21) - 1)) - (1 << 20) for a in range(3)], 1).double()
    org = torch.tensor([float(np.float32(o)) for o in origin], dtype=torch.float64)
    frac = acc_sums[:, 1:4].double() / (cnt * 4294967296.0)[:, None]
    xyz_t = (org + (kk + frac) * float(np.float32(vs))).float()
    rgb_t = torch.floor(acc_sums[:, 4:7].double() / (cnt * 16777216.0)[:, None] * 255.0 + 0.5).to(torch.uint8)
    assert torch.equal(xyz_t, cloud["xyz"].cpu()) and torch.equal(rgb_t, cloud["rgb"].cpu())
    assert torch.equal(acc_sums[:, 0].int(), cloud["count"].cpu())


def test_thin_slab_exports_onto_its_plane():
    """Density that depends on z only: an opaque slab one grid cell thick around z = c; a camera above it looking
    down -z.  Every point lies within one cell, one sample spacing and one voxel of c."""
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", 64, n_init_frames=2).to("cuda")
    rf = lt.tensorfs[0]
    G = 64
    idx = 36
    c = idx / (G - 1) * 4.0 - 2.0                    # aabb [-2, 2]; inside the unit cube contraction is the identity
    with torch.no_grad():
        for i in range(3):
            rf.density_plane[i].fill_(1.0 / 8 if i == 0 else 0.0)
            rf.density_line[i].fill_(0.0)
        rf.density_line[0].fill_(-30.0)
        rf.density_line[0][:, :, idx] = 30.0
        for i in range(2):
            lt.t_c2w[i].copy_(torch.tensor([0.05 * i, 0.0, 0.8]).cuda())
    vs = 1 / 256
    cloud = point_cloud(lt, 64, 48, voxel_size=vs, capacity=1 << 16)
    z = cloud["xyz"][:, 2].double().cpu()
    cell = 4.0 / (G - 1)
    step = float(rf.stepSize)
    assert len(z) > 500 and cloud["n_kept"] > 0.5 * 2 * 64 * 48
    assert float((z - c).abs().max()) <= cell + step + vs, (float(z.min()), float(z.max()), c)


def test_overflow_raises(scene):
    with pytest.raises(RuntimeError, match="capacity"):
        point_cloud(scene, W, H, voxel_size=1 / 128, min_acc=0.05, capacity=4)
