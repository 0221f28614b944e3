"""GPU: the mesh export (lrf_mesh_lattice / lrf_mesh_cells / lrf_mesh_extract / lrf_mesh_normals and
localrf_b200.export.mesh) against getDenseAlpha bit for bit, the float64 restatement of A, the numpy restatement of the
marching-cubes stages bit for bit, and analytic solids."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import localrf_b200 as L
import mesh_oracle as mo
import render64 as r64
from localrf_b200 import _lib
from localrf_b200.export import _mesh_table, mesh
from localrf_b200.ray_utils import contract

pytestmark = pytest.mark.gpu
CANARY = -12345.0


def _lt(n_fields=1, grid=64, **over):
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", grid, n_init_frames=2, density_shift=over.pop("density_shift", 2.0),
                      **over)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(2):
            lt.t_c2w[i].add_(0.3 * torch.randn(3, generator=g))
    for _ in range(n_fields - 1):
        lt.append_rf(2)
    return lt.to("cuda")


def _scene_struct(lt, w2rf, voxel, origin=(0.0, 0.0, 0.0), max_norm=1.0, level=0.005):
    n = len(lt.tensorfs)
    keep = dict(w2rf=torch.as_tensor(np.asarray(w2rf, np.float32), device="cuda").reshape(n, 3).contiguous(),
                fields=(_lib.LrfField * n)(*[rf._field() for rf in lt.tensorfs]),
                steps=(C.c_float * n)(*[float(rf.stepSize) for rf in lt.tensorfs]))
    s = _lib.LrfMeshScene(n_fields=n, fields=keep["fields"], step_size=keep["steps"],
                          world2rf=keep["w2rf"].data_ptr(), voxel_size=voxel, max_norm=max_norm, level=level)
    s.origin[:] = list(origin)
    return s, keep


def _lattice(s, lo, dims):
    v = torch.full((int(np.prod(dims)) + 64,), CANARY, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().lrf_mesh_lattice(C.byref(s), (C.c_int32 * 3)(*lo), (C.c_int32 * 3)(*dims), v.data_ptr(),
                                           None))
    torch.cuda.synchronize()
    assert (v[-64:] == CANARY).all()
    return v[:-64].reshape(*dims)


def _points(lo, dims, voxel, origin):
    ax = [np.float32(origin[a]) + np.arange(lo[a], lo[a] + dims[a]).astype(np.float32) * np.float32(voxel)
          for a in range(3)]
    return torch.from_numpy(np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3).astype(np.float64))


@pytest.mark.parametrize("mask", [False, True])
def test_lattice_equals_get_dense_alpha_bit_for_bit(mask):
    lt = _lt()
    rf = lt.tensorfs[0]
    if mask:
        rf.updateAlphaMask((32, 32, 32))
    k = 5
    dense = rf.getDenseAlpha((2 ** k + 1,) * 3)                # points -2 + 4 i / 2^k
    s, keep = _scene_struct(lt, [[0, 0, 0]], 4 / 2 ** k, max_norm=1.0)
    h = 2 ** (k - 2)                                           # the unit cube: lattice indices [-h, h]
    got = _lattice(s, (-h, -h, -h), (2 * h + 1,) * 3)
    want = dense[2 * h - h:2 * h + h + 1, 2 * h - h:2 * h + h + 1, 2 * h - h:2 * h + h + 1]
    assert torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32))
    assert float(got.max()) > 0.01


@pytest.mark.parametrize("variant", ["softplus", "relu", "mask", "pe"])
def test_lattice_matches_float64(variant):
    over = dict(fea_pe=2, view_pe=2) if variant == "pe" else {}
    lt = _lt(2, grid=48, **over)
    if variant == "relu":
        for rf in lt.tensorfs:
            rf.fea2denseAct = "relu"
    if variant == "mask":
        lt.tensorfs[1].updateAlphaMask((24, 24, 24))
    w2rf = np.array([[0.0, 0.0, 0.0], [-0.5, 0.25, 0.0]], np.float32)
    voxel, origin, max_norm = 1 / 16, (0.01, -0.02, 0.03), 1.5
    s, keep = _scene_struct(lt, w2rf, voxel, origin, max_norm)
    lo, dims = (-30, -28, -29), (50, 50, 49)
    got = _lattice(s, lo, dims).reshape(-1).double().cpu()
    fields = [r64.Field64.from_module(rf) for rf in lt.tensorfs]
    A, owner, flagged = mo.mesh_value64(fields, [float(rf.stepSize) for rf in lt.tensorfs], w2rf,
                                        _points(lo, dims, voxel, origin), max_norm)
    ok = ~flagged
    assert int(flagged.sum()) < 0.01 * len(A)
    assert (owner == 0).any() and (owner == 1).any() and (owner == -1).any()
    assert float((got - A)[ok].abs().max()) <= 2e-5 + 1e-5 * float(A.abs().max())
    assert (got[owner == -1] == 0).all()


def _extract(t):
    lib = _lib.lib()
    nb = lib.lrf_mesh_extract_scratch_bytes(t.capacity, t.max_triangles)
    scratch = torch.full((nb,), 0x5A, dtype=torch.uint8, device="cuda")
    half = t.capacity // 2
    xyz = torch.full((half + 8, 3), CANARY, dtype=torch.float32, device="cuda")
    faces = torch.full((t.max_triangles + 8, 3), -7, dtype=torch.int32, device="cuda")
    counts = torch.full((4,), -9, dtype=torch.int64, device="cuda")
    _lib.check(lib.lrf_mesh_extract(C.byref(t), xyz.data_ptr(), faces.data_ptr(), counts.data_ptr(),
                                    scratch.data_ptr(), nb, None))
    torch.cuda.synchronize()
    nv, nt = counts[:2].tolist()
    assert counts[2:].tolist() == [-9, -9] and (xyz[half:] == CANARY).all() and (faces[t.max_triangles:] == -7).all()
    assert (xyz[nv:half] == CANARY).all() and (faces[nt:t.max_triangles] == -7).all()
    return xyz[:nv].cpu().numpy(), faces[:nt].cpu().numpy()


def _cells(s, lo, dims, values, t):
    _lib.check(_lib.lib().lrf_mesh_cells(C.byref(s), (C.c_int32 * 3)(*lo), (C.c_int32 * 3)(*dims),
                                         values.data_ptr(), C.byref(t), None))


@pytest.mark.parametrize("seed", range(3))
def test_cells_and_extract_equal_the_restatement(seed):
    """Random lattice values with every case, exact level values, NaN and infinities; one brick and the same lattice
    in 2 x 3 x 2 bricks give the restatement's mesh bit for bit."""
    lt = _lt()
    rng = np.random.default_rng(seed)
    level = 0.5
    dims = (21, 22, 23)
    v = rng.random(dims).astype(np.float32)
    v[rng.random(dims) < 0.05] = level
    v[rng.random(dims) < 0.01] = np.nan
    v[rng.random(dims) < 0.01] = np.inf
    v[rng.random(dims) < 0.01] = -np.inf
    lo = (-7 + seed, 3, -(1 << 19))
    voxel, origin = 0.03125 * (seed + 1), (0.1, -0.2, 0.3)
    s, keep = _scene_struct(lt, [[0, 0, 0]], voxel, origin, level=level)
    want = mo.mesh_lattice(v, lo, level, origin, voxel)
    assert len(want[1]) > 5000
    t, store = _mesh_table(1 << 16, 1 << 16, "cuda")
    vt = torch.from_numpy(v).cuda().reshape(-1).contiguous()
    _cells(s, lo, dims, vt, t)
    got = _extract(t)
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and np.array_equal(got[1], want[1])
    t2, store2 = _mesh_table(1 << 16, 1 << 16, "cuda")
    for x0, x1 in ((0, 11), (10, 21)):
        for y0, y1 in ((0, 8), (7, 15), (14, 22)):
            for z0, z1 in ((0, 12), (11, 23)):
                sub = torch.from_numpy(np.ascontiguousarray(v[x0:x1, y0:y1, z0:z1])).cuda().reshape(-1)
                _cells(s, (lo[0] + x0, lo[1] + y0, lo[2] + z0), (x1 - x0, y1 - y0, z1 - z0), sub, t2)
    got2 = _extract(t2)
    assert np.array_equal(got2[0].view(np.uint32), want[0].view(np.uint32)) and np.array_equal(got2[1], want[1])


def _bytes(m):
    return b"".join(m[k].cpu().numpy().tobytes() for k in ("xyz", "normals", "rgb", "faces"))


@pytest.fixture(scope="module")
def two_fields():
    return _lt(2)


def test_brick_size_and_run_independence(two_fields):
    kw = dict(voxel_size=1 / 32, level=0.05, capacity=1 << 18, max_triangles=1 << 19)
    a = mesh(two_fields, _brick=64, **kw)
    assert len(a["faces"]) > 1000
    assert _bytes(a) == _bytes(mesh(two_fields, _brick=8, **kw)) == _bytes(mesh(two_fields, _brick=37, **kw))
    assert _bytes(a) == _bytes(mesh(two_fields, _brick=64, **kw))
    f = a["faces"].cpu().numpy()
    assert mo.is_closed_oriented(f)


def _cylinder(lt, rf, centre, r, half_h):
    """relu density S P(x, y) L(z): P, L ramps from 0 to 1 across one grid cell around the disc edge and the interval
    ends (component 0 of plane / line 0); S puts alpha = level at P L = 1/2."""
    G = rf.gridSize.tolist()[0]
    cell = 4.0 / (G - 1)
    c = torch.linspace(-2, 2, G, dtype=torch.float64)
    yy, xx = torch.meshgrid(c, c, indexing="ij")
    P = (0.5 + (r - torch.hypot(xx - centre[0], yy - centre[1])) / cell).clamp(0, 1)
    Lz = (0.5 + (half_h - (c - centre[2]).abs()) / cell).clamp(0, 1)
    S = -math.log(1 - 0.005) / (float(rf.stepSize) * 0.5)
    with torch.no_grad():
        for i in range(3):
            rf.density_plane[i].zero_()
            rf.density_line[i].zero_()
        rf.density_plane[0][0, 0] = P.float().cuda()
        rf.density_line[0][0, 0, :, 0] = (S * Lz).float().cuda()
    rf.fea2denseAct = "relu"
    return cell


def test_analytic_cylinder():
    lt = _lt(grid=128)
    rf = lt.tensorfs[0]
    r, hh = 0.5, 0.4
    w = lt.world2rf[0].detach().cpu().double()
    cell = _cylinder(lt, rf, (0.0, 0.0, 0.0), r, hh)
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(-x) for x in w))
    xyz, f = m["xyz"].cpu().numpy(), m["faces"].cpu().numpy()
    assert mo.is_closed_oriented(f) and mo.euler_characteristic(xyz, f) == 2
    vol = mo.signed_volume(xyz - (-w.numpy()).astype(np.float32), f)
    want = math.pi * r * r * 2 * hh
    assert abs(vol - want) <= 0.02 * want, (vol, want)
    loc = xyz.astype(np.float64) + w.numpy()
    n = m["normals"].cpu().numpy()
    rad = np.hypot(loc[:, 0], loc[:, 1])
    side = (np.abs(loc[:, 2]) < hh - 2 * cell) & (np.abs(rad - r) < cell)
    assert side.sum() > 200
    radial = loc[side, :2] / rad[side, None]
    assert (np.einsum("ij,ij->i", n[side, :2], radial) > 0.9).all()


def test_surface_stays_closed_across_the_owner_seam():
    lt = _lt(2, grid=128)
    w = [lt.world2rf[k].detach().cpu().double().numpy() for k in range(2)]
    with torch.no_grad():
        lt.world2rf[1].copy_(lt.world2rf[0] - torch.tensor([0.8, 0.0, 0.0], device="cuda"))
    w = [lt.world2rf[k].detach().cpu().double().numpy() for k in range(2)]
    centre_world = -w[0] + np.array([0.4, 0.0, 0.0])                   # on the seam between the two centres
    for k in range(2):
        _cylinder(lt, lt.tensorfs[k], tuple(centre_world + w[k]), 0.3, 0.3)
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(v) for v in -w[0]), max_norm=1.0)
    xyz, f = m["xyz"].cpu().numpy(), m["faces"].cpu().numpy()
    assert len(f) > 1000 and mo.is_closed_oriented(f) and mo.euler_characteristic(xyz, f) == 2


def test_normals_and_colours(two_fields):
    lt = two_fields
    m = mesh(lt, voxel_size=1 / 32, level=0.05, capacity=1 << 18, max_triangles=1 << 19)
    x = m["xyz"].double().cpu()
    w2rf = torch.stack([w.detach().float() for w in lt.world2rf]).cpu().numpy()
    fields = [r64.Field64.from_module(rf) for rf in lt.tensorfs]
    steps = [float(rf.stepSize) for rf in lt.tensorfs]
    h = (1 / 32) / 2
    g = torch.zeros_like(x)
    bad = torch.zeros(len(x), dtype=torch.bool)
    for a in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[a] = h
        hi, _, f1 = mo.mesh_value64(fields, steps, w2rf, x + e, 1.0)
        lo, _, f2 = mo.mesh_value64(fields, steps, w2rf, x - e, 1.0)
        g[:, a] = hi - lo
        bad |= f1 | f2
    gn = g.norm(dim=1)
    ok = ~bad & (gn > 1e-2)
    assert int(ok.sum()) > 0.5 * len(x)
    n64 = -g / gn[:, None]
    assert float((m["normals"].double().cpu() - n64)[ok].abs().max()) <= 1e-3

    # colours: the owner by float64 norms (near-ties skipped), then compute_appfeature + renderModule as torch ops
    wt = torch.as_tensor(w2rf, dtype=torch.float64)
    norms = (x[:, None] + wt[None]).abs().amax(-1)
    srt = norms.sort(dim=-1, stable=True)
    clear = (srt.values[:, 1] - srt.values[:, 0]) > 1e-5
    owner = srt.indices[:, 0]
    nrm = m["normals"]
    view = torch.where((nrm == 0).all(-1, keepdim=True), torch.tensor([0.0, 0.0, -1.0], device="cuda"), -nrm)
    with torch.no_grad():
        for k, rf in enumerate(lt.tensorfs):
            sel = ((owner == k) & clear).nonzero().reshape(-1).cuda()
            pts = m["xyz"][sel] + lt.world2rf[k].detach().float()
            feats = rf.compute_appfeature(rf.normalize_coord(contract(pts)))
            c = rf.renderModule(None, view[sel], feats, bool(lt.is_refining))
            want = torch.floor(255 * c + 0.5).to(torch.uint8)
            assert torch.equal(m["rgb"][sel], want)
    assert int(clear.sum()) > 0.9 * len(x)


def test_overflow_raises_and_names_the_parameter(two_fields):
    kw = dict(voxel_size=1 / 32, level=0.05)
    with pytest.raises(RuntimeError, match="capacity"):
        mesh(two_fields, capacity=64, **kw)
    with pytest.raises(RuntimeError, match="max_triangles"):
        mesh(two_fields, max_triangles=64, **kw)
