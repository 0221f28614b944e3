"""-m gpu: the VM lookups (lrf_density_feature, lrf_app_feature, lrf_app_products), their backward
(lrf_density_feature_backward, lrf_app_products_backward), the stand-alone MLP (lrf_mlp_forward), lrf_pack_bf16 and
lrf_repack_nchw_to_nhwc, called directly through the C ABI, against float64 (render64.py) or bitwise against torch.

Coordinates: uniform in [-1.1, 1.1]^3, and rows whose axes take exactly +-1, +-inf, +-0, NaN, the lattice points
2k / (size - 1) - 1 rounded to fp32 and their fp32 neighbours one ulp either side, and the largest fp32 coordinate
below 1 whose fp32 pixel coordinate rounds to size - 1.  The float64 side reads NaN as -1 (the header's rule: NaN
reads texel 0) and +-inf as +-2 (any clipped value reads the border texel).

Forward bar, per entry: |kernel - float64| <= c EPS A + slope dq.  A is render64._abs_sum (the sum of the absolute
values of every term the fp32 arithmetic adds).  c bounds the roundings along one term, counted linearly: the
bilinear weights carry 3 roundings, the 4-tap bilinear sum 4 more, the line's interpolation 3, the product 1 -- 11,
taken as 16 -- plus one per term of the sum that follows: 24 for the density feature (c = 40), 72 for the basis
product of the appearance feature (c = 88), none for the products (c = 16).  The fp32 pixel coordinate ((q + 1) / 2)
(size - 1) carries two roundings of EPS of itself each, so it reads the field at a point up to 2 EPS (|q| + 1) away
from q; slope dq (render64._slope) with twice that, dq = 4 EPS (|q| + 1), is what it can move the value.

Backward: parameter gradients within 2e-4 of each tensor's scale (sums of up to 2^20 atomically added fp32 terms);
d_xyz row by row within 2e-4 of its scale, skipping the rows with a pixel coordinate within TEXEL_MARGIN of a texel
floor (the position gradient jumps there, nothing else does); clipped axes give exactly 0.

Measured on an H100 80GB HBM3 at a 700 W power limit: forward at most 0.47 of its bar (products; density 0.32,
appearance feature 0.31, past 2^31 elements 0.24); parameter gradients at most 3.8e-5 of their scale, d_xyz 4.4e-6;
at most 0.34 % of the uniform rows skipped for d_xyz (640^3); MLP rgb within 1.6e-7 with no row below its margin; the
file runs in about 16 s."""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import render64 as R
from test_gpu_backward_edges import MARGIN_MLP, TEXEL_MARGIN, make_module, n_sms

pytestmark = pytest.mark.gpu
EPS = R.EPS
TOL = 2e-4
GUARD = 3                        # rows past M in every output, pre-filled with NaN: they must stay NaN
C_FWD = {"density": 40, "app_feature": 88, "products": 16}
WIDTH = {"density": 1, "app_feature": 27, "products": 72}
ENTRY = {"density": "lrf_density_feature", "app_feature": "lrf_app_feature", "products": "lrf_app_products"}
BWD_ENTRY = {"density": "lrf_density_feature_backward", "products": "lrf_app_products_backward"}
GRIDS = {"2": (2, 2, 2), "2x300x3": (2, 300, 3), "405264": (40, 52, 64), "300": (300, 300, 300),
         "640": (640, 640, 640)}
M_BIG = (1 << 20) + 3
COUNTS = [1, 127, 128, 129, 255, 256, 257]
MAX_SKIPPED = 0.01               # d_xyz rows skipped at a texel floor, of the uniform rows


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, math.nan, dtype=dtype, device="cuda")


def _lib():
    from localrf_b200 import _lib as L
    return L


def _keys(kind):
    pre = "density" if kind == "density" else "app"
    return [(f"{pre}_plane.{i}", f"{pre}_line.{i}") for i in range(3)]


# ---- coordinates ----------------------------------------------------------------------------------------------------
def _kernel_pixel(q, size):
    """The kernels' fp32 pixel coordinate ((q + 1) * 0.5) * (size - 1) (grid_coord, lrf_common.cuh)."""
    q = np.float32(q)
    return np.float32(np.float32(np.float32(q + np.float32(1)) * np.float32(0.5)) * np.float32(size - 1))


def near_top(size):
    """The smallest fp32 q < 1 whose fp32 pixel coordinate still rounds to size - 1 (from below)."""
    q = np.float32(1)
    while _kernel_pixel(np.nextafter(q, np.float32(0)), size) == np.float32(size - 1):
        q = np.nextafter(q, np.float32(0))
    assert q < 1 and _kernel_pixel(q, size) == size - 1
    return q


def coords(grid, M, seed, special=0.25):
    """fp32 [M, 3] on the GPU: the first M - n_special rows uniform in [-1.1, 1.1]^3, then rows whose axes each take,
    with probability 1/2, one of the special values of that axis -> (xyz, number of uniform rows)."""
    rng = np.random.default_rng(seed)
    q = (rng.random((M, 3)) * 2.2 - 1.1).astype(np.float32)
    n_sp = int(M * special) if M >= 16 else 0
    n_u = M - n_sp
    for a, size in enumerate(grid):
        k = rng.integers(0, size, n_sp)
        lat = (2.0 * k / (size - 1) - 1).astype(np.float32)
        fixed = np.array([1, -1, np.inf, -np.inf, -0.0, 0.0, np.nan, near_top(size)], np.float32)
        cat = rng.integers(0, len(fixed) + 3, n_sp)
        v = np.where(cat < len(fixed), fixed[np.minimum(cat, len(fixed) - 1)], lat)
        v = np.where(cat == len(fixed) + 1, np.nextafter(lat, np.float32(np.inf)), v)
        v = np.where(cat == len(fixed) + 2, np.nextafter(lat, np.float32(-np.inf)), v)
        pick = rng.random(n_sp) < 0.5
        q[n_u:, a] = np.where(pick, v, q[n_u:, a])
    return torch.from_numpy(q).cuda(), n_u


def ref_coords(xyz):
    """float64 coordinates the reference reads: NaN -> -1 (texel 0), +-inf -> +-2 (clipped)."""
    q = xyz.double()
    return torch.nan_to_num(q, nan=-1.0, posinf=2.0, neginf=-2.0)


def clipped(xyz):
    return ~(xyz.abs() < 1)           # |q| >= 1, +-inf and NaN: no position gradient


# ---- fields ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def field(gname, seed=0):
    """(module, Field64) of a random field on GRIDS[gname]: grids of 300 and up upsampled from 32 per axis."""
    grid = GRIDS[gname]
    fd = R.random_field(grid, seed=seed, safe_mlp=True, coarse=32 if max(grid) >= 300 else None)
    m = make_module(fd)
    return m, R.Field64.from_module(m, "cuda")


# ---- the kernels ----------------------------------------------------------------------------------------------------
def kernel_forward(m, kind, xyz, bf16=False):
    """One forward lookup -> [M, width] (guard rows checked NaN)."""
    L = _lib()
    M = xyz.shape[0]
    fs, keep = m._field_struct(None, need_mlp=False, grid16=bf16)
    out = nan(M + GUARD, WIDTH[kind])
    L.check(getattr(L.lib(), ENTRY[kind])(C.byref(fs), _p(xyz), M, _p(out), _stream()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[M:]).all()), "a guard row past M was written"
    return out[:M]


def _grads_of(m, kind):
    return (m.density_plane, m.density_line) if kind == "density" else (m.app_plane, m.app_line)


def kernel_backward(m, kind, xyz, gout, prefill=None, want_dxyz=True):
    """One backward call -> (d_planes + d_lines [6 tensors, parameter shapes], d_xyz [M, 3] or None)."""
    L = _lib()
    M = xyz.shape[0]
    planes, lines = _grads_of(m, kind)
    bufs = [torch.zeros_like(t, memory_format=torch.channels_last) for t in list(planes) + list(lines)]
    if prefill is not None:
        for b, p in zip(bufs, prefill):
            b.copy_(p)
    d_xyz = nan(M + GUARD, 3) if want_dxyz else None
    fs, keep = m._field_struct(None, need_mlp=False)
    pp = (C.c_void_p * 3)(*[t.data_ptr() for t in bufs[:3]])
    lp = (C.c_void_p * 3)(*[t.data_ptr() for t in bufs[3:]])
    L.check(getattr(L.lib(), BWD_ENTRY[kind])(C.byref(fs), _p(xyz), _p(gout), M, pp, lp, _p(d_xyz), _stream()))
    torch.cuda.synchronize()
    if d_xyz is not None:
        assert bool(torch.isnan(d_xyz[M:]).all()), "a guard row past M was written"
        d_xyz = d_xyz[:M]
    return bufs, d_xyz


# ---- float64 --------------------------------------------------------------------------------------------------------
def ref_values(F, kind, q):
    """float64 forward of one lookup kind at q [M, 3] -> [M, width]."""
    prods = [R._lookup(F.p[a].detach(), F.p[b].detach(), q, i) for i, (a, b) in enumerate(_keys(kind))]
    if kind == "density":
        return sum(p.sum(-1) for p in prods)[:, None]
    x = torch.cat(prods, -1)
    return x if kind == "products" else x @ F.p["basis_mat.weight"].detach().t()


def ref_bar(F, kind, q, finite):
    """The forward bar per entry: C_FWD EPS A + slope dq (module docstring)."""
    A = R._abs_sum(_keys(kind), q, F)
    if kind == "density":
        A = sum(a.sum(-1) for a in A)[:, None]
    else:
        A = torch.cat(A, -1)
        if kind == "app_feature":
            A = A @ F.p["basis_mat.weight"].detach().abs().t()
    dq = torch.where(finite, 4 * EPS * (q.abs() + 1), torch.zeros_like(q))
    return C_FWD[kind] * EPS * A + R._slope(lambda qq: ref_values(F, kind, qq), q, dq)


def ref_backward(F, kind, q, gout):
    """float64 autograd of the lookup: -> (6 parameter gradients, d_q [M, 3])."""
    qq = q.clone().requires_grad_(True)
    keys = _keys(kind)
    prods = [R._lookup(F.p[a], F.p[b], qq, i) for i, (a, b) in enumerate(keys)]
    out = sum(p.sum(-1) for p in prods) if kind == "density" else torch.cat(prods, -1)
    leaves = [qq] + [F.p[a] for a, _ in keys] + [F.p[b] for _, b in keys]
    gs = torch.autograd.grad((out * gout).sum(), leaves)
    return list(gs[1:]), gs[0]


def scale_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check_forward(tag, got, ref, bar):
    r = ((got.double() - ref).abs() / bar.clamp_min(1e-300))
    assert bool(torch.isfinite(got).all()), tag
    worst = float(r.max())
    print(f"{tag}: largest error {worst:.3f} of its bar")
    assert worst <= 1.0, (tag, worst)
    return worst


# ---- forward --------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _big_coords(gname):
    return coords(GRIDS[gname], M_BIG, seed=1)


@pytest.mark.parametrize("kind", ["density", "app_feature", "products"])
@pytest.mark.parametrize("gname", list(GRIDS))
def test_forward_vs_float64(gname, kind):
    m, F = field(gname)
    xyz, n_u = _big_coords(gname)
    got = kernel_forward(m, kind, xyz)
    q = ref_coords(xyz)
    with torch.no_grad():
        ref = ref_values(F, kind, q)
        bar = ref_bar(F, kind, q, torch.isfinite(xyz))
    check_forward(f"{gname} {kind}", got, ref, bar)
    # NaN reads texel 0 of its axis: exactly what -1 reads
    rows = torch.isnan(xyz).any(-1)
    assert int(rows.sum()) > 0
    sub = xyz[rows]
    assert torch.equal(got[rows], kernel_forward(m, kind, torch.where(torch.isnan(sub), -1.0, sub).contiguous()))


@pytest.mark.parametrize("gname", list(GRIDS))
def test_bf16_storage_equals_fp32_of_rounded_field(gname):
    """lrf_density_feature / lrf_app_feature on bf16 texels: bitwise the fp32 lookups of the bf16-rounded field."""
    grid = GRIDS[gname]
    fd = R.random_field(grid, seed=2, safe_mlp=True, coarse=32 if max(grid) >= 300 else None)
    m = make_module(fd)
    with torch.no_grad():
        for plist in (m.density_plane, m.density_line, m.app_plane, m.app_line):
            for p in plist:
                p.copy_(p.to(torch.bfloat16).float())
    xyz, _ = _big_coords(gname)
    for kind in ("density", "app_feature"):
        a, b = kernel_forward(m, kind, xyz, bf16=True), kernel_forward(m, kind, xyz)
        assert torch.equal(a, b), (gname, kind, scale_err(a, b))


@pytest.mark.parametrize("M", COUNTS)
def test_point_counts(M):
    """M rows alone: bitwise the first M rows of the 2^20 + 3 row call (each row is its own thread), guard rows NaN;
    the backward of M rows against float64."""
    m, F = field("405264")
    xyz, _ = _big_coords("405264")
    sub = xyz[:M].contiguous()
    for kind in ("density", "app_feature", "products"):
        assert torch.equal(kernel_forward(m, kind, sub), kernel_forward(m, kind, xyz)[:M]), kind
    g = torch.Generator(device="cuda").manual_seed(M)
    for kind in BWD_ENTRY:
        gout = torch.randn(M, *(() if kind == "density" else (72,)), generator=g, device="cuda")
        bufs, d_xyz = kernel_backward(m, kind, sub, gout)
        ref, d_ref = ref_backward(F, kind, ref_coords(sub), gout.double())
        err = max(scale_err(b, r) for b, r in zip(bufs, ref))
        keep = R._texel_margin(ref_coords(sub), F.grid) >= TEXEL_MARGIN
        if bool(keep.any()):
            err = max(err, scale_err(d_xyz[keep], d_ref[keep]))
        print(f"M {M} {kind}: {err:.1e}")
        assert err < TOL, (M, kind, err)


def test_app_products_past_2_31_elements():
    """M = floor(2^31 / 72) + 1 rows: m * 72 passes 2^31 elements.  Sampled rows and the last rows against float64."""
    M = (1 << 31) // 72 + 1
    need = (M + GUARD) * (72 + 3) * 4 + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB free")
    m, F = field("405264")
    g = torch.Generator(device="cuda").manual_seed(5)
    xyz = torch.rand(M, 3, generator=g, device="cuda") * 2.2 - 1.1
    out = kernel_forward(m, "products", xyz)
    rows = torch.cat([torch.randint(0, M, (1 << 14,), generator=g, device="cuda"),
                      torch.arange(M - 300, M, device="cuda")])
    q = xyz[rows].double()
    with torch.no_grad():
        check_forward("M past 2^31 / 72", out[rows], ref_values(F, "products", q),
                      ref_bar(F, "products", q, torch.ones_like(q, dtype=torch.bool)))
    del out


# ---- backward -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(BWD_ENTRY))
@pytest.mark.parametrize("gname", list(GRIDS))
def test_backward_vs_float64(gname, kind):
    m, F = field(gname)
    xyz, n_u = _big_coords(gname)
    M = xyz.shape[0]
    g = torch.Generator(device="cuda").manual_seed(7)
    gout = torch.randn(M, *(() if kind == "density" else (72,)), generator=g, device="cuda")
    bufs, d_xyz = kernel_backward(m, kind, xyz, gout)
    q = ref_coords(xyz)
    ref, d_ref = ref_backward(F, kind, q, gout.double())
    errs = {f"{w}.{i}": scale_err(b, r) for (w, i), b, r in
            zip([(w, i) for w in ("plane", "line") for i in range(3)], bufs, ref)}
    # clipped axes (|q| >= 1, +-inf, NaN): exactly no position gradient
    cl = clipped(xyz)
    assert bool((d_xyz[cl] == 0).all()), "a clipped axis has a position gradient"
    tm = R._texel_margin(q, F.grid)
    keep = tm >= TEXEL_MARGIN
    skipped = float((~keep[:n_u]).double().mean())
    errs["d_xyz"] = scale_err(d_xyz[keep], d_ref[keep])
    print(f"{gname} {kind}:", {k: f"{v:.1e}" for k, v in errs.items()},
          f"d_xyz rows skipped: {100 * skipped:.3f} % of the uniform rows, {int((~keep).sum())} in all")
    assert skipped <= MAX_SKIPPED
    assert max(errs.values()) < TOL, errs


@pytest.mark.parametrize("kind", list(BWD_ENTRY))
def test_backward_accumulates_and_zero_cotangent(kind):
    """Buffers pre-filled with P come back as P + the gradient; a zero grad_out adds exactly nothing (P bitwise) and
    gives d_xyz = 0."""
    m, F = field("405264")
    xyz, _ = coords(GRIDS["405264"], 50000, seed=3)
    g = torch.Generator(device="cuda").manual_seed(11)
    gout = torch.randn(xyz.shape[0], *(() if kind == "density" else (72,)), generator=g, device="cuda")
    g0, d0 = kernel_backward(m, kind, xyz, gout)
    P = [torch.randn(t.shape, generator=g, device="cuda") * t.abs().max() + 0.5 * t.abs().max() for t in g0]
    got, d1 = kernel_backward(m, kind, xyz, gout, prefill=P)
    for t, p, g_ in zip(got, P, g0):
        bar = 1e-4 * float(g_.abs().max()) + 2 * EPS * (p.abs() + g_.abs())
        assert bool(((t - p - g_).abs() <= bar).all())
    assert torch.equal(d1, d0)                    # d_xyz is overwritten, per row, with no atomics
    zero, dz = kernel_backward(m, kind, xyz, torch.zeros_like(gout), prefill=P)
    for t, p in zip(zero, P):
        assert torch.equal(t, p)
    assert bool((dz == 0).all())


def _integer_field(grid, seed):
    """A module whose plane / line texels are integers in [-3, 3]."""
    fd = R.random_field(grid, seed=seed, safe_mlp=True)
    rng = np.random.default_rng(seed)
    for k in R.GRID_KEYS:
        fd[k] = rng.integers(-3, 4, np.shape(fd[k])).astype(np.float64)
    return make_module(fd)


@pytest.mark.parametrize("kind", list(BWD_ENTRY))
@pytest.mark.parametrize("where", ["corner", "mid"])
def test_atomic_contention_exact(kind, where):
    """2^20 points on one lattice point that is exact in fp32 (q = -1 on a [2, 2, 2] grid; q = 0 on a [33, 17, 65]
    grid, 2^k + 1 texels per axis), integer texels and integer grad_out: every term is an integer and every partial
    sum stays below 2^24, so the accumulated texels equal the float64 sum bit for bit in any order of the atomics.  The
    buffers are pre-filled with integers (ACCUMULATE), and d_xyz = NULL leaves them bitwise the same."""
    grid, qv = ((2, 2, 2), -1.0) if where == "corner" else ((33, 17, 65), 0.0)
    m = _integer_field(grid, seed=4)
    M = 1 << 20
    xyz = torch.full((M, 3), qv, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(13)
    W = 1 if kind == "density" else 72
    gout = torch.randint(-3, 4, (M, W), generator=g, device="cuda").float()
    gout = gout[:, 0].contiguous() if kind == "density" else gout
    planes, lines = _grads_of(m, kind)
    P = [torch.randint(-1000, 1001, t.shape, generator=g, device="cuda").float() for t in list(planes) + list(lines)]
    got, d_xyz = kernel_backward(m, kind, xyz, gout, prefill=P)
    got_null, _ = kernel_backward(m, kind, xyz, gout, prefill=P, want_dxyz=False)
    # expected: one texel of each plane and one of each line, t = 0 on every axis
    gsum = gout.double().reshape(M, -1).sum(0)                     # [W]
    exp = [p.double().clone() for p in P]
    for i in range(3):
        W0, H0, L0 = grid[R.MAT0[i]], grid[R.MAT1[i]], grid[R.VEC[i]]
        x, y, l = (int(round((qv + 1) / 2 * (s - 1))) for s in (W0, H0, L0))
        Cn = planes[i].shape[1]
        gs = gsum if kind == "density" else gsum[i * Cn:(i + 1) * Cn]
        pl, ln = planes[i].detach().double()[0, :, y, x], lines[i].detach().double()[0, :, l, 0]
        exp[i][0, :, y, x] += gs * ln
        exp[3 + i][0, :, l, 0] += gs * pl
    assert max(float(e.abs().max()) for e in exp) < 2 ** 24
    for t, e, t2 in zip(got, exp, got_null):
        assert torch.equal(t.double(), e), float((t.double() - e).abs().max())
        assert torch.equal(t2, t)
    if where == "corner":
        assert bool((d_xyz == 0).all())


# ---- lrf_mlp_forward ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mlp_case():
    """A safe-MLP field, products from lrf_app_products at random points and random unit view directions for the
    largest count; float64 is taken on sampled rows."""
    m, F = field("405264")
    fs, _ = m._field_struct(None)
    prep = m.prepare(fs)
    M = 3 * (1 << 20) + 5
    g = torch.Generator(device="cuda").manual_seed(17)
    xyz = torch.rand(M, 3, generator=g, device="cuda") * 2 - 1
    feats = kernel_forward(m, "products", xyz).contiguous()
    vd = torch.randn(M, 3, generator=g, device="cuda")
    vd = (vd / vd.norm(dim=-1, keepdim=True)).contiguous()
    return m, F, prep, xyz, feats, vd


def mlp(prep, feats, vd):
    L = _lib()
    M = feats.shape[0]
    out = nan(M + GUARD, 3)
    L.check(L.lib().lrf_mlp_forward(_p(prep), _p(feats), _p(vd), M, _p(out), _stream()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[M:]).all()), "a guard row past M was written"
    return out[:M]


def check_mlp(tag, F, xyz, feats, vd, got):
    """rgb against render64._mlp (pe = 0) in float64: per entry within TOL_MLP = 1e-4 (the render forward's rgb bar)
    on the rows whose MLP pre-activations clear the tensor-core margin of test_gpu_render_edges.py."""
    with torch.no_grad():
        q = xyz.double()
        ref, marg = R._mlp(F, feats.double(), vd.double(), True, q, torch.zeros_like(q))
    keep = marg >= MARGIN_MLP[True]
    frac = 1 - float(keep.double().mean())
    err = float((got.double() - ref)[keep].abs().max())
    print(f"{tag}: rgb error {err:.1e} ({err / 1e-4:.3f} of the bar), {100 * frac:.2f} % of rows below the MLP margin")
    assert frac <= 0.01 and err <= 1e-4


@pytest.mark.parametrize("which", ["1", "127", "128", "129", "2x128sm+1", "3M+5"])
def test_mlp_forward_vs_float64(mlp_case, which):
    m, F, prep, xyz, feats, vd = mlp_case
    M = {"1": 1, "127": 127, "128": 128, "129": 129, "2x128sm+1": 2 * 128 * n_sms() + 1, "3M+5": feats.shape[0]}[which]
    got = mlp(prep, feats[:M].contiguous(), vd[:M].contiguous())
    rows = torch.arange(M, device="cuda")
    if M > 1 << 16:
        g = torch.Generator(device="cuda").manual_seed(19)
        rows = torch.cat([torch.randint(0, M, (1 << 16,), generator=g, device="cuda"),
                          torch.arange(M - 300, M, device="cuda")])
    check_mlp(f"mlp M {M}", F, xyz[rows], feats[rows], vd[rows], got[rows])


def test_mlp_rows_bitwise_alone_batched_permuted(mlp_case):
    m, F, prep, xyz, feats, vd = mlp_case
    n = 2 * 128 * n_sms() + 1
    whole = mlp(prep, feats[:n].contiguous(), vd[:n].contiguous())
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(23)).cuda()
    shuffled = mlp(prep, feats[perm].contiguous(), vd[perm].contiguous())
    assert torch.equal(shuffled, whole[perm])
    for r in (0, 127, 128, n - 1):
        assert torch.equal(mlp(prep, feats[r:r + 1].contiguous(), vd[r:r + 1].contiguous())[0], whole[r]), r


# ---- lrf_pack_bf16 --------------------------------------------------------------------------------------------------
def pack(src, dst, n):
    L = _lib()
    L.check(L.lib().lrf_pack_bf16(_p(src), _p(dst), n, _stream()))
    torch.cuda.synchronize()


def _check_pack(src, out):
    """Bitwise torch's round to nearest even, except that a NaN only has to stay a NaN."""
    ref = src.to(torch.bfloat16).view(torch.int16)
    o = out.view(torch.int16)
    isnan = torch.isnan(src)
    same = (o == ref) | isnan
    assert bool(same.all()), int((~same).sum())
    on = o[isnan].int() & 0xFFFF
    assert bool((((on & 0x7F80) == 0x7F80) & ((on & 0x7F) != 0)).all()), "a NaN did not stay a NaN"


def test_pack_bf16_exhaustive():
    """All 2^32 fp32 bit patterns, 2^28 at a time."""
    CH = 1 << 28
    base = torch.arange(CH, dtype=torch.int32, device="cuda")
    out = torch.empty(CH, dtype=torch.bfloat16, device="cuda")
    for c in range(16):
        hi = (c << 28) - (1 << 32) if c >= 8 else c << 28        # the top 4 bits as a signed 32-bit word
        src = (base | hi).view(torch.float32)
        pack(src, out, CH)
        _check_pack(src, out)


@pytest.mark.parametrize("n", [1, 7, 1001, 1 << 20 | 1])
def test_pack_bf16_odd_n_and_offsets(n):
    """Odd n, a source 4 bytes into its buffer and a destination 2 bytes into its: the elements past n untouched."""
    g = torch.Generator(device="cuda").manual_seed(n)
    raw = torch.randn(n + 1, generator=g, device="cuda") * 10.0 ** torch.randint(-30, 30, (n + 1,), generator=g,
                                                                                  device="cuda").float()
    src = raw[1:]
    dbuf = torch.full((n + 1 + GUARD,), -7.0, dtype=torch.bfloat16, device="cuda")
    dst = dbuf[1:]
    pack(src, dst, n)
    _check_pack(src, dst[:n])
    assert bool((dbuf[0] == -7.0) and (dst[n:] == -7.0).all())


# ---- lrf_repack_nchw_to_nhwc ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_,H,W", [(1, 5, 7), (8, 1, 1), (24, 1, 1), (27, 1, 1), (8, 13, 17), (24, 31, 1),
                                    (27, 3, 5), (1, 640, 640), (24, 640, 640)])
def test_repack_bitwise(C_, H, W):
    L = _lib()
    g = torch.Generator(device="cuda").manual_seed(C_ * 1000 + H * W)
    src = torch.randn(C_, H, W, generator=g, device="cuda")
    dst = nan(C_ * H * W + GUARD)
    L.check(L.lib().lrf_repack_nchw_to_nhwc(_p(src), _p(dst), C_, H, W, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(dst[:C_ * H * W].view(H, W, C_), src[None].permute(0, 2, 3, 1).contiguous()[0])
    assert bool(torch.isnan(dst[C_ * H * W:]).all())
