"""-m gpu: the schedule-time kernels (localrf_b200/csrc/lrf_sched.cu) at training sizes against float64 restatements
of the reference formulas (tests/sched_oracle.py).

Every sched launcher caps its grid at 16 blocks of 256 threads per SM (540,672 threads on a 132-SM H100), so the
full-size cases here run each grid-stride loop for several passes.  The density_L1 backward is checked on all three
of its paths: lines of at most 256 (register slot 0), 257..1024 (slots 1-3) and longer (the atomic tail loop).
Wherever a check depends on the data reaching some region (a clamp, a branch, the kept part of a mask), the test
asserts that it does, so a change of seed cannot make it vacuous."""
import ctypes as C
import math

import pytest
import torch

import localrf_b200 as L
from localrf_b200 import _lib
import sched_oracle as so
from gpu_helpers import oracle_field

pytestmark = pytest.mark.gpu

U = so.U32
THREADS_PER_SM = 16 * 256          # cta_count(..., 16) in lrf_sched.cu: at most 16 blocks of 256 threads per SM


class TVLoss(torch.nn.Module):
    """Interface of the reference's regulariser (utils/utils.py:293-312): what train.py:340 passes."""

    def __init__(self, TVLoss_weight=1):
        super().__init__()
        self.TVLoss_weight = TVLoss_weight

    def forward(self, x):
        tv = 0
        if x.size(2) > 1:
            tv = tv + torch.pow(x[:, :, 1:, :] - x[:, :, :-1, :], 2).mean()
        if x.size(3) > 1:
            tv = tv + torch.pow(x[:, :, :, 1:] - x[:, :, :, :-1], 2).mean()
        return self.TVLoss_weight * 2 * tv


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _grid_threads():
    return torch.cuda.get_device_properties(0).multi_processor_count * THREADS_PER_SM


def _passes(n):
    """grid-stride passes of the busiest thread of a sched launch over n work items"""
    return math.ceil(n / _grid_threads())


def _scale_err(a, ref):
    """max |a - ref| / max |ref| (the gradient metric of test_gpu_sched.py) and relative L2"""
    a, ref = a.double(), ref.double()
    d = a - ref
    return float(d.abs().max() / ref.abs().max().clamp_min(1e-300)), float(d.norm() / ref.norm().clamp_min(1e-300))


def _cl_param(t):
    return torch.nn.Parameter(t.contiguous(memory_format=torch.channels_last))


def _field(grid, **over):
    import bench
    torch.manual_seed(0)
    aabb = 2 * torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    return L.TensorVMSplit("cuda", aabb.cuda(), list(grid), **bench.field_kwargs(**over)).to("cuda")


@pytest.fixture(scope="module")
def _bench300():
    import bench
    return bench.build_scene("cuda", 300).tensorfs[0]


@pytest.fixture()
def field300(_bench300):
    """the 300^3 bench field (softplus, density_shift = -5); density grids, activation and mask restored after use"""
    m = _bench300
    params = [*m.density_plane, *m.density_line]
    saved = [p.detach().clone() for p in params]
    yield m
    with torch.no_grad():
        for p, s in zip(params, saved):
            p.copy_(s)
    m.fea2denseAct = "softplus"
    m.alphaMask = None
    m.zero_grad(set_to_none=True)


# ---- 1. density_L1 forward and backward -----------------------------------------------------------------------
# H100 80GB HBM3: loss value within 2.0e-7 relative (300^3 relu: 50 grid-stride passes of fp32 terms per thread;
# 3.1e-8 with softplus), gradients within 3.8e-6 of their tensor's max (density_line.0 of [1100, 700, 9]:
# 9 positions, each a sum over 770,000 texels of atomically added block partials)
VALUE_BAR = 1e-6
GRAD_BAR = 2e-5


def _l1_near_decisions(m, planes64, lines64, f, exact=False):
    """indices whose float64 feature lies within fp32 rounding of a clamp or branch decision of l1_dfeature: the
    feature is a sum of 24 fp32 products (rounding <= 16 u * sum |terms|), x = f + shift rounds once more, and
    log1pf(expf(x)) is good to a few ulps (16 u * |x| covers both).

    exact: the grids are integer multiples of 2^-14 below 2^-2 in magnitude, so every product is an integer multiple
    of 2^-28 below 2^24 of those units; if sum |terms| stays below 2^-4 as well, every partial sum of the kernel's f
    is one too, each fp32 operation is exact, and fp32 and float64 take every decision alike."""
    with torch.no_grad():
        terms = so.l1_abs_terms([p.detach() for p in planes64], [l.detach() for l in lines64])
        if exact:
            for t in (*planes64, *lines64):
                q = t.detach() * 2 ** 14
                assert torch.equal(q, q.round()) and float(q.abs().max()) < 2 ** 12
            assert float(terms.max()) < 2 ** -4
            return 0
        if m.fea2denseAct == "softplus":
            x = f + m.density_shift
            margin = 16 * U * (terms + x.abs())
            x_clamp = math.log(math.expm1(1e-5))              # softplus(x) = 1e-5
            near = ((x - 20).abs() <= margin) | ((x - x_clamp).abs() <= margin)
        else:
            margin = 16 * U * terms
            near = (f.abs() <= margin) | ((f - 1e-5).abs() <= margin)
        return int(near.sum())


def _check_l1(m, value_bar=VALUE_BAR, grad_bar=GRAD_BAR, exact=False):
    """density_L1 (value and the six gradients through loss * 1e-2) against float64 autograd; -> (f64, report)"""
    m.zero_grad(set_to_none=True)
    val = m.density_L1()
    (val * 1e-2).backward()
    planes64 = [p.detach().double().requires_grad_() for p in m.density_plane]
    lines64 = [l.detach().double().requires_grad_() for l in m.density_line]
    ref, f = so.density_l1(planes64, lines64, m.fea2denseAct, float(m.density_shift))
    (ref * 1e-2).backward()
    f = f.detach()
    assert _l1_near_decisions(m, planes64, lines64, f, exact) == 0
    verr = abs(float(val.detach()) - float(ref.detach())) / abs(float(ref.detach()))
    report = {"value": verr}
    assert verr <= value_bar, report
    for name, got, want in (*[(f"density_plane.{i}", p.grad, r.grad) for i, (p, r) in
                              enumerate(zip(m.density_plane, planes64))],
                            *[(f"density_line.{i}", l.grad, r.grad) for i, (l, r) in
                              enumerate(zip(m.density_line, lines64))]):
        assert got is not None and got.shape == want.shape, name
        assert float(want.abs().max()) > 0, name
        report[name] = _scale_err(got, want)
    print(f"\n  N = {f.numel()}, fwd passes = {_passes(f.numel())}: " +
          ", ".join(f"{k} {v[0]:.2e}/{v[1]:.2e}" if isinstance(v, tuple) else f"{k} {v:.2e}"
                    for k, v in report.items()))
    worst = max(v[0] for k, v in report.items() if k != "value")
    assert worst <= grad_bar, report
    return f, report


# grid -> line length of plane i is grid[vecMode[i]] = grid[2 - i]
@pytest.mark.parametrize("grid", [[1100, 700, 9], [1024, 256, 8], [1025, 257, 8]],
                         ids=["tail-slots012-slot0", "edges-1024-256", "edges-1025-257"])
def test_density_l1_backward_paths(grid):
    m = _field(grid)
    lens = [grid[2 - i] for i in range(3)]
    assert max(lens) > 256                       # a slots-1..3 path runs in every case
    _check_l1(m)


def test_density_l1_bench_field(field300):
    """the training shape: 300^3, softplus with shift -5; lines of 300 use register slots 0 and 1"""
    f, _ = _check_l1(field300)
    assert _passes(f.numel()) >= 40


def test_density_l1_relu_regions(field300):
    """relu: scaled so that every region of l1_dfeature is populated: f <= 0 (no gradient), 0 < f < 1e-5 (clamped:
    value sqrt(1e-5), no gradient) and f >= 1e-5.  Among 27 M features about 65 would lie within worst-case fp32
    rounding of 1e-5, so the scaled grids are also rounded to multiples of 2^-14: the kernel's features are then
    exact and the clamp decides every index as float64 does."""
    m = field300
    m.fea2denseAct = "relu"
    with torch.no_grad():                        # f scales with k^2: std ~0.05 -> ~2e-4
        for p in (*m.density_plane, *m.density_line):
            p.copy_(torch.round(p * (0.064 * 2 ** 14)) / 2 ** 14)
    f, _ = _check_l1(m, exact=True)
    n = f.numel()
    fr = [float((f <= 0).sum()) / n, float(((f > 0) & (f < 1e-5)).sum()) / n, float((f >= 1e-5).sum()) / n]
    print(f"  region fractions f<=0 {fr[0]:.3f}, clamped {fr[1]:.4f}, f>=1e-5 {fr[2]:.3f}")
    assert fr[0] >= 0.3 and fr[1] >= 0.01 and fr[2] >= 0.3, fr


def test_density_l1_softplus_linear_branch():
    """softplus above its threshold (x = f + shift > 20 returns x): a block of large components drives x past 20"""
    m = _field([96, 80, 300])
    with torch.no_grad():
        m.density_plane[0][0, 0, 20:60, 30:70] += 6.0       # plane 0: [grid[1], grid[0]]
        m.density_line[0][0, 0, 50:250, 0] += 6.0           # line 0: grid[2]
    f, _ = _check_l1(m)
    frac = float((f + m.density_shift > 20).sum()) / f.numel()
    print(f"  fraction with x > 20: {frac:.3f}")
    assert frac >= 0.1


# ---- 2. lrf_alpha_mask_build ------------------------------------------------------------------------------
# alpha = 1 - exp(-sigma step) is quantised to the fp32 spacing below 1.0 (6e-8); H100 80GB HBM3: 1.04e-7
ALPHA_TOL = 2.5e-7


def _add_dense_region(m, amp=2.0):
    """component 0 of density plane 0 and line 0 raised by amp: f ~ amp^2 where x < 1 and y, z in the middle half
    of the aabb (x starts at the face, so a lattice with gx = 1, which samples x = aabb min, reaches it)"""
    g = m._grid_host
    with torch.no_grad():
        m.density_plane[0][0, 0, g[1] // 4:3 * g[1] // 4, :3 * g[0] // 4] += amp
        m.density_line[0][0, 0, g[2] // 4:3 * g[2] // 4, 0] += amp


def _alpha_build(m, dims, want_mask):
    """one lrf_alpha_mask_build call on NaN-prefilled outputs -> (alpha [gx,gy,gz], mask [gz,gy,gx] or None, kept)"""
    dims = [int(d) for d in dims]
    alpha = torch.full(dims, float("nan"), device="cuda")
    mask = torch.full(dims[::-1], float("nan"), device="cuda") if want_mask else None
    kept = torch.zeros(1, dtype=torch.int64, device="cuda")
    fs, _ = m._field_struct(None, need_mlp=False)
    _lib.check(_lib.lib().lrf_alpha_mask_build(C.byref(fs), (C.c_int32 * 3)(*dims), float(m.stepSize),
                                               float(m.alphaMask_thres), _ptr(alpha), _ptr(mask), _ptr(kept),
                                               _stream()))
    torch.cuda.synchronize()
    return alpha, mask, int(kept)


@pytest.mark.parametrize("dims", [[150, 150, 150], [1, 37, 64]], ids=["150cubed", "dim1"])
def test_alpha_mask_build(field300, dims):
    m = field300
    _add_dense_region(m)
    alpha, mask, kept = _alpha_build(m, dims, True)
    n = alpha.numel()
    assert not alpha.isnan().any() and not mask.isnan().any()          # every element written
    a64 = so.dense_alpha64(m, dims)
    err = float((alpha.double() - a64).abs().max())
    pooled = so.pooled_alpha64(a64)
    thres = float(m.alphaMask_thres)
    ref = pooled >= thres
    near = (pooled - thres).abs() <= ALPHA_TOL
    assert bool(((mask == 0) | (mask == 1)).all())
    bad = int(((mask == 1) != ref)[~near].sum())
    print(f"\n  {dims}: {n} points, passes {_passes(n)}, alpha max err {err:.2e}, kept {kept / n:.3f}, "
          f"pooled within {ALPHA_TOL:g} of thres: {int(near.sum())}")
    assert err <= ALPHA_TOL
    assert bad == 0
    assert kept == int(mask.sum())
    assert 0.05 <= kept / n <= 0.6


def test_alpha_mask_build_masked_lattice(field300):
    """updateAlphaMask at the reference's gridSize / 2, then getDenseAlpha with that mask in place: alpha is exactly
    0 where the mask culls (compute_alpha, tensorBase.py:538-558) and the float64 alpha elsewhere.

    Which mask voxels carry weight at a point depends on fp32 rounding only where one of its voxel coordinates lies
    within 1e-3 of an integer (a "tie": the fp32 trilinear weight of a neighbour may be 0 or a tiny positive value).
    Away from ties the keep decision must equal oracle.alpha_mask_sample, which is pinned to the reference.  At a tie
    only the decisions that cannot flip are asserted: kept if a set voxel has float64 weight >= 1e-3, culled if no
    voxel around the nearest one is set.  So only [151, 149, 153] (96 % of its points off the ties) is compared with
    the oracle.  On the voxel-centre lattice (dims equal to the mask's) and on the gx = 1 lattice (the x = aabb min
    face) every point is a tie, and those two check the pinned decisions alone."""
    from oracle import oracle as orc
    m = field300
    _add_dense_region(m)
    m.updateAlphaMask((150, 150, 150))
    vol = m.alphaMask.alpha_volume.detach()                               # [1, 1, gz, gy, gx]
    vdims = torch.tensor(vol.shape[-3:][::-1], dtype=torch.float64, device="cuda")       # (gx, gy, gz)
    near_vox = torch.nn.functional.max_pool3d(vol, 3, 1, 1)[0, 0]
    of = oracle_field(m)
    aabb = m.aabb.detach().double()
    for dims, vs_oracle in (([151, 149, 153], True), ([150, 150, 150], False), ([1, 150, 150], False)):
        alpha, _, _ = _alpha_build(m, dims, False)
        assert not alpha.isnan().any()
        a64 = so.dense_alpha64(m, dims)
        assert float(a64.min()) > 20 * ALPHA_TOL            # an alpha of 0 can only come from the mask
        pts = so.lattice_points(m.aabb.detach(), dims)
        culled = alpha == 0
        vc = (pts.double() - aabb[0]) / (aabb[1] - aabb[0]) * (vdims - 1)
        tie = ((vc - vc.round()).abs() < 1e-3).any(-1)
        g = (2 * vc / (vdims - 1) - 1).view(1, -1, 1, 1, 3)
        v64 = torch.nn.functional.grid_sample(vol.double(), g, align_corners=True).view(dims)
        r = vc.round().long()
        around = near_vox[r[..., 2], r[..., 1], r[..., 0]]
        sure_keep, sure_cull = tie & (v64 >= 1e-3), tie & (around == 0)
        msg = (f"\n  {dims}: culled {float(culled.float().mean()):.3f}, ties {int(tie.sum())} "
               f"(pinned keep {int(sure_keep.sum())}, cull {int(sure_cull.sum())})")
        if vs_oracle:
            keep = torch.from_numpy(orc.alpha_mask_sample(of, pts.reshape(-1, 3).cpu().numpy()) > 0).cuda().view(dims)
            msg += f", disagreements with the oracle off the ties {int(((culled == keep) & ~tie).sum())}"
            assert float((~tie).float().mean()) >= 0.9
            assert int(((culled == keep) & ~tie).sum()) == 0
        else:
            assert bool(tie.all())
        print(msg)
        assert not bool((culled & sure_keep).any()) and bool(culled[sure_cull].all())
        assert int(sure_keep.sum()) > 0 and int(sure_cull.sum()) > 0
        assert 0.05 <= float(culled.float().mean()) <= 0.95
        err = float((alpha.double() - a64)[~culled].abs().max())
        assert err <= ALPHA_TOL, err


# ---- 3. lrf_upsample / up_sampling_VM ------------------------------------------------------------------------
def _upsample(src, H2, W2):
    """lrf_upsample of src [H, W, C] (fp32, contiguous) into a NaN-prefilled [H2, W2, C]"""
    H, W, Cc = src.shape
    dst = torch.full((H2, W2, Cc), float("nan"), device="cuda")
    _lib.check(_lib.lib().lrf_upsample(_ptr(src), H, W, _ptr(dst), H2, W2, Cc, _stream()))
    torch.cuda.synchronize()
    return dst


def _check_upsample(src, H2, W2, dst):
    """the blend of ATen's fp32 weights in fp32 rounds at most three times along any path, each time relative to a
    value of at most the largest tap: |out - float64 blend| <= 4 u max|tap| per element"""
    ref, tap = so.upsample64(src, H2, W2)
    assert not dst.isnan().any()
    excess = float(((dst.double() - ref).abs() - 4 * U * tap).max())
    assert excess <= 0, excess
    # what the reference runs: CUDA fp32 F.interpolate (its NHWC kernel may contract differently: reported only)
    x = src.permute(2, 0, 1)[None].contiguous(memory_format=torch.channels_last)
    ti = torch.nn.functional.interpolate(x, size=(H2, W2), mode="bilinear", align_corners=True)[0].permute(1, 2, 0)
    same = int((ti == dst).sum())
    print(f"\n  {tuple(src.shape)} -> ({H2}, {W2}): {dst.numel() // 4} threads, "
          f"max err / ulp-of-tap {float(((dst.double() - ref).abs() / (U * tap).clamp_min(1e-300)).max()):.2f}, "
          f"bit-identical to F.interpolate {same}/{dst.numel()}")


@pytest.mark.parametrize("H,W,H2,W2,Cc", [
    (64, 1, 137, 1, 8), (64, 1, 137, 1, 24),                  # lines
    (64, 64, 137, 129, 8), (64, 64, 137, 129, 24),            # planes, non-integer ratios
    (48, 40, 1, 40, 8), (1, 48, 5, 96, 8),                    # H2 = 1 (scale 0), H = 1
    (137, 129, 64, 64, 24),                                   # downsample
    (449, 449, 640, 640, 24),                                 # 2.46 M threads
])
def test_upsample(H, W, H2, W2, Cc):
    src = torch.randn(H, W, Cc, device="cuda", generator=torch.Generator("cuda").manual_seed(H * W + Cc))
    _check_upsample(src, H2, W2, _upsample(src, H2, W2))
    if H2 * W2 * Cc // 4 > _grid_threads():
        assert _passes(H2 * W2 * Cc // 4) >= 4


def test_upsample_identity_is_exact():
    src = torch.randn(37, 53, 24, device="cuda")
    dst = _upsample(src, 37, 53)
    assert torch.equal(dst.view(torch.int32), src.view(torch.int32))


def test_up_sampling_vm_nchw_source():
    """an NCHW-contiguous plane (the permute branch of up_sampling_VM) and the lines, through the module"""
    m = _field([16, 16, 16])
    planes = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(1, 24, 64, 48, device="cuda"))
                                     for _ in range(3)])
    lines = torch.nn.ParameterList([_cl_param(torch.randn(1, 24, 50, 1, device="cuda")) for _ in range(3)])
    assert not planes[0].is_contiguous(memory_format=torch.channels_last)
    srcs = [p.detach().permute(0, 2, 3, 1)[0].contiguous() for p in planes]
    lsrc = [l.detach().permute(0, 2, 3, 1)[0].contiguous() for l in lines]
    res = [70, 90, 110]
    planes, lines = m.up_sampling_VM(planes, lines, res)
    for i, (m0, m1) in enumerate(so.MAT_MODE):
        # sizes: plane i is [res[m1], res[m0]], line i is [res[vecMode[i]], 1]; the sources are [64, 48] / [50, 1]
        for got, src, (h2, w2) in ((planes[i], srcs[i], (res[m1], res[m0])),
                                   (lines[i], lsrc[i], (res[so.VEC_MODE[i]], 1))):
            assert got.shape == (1, 24, h2, w2) and got.is_contiguous(memory_format=torch.channels_last)
            _check_upsample(src, h2, w2, got.detach()[0].permute(1, 2, 0).contiguous())


# ---- 4. lrf_tv_sums / TV_loss_density / TV_loss_app -------------------------------------------------------------
@pytest.mark.parametrize("H,W,Cc", [(300, 300, 24), (300, 1, 24), (1, 300, 8), (1, 1, 4), (37, 53, 1),
                                    (37, 53, 3), (45, 300, 8)])
def test_tv_sums(H, W, Cc):
    """raw sums: each is a sum of non-negative fp32 terms (one rounding for the difference, one for the fused
    square-add) over at most `passes` terms per thread, two 5-level warp reductions and a float64 block total, so
    the relative error is at most (passes + 14) u"""
    x = torch.randn(H, W, Cc, device="cuda", generator=torch.Generator("cuda").manual_seed(H + 7 * W + 31 * Cc))
    sums = torch.zeros(2, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().lrf_tv_sums(_ptr(x), H, W, Cc, _ptr(sums), _stream()))
    got = sums.tolist()
    want = so.tv_sums64(x)
    bound = (_passes(x.numel()) + 14) * U
    for g, w in zip(got, want):
        if w == 0:
            assert g == 0
        else:
            assert abs(g - w) <= bound * w, (g, w, bound)
    print(f"\n  [{H},{W},{Cc}]: passes {_passes(x.numel())}, rel err " +
          ", ".join(f"{abs(g - w) / w:.2e}" if w else "exact 0" for g, w in zip(got, want)) + f" (bound {bound:.1e})")


TV_GRAD_BAR = 1e-6       # H100 80GB HBM3: 1.4e-7 of the tensor's max gradient


def _check_tv(planes, lines, call, grad_bar):
    """loss through the module's TV path (lrf_tv_sums / lrf_tv_sums_backward) against float64 autograd of the
    reference formulation"""
    for t in (*planes, *lines):
        t.grad = None
    reg = TVLoss(TVLoss_weight=0.5)
    val = call(reg)
    (val * 3.0).backward()
    p64 = [p.detach().double().requires_grad_() for p in planes]
    l64 = [l.detach().double().requires_grad_() for l in lines]
    ref = so.tv_total(p64, l64, reg)
    (ref * 3.0).backward()
    verr = abs(float(val.detach()) - float(ref.detach())) / abs(float(ref.detach()))
    assert all(t.grad is not None for t in (*planes, *lines))
    # a tensor with H = W = 1 has no differences: TVLoss returns 0 and autograd never reaches it
    refs = [r.grad if r.grad is not None else torch.zeros_like(r) for r in (*p64, *l64)]
    errs = [_scale_err(t.grad, r) for t, r in zip((*planes, *lines), refs) if r.abs().max() > 0]
    print(f"\n  value {verr:.2e}, grads " + ", ".join(f"{a:.1e}/{b:.1e}" for a, b in errs))
    assert verr <= 3e-7                          # H100 80GB HBM3: 5.1e-8
    assert max(a for a, _ in errs) <= grad_bar
    for t, r in zip((*planes, *lines), refs):
        if r.abs().max() == 0:
            assert float(t.grad.abs().max()) == 0


def test_tv_bench_field(field300):
    """300^2 x 24 appearance planes and 300 x 24 lines, 300^2 x 8 density planes"""
    m = field300
    _check_tv(list(m.app_plane), list(m.app_line), m.TV_loss_app, grad_bar=TV_GRAD_BAR)
    _check_tv(list(m.density_plane), list(m.density_line), m.TV_loss_density, grad_bar=TV_GRAD_BAR)
    assert _passes(m.app_plane[0].numel()) >= 4


@pytest.mark.parametrize("shapes", [
    ([(8, 1, 37), (8, 29, 1), (8, 1, 1)], [(8, 1), (8, 45), (8, 3)]),          # H = 1, W = 1, both
    ([(1, 37, 53), (1, 20, 33), (1, 64, 17)], [(1, 41), (1, 7), (1, 90)]),      # C = 1
    ([(3, 37, 53), (3, 20, 33), (3, 64, 17)], [(3, 41), (3, 7), (3, 90)]),      # C = 3
    ([(8, 45, 300), (8, 300, 45), (8, 128, 7)], [(8, 300), (8, 45), (8, 128)]),  # non-square
], ids=["H1-W1", "C1", "C3", "nonsquare"])
def test_tv_shapes(shapes):
    m = _field([16, 16, 16])
    g = torch.Generator("cuda").manual_seed(3)
    m.density_plane = torch.nn.ParameterList([_cl_param(torch.randn(1, c, h, w, device="cuda", generator=g))
                                              for c, h, w in shapes[0]])
    m.density_line = torch.nn.ParameterList([_cl_param(torch.randn(1, c, n, 1, device="cuda", generator=g))
                                             for c, n in shapes[1]])
    _check_tv(list(m.density_plane), list(m.density_line), m.TV_loss_density, grad_bar=TV_GRAD_BAR)


# ---- 5. lrf_sample_ray ----------------------------------------------------------------------------------------
def _sample_ray(rays, jitter, S, aabb, near, far, step):
    n = rays.shape[0]
    pts = torch.full((n, S, 3), float("nan"), device="cuda")
    z = torch.full((n, S), float("nan"), device="cuda")
    inside = torch.full((n, S), 7, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().lrf_sample_ray(_ptr(rays), _ptr(jitter), n, S, (C.c_float * 6)(*aabb.reshape(-1).tolist()),
                                         near, far, step, _ptr(pts), _ptr(z), _ptr(inside), _stream()))
    torch.cuda.synchronize()
    return pts, z, inside


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def test_sample_ray_grid_stride(field300):
    """4096 rays x 600 samples through the module's sample_ray (eval): bit-exact against the fp32 torch ops"""
    m = field300
    g = torch.Generator("cuda").manual_seed(11)
    o = 3.0 * torch.rand(4096, 3, device="cuda", generator=g) - 1.5
    d = torch.randn(4096, 3, device="cuda", generator=g)
    pts, z, inside = m.sample_ray(o, d, is_train=False, N_samples=600)
    rp, rz, rin = so.sample_ray32(o, d, m.aabb.detach(), m.near_far[0], m.near_far[1], float(m.stepSize), 600)
    assert _passes(4096 * 600) >= 4
    assert _bits_equal(z, rz) and _bits_equal(pts, rp)
    assert torch.equal(inside, rin)
    assert 0.1 <= float(inside.float().mean()) <= 0.9


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train-jitter"])
def test_sample_ray_edges(train):
    """zero and negative-zero direction components (the 1e-6 substitution), origins inside the box and outside the
    slab of a zero component, entry distances past `far`; train mode with a fixed per-ray jitter"""
    aabb = torch.tensor([[-2.0, -1.5, -1.0], [2.0, 1.5, 1.0]], device="cuda")
    near, far, step, S = 0.1, 3.5, 0.0137, 97
    g = torch.Generator("cuda").manual_seed(23)
    n = 6000
    o = (torch.rand(n, 3, device="cuda", generator=g) * 2 - 1) * torch.tensor([4.5, 4.0, 3.5], device="cuda")
    d = torch.randn(n, 3, device="cuda", generator=g)
    kind = torch.randint(0, 6, (n, 3), device="cuda", generator=g)       # 4: +0.0, 5: -0.0, else as drawn
    d = torch.where(kind == 4, torch.zeros_like(d), torch.where(kind == 5, torch.full_like(d, -0.0), d))
    rays = torch.cat([o, d], -1).contiguous()
    jitter = torch.rand(n, device="cuda", generator=g) if train else None
    pts, z, inside = _sample_ray(rays, jitter, S, aabb, near, far, step)
    rp, rz, rin = so.sample_ray32(o, d, aabb, near, far, step, S, jitter)
    assert _bits_equal(z, rz) and _bits_equal(pts, rp)
    assert torch.equal(inside, rin.to(torch.uint8))
    # the data reaches every edge this test is about
    neg0 = (d == 0) & torch.signbit(d)
    out_slab = (o < aabb[0]) | (o > aabb[1])
    inbox = ((o >= aabb[0]) & (o <= aabb[1])).all(-1)
    vec = torch.where(d == 0, torch.full_like(d, 1e-6), d)
    entry = torch.minimum((aabb[1] - o) / vec, (aabb[0] - o) / vec).amax(-1)
    for what, cnt in (("-0.0 component outside its slab", int((neg0 & out_slab).sum())),
                      ("+0.0 component outside its slab", int(((d == 0) & ~torch.signbit(d) & out_slab).sum())),
                      ("origin inside the box", int(inbox.sum())), ("entry past far", int((entry > far).sum())),
                      ("entry before near", int((entry < near).sum())),
                      ("entry between near and far", int(((entry >= near) & (entry <= far)).sum()))):
        assert cnt >= 50, what
    assert 0.01 <= float(inside.float().mean()) <= 0.9
