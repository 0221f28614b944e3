"""-m gpu: lrf_render_backward and lrf_render_backward_batch across the batch sizes, sample counts, grids and options
their C ABI accepts, against the float64 restatement of tests/render64.py with its hard decisions removed.

Three devices make the tight bars possible at any size:
  - zeroed cotangents: the backward is linear in grad_rgb, grad_depth and grad_directions, so a ray whose decision
    margins (render64.py) fall below their bounds gets zero cotangents and adds exactly nothing on either side; the
    excluded fraction is printed and asserted small, so a seed cannot make a case vacuous;
  - MLPs with no near-zero pre-activation (render64.random_field(safe_mlp=True)), checked with the `mlp` margin, for
    the cases with many shaded samples; one random-MLP case at small S on the CUDA-core path keeps masks that vary
    by sample (the golden fields of test_gpu_backward.py keep them on both paths);
  - d_rays compared row by row, skipping the rows with a texel-floor tie (only the position gradients jump there).

Error model of the bar.  Per tensor: max |kernel - float64| / max |float64|.  The CUDA-core path (LRF_BWD_TC=0) is
fp32 throughout: each gradient entry is a sum of up to a few thousand terms, each carrying a few roundings, so its
error is a few hundred EPS = 2^-24 of the tensor's scale at worst (1e-5).  The tensor-core path runs its four
per-sample products as three bf16 products of hi / lo operands (about 16 mantissa bits: 2^-16 = 1.5e-5 relative per
product, the same order after a 128-term sum).  Both are well under TOL = 2e-4, the bar the golden fields meet; a
corrupted tile, a lost pass or a dropped carry moves whole samples, O(1e-2) or more of a tensor's scale.
Measured on an H100 80GB HBM3 at a 700 W power limit: at most 3.7e-5 on any field tensor or d_rays row set (300^3
relu, S = 344; the 2^-16 products of the tensor-core path stay at the CUDA-core path's level), 1.3e-5 through the
training call, 2e-5 on the camera gradients; 1.0e-3 at S = 65535 (its own bar below)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import render64 as R

pytestmark = pytest.mark.gpu
TOL = 2e-4
MARGIN = 2.0 ** 6           # EPS units (render64.py): the contraction and mask margins below which a ray is zeroed
BOUND = 2.0                 # the propagated-bound margins (render64.BOUND_KEYS); the bound holds at 300^3 with the
                            # fp32 error at most 0.49 of it (test_render64_cpu.py::test_weight_error_bound_holds_at_300)
# the MLP margin counts 8 EPS per layer sum; the tensor-core path's three bf16 products leave 3 x 2^-16 = 96 times that
MARGIN_MLP = {True: BOUND * 96, False: BOUND}
MAX_EXCLUDED = 0.06         # measured <= 5.5 % (300^3, S = 344, relu: weights near 1e-3, features near 0)
TEXEL_MARGIN = 4.0          # texel-floor units (4 size EPS, render64.py); a pixel coordinate carries about 2 size EPS


def scale_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def n_sms():
    from localrf_b200 import _lib
    v = [C.c_int32() for _ in range(3)]
    _lib.check(_lib.lib().lrf_launch_info(*[C.byref(x) for x in v]))
    assert v[0].value == torch.cuda.get_device_properties(0).multi_processor_count
    return v[0].value


ztable, make_rays = R.ztable, R.make_rays


def make_module(fd):
    """A (product) TensorVMSplit holding fd's parameters (rounded to fp32)."""
    import localrf_b200 as L
    from gpu_helpers import field_kwargs
    from helpers import FIELD_KEYS, field_scalars
    sc = field_scalars(fd)
    aabb = torch.as_tensor(fd["aabb"], dtype=torch.float32)
    m = L.TensorVMSplit("cpu", aabb, sc["gridSize"], **field_kwargs(sc))
    if "alphaMask.alpha_volume" in fd:
        m.alphaMask = L.AlphaGridMask("cpu", aabb, torch.as_tensor(fd["alphaMask.alpha_volume"], dtype=torch.float32))
    sd = m.state_dict()
    for k in FIELD_KEYS:
        sd[k] = torch.as_tensor(np.asarray(fd[k]), dtype=torch.float32).reshape(sd[k].shape)
    m.load_state_dict(sd)
    return m.cuda()


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _unfold(m, bufs):
    """The kernel's buffers as float64 gradients keyed like render64.PARAM_KEYS (d_w1b unfolded in float64)."""
    d_dp, d_dl, d_ap, d_al, d_w1b, d_b1, d_w2, d_b2, d_w3, d_b3 = bufs
    w1, basis = m.renderModule.mlp[0].weight.detach().double(), m.basis_mat.weight.detach().double()
    vals = (*d_dp, *d_dl, *d_ap, *d_al, w1.t() @ d_w1b.double(), d_w1b.double() @ basis.t(), d_b1, d_w2, d_b2, d_w3,
            d_b3)
    return {k: v.double() for k, v in zip(R.PARAM_KEYS, vals)}


def _flat(bufs):
    return [t for b in bufs for t in (b if isinstance(b, list) else [b])]


def kernel_backward(m, rays, z, white_bg, g_rgb, g_depth, prefill=None, scratch_byte=0, d_rays_fill=math.nan):
    """lrf_render_backward called directly -> (float64 gradients keyed like PARAM_KEYS plus "rays", raw buffers)."""
    from localrf_b200 import _lib
    from localrf_b200.tensorf import _field_grad_buffers
    lib = _lib.lib()
    n = rays.shape[0]
    fs, _ = m.field_and_prepared(z, fp32=True)
    bp = m._prepared_backward()
    bufs, g = _field_grad_buffers(m, torch.device("cuda"))
    if prefill is not None:
        for b, p in zip(_flat(bufs), prefill):
            b.copy_(p)
    d_rays = torch.full((n, 6), d_rays_fill, device="cuda")
    g.d_rays = d_rays.data_ptr()
    need = lib.lrf_backward_scratch_bytes(n, z.numel())
    scratch = torch.full((need,), scratch_byte, dtype=torch.uint8, device="cuda")
    _lib.check(lib.lrf_render_backward(C.byref(fs), _ptr(bp), _ptr(rays), n, int(white_bg), _ptr(g_rgb),
                                       _ptr(g_depth), C.byref(g), _ptr(scratch), need, _stream()))
    torch.cuda.synchronize()
    out = _unfold(m, bufs)
    out["rays"] = d_rays
    return out, bufs


def cotangents(n, seed, keep=None):
    g = torch.Generator().manual_seed(seed)
    c_rgb, c_depth = torch.randn(n, 3, generator=g), 0.05 * torch.randn(n, generator=g)
    if keep is not None:
        c_rgb, c_depth = c_rgb * keep[:, None], c_depth * keep
    return c_rgb.cuda().contiguous(), c_depth.cuda().contiguous()


def excluded(ex, tc):
    """Rays to drop: any decision margin below its bound."""
    per = {k: ex[k] < (MARGIN_MLP[tc] if k == "mlp" else BOUND if k in R.BOUND_KEYS else MARGIN)
           for k in R.MARGIN_KEYS}
    print("rays below each margin:", {k: int(v.sum()) for k, v in per.items()})
    return torch.stack(list(per.values())).any(0)


def compare(tag, got, ref, skip_rows, tol=TOL):
    errs = {k: scale_err(got[k], ref[k]) for k in R.PARAM_KEYS}
    keep = ~skip_rows
    print(f"d_rays rows compared: {int(keep.sum())} of {keep.numel()}")
    if bool(keep.any()):
        errs["rays"] = scale_err(got["rays"][keep], ref["rays"][keep])
    print(tag, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < tol, (tag, errs)
    return errs


def _mask(dims, seed):
    rng = np.random.default_rng(seed)
    return (rng.random((1, 1, *dims)) > 0.3).astype(np.float64)


# (grid, S, act, white_bg, mask, thres, safe MLP, n rays, far z table); both shade paths unless noted
CASES = {
    "g2_S2": ((2, 2, 2), 2, "softplus", True, False, 1e-3, True, 512, True),
    "g2_S33_relu_mask": ((2, 2, 2), 33, "relu", False, True, 1e-3, True, 512, True),
    "g405264_S31_mask": ((40, 52, 64), 31, "softplus", False, True, 1e-3, True, 1024, True),
    "g405264_S32_relu": ((40, 52, 64), 32, "relu", True, False, 1e-3, True, 1024, True),
    "g405264_S33_thres0": ((40, 52, 64), 33, "softplus", True, False, 0.0, True, 1024, False),
    "g300_S344_mask": ((300, 300, 300), 344, "softplus", True, True, 1e-3, True, 4096, True),
    "g300_S344_relu": ((300, 300, 300), 344, "relu", False, False, 1e-3, True, 4096, True),
    "g300_S344_thres0": ((300, 300, 300), 344, "softplus", True, False, 0.0, True, 2048, False),
    "g640_S738_thres0": ((640, 640, 640), 738, "softplus", False, False, 0.0, True, 2048, False),
    "g405264_S65535": ((40, 52, 64), 65535, "softplus", True, False, 1e-3, True, 4, 0.6),
}


def _run_case(grid, S, act, white_bg, mask, thres, safe, n, far, tc, seed=0, monkeypatch=None, shift=-2.0,
              coarse=None):
    monkeypatch.setenv("LRF_BWD_TC", "1" if tc else "0")
    # grids of 300^3 and more: upsampled from 32 per axis, as training grows them (steep grids: the smaller cases)
    fd = R.random_field(grid, act=act, shift=shift, thres=thres, seed=seed, safe_mlp=safe,
                        coarse=coarse or (32 if max(grid) >= 300 else None),
                        mask=_mask((17, 19, 23), seed) if mask else None)
    m = make_module(fd)
    F = R.Field64.from_module(m, "cuda")
    rays = make_rays(n, seed + 1, spread=2.5 if far is True or far is False else 0.2).cuda()
    z = ztable(S, far).cuda()
    with torch.no_grad():
        ex = {}
        step = max(1, R.CHUNK_SAMPLES // S)
        for r0 in range(0, n, step):
            _, _, e = R.field_forward(F, rays[r0:r0 + step].double(), z.double(), white_bg, True)
            for k, v in e.items():
                ex.setdefault(k, []).append(v)
        ex = {k: torch.cat(v) for k, v in ex.items()}
    drop = excluded(ex, tc)
    frac = float(drop.double().mean())
    print(f"excluded {int(drop.sum())} of {n} rays ({100 * frac:.2f} %); shaded samples {int(ex['n_app'].sum())}")
    if safe:
        assert float(ex["mlp"].min()) > 1e4, "the safe MLP has a pre-activation near 0"
    assert frac <= MAX_EXCLUDED or n <= 4 and frac == 0
    keep = (~drop).float().cpu()
    g_rgb, g_depth = cotangents(n, seed + 2, keep)
    got, _ = kernel_backward(m, rays, z, white_bg, g_rgb, g_depth)
    ref, _ = R.field_backward(F, rays, z, white_bg, g_rgb, g_depth, want_margins=False)
    return got, ref, ex, drop, (m, F, rays, z, g_rgb, g_depth)


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("shade", ["wgmma", "cuda_cores"])
def test_backward_vs_float64(case, shade, monkeypatch):
    grid, S, act, white_bg, mask, thres, safe, n, far = CASES[case]
    got, ref, ex, drop, _ = _run_case(grid, S, act, white_bg, mask, thres, safe, n, far, shade == "wgmma",
                                      monkeypatch=monkeypatch)
    # the transmittance product and the suffix sum of the density backward run sequentially over the S samples of a
    # ray, one rounding per sample each: their relative error is bounded by 2 S EPS (7.8e-3 at S = 65535; measured
    # 1.0e-3, the rounding errors partly cancelling); below S = 1600 the bound is under TOL
    compare(f"{case} {shade}", got, ref, ex["texel"] < TEXEL_MARGIN, tol=max(TOL, 2 * S * R.EPS))


def test_random_mlp_small_S_cuda_cores(monkeypatch):
    """A random MLP (ReLU masks that vary by sample) at S = 26 on the CUDA-core path, where the ReLU margins exclude
    few rays (3.7 %: grids upsampled from 8 per axis, so the products' slope adds little to the pre-activations'
    error; on steep grids the position error excludes 19 %)."""
    got, ref, ex, drop, _ = _run_case((40, 52, 64), 26, "softplus", True, False, 1e-3, False, 2048, True, False,
                                      seed=5, monkeypatch=monkeypatch, shift=2.0, coarse=8)
    compare("random MLP S 26", got, ref, ex["texel"] < TEXEL_MARGIN)


@pytest.mark.parametrize("count", ["62", "63", "64", "65", "128", "64sm", "64sm+2"])
@pytest.mark.parametrize("shade", ["wgmma", "cuda_cores"])
def test_shade_tile_fills(count, shade, monkeypatch):
    """weight_thres = 0, no mask and a low-density field: every sample has w > 0, so the shade kernel's list holds
    exactly n S samples -- full and partial last tiles, one tile per CTA and a second round of tiles."""
    sm = n_sms()
    n, S = {"62": (2, 31), "63": (1, 63), "64": (2, 32), "65": (1, 65), "128": (4, 32), "64sm": (2 * sm, 32),
            "64sm+2": (32 * sm + 1, 2)}[count]
    monkeypatch.setenv("LRF_BWD_TC", "1" if shade == "wgmma" else "0")
    fd = R.random_field((40, 52, 64), shift=-6.0, thres=0.0, seed=3, safe_mlp=True)
    m = make_module(fd)
    F = R.Field64.from_module(m, "cuda")
    rays = make_rays(n, 4, spread=1.0).cuda()
    z = ztable(S, far=False).cuda()
    g_rgb, g_depth = cotangents(n, 6)
    ref, fwd = R.field_backward(F, rays, z, True, g_rgb, g_depth)
    assert int((fwd["w"] > 0).sum()) == n * S == int(fwd["n_app"].sum())
    assert not bool(excluded(fwd, shade == "wgmma").any())
    got, _ = kernel_backward(m, rays, z, True, g_rgb, g_depth)
    compare(f"{n * S} shaded samples {shade}", got, ref, fwd["texel"] < TEXEL_MARGIN)


# ---- scale without a reference: grid-stride passes, chunking, ABI promises -----------------------------------------
@pytest.fixture(scope="module")
def field_small():
    fd = R.random_field((40, 52, 64), shift=-2.0, thres=1e-3, seed=7, safe_mlp=True)
    return make_module(fd)


def _sum_err(parts, whole):
    return max(scale_err(sum(p[k] for p in parts), whole[k]) for k in R.PARAM_KEYS)


@pytest.mark.parametrize("which", ["-1", "0", "+1", "2x+37"])
def test_render_backward_grid_stride(field_small, which):
    """n = 64 n_sms - 1 .. 2 (64 n_sms) + 37 rays: the march and density kernels' grid-stride loops run a second pass.
    Each ray's d_rays equals its row rendered in chunks of 4096 and alone (within the order of the per-ray atomics of
    lrf_render_backward), and the parameter gradients are the sum of the chunks' (within fp32 atomic order)."""
    sm = n_sms()
    n = {"-1": 64 * sm - 1, "0": 64 * sm, "+1": 64 * sm + 1, "2x+37": 128 * sm + 37}[which]
    m = field_small
    rays = make_rays(n, 11).cuda()
    z = ztable(72).cuda()
    g_rgb, g_depth = cotangents(n, 12)
    whole, _ = kernel_backward(m, rays, z, True, g_rgb, g_depth)
    assert bool(torch.isfinite(whole["rays"]).all())
    parts = [kernel_backward(m, rays[a:a + 4096], z, True, g_rgb[a:a + 4096], g_depth[a:a + 4096])[0]
             for a in range(0, n, 4096)]
    d_parts = torch.cat([p["rays"] for p in parts])
    err = float((d_parts - whole["rays"]).abs().max() / whole["rays"].abs().max())
    assert err < 1e-6, err
    e = _sum_err(parts, whole)
    print(f"n {n}: d_rays chunked {err:.1e}, parameters {e:.1e}")
    assert e < 1e-4                        # measured <= 2.5e-5: sums of thousands of atomics, in another order
    for r in (0, min(64 * sm, n - 1), n - 1):
        alone, _ = kernel_backward(m, rays[r:r + 1], z, True, g_rgb[r:r + 1], g_depth[r:r + 1])
        assert float((alone["rays"][0] - whole["rays"][r]).abs().max()) <= 1e-6 * float(whole["rays"].abs().max())


def test_render_backward_abi_promises(field_small):
    """Scratch filled with 0xFF gives what zeroed scratch gives, parameter buffers pre-filled with P receive P + the
    gradient, and a NaN-filled d_rays is overwritten everywhere."""
    m = field_small
    n = 3000
    rays = make_rays(n, 21).cuda()
    z = ztable(72).cuda()
    g_rgb, g_depth = cotangents(n, 22)
    a, bufs = kernel_backward(m, rays, z, False, g_rgb, g_depth, scratch_byte=0)
    b, _ = kernel_backward(m, rays, z, False, g_rgb, g_depth, scratch_byte=0xFF)
    assert bool(torch.isfinite(a["rays"]).all()) and bool(torch.isfinite(b["rays"]).all())
    assert scale_err(b["rays"], a["rays"]) < 1e-6
    assert max(scale_err(b[k], a[k]) for k in R.PARAM_KEYS) < 1e-4
    gen = torch.Generator(device="cuda").manual_seed(3)
    P = [torch.randn(t.shape, generator=gen, device="cuda") * t.abs().max() for t in _flat(bufs)]
    c, cb = kernel_backward(m, rays, z, False, g_rgb, g_depth, prefill=P)
    check_prefill(_flat(cb), P, _flat(bufs))


def check_prefill(got, P, g0s):
    """Buffers pre-filled with P hold P + the gradient: entry by entry within the atomic order of the gradient's own
    sum (1e-4 of its scale, the bar of the sums of chunks; measured <= 2.5e-5) plus the rounding of P + g."""
    for t, p, g0 in zip(got, P, g0s):
        bar = 1e-4 * float(g0.abs().max()) + 2 * R.EPS * (p.abs() + g0.abs())
        assert bool(((t - p - g0).abs() <= bar).all())


# ---- the training call --------------------------------------------------------------------------------------------
def batch_backward(m, z, ids, W, H, fov360, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs, white_bg=True,
                   use_intr=True, null=(), scratch_byte=0, d_rays_fill=math.nan, prefill=None):
    """lrf_render_backward_batch called directly -> dict: float64 field gradients (PARAM_KEYS), "rays" (d_rays or
    None), the camera gradients (None where NULL) and "scratch_rays"."""
    import localrf_b200 as L
    from localrf_b200.local_tensorfs import _train_batch
    from localrf_b200.tensorf import _field_grad_buffers
    lib = L._lib.lib()
    n, V = ids.shape[0], c2w.shape[0]
    fs, _ = m.field_and_prepared(z, fp32=True)
    bp = m._prepared_backward()
    b = _train_batch(ids, W, H, fov360, c2w, intr, E, w2, white_bg)
    if not use_intr:
        b.intrinsics = None
        b.focal, b.cx, b.cy = (float(v) for v in intr.cpu())
    bufs, g = _field_grad_buffers(m, torch.device("cuda"))
    if prefill is not None:
        for b_, p in zip(_flat(bufs), prefill):
            b_.copy_(p)
    out = {"rays": None if "d_rays" in null else torch.full((n, 6), d_rays_fill, device="cuda")}
    if out["rays"] is not None:
        g.d_rays = out["rays"].data_ptr()
    shapes = dict(d_cam2world=(V, 3, 4), d_intrinsics=(3,), d_exposure=(V, 3, 3), d_world2rf=(3,))
    cg = L._lib.LrfCameraGrads()
    for k, s in shapes.items():
        out[k] = None if k in null else torch.full(s, math.nan, device="cuda")
        if out[k] is not None:
            setattr(cg, k, out[k].data_ptr())
    nbytes = lib.lrf_backward_batch_scratch_bytes(n, z.numel(), V)
    scratch = torch.full((nbytes,), scratch_byte, dtype=torch.uint8, device="cuda")
    L._lib.check(lib.lrf_render_backward_batch(C.byref(fs), _ptr(bp), C.byref(b), _ptr(x), _ptr(g_rgb),
                                               _ptr(g_depth), _ptr(g_dirs), C.byref(g), C.byref(cg), _ptr(scratch),
                                               nbytes, _stream()))
    torch.cuda.synchronize()
    out.update(_unfold(m, bufs))
    out["bufs"] = [t.clone() for t in _flat(bufs)]
    out["scratch_rays"] = scratch[: n * 24].view(torch.float32).view(n, 6).clone()
    return out


def _cameras(V, seed, W, H):
    g = torch.Generator().manual_seed(seed)
    c2w = torch.zeros(V, 3, 4)
    for v in range(V):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
        c2w[v, :, :3] = q
        c2w[v, :, 3] = 0.3 * torch.randn(3, generator=g)
    intr = torch.tensor([0.8 * W, 0.5 * W + 0.25, 0.5 * H - 0.375])
    return c2w.cuda().contiguous(), intr.cuda()


def _train_inputs(V, rpv, W, H, seed, exposure):
    """Ray ids, cameras, intrinsics, exposure (or None), world2rf and a pre-exposure colour x that puts E x exactly
    at 0 and at 1 on some channels: E = diag(2, 0.5, 1) (powers of two, so the kernel's fmas are exact there) or
    the identity."""
    g = torch.Generator().manual_seed(seed)
    n = V * rpv
    ids = torch.randint(0, W * H, (n,), generator=g) + torch.arange(V).repeat_interleave(rpv) * W * H
    c2w, intr = _cameras(V, seed + 1, W, H)
    E = torch.diag(torch.tensor([2.0, 0.5, 1.0])).expand(V, 3, 3).contiguous().cuda() if exposure else None
    x = torch.rand(n, 3, generator=g) * 1.2 - 0.1
    d = torch.tensor([2.0, 0.5, 1.0]) if exposure else torch.ones(3)
    x[0::7, 0] = 0.0
    x[1::7, 1] = 1.0 / d[1]
    x[2::7, 2] = 1.0 / d[2]
    x[3::7, 0] = 1.0 / d[0]
    w2 = torch.tensor([0.05, -0.02, 0.01]).cuda()
    g_rgb = torch.randn(n, 3, generator=g)
    g_depth = 0.05 * torch.randn(n, generator=g)
    g_dirs = 0.1 * torch.randn(n, 3, generator=g)
    return ids.cuda(), c2w, intr, E, w2, x.cuda().contiguous(), g_rgb, g_depth, g_dirs


TRAIN_CASES = {   # (n_views, rays per view, fov360, intrinsics pointer, exposure)
    "v1_r1": (1, 1, False, True, True),
    "v3_r255_fov360": (3, 255, True, True, False),
    "v3_r256_focal": (3, 256, False, False, True),
    "v3_r257": (3, 257, False, True, False),
    "v16_r257_focal": (16, 257, False, False, False),
    "v16_r1000_fov360": (16, 1000, True, False, True),
    "v1_r1000": (1, 1000, False, True, True),
}


def _train_case(m, F, z, V, rpv, fov360, use_intr, exposure, seed, tc):
    W, H = 96, 64
    ids, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs = _train_inputs(V, rpv, W, H, seed, exposure)
    n = V * rpv
    # the margins of the float64 forward first (they do not depend on the cotangents), then the cotangents
    _, fwd = R.train_backward(F, z, ids, W, H, fov360, intr, c2w, w2, E, x, True, g_rgb, g_depth, g_dirs)
    drop = excluded(fwd, tc) | (fwd["texel"] < TEXEL_MARGIN) | (fwd["clamp"] < MARGIN)
    frac = float(drop.double().mean())
    print(f"excluded {int(drop.sum())} of {n} rays ({100 * frac:.2f} %)")
    assert frac <= MAX_EXCLUDED or n <= 3 and frac < 1
    keep = (~drop).double().cpu()
    g_rgb, g_depth, g_dirs = g_rgb * keep[:, None], g_depth * keep, g_dirs * keep[:, None]
    ref, fwd = R.train_backward(F, z, ids, W, H, fov360, intr, c2w, w2, E, x, True, g_rgb, g_depth, g_dirs)
    f32 = lambda t: t.float().cuda().contiguous()
    got = batch_backward(m, z, ids, W, H, fov360, c2w, intr, E, w2, x, f32(g_rgb), f32(g_depth), f32(g_dirs),
                         use_intr=use_intr)
    return got, ref, fwd, (ids, c2w, intr, E, w2, x, f32(g_rgb), f32(g_depth), f32(g_dirs), W, H)


@pytest.fixture(scope="module")
def train_field():
    fd = R.random_field((40, 52, 64), shift=-2.0, thres=1e-3, seed=9, safe_mlp=True)
    m = make_module(fd)
    return m, R.Field64.from_module(m, "cuda"), ztable(72).cuda()


@pytest.mark.parametrize("case", list(TRAIN_CASES))
@pytest.mark.parametrize("shade", ["wgmma", "cuda_cores"])
def test_train_call_vs_float64(train_field, case, shade, monkeypatch):
    """lrf_render_backward_batch end to end from cam2world, intrinsics (pointer, or NULL with focal / cx / cy),
    exposure (or NULL) and world2rf, against the float64 restatement; E x sits exactly on 0 and 1 on some channels
    (both bounds pass the gradient).  Camera gradients: the same bar as the field's (they are fp64 sums of the
    d_rays rows, whose error the field's bar already bounds)."""
    monkeypatch.setenv("LRF_BWD_TC", "1" if shade == "wgmma" else "0")
    m, F, z = train_field
    V, rpv, fov360, use_intr, exposure = TRAIN_CASES[case]
    got, ref, fwd, _ = _train_case(m, F, z, V, rpv, fov360, use_intr, exposure, 31, shade == "wgmma")
    assert float((got["scratch_rays"].double() - fwd["rays"]).abs().max()) < 1e-5     # the rays it marched
    errs = compare(f"{case} {shade}", got, ref, fwd["texel"] < TEXEL_MARGIN)
    cam = {k: scale_err(got[k], ref[k]) for k in ("d_cam2world", "d_exposure", "d_world2rf")}
    if fov360:
        assert float(got["d_intrinsics"].abs().max()) == 0.0
    else:
        cam["d_intrinsics"] = scale_err(got["d_intrinsics"], ref["d_intrinsics"])
    print("camera:", {k: f"{v:.1e}" for k, v in cam.items()})
    assert max(cam.values()) < TOL, cam


def test_train_call_prologue_second_pass(monkeypatch):
    """n = 2048 n_sms + 1 rays at S = 2 on a [2, 2, 2] grid: ray_prologue_kernel's grid-stride loop runs twice."""
    sm = n_sms()
    fd = R.random_field((2, 2, 2), shift=-2.0, thres=1e-3, seed=13, safe_mlp=True)
    m = make_module(fd)
    F = R.Field64.from_module(m, "cuda")
    got, ref, fwd, _ = _train_case(m, F, ztable(2).cuda(), 1, 2048 * sm + 1, False, True, True, 41, True)
    compare("prologue 2 passes", got, ref, fwd["texel"] < TEXEL_MARGIN)
    cam = {k: scale_err(got[k], ref[k]) for k in ("d_cam2world", "d_exposure", "d_world2rf", "d_intrinsics")}
    print("camera:", {k: f"{v:.1e}" for k, v in cam.items()})
    assert max(cam.values()) < TOL, cam


def test_train_call_null_outputs_and_abi_promises(train_field):
    """Each optional output NULL in turn leaves the others bitwise unchanged (the field's parameter gradients, which
    are atomic sums, within their order); grad_directions = NULL is bitwise grad_directions = 0; scratch filled with
    0xFF gives the same bits as zeroed scratch; a NaN-filled d_rays and NaN-filled camera outputs are overwritten;
    parameter buffers pre-filled with P receive P + the gradient."""
    m, F, z = train_field
    ids, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs = _train_inputs(4, 300, 96, 64, 51, True)
    f32 = lambda t: t.float().cuda().contiguous()
    args = (m, z, ids, 96, 64, False, c2w, intr, E, w2, x, f32(g_rgb), f32(g_depth))
    full = batch_backward(*args, f32(g_dirs))
    det = ("rays", "d_cam2world", "d_intrinsics", "d_exposure", "d_world2rf")
    for k in det:
        assert bool(torch.isfinite(full[k]).all()), k
    for k in ("d_rays",) + det[1:]:
        part = batch_backward(*args, f32(g_dirs), null=(k,))
        for j in det:
            if j != (k if k != "d_rays" else "rays"):
                assert torch.equal(part[j], full[j]), (k, j)
        assert max(scale_err(part[j], full[j]) for j in R.PARAM_KEYS) < 1e-4, k
    a = batch_backward(*args, None)
    b = batch_backward(*args, torch.zeros(ids.shape[0], 3, device="cuda"))
    for j in det:
        assert torch.equal(a[j], b[j]), j
    c = batch_backward(*args, f32(g_dirs), scratch_byte=0xFF)
    for j in det:
        assert torch.equal(c[j], full[j]), j
    assert max(scale_err(c[j], full[j]) for j in R.PARAM_KEYS) < 1e-4
    gen = torch.Generator(device="cuda").manual_seed(5)        # the field's buffers accumulate here as well
    P = [torch.randn(t.shape, generator=gen, device="cuda") * t.abs().max() for t in full["bufs"]]
    d = batch_backward(*args, f32(g_dirs), prefill=P)
    check_prefill(d["bufs"], P, full["bufs"])
    for j in det:
        assert torch.equal(d[j], full[j]), j


@pytest.mark.parametrize("shade", ["wgmma", "cuda_cores"])
def test_train_call_rows_bitwise_across_chunks(train_field, shade, monkeypatch):
    """d_rays of the batch path is summed in a fixed order (no float atomics), and every wgmma / FMA row is
    independent of the other rows: a ray's row is bitwise the same rendered in one call of 2 (64 n_sms) + 37 rays
    (past the first grid-stride pass), in chunks of 4096 and alone.  The parameter gradients are the sum of the
    chunks' within fp32 atomic order."""
    monkeypatch.setenv("LRF_BWD_TC", "1" if shade == "wgmma" else "0")
    m, F, z = train_field
    sm = n_sms()
    n = 128 * sm + 37
    ids, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs = _train_inputs(1, n, 96, 64, 61, True)
    f32 = lambda t: t.float().cuda().contiguous()
    g_rgb, g_depth, g_dirs = f32(g_rgb), f32(g_depth), f32(g_dirs)
    run = lambda a, b: batch_backward(m, z, ids[a:b].contiguous(), 96, 64, False, c2w, intr, E, w2,
                                      x[a:b].contiguous(), g_rgb[a:b].contiguous(), g_depth[a:b].contiguous(),
                                      g_dirs[a:b].contiguous())
    whole = run(0, n)
    parts = [run(a, min(n, a + 4096)) for a in range(0, n, 4096)]
    assert torch.equal(torch.cat([p["rays"] for p in parts]), whole["rays"])
    for r in (0, 64 * sm - 1, 64 * sm, n - 1):
        assert torch.equal(run(r, r + 1)["rays"][0], whole["rays"][r]), r
    e = _sum_err(parts, whole)
    print(f"parameters, sum of chunks: {e:.1e}")
    assert e < 1e-4
