"""-m gpu: lrf_render across the batch sizes, sample counts, grids, options and outputs its C ABI accepts, against the
float64 restatement of tests/render64.py with its hard decisions removed, and bitwise against itself where the ABI
promises an exact result.

What the cases reach in the kernel (localrf_b200/csrc/lrf_render.cu):
  - producer counts: with the floater filter each producer warp keeps an S-float alpha table in shared memory, so
    the launch runs fewer producers as S grows (smem_total below restates the layout): 8 up to S = 1064, 7 from
    1065, ..., 1 from 4601 to 9312, and S = 9313 is refused; with positional encodings 473 / 2233 / 4577;
  - slot waits and mid-launch tile padding: an opaque field whose rays shade 1 to 3 samples, one producer, and a
    threshold above every weight (no tile at all);
  - early termination after the 32-sample block in which T falls below 1e-10, and the zeroed weight tail;
  - fewer CTAs than SMs below 8 n_sms rays, and the ray counter past the first round;
  - the outputs LocalTensorfs and the multi-GPU path use: pix, accumulate, blend with blend_stride, finalize with and
    without exposure over 1 to 16 views, explicit rays with exposure, the intrinsics pointer, directions and ij,
    stats, weights on both paths; bf16 grid storage and the positional-encoding instantiation.

Bars.  rgb and depth: per tensor, max |kernel - float64| / max |float64| < max(1e-4, 2 S EPS) -- the second term is
the sequential transmittance product's relative error bound (the backward suite's rule).  Weights: |dw| <= max(1e-4
max(|w|, 5e-3), w_err), w_err the propagated fp32 bound of render64 (it holds with room at 300^3,
test_render64_cpu.py::test_weight_error_bound_holds_at_300).  A ray is compared only if it clears the margins that
act in the forward (thres, floater, relu / softplus, mlp -- with the tensor-core factor --, mask; not the
contraction, which is continuous); the excluded fraction is printed and asserted small.
Measured on an H100 80GB HBM3 at a 700 W power limit: rgb at most 1.3e-6 and depth 3.3e-5 of their scale (300^3 relu,
S = 344), 1.0e-3 rgb at S = 65535 (bar 7.8e-3), weights at most 0.25 of their bar, at most 5.5 % of a case's rays
excluded, directions within 0.4 EPS (lean) and 11.6 EPS (360); the file runs in about 15 s."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import render64 as R
from test_gpu_backward_edges import BOUND, MARGIN, MARGIN_MLP, make_module, n_sms

pytestmark = pytest.mark.gpu
TOL = 1e-4
GUARD = 3                   # rows past n_rays in every output buffer, pre-filled with NaN: they must stay NaN
MAX_EXCLUDED = 0.08
OPTIN_H100 = 232448         # the H100's opt-in shared memory per block; the producer-count steps below are for it


# ---- the render kernel's shared-memory layout (smem_v3 in lrf_render.cu), for the producer counts -----------------
def smem_total(S, floater, nprod, pe):
    oper1, oper2, tail = 16 * 10 * 128, 16 * 16 * 128, 656 * 4
    prep = 2 * oper1 + 2 * oper2 + tail
    pe_res = 2 * 16 * 10 * 32 + 2 * oper2 + tail
    off = ((pe_res + 1023) & ~1023) + 2 * 16384 if pe else prep
    off = (off + 1023) & ~1023
    off += 4 * oper1 + 2 * 128 + 2 * 128 * 4 + (2 * 64 * 33 * 4 if pe else 0)
    off = (off + 15) & ~15
    off += 8 * 3 * 80                                   # 8 producers x 3 ray slots of 80 bytes
    off = (off + 15) & ~15
    per = 64 * 7 + (((S + 3) & ~3) * 4 if floater else 0)
    off += nprod * ((per + 15) & ~15)
    off = (off + 15) & ~15
    return (off + 56 + 15) & ~15


def n_producers(S, floater, pe, optin):
    return next((n for n in range(8, 0, -1) if smem_total(S, floater, n, pe) <= optin), 0)


def optin():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# ---- calling lrf_render directly ------------------------------------------------------------------------------------
def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, math.nan, dtype=dtype, device="cuda")


def render(m, z, n, rays=None, gen=None, white_bg=True, floater=0.0, refine=True, weights=True, stats=None,
           pix=None, rgb=None, depth=None, blend=None, blend_stride=0, exposure=None, n_views=1, accumulate=0,
           finalize=0, dirs=None, ij=None, fp32=True):
    """One lrf_render launch.  Outputs not given are allocated with GUARD extra rows of NaN.  gen: the ray-generation
    fields (ray_ids, W, H, fov360, focal, cx, cy, intrinsics, cam2world, world2rf).  -> (return code, outputs)."""
    from localrf_b200 import _lib
    fs, prep = m.field_and_prepared(z, fp32=fp32)
    S = z.numel()
    out = {"pix": pix, "stats": stats, "dirs": dirs, "ij": ij}
    if pix is None:
        out["rgb"] = rgb if rgb is not None else nan(n + GUARD, 3)
        out["depth"] = depth if depth is not None else nan(n + GUARD)
    out["weights"] = nan(n + GUARD, S) if weights else None
    b = _lib.LrfBatch(n_rays=n, rays=_p(rays), n_views=n_views, white_bg=int(white_bg), floater_thresh=float(floater),
                      refine=int(refine), blend=_p(blend), blend_stride=blend_stride, exposure=_p(exposure),
                      accumulate=accumulate, finalize=finalize)
    if gen is not None:
        b.ray_ids, b.W, b.H, b.fov360 = _p(gen["ids"]), gen["W"], gen["H"], int(gen["fov360"])
        b.focal, b.cx, b.cy = gen.get("focal", 0.0), gen.get("cx", 0.0), gen.get("cy", 0.0)
        b.intrinsics, b.cam2world, b.world2rf = _p(gen.get("intr")), _p(gen["c2w"]), _p(gen.get("w2rf"))
    o = _lib.LrfOutputs(rgb=_p(out.get("rgb")), depth=_p(out.get("depth")), weights=_p(out["weights"]),
                        directions=_p(dirs), ij=_p(ij), pix=_p(pix), stats=_p(stats))
    rc = _lib.lib().lrf_render(C.byref(fs), C.c_void_p(prep.data_ptr()), C.byref(b), C.byref(o), _stream())
    torch.cuda.synchronize()
    return rc, out


def rendered(m, z, n, **kw):
    rc, out = render(m, z, n, **kw)
    assert rc == 0, rc
    for k in ("rgb", "depth", "weights"):
        if out.get(k) is not None:
            assert bool(torch.isnan(out[k][n:]).all()), f"{k}: a guard row past n_rays was written"
            assert bool(torch.isfinite(out[k][:n]).all()), f"{k}: a row was not written"
    return out


def bf16_field64(m):
    """The float64 restatement of a module on its bf16-rounded grids (what bf16 storage renders)."""
    F = R.Field64.from_module(m, "cuda")
    with torch.no_grad():
        for k in R.GRID_KEYS:
            F.p[k].copy_(F.p[k].to(torch.bfloat16).double())
    return F


# The decisions that move the forward's colour: the contraction is not one of them (both branches give 1 at max|p| =
# 1, and its argmax only routes the gradient), nor are the texel floors (the lookups are continuous there).
FORWARD_KEYS = tuple(k for k in R.MARGIN_KEYS if k != "contract")


def excluded(fw):
    per = {k: fw[k] < (MARGIN_MLP[True] if k == "mlp" else BOUND if k in R.BOUND_KEYS else MARGIN)
           for k in FORWARD_KEYS}
    print("rays below each margin:", {k: int(v.sum()) for k, v in per.items() if int(v.sum())})
    return torch.stack(list(per.values())).any(0)


def scale_err(a, b, floor=1e-30):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(floor))


def compare(tag, out, fw, n, S, keep, weights=True, max_excluded=MAX_EXCLUDED):
    frac = 1 - float(keep.double().mean())
    tol = max(TOL, 2 * S * R.EPS)
    e_rgb = scale_err(out["rgb"][:n][keep], fw["rgb"][keep], 0.1)      # (a background-only rgb may be ~0)
    e_dep = scale_err(out["depth"][:n][keep], fw["depth"][keep])
    msg = f"{tag}: excluded {100 * frac:.2f} %, rgb {e_rgb:.1e} depth {e_dep:.1e} (bar {tol:.1e})"
    if weights:
        dw = (out["weights"][:n][keep].double() - fw["w"][keep]).abs()
        bar = torch.maximum(1e-4 * fw["w"][keep].abs().clamp_min(5e-3), fw["w_err"][keep])
        e_w = float((dw / bar).max())
        msg += f" weights {e_w:.2f} of their bar"
        assert e_w <= 1.0, msg
    print(msg)
    assert frac <= max_excluded or n <= 9 and frac < 1, msg
    assert e_rgb < tol and e_dep < tol, msg


# (grid, S, act, white_bg, mask, thres, floater, (fea_pe, view_pe), refine, n rays, far, shift, bf16)
BASE = dict(grid=(40, 52, 64), S=344, act="softplus", white_bg=True, mask=False, thres=1e-3, floater=0.0, pe=(0, 0),
            refine=True, n=1024, far=True, shift=-2.0, bf16=False, scale=None, seed=0)
CASES = {
    "g2_S2": dict(grid=(2, 2, 2), S=2, n=512),
    "g405264_S31_mask_relu": dict(S=31, act="relu", mask=True, white_bg=False),
    "g405264_S32": dict(S=32, thres=0.0, far=False),
    "g405264_S33_mask": dict(S=33, mask=True),
    "g300_S344_relu": dict(grid=(300, 300, 300), S=344, act="relu", n=2048),
    "g300_S344_mask_floater": dict(grid=(300, 300, 300), S=344, mask=True, floater=0.5, shift=0.0, n=2048,
                                   white_bg=False),
    "g640_S738_floater": dict(grid=(640, 640, 640), S=738, floater=0.5, shift=0.0, n=1024),
    "g405264_S65535": dict(S=65535, n=4, far=0.6),
    "floater_S1064_8prod": dict(S=1064, floater=0.5, shift=0.0, n=512),
    "floater_S1065_7prod": dict(S=1065, floater=0.5, shift=0.0, n=512),
    "floater_S4600_2prod": dict(S=4600, floater=0.5, shift=2.0, far=False, n=128),
    "floater_S4601_1prod": dict(S=4601, floater=0.5, shift=2.0, far=False, n=128),
    "floater_S9312_1prod": dict(S=9312, floater=0.5, shift=2.0, far=False, n=64),
    "pe22_floater_S472": dict(S=472, floater=0.5, pe=(2, 2), shift=0.0, n=512),
    "pe22_floater_S473": dict(S=473, floater=0.5, pe=(2, 2), shift=0.0, n=512),
    "pe22_floater_S2233_1prod": dict(S=2233, floater=0.5, pe=(2, 2), shift=2.0, far=False, n=128),
    "pe22_floater_S4576_norefine": dict(S=4576, floater=0.5, pe=(2, 2), refine=False, shift=2.0, far=False, n=64),
    "pe11": dict(S=72, pe=(1, 1)),
    "pe04_relu": dict(S=72, pe=(0, 4), act="relu"),
    "pe30_norefine": dict(S=72, pe=(3, 0), refine=False, mask=True),
    "pe88": dict(S=72, pe=(8, 8)),
    "pe88_norefine_thres0": dict(S=72, pe=(8, 8), refine=False, thres=0.0, far=False),
    "thres0": dict(S=96, thres=0.0, far=False, shift=-4.0),
    "thres_above_every_weight": dict(S=96, thres=1.0),
    "opaque_S344": dict(S=344, shift=4.0, scale=300.0, n=4096),
    "opaque_S344_floater": dict(S=344, shift=4.0, scale=300.0, floater=0.5, n=2048),
    "bf16_S344": dict(S=344, bf16=True),
    "bf16_g300_floater_S1065": dict(grid=(300, 300, 300), S=1065, floater=0.5, shift=0.0, bf16=True, n=256),
    "bf16_opaque_relu": dict(S=96, act="relu", shift=4.0, scale=300.0, bf16=True, white_bg=False),
}


def make_case(c, seed=0):
    c = {**BASE, **c}
    fd = R.random_field(c["grid"], act=c["act"], shift=c["shift"], thres=c["thres"], seed=seed, safe_mlp=True,
                        coarse=32 if max(c["grid"]) >= 300 else None, fea_pe=c["pe"][0], view_pe=c["pe"][1],
                        mask=(np.random.default_rng(seed).random((1, 1, 17, 19, 23)) > 0.3).astype(np.float64)
                        if c["mask"] else None)
    if c["scale"] is not None:
        fd["distance_scale"] = np.asarray(c["scale"])
    m = make_module(fd)
    if c["bf16"]:
        m.set_grid_storage("bf16")
    F = bf16_field64(m) if c["bf16"] else R.Field64.from_module(m, "cuda")
    return c, m, F


def check_stats(tag, stats, prior, fw, ok_rays):
    """stats adds {marched, shaded} to its prior contents; exact where every ray clears the decisions that set the
    counts (the mask for the marched samples, the threshold and the floater cut for the shaded ones, the early
    termination for both)."""
    got = (stats.cpu() - prior.cpu()).tolist()
    want = [int(fw["n_march"].sum()), int(fw["n_shade"].sum())]
    print(f"{tag}: stats {got} float64 {want} (exact: {bool(ok_rays.all())})")
    if bool(ok_rays.all()):
        assert got == want, (tag, got, want)


def count_margins_clear(fw):
    ok = fw["term"] >= BOUND
    for k in ("thres", "floater", "mask", "relu_f", "softplus"):
        ok &= fw[k] >= (BOUND if k in R.BOUND_KEYS else MARGIN)
    return ok


@pytest.mark.parametrize("case", list(CASES))
def test_render_vs_float64(case):
    c, m, F = make_case(CASES[case])
    n, S = c["n"], c["S"]
    if c["floater"] and optin() == OPTIN_H100:
        print(f"{case}: {n_producers(S, True, c['pe'] != (0, 0), optin())} producer warps")
    rays = R.make_rays(n, 1, spread=2.5 if c["far"] is True or c["far"] is False else 0.2).cuda()
    z = R.ztable(S, c["far"]).cuda()
    fw = R.forward_chunked(F, rays, z, c["white_bg"], c["floater"], c["refine"])
    assert float(fw["mlp"].min()) > MARGIN_MLP[True], "the safe MLP has a pre-activation near 0"
    keep = ~excluded(fw)
    prior = torch.tensor([123456789, 987654321], dtype=torch.int64, device="cuda")
    stats = prior.clone()
    out = rendered(m, z, n, rays=rays, white_bg=c["white_bg"], floater=c["floater"], refine=c["refine"],
                   stats=stats, fp32=not c["bf16"])
    compare(case, out, fw, n, S, keep)
    check_stats(case, stats, prior, fw, count_margins_clear(fw))
    w = out["weights"][:n]
    if c["floater"]:
        assert int(fw["k_end"].min()) == S                       # the filter marches and writes every sample
    else:                                                        # the terminated tail is exactly 0
        tail = torch.arange(S, device="cuda")[None] >= fw["k_end"][:, None]
        bad = ((w != 0) & tail).any(-1) & (fw["term"] >= BOUND) & keep
        for r in torch.nonzero(bad)[:4, 0].tolist():
            nz = torch.nonzero(w[r] != 0)[-1, 0].item()
            print(f"ray {r}: k_end {int(fw['k_end'][r])}, last written weight at {nz} ({float(w[r, nz]):.3e}); "
                  f"margins", {k: f"{float(fw[k][r]):.2e}" for k in R.MARGIN_KEYS + ("term",)})
        assert not bool(bad.any()), "weights written past the block where T fell below 1e-10"
        print(f"rays terminated before S: {int((fw['k_end'] < S).sum())}")
    if c["thres"] >= 1.0:                                        # nothing shaded: rgb is the background only
        assert int(fw["n_shade"].sum()) == 0 and int((stats - prior)[1]) == 0
        bg = (1.0 - fw["w"].sum(-1)) if c["white_bg"] else torch.zeros(n, dtype=torch.float64, device="cuda")
        assert float((out["rgb"][:n].double() - bg[:, None]).abs().max()) < 1e-5
    if case.startswith("opaque"):
        shaded = fw["n_shade"].double()
        print(f"shaded samples per ray: mean {float(shaded.mean()):.2f}, max {int(shaded.max())}")
        assert float(shaded.mean()) <= 3.0


@pytest.mark.parametrize("which", ["1", "7", "8", "9", "8sm-1", "8sm", "8sm+1", "64sm+1", "4096", "2048sm+1"])
def test_render_batch_sizes_vs_float64(which):
    """Fewer CTAs than SMs below 8 n_sms rays (cta_count(n, 8, ...)), one round of the ray counter, several rounds."""
    sm = n_sms()
    n = {"1": 1, "7": 7, "8": 8, "9": 9, "8sm-1": 8 * sm - 1, "8sm": 8 * sm, "8sm+1": 8 * sm + 1,
         "64sm+1": 64 * sm + 1, "4096": 4096, "2048sm+1": 2048 * sm + 1}[which]
    S = 2 if n > 100000 else 72
    c, m, F = make_case(dict(grid=(2, 2, 2) if S == 2 else (40, 52, 64), S=S), seed=3)
    rays = R.make_rays(n, 5).cuda()
    z = R.ztable(S).cuda()
    fw = R.forward_chunked(F, rays, z, True)
    keep = ~excluded(fw)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    out = rendered(m, z, n, rays=rays, stats=stats)
    compare(f"n = {n}", out, fw, n, S, keep)
    check_stats(f"n = {n}", stats, torch.zeros_like(stats), fw, count_margins_clear(fw))


# ---- exact, without a reference -------------------------------------------------------------------------------------
INDEP = {"1prod_floater_S4601": dict(S=4601, floater=0.5, shift=0.0, n=300),
         "8prod_S344": dict(S=344, n=3000),
         "pe22_floater": dict(S=200, floater=0.5, pe=(2, 2), n=2000),
         "bf16_opaque": dict(S=344, shift=4.0, scale=300.0, bf16=True, n=3000)}


@pytest.mark.parametrize("case", list(INDEP))
def test_batch_independence_bitwise(case):
    """A ray's rgb, depth and weights are the same bits rendered in one batch, in uneven chunks, in a permuted batch
    and alone (composition is fixed point, every other step is per ray)."""
    c, m, _ = make_case(INDEP[case], seed=7)
    n, S = c["n"], c["S"]
    rays = R.make_rays(n, 8).cuda()
    z = R.ztable(S).cuda()
    kw = dict(white_bg=c["white_bg"], floater=c["floater"], refine=c["refine"], fp32=not c["bf16"])
    whole = rendered(m, z, n, rays=rays, **kw)
    cuts = [0, 1, n // 3, n // 3 + 37, n]
    parts = [rendered(m, z, b - a, rays=rays[a:b].contiguous(), **kw) for a, b in zip(cuts[:-1], cuts[1:])]
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1)).cuda()
    shuf = rendered(m, z, n, rays=rays[perm].contiguous(), **kw)
    for k in ("rgb", "depth", "weights"):
        assert torch.equal(torch.cat([p[k][:b - a] for p, a, b in zip(parts, cuts[:-1], cuts[1:])]), whole[k][:n]), k
        assert torch.equal(shuf[k][:n], whole[k][:n][perm]), k
    for r in (0, n // 2, n - 1):
        alone = rendered(m, z, 1, rays=rays[r:r + 1].contiguous(), **kw)
        for k in ("rgb", "depth", "weights"):
            assert torch.equal(alone[k][0], whole[k][r]), (k, r)


@pytest.fixture(scope="module")
def small_field():
    c, m, F = make_case(dict(S=96), seed=11)
    return m, F, R.ztable(96).cuda()


def test_weights_null_and_floater_writes_all(small_field):
    """weights = NULL gives the same rgb and depth bits; the floater path writes all S weights."""
    m, F, z = small_field
    n = 1000
    rays = R.make_rays(n, 12).cuda()
    for fl in (0.0, 0.5):
        a = rendered(m, z, n, rays=rays, floater=fl)
        b = rendered(m, z, n, rays=rays, floater=fl, weights=False)
        assert torch.equal(a["rgb"][:n], b["rgb"][:n]) and torch.equal(a["depth"][:n], b["depth"][:n])
    assert bool(torch.isfinite(a["weights"][:n]).all())


def test_pix_and_accumulate_bitwise(small_field):
    """pix holds the rgb / depth bits interleaved; accumulate onto P is P plus the non-accumulated launch, one fp32
    add (finalize 0), in both layouts; the fourth column of pix and the guard rows are left alone."""
    m, F, z = small_field
    n = 2000
    rays = R.make_rays(n, 13).cuda()
    ref = rendered(m, z, n, rays=rays)
    pix = nan(n + GUARD, 4)
    rendered(m, z, n, rays=rays, pix=pix)
    assert torch.equal(pix[:n, :3], ref["rgb"][:n]) and torch.equal(pix[:n, 3], ref["depth"][:n])
    assert bool(torch.isnan(pix[n:]).all())
    gen = torch.Generator(device="cuda").manual_seed(2)
    P = torch.rand(n + GUARD, 4, generator=gen, device="cuda") * 4 - 2
    pix = P.clone()
    rendered(m, z, n, rays=rays, pix=pix, accumulate=1)
    assert torch.equal(pix[:n, :3], P[:n, :3] + ref["rgb"][:n]) and torch.equal(pix[:n, 3], P[:n, 3] + ref["depth"][:n])
    assert torch.equal(pix[n:], P[n:])
    rgb, depth = P[:, :3].contiguous(), P[:, 3].contiguous()
    rgb[n:], depth[n:] = math.nan, math.nan
    rendered(m, z, n, rays=rays, rgb=rgb, depth=depth, accumulate=1, weights=False)
    assert torch.equal(rgb[:n], P[:n, :3] + ref["rgb"][:n]) and torch.equal(depth[:n], P[:n, 3] + ref["depth"][:n])


def _cameras(V, seed, W, H):
    g = torch.Generator().manual_seed(seed)
    c2w = torch.zeros(V, 3, 4)
    for v in range(V):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
        c2w[v, :, :3] = q
        c2w[v, :, 3] = 0.3 * torch.randn(3, generator=g)
    return c2w.cuda().contiguous(), torch.tensor([0.8 * W, 0.5 * W + 0.25, 0.5 * H - 0.375]).cuda()


def _exposures(V, seed):
    """Per-view 3x3 exposures, each its own, that push the first channel above 1, the second below 0 and leave the
    third inside (both clamp bounds)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.tensor([[4.0, 0.0, 0.0], [0.0, -0.5, 0.0], [0.2, 0.2, 0.6]])
    E = base * (1 + 0.05 * torch.arange(V).view(V, 1, 1)) + 0.05 * torch.randn(V, 3, 3, generator=g)
    return E.cuda().contiguous()


@pytest.mark.parametrize("V", [1, 3, 16])
def test_exposure_equals_exposure_clamp(small_field, V):
    """finalize with exposure (explicit rays, n_views views) equals lrf_exposure_clamp of the finalize = 0 output
    bitwise, for per-view exposures that clamp at both bounds and for a NULL exposure (clamp only)."""
    from localrf_b200 import _lib
    m, F, z = small_field
    n = V * 257
    rays = R.make_rays(n, 14).cuda()
    lin = rendered(m, z, n, rays=rays, n_views=V, exposure=None)["rgb"][:n].contiguous()
    for E in (_exposures(V, V), None):
        got = rendered(m, z, n, rays=rays, n_views=V, exposure=E, finalize=1)["rgb"][:n]
        want = torch.empty(n, 3, device="cuda")
        _lib.check(_lib.lib().lrf_exposure_clamp(_p(lin), _p(E), n, V, _p(want), _stream()))
        torch.cuda.synchronize()
        assert torch.equal(got, want), V
        if E is not None:
            assert float(want.min()) == 0.0 and float(want.max()) == 1.0       # both bounds reached
            assert not torch.equal(want, lin.clamp(0, 1))


@pytest.mark.parametrize("mode", ["lean", "fov360", "intrinsics"])
def test_three_fields_into_pix_vs_float64(mode):
    """Ray-generation mode, three fields rendered into pix as LocalTensorfs does (blend[v * 3 + f], accumulate on the
    second and third, finalize with per-view exposure on the third): the pix bits equal the sum of the three
    non-accumulated launches and lrf_exposure_clamp of it; the result, the directions and ij against the float64
    restatement (directions within 4 EPS, 16 for 360 directions; ij exact)."""
    from localrf_b200 import _lib
    V, rpv, W, H, S = 4, 300, 96, 64, 96
    n = V * rpv
    ms, Fs = [], []
    for f in range(3):
        _, m, F = make_case(dict(S=S), seed=20 + f)
        ms.append(m)
        Fs.append(F)
    z = R.ztable(S).cuda()
    c2w, intr = _cameras(V, 5, W, H)
    g = torch.Generator().manual_seed(6)
    ids = (torch.randint(0, W * H, (n,), generator=g) + torch.arange(V).repeat_interleave(rpv) * W * H).cuda()
    blend = (0.2 + 0.8 * torch.rand(V, 3, generator=g)).cuda().contiguous()
    E = _exposures(V, 7)
    w2rf = [torch.tensor([0.05 * f, -0.02, 0.01]).cuda() for f in range(3)]
    gen = dict(ids=ids, W=W, H=H, fov360=mode == "fov360", c2w=c2w)
    if mode == "intrinsics":
        gen["intr"] = intr
    else:
        gen["focal"], gen["cx"], gen["cy"] = (float(v) for v in intr.cpu())
    pix = nan(n + GUARD, 4)
    dirs, ij = nan(n + GUARD, 3), torch.full((n + GUARD, 2), -7, dtype=torch.int64, device="cuda")
    solo = []
    for f in range(3):
        kw = dict(gen={**gen, "w2rf": w2rf[f]}, blend=blend[:, f:], blend_stride=3, n_views=V, weights=False)
        rendered(ms[f], z, n, pix=pix, accumulate=int(f > 0), finalize=int(f == 2), exposure=E if f == 2 else None,
                 dirs=dirs if f == 0 else None, ij=ij if f == 0 else None, **kw)
        solo.append(rendered(ms[f], z, n, **kw))
    lin = (solo[0]["rgb"][:n] + solo[1]["rgb"][:n]) + solo[2]["rgb"][:n]
    want = torch.empty(n, 3, device="cuda")
    _lib.check(_lib.lib().lrf_exposure_clamp(_p(lin.contiguous()), _p(E), n, V, _p(want), _stream()))
    torch.cuda.synchronize()
    assert torch.equal(pix[:n, :3], want)
    assert torch.equal(pix[:n, 3], (solo[0]["depth"][:n] + solo[1]["depth"][:n]) + solo[2]["depth"][:n])
    assert bool(torch.isnan(pix[n:]).all()) and bool(torch.isnan(dirs[n:]).all()) and bool((ij[n:] == -7).all())
    ref = R.render_views(Fs, z, ids, W, H, mode == "fov360", intr, c2w, w2rf, blend, E, True)
    keep = ~excluded(ref)
    frac = 1 - float(keep.double().mean())
    e_rgb, e_dep = scale_err(pix[:n, :3][keep], ref["rgb"][keep]), scale_err(pix[:n, 3][keep], ref["depth"][keep])
    e_dir = float((dirs[:n].double() - ref["dirs"]).abs().max() / (R.EPS * ref["dirs"].abs().max()))
    print(f"{mode}: excluded {100 * frac:.2f} %, rgb {e_rgb:.1e} depth {e_dep:.1e}, directions {e_dir:.1f} EPS")
    # lean: a subtraction and a division (a few EPS); 360: sin / cos of angles up to 3 pi, whose own rounding is
    # 3 pi EPS
    assert frac <= MAX_EXCLUDED and e_rgb < TOL and e_dep < TOL and e_dir <= (16.0 if mode == "fov360" else 4.0)
    assert torch.equal(ij[:n], ref["ij"])


def test_explicit_rays_leave_directions_and_ij(small_field):
    """With explicit rays the directions and ij buffers are not written."""
    m, F, z = small_field
    n = 500
    dirs, ij = nan(n, 3), torch.full((n, 2), -7, dtype=torch.int64, device="cuda")
    rendered(m, z, n, rays=R.make_rays(n, 15).cuda(), dirs=dirs, ij=ij)
    assert bool(torch.isnan(dirs).all()) and bool((ij == -7).all())


def test_empty_and_refused_launches(small_field):
    """n_rays = 0 returns LRF_OK and writes nothing; with the floater filter the first S whose alpha tables no longer
    fit one producer (9313 without encodings, 4577 with) is LRF_ERR_UNSUPPORTED and leaves every output untouched,
    and the S just below it renders."""
    m, F, z = small_field
    stats = torch.full((2,), 5, dtype=torch.int64, device="cuda")
    rc, out = render(m, z, 0, rays=R.make_rays(1, 1).cuda(), stats=stats)
    assert rc == 0 and bool(torch.isnan(out["rgb"]).all()) and bool(torch.isnan(out["weights"]).all())
    assert stats.tolist() == [5, 5]
    if optin() != OPTIN_H100:
        pytest.skip(f"opt-in shared memory {optin()} B, not the H100's {OPTIN_H100}: the limits below are the H100's")
    count = lambda S, pe: n_producers(S, True, pe, optin())
    steps = {pe: [S for S in range(3, 10000) if count(S, pe) != count(S - 1, pe)] for pe in (False, True)}
    assert steps[False] == [1065, 1233, 1457, 1773, 2245, 3029, 4601, 9313], steps
    assert steps[True] == [473, 557, 669, 825, 1061, 1449, 2233, 4577], steps
    for pe, limit in ((False, 9313), (True, 4577)):
        _, mm, _ = make_case(dict(S=limit, pe=(2, 2) if pe else (0, 0)), seed=2)
        rays = R.make_rays(8, 3).cuda()
        stats = torch.full((2,), 5, dtype=torch.int64, device="cuda")
        rc, out = render(mm, R.ztable(limit).cuda(), 8, rays=rays, floater=0.5, stats=stats)
        assert rc == -2, rc
        assert all(bool(torch.isnan(out[k]).all()) for k in ("rgb", "depth", "weights")) and stats.tolist() == [5, 5]
        rc, out = render(mm, R.ztable(limit - 1).cuda(), 8, rays=rays, floater=0.5)
        assert rc == 0 and bool(torch.isfinite(out["rgb"][:8]).all())
