"""CPU: the float64 restatement of tests/render64.py pinned to the reference's autograd golden and to the oracle's
analytic backward, and each of its decision margins shown to flag a ray built to sit exactly on that decision."""
import math

import numpy as np
import pytest
import torch

import render64 as R
from helpers import full_field_dict, load_golden
from oracle import oracle as orc


def scale_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def _cot(n, seed=11):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, 3)), 0.05 * rng.standard_normal(n)


def test_grads_field_golden():
    """The reference's own fp32 autograd (grads_field): every gradient within 2e-5 of its scale, the rgb within 1e-5.
    The golden is fp32, so this is the fp32-vs-fp64 level (measured <= 3.6e-6); no sample of it lies near a decision."""
    g = load_golden("grads_field")
    F = R.Field64(full_field_dict(g))
    grads, fwd = R.field_backward(F, g["rays"], g["z"], True, g["c_rgb"], g["c_depth"])
    assert scale_err(fwd["rgb"], g["out.rgb"]) < 1e-5 and scale_err(fwd["depth"], g["out.depth"]) < 1e-5
    errs = {k: scale_err(grads[k].numpy(), g["grad." + k]) for k in R.PARAM_KEYS + ["rays"]}
    print("grads_field vs float64:", {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < 2e-5, errs


@pytest.mark.parametrize("name,white_bg", [("cfg1_64", True), ("cfg1_64", False), ("relu_32", True),
                                           ("alphamask_32", False), ("opaque_32", True)])
def test_vs_oracle_backward(name, white_bg):
    """The oracle's fp32 analytic backward on the golden fields: every tensor within 1e-4 of its scale on the rays
    clear of every decision (render64.clear; the others get zero cotangents on both sides)."""
    g = load_golden(name)
    fd = full_field_dict(g)
    n = min(g["rays"].shape[0], 192)
    rays = np.ascontiguousarray(g["rays"][:n])
    z = g["z"] if "z" in g else g["eval.z"]
    c_rgb, c_depth = _cot(n)
    F = R.Field64(fd)
    with torch.no_grad():
        _, _, ex = R.field_forward(F, torch.from_numpy(rays).double(), torch.from_numpy(z).double(), white_bg, True)
    keep = R.clear(ex).numpy()
    print(name, "rays excluded:", int((~keep).sum()), "of", n)
    assert keep.mean() > 0.9
    c_rgb = c_rgb * keep[:, None]; c_depth = c_depth * keep
    grads, fwd = R.field_backward(F, rays, z, white_bg, c_rgb, c_depth)
    ref = orc.field_backward(orc.Field(fd), fd, rays, z, c_rgb.astype(np.float32), c_depth.astype(np.float32),
                             white_bg=white_bg)
    errs = {k: scale_err(grads[k].numpy(), ref[k]) for k in ref}
    print(name, "oracle vs float64:", {k: f"{v:.1e}" for k, v in errs.items()})
    # opaque_32: alpha -> 1 makes dL/dalpha a difference of large terms in fp32 (test_gpu_backward.py's 1e-3)
    assert max(errs.values()) < (1e-3 if name == "opaque_32" else 1e-4), errs


@pytest.mark.parametrize("act,seed", [("relu", 0), ("softplus", 1)])
def test_weight_error_bound_holds_at_300(act, seed):
    """The propagated bound w_err of render64 holds for an fp32 implementation at training size: the oracle's fp32
    weights (its own rounding order, no FMA) differ from the float64 weights by at most w_err on every sample of every
    ray clear of the relu / softplus / contraction / mask decisions, at 300^3 with S = 344 and the far distance table
    -- where the fp32 error of w grows along the ray to ~1e-3 relative through the feature's slope and the product."""
    fd = R.random_field((300, 300, 300), act=act, seed=seed, safe_mlp=True)
    for k, v in fd.items():                                    # the fp32 parameters both sides read
        if isinstance(v, np.ndarray) and v.dtype == np.float64 and v.ndim:
            fd[k] = v.astype(np.float32).astype(np.float64)
    rays, z = R.make_rays(512, 1), R.ztable(344)
    F = R.Field64(fd)
    with torch.no_grad():
        _, _, ex = R.field_forward(F, rays.double(), z.double(), True, True)
    w32 = orc.field_forward(orc.Field(fd), rays.numpy(), z.numpy())["weights"]
    ok = torch.ones(512, dtype=torch.bool)
    for k in ("relu_f", "softplus", "contract", "mask"):
        ok &= ex[k] >= 1.0
    ratio = (torch.from_numpy(w32).double() - ex["w"]).abs() / ex["w_err"]
    worst = float(ratio[ok].max())
    rel = float(((torch.from_numpy(w32).double() - ex["w"]).abs() / ex["w"].clamp_min(1e-30))[ok][ex["w"][ok] > 1e-4].max())
    print(f"{act}: rays checked {int(ok.sum())} of 512; max |w32 - w64| / w_err = {worst:.3f}; "
          f"largest relative w error (w > 1e-4) {rel:.1e}")
    assert int(ok.sum()) > 450 and worst <= 1.0


# ---- each margin flags a ray built to sit on its decision ---------------------------------------------------------
def _field(**kw):
    return R.random_field(**kw)


Z = torch.linspace(0.1, 2.5, 40, dtype=torch.float64)


def _margins(fd, rays, z=Z, white_bg=True):
    with torch.no_grad():
        _, _, ex = R.field_forward(R.Field64(fd), torch.as_tensor(rays, dtype=torch.float64), z, white_bg, True)
    return ex


def _rays(n=8, seed=1):
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((n, 3))
    return np.concatenate([0.2 * rng.standard_normal((n, 3)), d], -1)


def test_margin_thres():
    fd = _field()
    rays = _rays()
    ex = _margins(fd, rays)
    assert float(ex["thres"].min()) > 1.0
    fd["rayMarch_weight_thres"] = float(ex["w"][3, 5])          # ray 3's sample 5 now sits on the switch
    ex2 = _margins(fd, rays)
    assert float(ex2["thres"][3]) == 0.0 and float(ex2["thres"].max()) > 1.0


def test_margin_contract_boundary_and_argmax_tie():
    fd = _field()
    z = torch.tensor([0.1, 0.5, 0.9, 1.3], dtype=torch.float64)
    rays = np.array([[0.0, 0.0, 0.0, 1.0, 0.0, 0.0],          # p = (0.9 + 0.1, 0, 0) = 1: on max|p| <= 1
                     [0.1, 0.0, 0.0, 2.0, 0.0, 0.0],
                     [1.5, 1.5, 0.0, 0.0, 0.0, 3.0],          # |p_x| = |p_y| = 1.5 > 1: argmax tie
                     [0.3, 0.2, 0.1, 0.3, 1.0, 0.2]])
    ex = _margins(fd, rays, z)
    c = ex["contract"]
    assert float(c[1]) < 1.0 and float(c[2]) == 0.0 and float(c[3]) > 1e3, c


def test_margin_alpha_mask_cell_boundary():
    vol = np.zeros((1, 1, 5, 5, 5))
    vol[0, 0, 2, 2, 3] = 1.0                                   # [D][H][W]: the voxel at x = 3, y = 2, z = 2
    fd = _field(mask=vol)
    # lattice coordinate x = 2 exactly (p_x = -2 + 4 * 2 / 4 = 0): the x = 3 corner has weight 0 -> value 0
    z = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)
    rays = np.array([[0.0, 0.0, -0.1, 0.0, 0.0, 1.0],          # (0, 0, 0): x on the lattice, value 0
                     [0.5, 0.0, -0.1, 0.0, 0.0, 1.0],          # (0.5, 0, 0): value > 0, well away
                     [-1.3, -1.3, -1.3, 0.0, 0.0, 1.0]])       # far from the voxel: value 0, not on a boundary
    ex = _margins(fd, rays, z)
    m = ex["mask"]
    assert float(m[0]) == 0.0 and float(m[1]) > 1e3 and float(m[2]) > 1e3, m


def test_margin_relu_and_softplus():
    fd = _field(act="relu")
    for i in range(3):
        fd[f"density_line.{i}"][:] = 0.0                        # f = 0 exactly everywhere
    ex = _margins(fd, _rays())
    assert float(ex["relu_f"].max()) == 0.0 and math.isinf(float(ex["softplus"].min()))
    fd = _field(act="softplus")
    rays = _rays()
    F = R.Field64(fd)
    with torch.no_grad():
        # the density feature of ray 2's sample 7, then the shift that puts f + shift on 20
        rc = torch.as_tensor(rays[2:3], dtype=torch.float64)
        o, d = rc[:, :3], rc[:, 3:] / rc[:, 3:].norm()
        p = o + d * Z[7]
        am = p.abs().amax(-1, keepdim=True)
        pc = torch.where(am <= 1, p, (2 * am - 1) / am ** 2 * p)
        q = pc / 2
        fe = sum(R._lookup(F.p[f"density_plane.{i}"], F.p[f"density_line.{i}"], q, i).sum() for i in range(3))
    fd["density_shift"] = 20.0 - float(fe)
    ex = _margins(fd, rays)
    assert float(ex["softplus"][2]) < 1.0 and math.isinf(float(ex["relu_f"].min()))


def test_margin_mlp_preactivation():
    fd = _field(thres=0.0)
    rays = _rays()
    F = R.Field64(fd)
    with torch.no_grad():
        rc = torch.as_tensor(rays[4:5], dtype=torch.float64)
        o, d = rc[:, :3], rc[:, 3:] / rc[:, 3:].norm()
        p = o + d * Z[3]
        am = p.abs().amax(-1, keepdim=True)
        pc = torch.where(am <= 1, p, (2 * am - 1) / am ** 2 * p)
        feats = torch.cat([R._lookup(F.p[f"app_plane.{i}"], F.p[f"app_line.{i}"], pc / 2, i) for i in range(3)], -1)
        x = feats @ F.p["basis_mat.weight"].t()
        a = float((x @ F.p["renderModule.mlp.0.weight"].t())[0, 17])
    fd["renderModule.mlp.0.bias"][17] = -a                     # unit 17's pre-activation on that sample: 0
    ex = _margins(fd, rays)
    assert float(ex["mlp"][4]) < 1.0 and float(ex["mlp"].max()) > 1.0


def test_margin_texel_floor():
    fd = _field(grid=(33, 11, 13))
    # x = 0.5 on every sample: q_x = 0.25, pixel (1.25 / 2) * 32 = 20 exactly
    rays = np.array([[0.5, 0.3, 0.2, 0.0, 0.0, 0.4], [0.52, 0.3, 0.2, 0.0, 0.0, 0.4]])
    z = torch.linspace(0.1, 0.85, 9, dtype=torch.float64)     # no integer pixel on the y and z axes
    ex = _margins(fd, rays, z)
    assert float(ex["texel"][0]) == 0.0 and float(ex["texel"][1]) > 1e3
    assert float(R.min_margin(ex)[0]) > 0                    # the texel floor is not one of the decisions


def test_clamp_margin_and_exact_bounds():
    """E x exactly 0 or 1 is not a margin (both implementations compute it exactly and pass the gradient at both
    bounds: ray 0's margin is that of its third channel, 0.5); E x within a rounding of 1 is."""
    fd = _field(thres=0.0)
    F = R.Field64(fd)
    W, H = 8, 6
    ids = torch.arange(4, dtype=torch.int64)
    c2w = torch.eye(3, 4, dtype=torch.float64)[None]
    x = torch.tensor([[0.0, 1.0, 0.5], [0.3, 0.2, 0.1], [1 + 1e-9, 0.5, 0.5], [0.2, 0.2, 0.2]], dtype=torch.float64)
    grads, fwd = R.train_backward(F, torch.linspace(0.1, 1.0, 6), ids, W, H, False, [5.0, 4.0, 3.0], c2w,
                                  [0.0, 0.0, 0.0], None, x, True, torch.ones(4, 3), torch.zeros(4), None)
    cl = fwd["clamp"]
    assert float(cl[0]) >= 2 ** 24 and float(cl[1]) > 1e3 and float(cl[2]) < 100
    # g' = g on both bounds: the identity exposure's gradient is the sum of x over the rays that pass
    dE = grads["d_exposure"][0]
    assert torch.allclose(dE[0], x[[0, 1, 3]].sum(0)) and torch.allclose(dE[1], x.sum(0))


# ---- the floater filter and the positional encodings against the reference's goldens --------------------------------
@pytest.mark.parametrize("name,case,floater,refine", [("cfg1_64", "eval_floater", 0.5, True),
                                                      ("opaque_32", "eval_floater", 0.5, True),
                                                      ("aniso_pe", "refine", 0.5, True),
                                                      ("aniso_pe", "norefine", 0.0, False)])
def test_forward_vs_reference_golden(name, case, floater, refine):
    """The reference's own fp32 forward (floater_thresh 0.5; fea_pe = view_pe = 2 with refine on and off): rgb and
    depth within 1e-5 of their scale and weights within 1e-6, on the rays clear of every decision (measured <= 3.3e-7
    and 1.1e-7; the excluded rays are the MLP's near-zero pre-activations of these random MLPs).  The filter cuts
    samples on many rays, so the pin is not that of the unfiltered forward."""
    g = load_golden(name)
    F = R.Field64(full_field_dict(g))
    out = R.forward_chunked(F, g["rays"], g[case + ".z"], True, floater, refine)
    keep = R.clear(out).numpy()
    print(name, case, "rays excluded:", int((~keep).sum()), "of", keep.size)
    assert keep.mean() > 0.6
    errs = (scale_err(out["rgb"].numpy()[keep], g[case + ".rgb"][keep]),
            scale_err(out["depth"].numpy()[keep], g[case + ".depth"][keep]),
            float(np.abs(out["w"].numpy()[keep] - g[case + ".weights"][keep]).max()))
    print(f"{name} {case}: rgb {errs[0]:.1e} depth {errs[1]:.1e} weights {errs[2]:.1e}")
    assert errs[0] < 1e-5 and errs[1] < 1e-5 and errs[2] < 1e-6
    if floater:
        plain = R.forward_chunked(F, g["rays"], g[case + ".z"], True, 0.0, refine)
        moved = (plain["w"] - out["w"]).abs().amax(-1) > 1e-3
        assert int(moved.sum()) >= 0.2 * keep.size
        assert torch.equal(plain["depth"], out["depth"])            # depth keeps the pre-filter weights


def _floater_setup():
    fd = _field(shift=0.0)
    rays = _rays()
    ex = _margins(fd, rays)
    ks = torch.arange(Z.shape[0], dtype=torch.float64)
    idx = (ex["w"] * ks).sum(-1)
    return fd, rays, idx


def test_margin_floater():
    """floater_thresh that puts ray 2's cut idx thresh exactly on an integer: its margin is 0; half way between two
    integers the margin is large."""
    fd, rays, idx = _floater_setup()
    k = math.floor(float(idx[2])) - 1
    assert 1 <= k < Z.shape[0] - 1
    F = R.Field64(fd)
    on = R.forward_chunked(F, rays, Z, True, floater=k / float(idx[2]))
    assert float(on["floater"][2]) < 1.0 and float(on["floater"].max()) > 1.0
    off = R.forward_chunked(F, rays, Z, True, floater=(k + 0.5) / float(idx[2]))
    assert float(off["floater"][2]) > 1e3
    assert math.isinf(float(R.forward_chunked(F, rays, Z, True)["floater"].min()))     # no filter: no decision


def test_margin_thres_after_floater():
    """With the filter, `thres` is measured on the filtered weights: a threshold equal to a filtered weight that
    differs from the unfiltered one sits on the switch."""
    fd, rays, idx = _floater_setup()
    fl = 0.5
    F = R.Field64(fd)
    out = R.forward_chunked(F, rays, Z, True, floater=fl)
    plain = _margins(fd, rays)
    r, k = [int(v) for v in torch.nonzero((out["w"] - plain["w"]).abs() > 1e-3)[-1]]
    fd["rayMarch_weight_thres"] = float(out["w"][r, k])
    out2 = R.forward_chunked(R.Field64(fd), rays, Z, True, floater=fl)
    assert float(out2["thres"][r]) == 0.0 and float(out2["thres"].max()) > 1.0


def test_margin_mlp_positional_encodings():
    """fea_pe = 3, view_pe = 2: a layer-1 unit whose pre-activation (encoded input, refine on) is 0 on one sample is
    flagged; with refine off the encoded inputs are zeros, and the same unit's pre-activation moves off 0."""
    fd = _field(thres=0.0, fea_pe=3, view_pe=2, safe_mlp=True)
    rays = _rays()
    F = R.Field64(fd)
    with torch.no_grad():
        rc = torch.as_tensor(rays[4:5], dtype=torch.float64)
        o, d = rc[:, :3], rc[:, 3:] / rc[:, 3:].norm()
        p = o + d * Z[3]
        am = p.abs().amax(-1, keepdim=True)
        pc = torch.where(am <= 1, p, (2 * am - 1) / am ** 2 * p)
        feats = torch.cat([R._lookup(F.p[f"app_plane.{i}"], F.p[f"app_line.{i}"], pc / 2, i) for i in range(3)], -1)
        x = feats @ F.p["basis_mat.weight"].t()
        enc = torch.cat([x, R._pe(x, 3)], -1)
        a = float((enc @ F.p["renderModule.mlp.0.weight"].t())[0, 17])
    fd["renderModule.mlp.0.bias"][17] = -a
    on = R.forward_chunked(R.Field64(fd), rays, Z, True)
    assert float(on["mlp"][4]) < 1.0 and float(on["mlp"].max()) > 1.0
    off = R.forward_chunked(R.Field64(fd), rays, Z, True, refine=False)
    assert float(off["mlp"][4]) > float(on["mlp"][4])


def test_margin_term_and_counts():
    """A distance scale that puts ray 1's transmittance at the end of the first 32-sample block on 1e-10 (fp32) is
    flagged by `term`; below it the march stops after that block (k_end = 32: the marched and shaded counts only
    reach the first block), above it the ray marches all 40 samples."""
    fd, rays = _field(), _rays()

    def tb(scale):
        fd["distance_scale"] = scale
        return R.forward_chunked(R.Field64(fd), rays, Z, True)

    lo, hi = math.log(1.0), math.log(1e5)
    for _ in range(70):                       # T at the block end falls as the scale grows
        mid = 0.5 * (lo + hi)
        out = tb(math.exp(mid))
        if int(out["k_end"][1]) == 32:
            hi = mid
        else:
            lo = mid
    on = tb(math.exp(hi))
    assert int(on["k_end"][1]) == 32 and float(on["term"][1]) < 1.0
    above = tb(math.exp(lo) * 0.5)
    assert int(above["k_end"][1]) == 40 and float(above["term"][1]) > 1.0
    below = tb(math.exp(hi) * 2)
    assert int(below["k_end"][1]) == 32 and float(below["term"][1]) > 1.0
    assert int(below["n_march"][1]) == 32 and int(above["n_march"][1]) == 39
    assert int(below["n_shade"][1]) == int((below["w"][1, :32] > float(fd["rayMarch_weight_thres"])).sum())


# ---- field_backward with the floater filter and refine: against central differences -------------------------------
def _directional(F, rays, z, g_rgb, g_depth, floater, refine, v, v_rays, h):
    """(L(theta + h v) - L(theta - h v)) / 2h, L = sum(rgb g_rgb) + sum(depth g_depth), and the hard decisions (the
    filtered alphas' zeros and the shading switch) at both ends."""
    vals, cuts = [], []
    with torch.no_grad():
        for s in (1.0, -1.0):
            for k in R.PARAM_KEYS:
                F.p[k].add_(s * h * v[k])
            rgb, depth, ex = R.field_forward(F, rays + s * h * v_rays, z, True, False, floater, refine)
            for k in R.PARAM_KEYS:
                F.p[k].sub_(s * h * v[k])
            vals.append(float((rgb * g_rgb).sum() + (depth * g_depth).sum()))
            cuts.append(((ex["w"] == 0), ex["w"] > F.thres))
    return (vals[0] - vals[1]) / (2 * h), cuts


@pytest.mark.parametrize("floater,refine,pe", [(0.5, True, (0, 0)), (0.5, True, (2, 1)), (0.0, False, (3, 0)),
                                               (0.3, False, (2, 2))])
def test_field_backward_floater_refine_vs_central_differences(floater, refine, pe):
    """field_backward(floater, refine) on a small field: the gradient's projection on random directions (every
    parameter and the ray origins at once) equals a float64 central difference within 1e-6 relative, on rays whose every
    decision clears its margin (render64.clear) and whose filter cut and shading switch stay put across +-h."""
    fd = R.random_field((9, 11, 13), shift=0.0, seed=5, fea_pe=pe[0], view_pe=pe[1], safe_mlp=True)
    F = R.Field64(fd)
    rays = torch.as_tensor(_rays(16, seed=3), dtype=torch.float64)
    fw = R.forward_chunked(F, rays, Z, True, floater=floater, refine=refine)
    keep = R.clear(fw, bound=4.0, margin=256.0) & (fw["texel"] >= 4.0)
    assert int(keep.sum()) >= 8, int(keep.sum())
    g_rgb, g_depth = (torch.as_tensor(c, dtype=torch.float64) for c in _cot(16, seed=7))
    g_rgb, g_depth = g_rgb * keep[:, None], g_depth * keep
    grads, _ = R.field_backward(F, rays, Z, True, g_rgb, g_depth, want_margins=False, floater=floater, refine=refine)
    gen = torch.Generator().manual_seed(9)
    for trial in range(3):
        v = {k: torch.randn(F.p[k].shape, generator=gen, dtype=torch.float64) for k in R.PARAM_KEYS}
        # origins only: the MLP reads the view direction detached (as the reference does), so d's gradient is partial
        v_rays = torch.randn(rays.shape, generator=gen, dtype=torch.float64) * keep[:, None]
        v_rays[:, 3:] = 0
        proj = sum(float((grads[k] * v[k]).sum()) for k in R.PARAM_KEYS) + float((grads["rays"] * v_rays).sum())
        fd_, cuts = _directional(F, rays, Z, g_rgb, g_depth, floater, refine, v, v_rays, 1e-6)
        for a, b in zip(cuts[0], cuts[1]):
            assert torch.equal(a[keep], b[keep]), "a decision moved within +-h"
        print(f"floater {floater} refine {refine} pe {pe}: projection {proj:.6e}, central difference {fd_:.6e}")
        assert abs(proj - fd_) <= 1e-6 * max(abs(proj), 1.0), (trial, proj, fd_)
