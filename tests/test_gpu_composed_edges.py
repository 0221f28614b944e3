"""-m gpu: the composed training path (TensorBase._forward_autograd: the lookups' CUDA backward through _VMLookup plus
fp32 torch ops) against the float64 restatement of tests/render64.py, for the fields that train through it: positional
encodings fea_pe / view_pe 1..8 (with and without `refine`), and pe = 0 with the floater filter or return_weights
while autograd records; and LocalTensorfs's training call of such a field (LocalTensorfs._forward_autograd: torch ray
generation, world2rf, exposure and clamp around it) against render64.train_backward.  It is also the path the fused
backward's own tests compare against.

The bars, the zeroed cotangents of rays below their margins and the excluded-fraction cap are those of
test_gpu_backward_edges.py (CUDA-core arithmetic: the fp32 MLP margin).  Matmuls run in fp32 (TF32 off) here, as the
bar assumes.
Measured on an H100 80GB HBM3 at a 700 W power limit: every tensor within 5.7e-5 of its scale up to fea_pe = 3 and
3.9e-4 at fea_pe = 8 (its own bar, below); the training call's field, pose, intrinsics, exposure and world2rf
gradients within 2.3e-5; at most 4.5 % of a case's rays excluded; the file runs in about 35 s."""
import numpy as np
import pytest
import torch

import render64 as R
from test_gpu_backward_edges import (MARGIN, MARGIN_MLP, MAX_EXCLUDED, TEXEL_MARGIN, TOL, compare, excluded,
                                     make_module, scale_err)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fp32_matmuls():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


GRIDS = {"405264": (40, 52, 64), "300": (300, 300, 300)}
PE_CASES = {   # (fea_pe, view_pe, act, refine)
    "pe1_1": (1, 1, "softplus", True),
    "pe2_2": (2, 2, "softplus", True),
    "pe0_4_relu": (0, 4, "relu", True),
    "pe3_0_norefine": (3, 0, "softplus", False),
    "pe8_8": (8, 8, "softplus", True),
}


def _run(grid, S, fea_pe, view_pe, act, refine, floater=0.0, return_weights=False, n=None, seed=0):
    # grids of 300^3 upsampled from 32 per axis; relu on the steep 40 x 52 x 64 grid from 8 per axis, where the
    # features' slope otherwise puts 7 % of the rays near relu's switch at S = 344
    coarse = 32 if max(grid) >= 300 else 8 if act == "relu" else None
    fd = R.random_field(grid, act=act, shift=-2.0, thres=1e-3, seed=seed, safe_mlp=True, fea_pe=fea_pe,
                        view_pe=view_pe, coarse=coarse)
    m = make_module(fd)
    F = R.Field64.from_module(m, "cuda")
    n = n or (1024 if S <= 72 else 512)
    rays = R.make_rays(n, seed + 1).cuda()
    z = R.ztable(S).cuda()
    fw = R.forward_chunked(F, rays, z, True, floater=floater, refine=refine)
    drop = excluded(fw, False)
    frac = float(drop.double().mean())
    print(f"excluded {int(drop.sum())} of {n} rays ({100 * frac:.2f} %); shaded samples {int(fw['n_app'].sum())}")
    assert float(fw["mlp"].min()) >= MARGIN_MLP[False], "the safe MLP has a pre-activation near 0"
    assert frac <= MAX_EXCLUDED
    g = torch.Generator().manual_seed(seed + 2)
    keep = (~drop).double().cpu()
    g_rgb = (torch.randn(n, 3, generator=g, dtype=torch.float64) * keep[:, None])
    g_depth = (0.05 * torch.randn(n, generator=g, dtype=torch.float64) * keep)
    # the composed path: TensorVMSplit under autograd (explicit z, white background: no coin)
    r = rays.clone().requires_grad_(True)
    called = []
    orig = m._forward_autograd
    m._forward_autograd = lambda *a, **k: called.append(1) or orig(*a, **k)
    rgb, depth = m(r, white_bg=True, is_train=False, z_vals=z, floater_thresh=floater, refine=refine,
                   return_weights=return_weights)
    assert called, "the call did not take the composed path"
    ((rgb * g_rgb.float().cuda()).sum() + (depth * g_depth.float().cuda()).sum()).backward()
    torch.cuda.synchronize()
    got = {name: p.grad if p.grad is not None else torch.zeros_like(p) for name, p in m.named_parameters()}
    got["rays"] = r.grad
    ref, _ = R.field_backward(F, rays, z, True, g_rgb, g_depth, want_margins=False, floater=floater, refine=refine)
    if return_weights:
        assert float((m.last_weights.double() - fw["w"]).abs().max()) < 1e-4
    return got, ref, fw


@pytest.mark.parametrize("S", [72, 344])
@pytest.mark.parametrize("gname", list(GRIDS))
@pytest.mark.parametrize("case", list(PE_CASES))
def test_positional_encodings_vs_float64(case, gname, S):
    """The bar grows with the feature encoding's top frequency: d sin(2^f x) / dx = 2^f cos(2^f x), and fp32 evaluates
    the cos at 2^f times x's rounding error, so the gradients upstream of the encoding (appearance grids, basis, layer
    1) carry 2^f more relative error at f = fea_pe - 1.  The bar is TOL through fea_pe = 6 and doubles with each
    frequency beyond, 4 TOL at fea_pe = 8 -- a scaling derived, not measured, between fea_pe = 3 (measured at most
    5.7e-5 of the scale) and 8 (3.9e-4 at 40 x 52 x 64, S = 72)."""
    fea_pe, view_pe, act, refine = PE_CASES[case]
    got, ref, fw = _run(GRIDS[gname], S, fea_pe, view_pe, act, refine)
    compare(f"{case} {gname} S {S}", got, ref, fw["texel"] < TEXEL_MARGIN, tol=TOL * max(1, 2 ** (fea_pe - 6)))


@pytest.mark.parametrize("gname", list(GRIDS))
@pytest.mark.parametrize("opt", ["floater", "return_weights"])
def test_pe0_options_take_composed_path_vs_float64(opt, gname):
    """pe = 0 with floater_thresh = 0.5 or return_weights=True: the fused backward covers neither, so autograd goes
    through the composed path."""
    got, ref, fw = _run(GRIDS[gname], 72, 0, 0, "softplus", True, floater=0.5 if opt == "floater" else 0.0,
                        return_weights=opt == "return_weights")
    compare(f"pe0 {opt} {gname}", got, ref, fw["texel"] < TEXEL_MARGIN)


# ---- LocalTensorfs: the training call of a field with positional encodings ----------------------------------------
def _scene(fd, fov360, V, seed):
    """A LocalTensorfs whose (only, training) field holds fd's parameters, V + 1 frames with random poses, clamping
    exposures (a channel pushed past 1 and one below 0 on most rays) and a non-zero world2rf; refining, so the
    feature encoding is on."""
    import localrf_b200 as L
    from gpu_helpers import field_kwargs
    from helpers import FIELD_KEYS, field_scalars
    sc = field_scalars(fd)
    aabb = torch.as_tensor(fd["aabb"], dtype=torch.float32).cuda()
    lt = L.LocalTensorfs(camera_prior=None, fov=360 if fov360 else 85.6, n_init_frames=V + 1, n_overlap=30,
                         WH=(96, 64), n_iters_per_frame=600, n_iters_reg=100, lr_R_init=5e-3, lr_t_init=5e-4,
                         lr_i_init=1e-3, lr_exposure_init=1e-3, rf_lr_init=2e-2, rf_lr_basis=1e-3,
                         lr_decay_target_ratio=0.1, N_voxel_list={}, update_AlphaMask_list=[], lr_upsample_reset=True,
                         device="cuda", aabb=aabb, gridSize=sc["gridSize"], **field_kwargs(sc)).cuda()
    rf = lt.tensorfs[-1]
    sd = rf.state_dict()
    for k in FIELD_KEYS:
        sd[k] = torch.as_tensor(np.asarray(fd[k]), dtype=torch.float32).reshape(sd[k].shape)
    rf.load_state_dict(sd)
    gen = torch.Generator().manual_seed(seed)
    clamp = torch.tensor([[3.0, 0.1, 0.0], [0.05, 1.2, 0.0], [-2.0, 0.1, 1.0]])
    with torch.no_grad():
        for i in range(V + 1):
            lt.t_c2w[i].copy_((0.3 * torch.randn(3, generator=gen)).cuda())
            lt.r_c2w[i].add_((0.3 * torch.randn(3, 2, generator=gen)).cuda())
            lt.exposure[i].copy_((clamp + 0.05 * torch.randn(3, 3, generator=gen)).cuda())
        lt.world2rf[-1].copy_(torch.tensor([0.05, -0.02, 0.01]).cuda())
        lt.focal_offset.fill_(1.1)
        lt.center_rel.copy_(torch.tensor([0.52, 0.47]).cuda())
    lt.is_refining = True
    return lt


LOCAL_CASES = {   # (fov360, views, rays per view)
    "v1": (False, 1, 1024),
    "v16": (False, 16, 64),
    "v1_fov360": (True, 1, 1024),
    "v16_fov360": (True, 16, 64),
}


@pytest.mark.parametrize("case", list(LOCAL_CASES))
def test_local_training_call_vs_float64(case):
    """LocalTensorfs.forward(is_train=True) on a field with fea_pe = view_pe = 2: every training call of such a field
    runs LocalTensorfs._forward_autograd (torch ray generation from cam2world and the intrinsics, world2rf, the
    exposure matmul and the clamp) around TensorBase._forward_autograd.  Against render64.train_backward: the field's
    gradients, and those of the poses (r_c2w, t_c2w), the intrinsics (init_focal, focal_offset, center_rel), the
    exposures and world2rf -- render64's d_cam2world / d_intrinsics chained through get_cam2world and focal / center
    by fp32 autograd.  Rays below a field margin, at a texel floor or with E x within MARGIN of a clamp bound get zero
    cotangents (the excluded-fraction cap of test_gpu_backward_edges.py); E x clamps at both bounds on the others."""
    fov360, V, rpv = LOCAL_CASES[case]
    fd = R.random_field((40, 52, 64), shift=-2.0, thres=1e-3, seed=3, safe_mlp=True, fea_pe=2, view_pe=2)
    lt = _scene(fd, fov360, V, seed=5)
    rf = lt.tensorfs[-1]
    F = R.Field64.from_module(rf, "cuda")
    W, H, n = 96, 64, V * rpv
    z = R.ztable(72).cuda()
    rf.sample_table = lambda *a, **k: z
    views = torch.arange(1, V + 1, device="cuda")
    gen = torch.Generator().manual_seed(7)
    ids = (torch.randint(0, W * H, (V, rpv), generator=gen).cuda() + views[:, None] * W * H).reshape(-1)
    with torch.no_grad():
        c2w = lt.get_cam2world(views).double()
        intr = torch.cat([lt.focal(W).reshape(1), lt.center(W, H)]).double()
        E = torch.stack([lt.exposure[int(v)] for v in views]).double()
        w2 = lt.world2rf[-1].double()
    x = R.render_views([F], z, ids, W, H, fov360, intr, c2w, [w2], None, None, True, finalize=False)["rgb"]
    g_rgb = torch.randn(n, 3, generator=gen, dtype=torch.float64)
    g_depth = 0.05 * torch.randn(n, generator=gen, dtype=torch.float64)
    g_dirs = 0.1 * torch.randn(n, 3, generator=gen, dtype=torch.float64)
    _, fwd = R.train_backward(F, z, ids, W, H, fov360, intr, c2w, w2, E, x, True, g_rgb, g_depth, g_dirs)
    drop = (excluded(fwd, False) | (fwd["texel"] < TEXEL_MARGIN) | (fwd["clamp"] < MARGIN)).cpu()
    frac = float(drop.double().mean())
    y = torch.einsum("nab,nb->na", E[torch.arange(n, device="cuda") // rpv], x)[~drop.cuda()]
    print(f"excluded {int(drop.sum())} of {n} rays ({100 * frac:.2f} %); kept channels above 1: "
          f"{int((y > 1).sum())}, below 0: {int((y < 0).sum())}")
    assert frac <= MAX_EXCLUDED and int((y > 1).sum()) > 0 and int((y < 0).sum()) > 0
    keep = (~drop).double()
    g_rgb, g_depth, g_dirs = g_rgb * keep[:, None], g_depth * keep, g_dirs * keep[:, None]
    ref, _ = R.train_backward(F, z, ids, W, H, fov360, intr, c2w, w2, E, x, True, g_rgb, g_depth, g_dirs)

    called = []
    orig = lt._forward_autograd
    lt._forward_autograd = lambda *a, **k: called.append(1) or orig(*a, **k)
    lt.zero_grad()
    rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True, white_bg=True)
    assert called, "the training call did not take the composed path"
    f32 = lambda t: t.float().cuda()
    ((rgb * f32(g_rgb)).sum() + (depth * f32(g_depth)).sum() + (dirs * f32(g_dirs)).sum()).backward()
    torch.cuda.synchronize()

    grad = lambda p: p.grad if p.grad is not None else torch.zeros_like(p)
    errs = {k: scale_err(grad(p), ref[k]) for k, p in rf.named_parameters() if k in R.PARAM_KEYS}
    # the camera leaves: render64's cam2world / intrinsics gradients through the fp32 graphs that build them
    poses = [lt.r_c2w[int(v)] for v in views] + [lt.t_c2w[int(v)] for v in views]
    ref_pose = torch.autograd.grad(lt.get_cam2world(views), poses, ref["d_cam2world"].float())
    errs["r_c2w"] = scale_err(torch.stack([grad(p) for p in poses[:V]]), torch.stack(ref_pose[:V]))
    errs["t_c2w"] = scale_err(torch.stack([grad(p) for p in poses[V:]]), torch.stack(ref_pose[V:]))
    errs["exposure"] = scale_err(torch.stack([grad(lt.exposure[int(v)]) for v in views]), ref["d_exposure"])
    errs["world2rf"] = scale_err(grad(lt.world2rf[-1]), ref["d_world2rf"])
    intr_leaves = [lt.init_focal, lt.focal_offset, lt.center_rel]
    if fov360:                          # the 360 directions read no intrinsics
        assert float(ref["d_intrinsics"].abs().max()) == 0.0
        assert all(float(grad(p).abs().max()) == 0.0 for p in intr_leaves)
    else:
        ref_intr = torch.autograd.grad(torch.cat([lt.focal(W).reshape(1), lt.center(W, H)]), intr_leaves,
                                       ref["d_intrinsics"].float())
        errs["intrinsics"] = scale_err(torch.cat([grad(p).reshape(-1) for p in intr_leaves]),
                                       torch.cat([r.reshape(-1) for r in ref_intr]))
    print(case, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs
