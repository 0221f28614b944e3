"""-m gpu: the training call of LocalTensorfs.forward as one autograd node (_TrainRenderFn: lrf_render in ray-generation
mode + lrf_exposure_clamp forward, lrf_render_backward_batch backward).  `_forward_autograd` is patched to raise, so
the node is what runs, except where the composed path is the reference being compared with.

Metric: max |dg| / max |g_ref| per tensor (scale error), as in test_gpu_grads.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import camera_oracle
from helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu


def scale_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))


def _no_composed(lt, monkeypatch):
    def boom(*a, **k):
        raise AssertionError("LocalTensorfs._forward_autograd ran; the training node was expected")
    monkeypatch.setattr(lt, "_forward_autograd", boom)


def _golden_scene():
    from gpu_helpers import local_from_golden
    g = load_golden("grads_local")
    lt = local_from_golden(g)
    z = torch.from_numpy(g["z"]).cuda()
    lt.tensorfs[-1].sample_table = lambda *a, **k: z
    ids = torch.from_numpy(g["ray_ids"]).cuda()
    views = torch.from_numpy(g["view_ids"]).cuda()
    return g, lt, z, ids, views


def test_grads_local_golden_through_node(monkeypatch):
    """Every parameter gradient of the reference's autograd golden (poses, intrinsics, exposure, world2rf.2 and the
    newest field) within the 3e-4 bar of test_scene_gradients_vs_reference."""
    g, lt, z, ids, views = _golden_scene()
    _no_composed(lt, monkeypatch)
    rgb, depth, dirs, ij = lt(ids, views, int(g["W"]), int(g["H"]), is_train=True)
    assert rgb.grad_fn is not None and type(rgb.grad_fn).__name__.startswith("_TrainRenderFn")
    assert rel_err(rgb.detach().cpu().numpy(), g["out.rgb"]) < 1e-4
    assert rel_err(depth.detach().cpu().numpy(), g["out.depth"]) < 1e-4
    loss = (rgb * torch.from_numpy(g["c_rgb"]).cuda()).sum() + (depth * torch.from_numpy(g["c_depth"]).cuda()).sum()
    loss.backward()
    errs = {}
    for name, p in lt.named_parameters():
        key = "grad." + name
        if key in g:
            assert p.grad is not None, name
            errs[name] = scale_err(p.grad.cpu().numpy(), g[key])
    print("grads_local scale errors:", {k: f"{v:.1e}" for k, v in errs.items()})
    assert "world2rf.2" in errs and len(errs) >= 30
    assert max(errs.values()) < 3e-4, errs


def _inputs(lt, ids, views, W, H, bg=True):
    """(rays_i, c2w, intr, E, w2) as the node passes them to the kernels (fp32, contiguous, detached)."""
    idl = views.tolist()
    c2w = lt.get_cam2world(idl).detach().contiguous()
    intr = torch.cat([lt.focal(W).reshape(1), lt.center_rel[0:1] * W, lt.center_rel[1:2] * H]).detach().contiguous()
    E = torch.stack([lt.exposure[v] for v in idl]).detach().contiguous()
    return ids.to(torch.int64).contiguous(), c2w, intr, E, lt.world2rf[-1].detach().contiguous()


def _batch_backward(lt, z, ids, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs, W, H, bg=True, fov360=False):
    """lrf_render_backward_batch called directly -> (scratch rays [n,6], d_rays [n,6], camera grads dict)."""
    import localrf_b200 as L
    from localrf_b200.local_tensorfs import _train_batch
    from localrf_b200.tensorf import _field_grad_buffers
    rf, dev, n, V = lt.tensorfs[-1], ids.device, ids.shape[0], c2w.shape[0]
    lib = L._lib.lib()
    fs, _ = rf.field_and_prepared(z, fp32=True)
    bp = rf._prepared_backward()
    b = _train_batch(ids, W, H, fov360, c2w, intr, E, w2, bg)
    bufs, g = _field_grad_buffers(rf, dev)
    d_rays = torch.empty(n, 6, device=dev)
    g.d_rays = d_rays.data_ptr()
    out = dict(d_cam2world=torch.empty(V, 3, 4, device=dev), d_intrinsics=torch.empty(3, device=dev),
               d_exposure=torch.empty(V, 3, 3, device=dev), d_world2rf=torch.empty(3, device=dev))
    cg = L._lib.LrfCameraGrads()
    for k, t in out.items():
        setattr(cg, k, t.data_ptr())
    nbytes = lib.lrf_backward_batch_scratch_bytes(n, z.numel(), V)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    L._lib.check(lib.lrf_render_backward_batch(C.byref(fs), P(bp), C.byref(b), P(x), P(g_rgb), P(g_depth), P(g_dirs),
                                               C.byref(g), C.byref(cg), P(scratch), nbytes,
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    rays = scratch[: n * 24].view(torch.float32).view(n, 6).clone()
    return rays, d_rays, out


def test_scratch_rays_bitwise_and_camera_grads_vs_oracle(monkeypatch):
    """The rays the backward writes to scratch, rendered through explicit-ray lrf_render, give bitwise the node's
    pre-exposure rgb and its depth (so the backward marched exactly the forward's rays); the camera gradients equal
    the float64 restatement fed with the d_rays of that same call, and the node's own backward gives bitwise the
    same camera gradients."""
    g, lt, z, ids, views = _golden_scene()
    _no_composed(lt, monkeypatch)
    W, H = int(g["W"]), int(g["H"])
    with torch.no_grad():
        for e in lt.exposure:                      # a non-identity exposure that clamps some channels at both ends
            e.copy_(torch.tensor([[4.0, 0.1, 0.0], [0.05, 1.2, 0.0], [-4.0, 0.1, 1.0]], device="cuda"))
    rays_i, c2w, intr, E, w2 = _inputs(lt, ids, views, W, H)
    n = rays_i.shape[0]
    gen = torch.Generator().manual_seed(4)
    g_rgb = torch.randn(n, 3, generator=gen).cuda()
    g_depth = (0.05 * torch.randn(n, generator=gen)).cuda()
    g_dirs = (0.1 * torch.randn(n, 3, generator=gen)).cuda()
    rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True)
    # the forward's pre-exposure colour, as the node saved it
    x = rgb.grad_fn.saved_tensors[-1].detach()
    y = torch.einsum("nab,nb->na", E.repeat_interleave(n // E.shape[0], 0), x)
    assert bool((y < 0).any()) and bool((y > 1).any()), "the case must clamp at both bounds"
    rays, d_rays, cam = _batch_backward(lt, z, rays_i, c2w, intr, E, w2, x, g_rgb, g_depth, g_dirs, W, H)
    rf = lt.tensorfs[-1]
    rgb_e, depth_e = rf._render_fused(rays, z, True, 0.0, False, None, fp32=True)
    assert torch.equal(rgb_e, x) and torch.equal(depth_e, depth.detach())
    ref = camera_oracle.camera_backward(d_rays.cpu().numpy(), x.cpu().numpy(), g_rgb.cpu().numpy(),
                                        rays_i.cpu().numpy(), W, H, c2w.cpu().numpy(), intr.cpu().numpy(),
                                        E.cpu().numpy(), g_dirs.cpu().numpy())
    errs = {k: scale_err(cam[k].cpu().numpy(), ref[k]) for k in cam}
    print("camera gradients vs float64 restatement:", {k: f"{v:.1e}" for k, v in errs.items()})
    # the kernel accumulates in fp64 but from its fp32 directions; the restatement recomputes them in float64 from
    # the ray ids (6e-8 relative apart), and the focal gradient is a sum with cancellation: 1e-4 of the scale
    assert max(errs.values()) < 1e-4, errs
    # the node's backward: the same kernels on the same inputs -> the same bits (d_rays has no float atomics either)
    c2w_l = c2w.clone().requires_grad_(True)
    intr_l = intr.clone().requires_grad_(True)
    E_l = E.clone().requires_grad_(True)
    w2_l = w2.clone().requires_grad_(True)
    from localrf_b200.local_tensorfs import _TrainRenderFn
    out = _TrainRenderFn.apply(rf, z, True, rays_i, W, H, False, [], c2w_l, intr_l, E_l, w2_l, *rf._grad_params())
    assert torch.equal(out[0], rgb.detach()) and torch.equal(out[2], dirs.detach()) and torch.equal(out[3], ij)
    torch.autograd.backward([out[0], out[1], out[2]], [g_rgb, g_depth, g_dirs])
    for k, leaf in (("d_cam2world", c2w_l), ("d_intrinsics", intr_l), ("d_exposure", E_l), ("d_world2rf", w2_l)):
        assert torch.equal(leaf.grad, cam[k]), k


def test_node_outputs_equal_fused_no_grad_call(monkeypatch):
    """rgb, depth, directions and ij of the node are bitwise those of the no-grad fused call on the same table."""
    g, lt, z, ids, views = _golden_scene()
    _no_composed(lt, monkeypatch)
    W, H = int(g["W"]), int(g["H"])
    got = lt(ids, views, W, H, is_train=True)
    with torch.no_grad():
        want = lt(ids, views, W, H, is_train=True)
    for a, b in zip(got, want):
        assert torch.equal(a.detach(), b)


def test_two_backwards_bitwise_equal(monkeypatch):
    g, lt, z, ids, views = _golden_scene()
    _no_composed(lt, monkeypatch)
    W, H = int(g["W"]), int(g["H"])
    c = torch.from_numpy(g["c_rgb"]).cuda()
    grads = []
    for _ in range(2):
        lt.zero_grad()
        rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True)
        ((rgb * c).sum() + depth.sum() + 0.1 * dirs.sum()).backward()
        grads.append({n: p.grad.clone() for n, p in lt.named_parameters()
                      if p.grad is not None and not n.startswith("tensorfs")})
    assert set(grads[0]) == set(grads[1]) and len(grads[0]) >= 15
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), k


@pytest.mark.parametrize("what", ["pose", "exposure", "field", "world2rf"])
def test_inplace_change_between_forward_and_backward_raises(what, monkeypatch):
    g, lt, z, ids, views = _golden_scene()
    _no_composed(lt, monkeypatch)
    rgb, depth, dirs, ij = lt(ids, views, int(g["W"]), int(g["H"]), is_train=True)
    v = int(views[0])
    with torch.no_grad():
        {"pose": lambda: lt.t_c2w[v].add_(1e-3), "exposure": lambda: lt.exposure[v].mul_(1.01),
         "field": lambda: lt.tensorfs[-1].density_plane[0].add_(1e-3),
         "world2rf": lambda: lt.world2rf[-1].add_(1e-3)}[what]()
    with pytest.raises(RuntimeError):
        (rgb.sum() + depth.sum()).backward()


def test_fov360_and_test_id(monkeypatch):
    """fov 360: the directions do not use the intrinsics, so their gradient is zero; test_id: the exposure is the
    detached neighbour average, so the exposure leaves get no gradient."""
    from gpu_helpers import local_from_golden
    g = load_golden("local3_fov360")
    lt = local_from_golden(g)
    _no_composed(lt, monkeypatch)
    W, H = int(g["W"]), int(g["H"])
    ids = torch.from_numpy(g["ray_ids"]).cuda()
    n_views = 2
    ids = ids[: (ids.shape[0] // n_views) * n_views]
    views = torch.tensor([1, 2], device="cuda")
    rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True)
    (rgb.sum() + depth.sum() + dirs.sum()).backward()
    for p in (lt.init_focal, lt.focal_offset, lt.center_rel):
        assert p.grad is not None and torch.count_nonzero(p.grad) == 0
    assert lt.t_c2w[1].grad is not None and torch.count_nonzero(lt.t_c2w[1].grad) > 0
    lt.zero_grad()
    rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True, test_id=True)
    (rgb.sum() + depth.sum()).backward()
    assert all(e.grad is None or torch.count_nonzero(e.grad) == 0 for e in lt.exposure)
    assert lt.t_c2w[1].grad is not None


# ---- 300^3, 16 views x 256 rays, against the composed path ------------------------------------------------------
def _make300():
    import bench
    import localrf_b200 as L
    lt = bench._scene(L.LocalTensorfs, "cpu", 300, n_init_frames=20).to("cuda")
    gen = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for i in range(20):
            lt.t_c2w[i].copy_((0.05 * torch.randn(3, generator=gen)).cuda())
            lt.r_c2w[i].add_((0.05 * torch.randn(3, 2, generator=gen)).cuda())
            lt.exposure[i].copy_((torch.eye(3) * 1.5 + 0.3 * torch.randn(3, 3, generator=gen)).cuda())
    lt.is_refining = True
    return lt


@pytest.fixture(scope="module")
def scene300():
    return _make300()


def _batch300(seed=3):
    import bench
    gen = torch.Generator().manual_seed(seed)
    views = list(range(4, 18)) + [17, 17]                    # 16 views, train.py's forced duplicate last views
    px = torch.randint(0, bench.IMG_W * bench.IMG_H, (16, 256), generator=gen)
    ids = (px + torch.tensor(views)[:, None] * bench.IMG_W * bench.IMG_H).reshape(-1)
    return ids.cuda(), torch.tensor(views).cuda(), bench.IMG_W, bench.IMG_H


def _run(lt, ids, views, W, H, composed, monkeypatch, cs, seed=11):
    monkeypatch.setenv("LRF_TRAIN_PATH", "composed" if composed else "fused")
    lt.zero_grad()
    torch.manual_seed(seed)
    rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True, white_bg=False)
    state = (torch.get_rng_state(), torch.cuda.get_rng_state())
    c_rgb, c_depth, c_dir = cs
    ((rgb * c_rgb).sum() + (depth * c_depth).sum() + (dirs * c_dir).sum()).backward()
    grads = {n: p.grad.detach().clone() for n, p in lt.named_parameters() if p.grad is not None}
    return (rgb.detach(), depth.detach(), dirs.detach(), ij), grads, state


def test_fullsize_vs_composed_path(scene300, monkeypatch):
    """The node against LocalTensorfs._forward_autograd (torch ops around _RenderFn) at 300^3, 16 x 256 rays, with a
    non-identity exposure clamping at both bounds, non-zero grad_directions and duplicate views.

    The two paths generate the rays with different fp32 arithmetic (torch's bmm vs the kernel's fmas), so their
    rays differ by a few ulps and, as test_fused_backward_matches_composed_path_fullsize explains, the field's hard
    switches (the shading threshold, the MLP's ReLUs) flip for a few samples: single rays' rgb and the sparse field
    gradients differ by the size of a few switched samples (bar 0.1, as there).  The camera gradients are sums over
    the rays of a view, where a few switched samples are small next to the total.  They are measured against the
    largest gradient of their family (every view's rotation, translation or exposure; the intrinsics; world2rf),
    because a view whose gradients are small by chance has its own scale set by the same switched samples
    (measured: per-tensor up to 1.3e-2 on two such views; of the family's scale 1.0e-2 on the rotations, 9e-3 on
    center_rel, <= 4e-3 elsewhere, 6e-7 on the exposure).  Bar: 2e-2 of the family's scale.
    The directions and ij are exact products of the same fp32 values: bitwise equal."""
    lt = scene300
    ids, views, W, H = _batch300()
    n = ids.shape[0]
    gen = torch.Generator().manual_seed(2)
    cs = (torch.randn(n, 3, generator=gen).cuda(), (0.05 * torch.randn(n, generator=gen)).cuda(),
          (0.1 * torch.randn(n, 3, generator=gen)).cuda())
    (o_c, g_c, st_c) = _run(lt, ids, views, W, H, True, monkeypatch, cs)
    (o_f, g_f, st_f) = _run(lt, ids, views, W, H, False, monkeypatch, cs)
    assert torch.equal(st_c[0], st_f[0]) and torch.equal(st_c[1], st_f[1]), "RNG state after the call"
    assert torch.equal(o_c[2], o_f[2]) and torch.equal(o_c[3], o_f[3])
    d_rgb = (o_f[0] - o_c[0]).abs().max(dim=-1).values
    print("rgb: median", float(d_rgb.median()), "max", float(d_rgb.max()))
    assert float(d_rgb.median()) < 1e-5 and float(d_rgb.max()) < 3e-2
    assert rel_err(o_f[1].cpu().numpy(), o_c[1].cpu().numpy()) < 1e-3
    assert set(g_c) == set(g_f)
    errs = {k: scale_err(g_f[k].cpu().numpy(), g_c[k].cpu().numpy()) for k in g_c}
    print("scale errors vs composed:", {k: f"{v:.1e}" for k, v in errs.items()})
    cam = {k: v for k, v in errs.items() if not k.startswith("tensorfs")}
    assert any(k.startswith("exposure") for k in cam) and "world2rf.0" in cam and "focal_offset" in cam
    fam_err = {}
    for fam in ("r_c2w.", "t_c2w.", "exposure.", "init_focal", "focal_offset", "center_rel", "world2rf."):
        keys = [k for k in cam if k.startswith(fam)]
        scale = max(float(g_c[k].abs().max()) for k in keys)
        fam_err[fam] = max(float((g_f[k] - g_c[k]).abs().max()) for k in keys) / max(scale, 1e-12)
    print("camera errors vs composed, of the family's scale:", {k: f"{v:.1e}" for k, v in fam_err.items()})
    assert max(fam_err.values()) < 2e-2, fam_err
    assert max(errs.values()) < 0.1, errs


def test_short_training_loop_tracks_composed_path(monkeypatch):
    """Six train.py-shaped steps (rgb L1 loss + the density L1 regulariser, optimizer_step with poses and exposure)
    from the same state through each path.  Bars: losses within 1e-3 relative; each pose / exposure tensor's total
    change within 5 % (L2) of the composed path's change -- Adam's first steps are nearly sign(g) lr per element, so
    an element whose gradient is close to zero may step differently; a wrong camera gradient moves O(1)."""
    runs = {}
    ids, views, W, H = _batch300(5)
    target = torch.full((ids.shape[0], 3), 0.4, device="cuda")
    base = {n: p.detach().clone() for n, p in _make300().named_parameters() if not n.startswith("tensorfs")}
    for composed in (True, False):
        monkeypatch.setenv("LRF_TRAIN_PATH", "composed" if composed else "fused")
        lt = _make300()
        torch.manual_seed(0)
        losses = []
        for _ in range(6):
            rgb, depth, dirs, ij = lt(ids, views, W, H, is_train=True)
            tv, l1 = lt.get_reg_loss(None, 0, 0, 8e-5)
            loss = (rgb - target).abs().mean() + l1
            lt.optimizer_step(loss, optimize_poses=True)
            losses.append(float(loss.detach()))
        runs[composed] = (losses, {n: p.detach().clone() for n, p in lt.named_parameters()})
    lc, lf = runs[True][0], runs[False][0]
    print("losses composed", lc, "node", lf)
    assert max(abs(a - b) / abs(a) for a, b in zip(lc, lf)) < 1e-3
    for v in (4, 10, 17):
        for name in (f"t_c2w.{v}", f"r_c2w.{v}", f"exposure.{v}"):
            pc, pf = runs[True][1][name], runs[False][1][name]
            step = float((pc - base[name]).norm())
            diff = float((pf - pc).norm())
            print(name, "change", step, "difference", diff)
            assert step > 0 and diff < 0.05 * step, name
