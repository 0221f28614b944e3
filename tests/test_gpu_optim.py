"""-m gpu: localrf_b200.adam_step (one lrf_adam_step launch) against torch.optim.Adam.step on the same GPU.

The oracle is a deep copy of the same optimisers stepped one by one with `o.step()`.  Parameters, exp_avg and
exp_avg_sq are compared as int32 bit patterns, `step` and `state_dict()` exactly: the kernel has to round as
torch 2.11's foreach sequence does, so there is no tolerance anywhere in this file."""
import copy

import pytest
import torch

from localrf_b200 import optim

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def scene_tensors(gen, grid=(20, 24, 28)):
    """One tensor of every class the scene model optimises, with its own layout."""
    gx, gy, gz = grid
    r = lambda *s: torch.randn(*s, generator=gen)
    ts = [_cl(0.1 * r(1, 8, gy, gx)), _cl(0.1 * r(1, 24, gz, gx)),        # channel-last planes
          _cl(0.1 * r(1, 8, gz, 1)), _cl(0.1 * r(1, 24, gx, 1)),          # [1,C,L,1] lines
          r(27, 72) * 0.1, r(128, 27) * 0.1, r(128), r(3, 131) * 0.1, r(3),  # Linear weights and biases
          torch.eye(3, 2) + 0.01 * r(3, 2), 0.01 * r(3), torch.eye(3) + 0.01 * r(3, 3),   # per-frame
          torch.ones(1), 0.5 * torch.ones(2)]                               # focal_offset, center_rel
    return [torch.nn.Parameter(t.to(DEV)) for t in ts]


def special_grad(p, gen, step):
    """Random gradient with zeros, denormals, +-1e-30 and +-1e20 (g*g overflows to inf) mixed in."""
    g = torch.randn(p.shape, generator=gen)
    sel = torch.randint(0, 10, p.shape, generator=gen)
    sign = torch.where(torch.rand(p.shape, generator=gen) < 0.5, -1.0, 1.0)
    g = torch.where(sel == 0, torch.zeros_like(g), g)
    g = torch.where(sel == 1, sign * 1e-40, g)                 # denormal
    g = torch.where(sel == 2, sign * 1e-30, g)
    g = torch.where(sel == 3, sign * 1e20, g)
    g = torch.where(sel == 4, g * 1e-3 * (step + 1), g)
    return torch.empty_like(p).copy_(g.to(DEV))                # p's layout, as autograd gives it


def bits(t):
    return t.detach().view(torch.int32) if t.dtype == torch.float32 else t.detach().view(torch.int64)


def same_tensor(a, b):
    """Same bits and, for dense tensors, the same layout (deepcopy makes a strided parameter contiguous)."""
    layout = a.stride() == b.stride() or not optim._dense(a)
    return a.shape == b.shape and layout and a.device == b.device and torch.equal(bits(a), bits(b))


def params_of(opts):
    return [p for o in opts for g in o.param_groups for p in g["params"]]


def assert_same(opts, refs):
    for o, r in zip(opts, refs, strict=True):
        for p, q in zip(params_of([o]), params_of([r]), strict=True):
            assert same_tensor(p, q)
            sp, sq = o.state.get(p, {}), r.state.get(q, {})
            assert list(sp) == list(sq)
            for k in sp:
                assert same_tensor(sp[k], sq[k]), k
        a, b = o.state_dict(), r.state_dict()
        assert a["param_groups"] == b["param_groups"]
        assert list(a["state"]) == list(b["state"])
        for i in a["state"]:
            assert list(a["state"][i]) == list(b["state"][i])
            for k in a["state"][i]:
                assert same_tensor(a["state"][i][k], b["state"][i][k]), (i, k)


def set_grads(opts, refs, grads):
    for p, q, g in zip(params_of(opts), params_of(refs), grads, strict=True):
        p.grad = None if g is None else g
        q.grad = None if g is None else g.clone(memory_format=torch.preserve_format)


def scene_optimizers(gen):
    ps = scene_tensors(gen)
    field = torch.optim.Adam([{"params": ps[0:4], "lr": 2e-2}, {"params": ps[4:9], "lr": 1e-3}], betas=(0.9, 0.99))
    frame = [torch.optim.Adam([p], betas=(0.9, 0.99), lr=lr) for p, lr in zip(ps[9:12], (5e-3, 5e-4, 1e-3))]
    intr = torch.optim.Adam(ps[12:14], betas=(0.9, 0.99), lr=1e-3)
    return [field] + frame + [intr]


class CountingLib:
    """Stands in for the loaded library and counts lrf_adam_step calls."""

    def __init__(self, L):
        self.L, self.calls = L, 0

    def __getattr__(self, name):
        return getattr(self.L, name)

    def lrf_adam_step(self, *args):
        self.calls += 1
        return self.L.lrf_adam_step(*args)


@pytest.fixture
def counting(monkeypatch):
    from localrf_b200 import _lib
    c = CountingLib(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: c)
    return c


def test_scene_tensors_20_steps(counting):
    """Every tensor class, 20 steps, lr decayed between them; the centre-rel parameter gets its first gradient at
    step 3 and focal_offset never gets one (no state is created for it)."""
    gen = torch.Generator().manual_seed(0)
    opts = scene_optimizers(gen)
    refs = copy.deepcopy(opts)
    ps = params_of(opts)
    for step in range(20):
        grads = [special_grad(p, gen, step) for p in ps]
        grads[-2] = None                                         # focal_offset: never a gradient
        if step < 3:
            grads[-1] = None                                     # center_rel: from step 3 on
        set_grads(opts, refs, grads)
        optim.adam_step(opts)
        for r in refs:
            r.step()
        assert_same(opts, refs)
        for o, r in zip(opts, refs):
            for og, rg in zip(o.param_groups, r.param_groups):
                og["lr"] *= 0.93
                rg["lr"] *= 0.93
    assert counting.calls == 20
    assert len(opts[-1].state) == 1 and opts[-1].state[ps[-1]]["step"].item() == 17.0


def test_field_640_and_back_to_back(counting):
    """A 640^3 field (39.3 M parameters: every chunk runs many passes), then a second adam_step with a different
    table enqueued right behind it with no synchronisation between them."""
    gen = torch.Generator(device=DEV).manual_seed(1)
    G = 640
    shapes = [(1, 8, G, G)] * 3 + [(1, 24, G, G)] * 3
    big = [torch.nn.Parameter(_cl(0.1 * torch.randn(s, device=DEV, generator=gen))) for s in shapes]
    big += [torch.nn.Parameter(_cl(0.1 * torch.randn(1, c, G, 1, device=DEV, generator=gen)))
            for c in (8, 8, 8, 24, 24, 24)]
    field = [torch.optim.Adam([{"params": big[:3] + big[6:9], "lr": 2e-2},
                               {"params": big[3:6] + big[9:], "lr": 2e-2}], betas=(0.9, 0.99))]
    small = scene_optimizers(torch.Generator().manual_seed(2))
    field_ref, small_ref = copy.deepcopy(field), copy.deepcopy(small)
    cg = torch.Generator().manual_seed(3)
    for step in range(2):
        set_grads(field, field_ref, [torch.randn(p.shape, device=DEV, generator=gen).contiguous(
            memory_format=torch.channels_last) for p in params_of(field)])
        set_grads(small, small_ref, [special_grad(p, cg, step) for p in params_of(small)])
        optim.adam_step(field)
        optim.adam_step(small)
        for r in field_ref + small_ref:
            r.step()
    assert_same(field, field_ref)
    assert_same(small, small_ref)
    assert counting.calls == 4


def test_repeatable():
    gen = torch.Generator().manual_seed(4)
    base = scene_optimizers(gen)
    grads = [[special_grad(p, gen, s) for p in params_of(base)] for s in range(3)]
    runs = []
    for _ in range(2):
        opts = copy.deepcopy(base)
        for g in grads:
            for p, gg in zip(params_of(opts), g):
                p.grad = gg.clone(memory_format=torch.preserve_format)
            optim.adam_step(opts)
        runs.append(opts)
    assert_same(*runs)


@pytest.mark.parametrize("order", ["fused_then_torch", "torch_then_fused", "load_state_dict"])
def test_switching(order):
    gen = torch.Generator().manual_seed(5)
    opts = scene_optimizers(gen)
    refs = copy.deepcopy(opts)
    ps = params_of(opts)
    for step in range(6):
        set_grads(opts, refs, [special_grad(p, gen, step) for p in ps])
        first = step < 3
        if order == "load_state_dict" and step == 3:
            # a fresh optimiser set over the same parameters, loaded from the torch-stepped state
            fresh = []
            for o, r in zip(opts, refs):
                n = torch.optim.Adam([{k: v for k, v in g.items() if k != "params"} | {"params": g["params"]}
                                      for g in o.param_groups])
                n.load_state_dict(copy.deepcopy(r.state_dict()))   # (load_state_dict keeps tensors as given)
                fresh.append(n)
            opts = fresh
        use_fused = {"fused_then_torch": first, "torch_then_fused": not first, "load_state_dict": not first}[order]
        if use_fused:
            optim.adam_step(opts)
        else:
            for o in opts:
                o.step()
        for r in refs:
            r.step()
        assert_same(opts, refs)


def _fallback_cases():
    p = lambda *s: torch.nn.Parameter(torch.randn(*s, device=DEV))
    cases = {
        "amsgrad": lambda: [torch.optim.Adam([p(3, 2)], amsgrad=True)],
        "maximize": lambda: [torch.optim.Adam([p(3, 2)], maximize=True)],
        "weight_decay": lambda: [torch.optim.Adam([p(3, 2)], weight_decay=1e-2)],
        "foreach_false": lambda: [torch.optim.Adam([p(3, 2)], foreach=False)],
        "fused": lambda: [torch.optim.Adam([p(3, 2)], fused=True)],
        "capturable": lambda: [torch.optim.Adam([p(3, 2)], capturable=True)],
        "differentiable": lambda: [torch.optim.Adam([p(3, 2)], differentiable=True)],
        "tensor_lr": lambda: [torch.optim.Adam([p(3, 2)], lr=torch.tensor(1e-3))],
        "tensor_betas": lambda: [torch.optim.Adam([p(3, 2)], betas=(torch.tensor(0.9), torch.tensor(0.99)))],
        "cpu": lambda: [torch.optim.Adam([torch.nn.Parameter(torch.randn(3, 2))])],
        "fp64": lambda: [torch.optim.Adam([torch.nn.Parameter(torch.randn(3, 2, device=DEV, dtype=torch.float64))])],
        "strided": lambda: [torch.optim.Adam([torch.nn.Parameter(torch.randn(4, 6, device=DEV)[:, ::2])])],
        "twice": lambda: (lambda q: [torch.optim.Adam([q], lr=1e-3), torch.optim.Adam([q], lr=2e-3)])(p(3, 2)),
        "subclass": lambda: [type("MyAdam", (torch.optim.Adam,), {})([p(3, 2)])],
        "pre_hook": lambda: [_hooked(torch.optim.Adam([p(3, 2)]), "pre")],
        "post_hook": lambda: [_hooked(torch.optim.Adam([p(3, 2)]), "post")],
    }
    return cases


def _hooked(o, kind):
    hook = lambda *a: None
    (o.register_step_pre_hook if kind == "pre" else o.register_step_post_hook)(hook)
    return o


@pytest.mark.parametrize("case", list(_fallback_cases()) + ["global_pre_hook", "global_post_hook", "grad_layout"])
def test_fallback(case, counting):
    """Each condition sends the optimiser through its own step(): torch's result, no lrf_adam_step call.  A plain
    optimiser in the same call still takes the kernel."""
    from torch.optim.optimizer import register_optimizer_step_post_hook, register_optimizer_step_pre_hook
    torch.manual_seed(6)
    handle = None
    if case in _fallback_cases():
        odd = _fallback_cases()[case]()
    else:
        odd = [torch.optim.Adam([torch.nn.Parameter(torch.randn(3, 2, device=DEV))])]
        if case == "global_pre_hook":
            handle = register_optimizer_step_pre_hook(lambda *a: None)
        elif case == "global_post_hook":
            handle = register_optimizer_step_post_hook(lambda *a: None)
    plain = torch.optim.Adam([torch.nn.Parameter(torch.randn(5, device=DEV))])
    opts = odd + [plain]
    try:
        refs = copy.deepcopy(opts)
        for step in range(2):
            grads = []
            for q in params_of(opts):
                g = torch.randn(q.shape, dtype=q.dtype, device=q.device)
                if case == "grad_layout" and q.dim() == 2:
                    g = g.t().contiguous().t()                   # a column-major gradient of a row-major p
                grads.append(g)
            for a, b, g in zip(params_of(opts), params_of(refs), grads):
                a.grad, b.grad = g, g.clone()
            try:
                for r in refs:
                    r.step()
            except Exception as e:                               # torch refuses this configuration ...
                with pytest.raises(type(e)):                     # ... and so does adam_step, the same way
                    optim.adam_step(opts)
                return
            optim.adam_step(opts)
            assert_same(opts, refs)
        expect = 0 if handle is not None else 2                  # global hooks: nothing takes the kernel
        assert counting.calls == expect
    finally:
        if handle is not None:
            handle.remove()


# ---- LocalTensorfs.optimizer_step -------------------------------------------------------------------------------

def _reference_optimizer_step(self, loss, optimize_poses):
    """LocalTensorfs.optimizer_step as the reference orders it (local_tensorfs.py:193-290): the field's step, the
    schedule events, then the pose, exposure and intrinsics steps, each optimiser with its own step()."""
    from localrf_b200.utils import N_to_reso
    it = self.rf_iter[-1]
    if it == 0:
        self.lr_factor = 1
        self.n_iters = self.n_iters_per_frame
        self.n_iters_reg = self.n_iters_reg_per_frame
    elif it == 1:
        n_train = (self.blending_weights[:, -1] > 0).sum()
        self.n_iters = int(self.n_iters_per_frame * n_train)
        self.n_iters_reg = int(self.n_iters_reg_per_frame * n_train)
        self.lr_factor = self.lr_decay_target_ratio ** (1 / self.n_iters)
        self.N_voxel_list = {int(k * n_train): v for k, v in self.N_voxel_per_frame_list.items()}
        self.update_AlphaMask_list = [int(u * n_train) for u in self.update_AlphaMask_per_frame_list]
    self.regularize = self.rf_iter[-1] < self.n_iters_reg

    def decay(opt):
        for group in opt.param_groups:
            group["lr"] *= self.lr_factor

    live = self._live_pose_ids()
    for i in live:
        if optimize_poses:
            decay(self.r_optimizers[i]); decay(self.t_optimizers[i])
            self.r_optimizers[i].zero_grad(); self.t_optimizers[i].zero_grad()
        if self.lr_exposure_init > 0:
            decay(self.exp_optimizers[i])
            self.exp_optimizers[i].zero_grad()
    tune_intrinsics = self.lr_i_init > 0 and self.blending_weights.shape[1] == 1 and self.is_refining
    if tune_intrinsics:
        decay(self.intrinsic_optimizer)
        self.intrinsic_optimizer.zero_grad()
    self.rf_optimizer.zero_grad()
    loss.backward()
    self.rf_optimizer.step()
    if self.is_refining:
        decay(self.rf_optimizer)
    if self.rf_iter[-1] in self.N_voxel_list:
        reso = N_to_reso(self.N_voxel_list[self.rf_iter[-1]], self.tensorfs[-1].aabb)
        self.tensorfs[-1].upsample_volume_grid(reso)
        if self.lr_upsample_reset:
            groups = self.tensorfs[-1].get_optparam_groups(self.rf_lr_init, self.rf_lr_basis)
            self.rf_optimizer = torch.optim.Adam(groups, betas=(0.9, 0.99))
    if self.rf_iter[-1] in self.update_AlphaMask_list:
        self.tensorfs[-1].updateAlphaMask(tuple((self.tensorfs[-1].gridSize / 2).int()))
    for i in live:
        if optimize_poses:
            self.r_optimizers[i].step(); self.t_optimizers[i].step()
        if self.lr_exposure_init > 0:
            self.exp_optimizers[i].step()
    if tune_intrinsics:
        self.intrinsic_optimizer.step()
    if self.is_refining:
        self.rf_iter[-1] += 1
    return self.rf_iter[-1] >= self.n_iters - 1


def _reference_poses_only(self, loss):
    live = self._live_pose_ids()
    for i in live:
        self.r_optimizers[i].zero_grad(); self.t_optimizers[i].zero_grad()
    loss.backward()
    for i in live:
        self.r_optimizers[i].step(); self.t_optimizers[i].step()


def _local(lr_exposure_init, lr_upsample_reset):
    import bench
    import localrf_b200 as L
    torch.manual_seed(0)
    aabb = 2 * torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    lt = L.LocalTensorfs(camera_prior=None, fov=85.6, n_init_frames=4, n_overlap=30, WH=(64, 48),
                         n_iters_per_frame=600, n_iters_reg=100, lr_R_init=5e-3, lr_t_init=5e-4, lr_i_init=1e-3,
                         lr_exposure_init=lr_exposure_init, rf_lr_init=2e-2, rf_lr_basis=1e-3,
                         lr_decay_target_ratio=0.1, N_voxel_list={0.5: 28 ** 3}, update_AlphaMask_list=[0.75],
                         lr_upsample_reset=lr_upsample_reset, device=DEV, aabb=aabb.cuda(), gridSize=[24, 24, 24],
                         **bench.field_kwargs()).cuda()
    lt.is_refining = True
    return lt


def _loss(lt, it):
    """A loss whose gradients are exact functions of the parameters (no atomics), so that the two models see the
    same gradients bit for bit: products with fixed random weights, a square and the pose chain."""
    gen = torch.Generator(device=DEV).manual_seed(100 + it)
    total = 0
    for p in lt.tensorfs[-1].parameters():
        if p.requires_grad:
            w = torch.randn(p.shape, device=DEV, generator=gen)
            total = total + (p * w).sum() + 0.5 * (p * p).sum()
    c2w = lt.get_cam2world(starting_id=0)
    total = total + (c2w * torch.randn(c2w.shape, device=DEV, generator=gen)).sum()
    total = total + (torch.stack(list(lt.exposure)) ** 2).sum() * 0.1
    total = total + lt.focal(64).sum() * 1e-3 + (lt.center(64, 48) ** 2).sum() * 1e-4
    return total


def _all_optimizers(lt):
    opts = [lt.rf_optimizer] + lt.r_optimizers + lt.t_optimizers + lt.exp_optimizers
    return opts + ([lt.intrinsic_optimizer] if hasattr(lt, "intrinsic_optimizer") else [])


@pytest.mark.parametrize("lr_exposure_init", [1e-3, 0.0])
@pytest.mark.parametrize("lr_upsample_reset", [True, False])
def test_local_tensorfs_optimizer_step(lr_exposure_init, lr_upsample_reset, counting):
    """Iterations of LocalTensorfs.optimizer_step against the reference's order with per-optimiser steps: an
    upsample iteration, an alpha-mask iteration, optimize_poses=False, intrinsics tuned while refining,
    append_frame and append_rf mid-run, and optimizer_step_poses_only."""
    models = [_local(lr_exposure_init, lr_upsample_reset) for _ in range(2)]
    plan = [("step", True), ("step", True), ("step", False), ("step", True), ("append_frame", True),
            ("poses_only", None), ("append_rf", True), ("step", True)]
    kernel_calls = 0
    for it, (what, poses) in enumerate(plan):
        for k, lt in enumerate(models):
            torch.manual_seed(1000 + it)                       # append_rf initialises the new field from it
            if what == "append_frame":
                lt.append_frame()
            if what == "append_rf":
                lt.append_frame()
                lt.append_rf()
            loss = _loss(lt, it)
            if what == "poses_only":
                (lt.optimizer_step_poses_only if k == 0 else lambda l: _reference_poses_only(lt, l))(loss)
            elif k == 0:
                lt.optimizer_step(loss, optimize_poses=poses)
            else:
                _reference_optimizer_step(lt, loss, optimize_poses=poses)
        kernel_calls += 1
        assert counting.calls == kernel_calls, it              # one launch per step
        a, b = models
        for (na, pa), (nb, pb) in zip(a.named_parameters(), b.named_parameters(), strict=True):
            assert na == nb and same_tensor(pa, pb), (it, na)
        assert a.rf_iter == b.rf_iter and a.is_refining == b.is_refining
        assert_same(_all_optimizers(a), _all_optimizers(b))
    assert models[0].tensorfs[0].gridSize.tolist() != [24, 24, 24]   # the upsample ran
    assert models[0].tensorfs[0].alphaMask is not None               # and the alpha mask


def test_optimizer_step_one_launch_no_sync():
    """One steady-state optimizer_step: exactly one optimiser kernel and no other foreach kernel, and no
    synchronisation (set_sync_debug_mode("error") raises on one)."""
    from torch.profiler import ProfilerActivity, profile
    lt = _local(1e-3, True)
    for it in range(2):                      # iteration 1 reads the blending weights on the host
        lt.optimizer_step(_loss(lt, it), optimize_poses=True)
    loss = _loss(lt, 2)
    lt.rf_iter[-1] = 5                       # past the schedule events
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda.set_sync_debug_mode("error")
        try:
            lt.optimizer_step(loss, optimize_poses=True)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert sum("adam_kernel" in n for n in names) == 1, names
    assert not any("multi_tensor_apply" in n for n in names), names
