"""Host-side mirror of the reference's scene model (local_tensorfs.py:31-499).

`LocalTensorfs` keeps the reference's constructor kwargs, attributes, `state_dict` key set
(`blending_weights, init_focal, focal_offset, center_rel, r_c2w.i, t_c2w.i, exposure.i, world2rf.k,
tensorfs.k.*`) and method signatures, so the reference's train.py / renderer.py can import it
unchanged.  `forward` is the CUDA path: every active field is ONE fused kernel launch over the
whole ray batch (ray generation, march, shading, blend accumulation; exposure + clamp ride on the
last field's launch).  Differences that are deliberate:

  * fields are never parked on the CPU (180 GB of HBM holds every field of a scene); the
    reference's CPU<->GPU shuffle (local_tensorfs.py:132,432-434,476-479) has no equivalent;
  * `chunk` does not bound memory any more (the kernel materialises nothing per sample); it is
    honoured only in train mode, where each chunk draws its own jitter like the reference;
  * `sixD_to_mtx` uses the per-view cross product for every batch size (see utils.py).
"""
import ctypes as C
import math
import os
import re

import torch

from . import _lib
from .optim import adam_step, zero_grad
from .tensorf import (AlphaGridMask, TensorVMSplit, _check_field_state, _field_grad_buffers, _field_grads,
                      _field_state, _key, _memo, _ptr, _require_cuda, _stream)
from .utils import N_to_reso, mtx_to_sixD, sixD_to_mtx


def ids2pixel_view(W, H, ids):
    """local_tensorfs.py:14-21."""
    return ids % W, (ids // W) % H, ids // (W * H)


def ids2pixel(W, H, ids):
    """local_tensorfs.py:23-29."""
    return ids % W, (ids // W) % H


class _LaunchPlan:
    """Everything a fused `LocalTensorfs.forward` call derives from the module state: one entry per lrf_render
    launch (field, distance table, LrfBatch, first ray of its chunk, whether it is the chunk's last launch) and the
    device copies of cameras / intrinsics / exposure / blending rows the batches point at.  An eval call without
    autograd caches its plan, so a repeated call (the renderer's per-frame or per-batch loop) only re-checks the
    guards, allocates outputs and enqueues the launches.

    `guards` = (container, index, tensor, version): the plan is valid while every guarded slot still
    holds the same tensor object at the same version (optimiser steps, load_state_dict, append_* all
    bump one of them).  Field parameters are guarded by TensorBase.field_and_prepared's own memo."""
    __slots__ = ("guards", "launches", "keep", "dev", "key_refs")

    def valid(self):
        for cont, idx, t, ver in self.guards:
            cur = cont[idx]
            if ver == "eq":                          # plain value (e.g. nSamples)
                if cur != t:
                    return False
            elif cur is not t or (ver is not None and t._version != ver):
                return False
        return True


def _uva_pointer(t):
    """Device-usable address of a tensor the kernel may touch directly: CUDA memory, or PINNED host
    memory (zero-copy over PCIe: under unified addressing the device address equals the host one)."""
    if t.is_cuda:
        return t.data_ptr()
    if not t.is_pinned():
        raise RuntimeError("localrf_b200: host tensors handed to the render path must be pinned "
                           "(page-locked) memory; pageable memory is not device-accessible")
    return t.data_ptr()


def _ray_ids(ray_ids):
    """(contiguous int64 ids, their device-usable address).  The address is that of the tensor the kernel reads: an
    int32 or strided pinned batch converts to a pageable copy, which is refused like pageable ids."""
    if ray_ids.dtype != torch.int64 or not ray_ids.is_contiguous():
        ray_ids = ray_ids.to(torch.int64).contiguous()
    return ray_ids, _uva_pointer(ray_ids)


def _chunks(n, n_views, budget):
    """(lo, hi, v_lo, v_hi) of consecutive chunks of whole views, at most `budget` rays each (but at least one view);
    one chunk when n <= budget.  Chunks stay on view boundaries because the kernel derives a ray's view from its
    position in the launch."""
    per_view = n // n_views
    step = n if n <= budget else max(per_view, (budget // per_view) * per_view)
    for lo in range(0, n, step):
        hi = min(lo + step, n)
        yield lo, hi, lo // per_view, hi // per_view


def _ray_batch(ids_ptr, n_rays, W, H, fov360, intr, cam2world, w2rf, v_lo, v_hi, exposure=None, blend=None, k=0,
               **flags):
    """LrfBatch in ray-generation mode: `n_rays` ids at `ids_ptr` over the views [v_lo, v_hi) of cam2world [V,3,4],
    of exposure [V,3,3] and of column k of blend [V, n_fields] (the last two when given); `flags` are the remaining
    scalar fields (white_bg, accumulate, finalize, floater_thresh, refine).  All tensors contiguous fp32 on the
    device."""
    b = _lib.LrfBatch(n_rays=n_rays, ray_ids=ids_ptr, W=int(W), H=int(H), fov360=int(fov360),
                      intrinsics=intr.data_ptr(), cam2world=cam2world.data_ptr() + 48 * v_lo, n_views=v_hi - v_lo,
                      world2rf=w2rf.data_ptr(), **flags)
    if exposure is not None:
        b.exposure = exposure.data_ptr() + 36 * v_lo
    if blend is not None:
        b.blend = blend.data_ptr() + 4 * (v_lo * blend.shape[1] + k)
        b.blend_stride = blend.shape[1]
    return b


def _train_batch(ray_ids, W, H, fov360, cam2world, intr, exposure, w2rf, bg):
    """LrfBatch of the training call: one field, no blend, finalize = 0 (the exposure and the clamp run in
    lrf_exposure_clamp), every view of cam2world.  All tensors contiguous fp32 (ray_ids int64) on the device."""
    return _ray_batch(ray_ids.data_ptr(), ray_ids.shape[0], W, H, fov360, intr, cam2world, w2rf, 0, cam2world.shape[0],
                      exposure=exposure, white_bg=int(bg))


class _TrainRenderFn(torch.autograd.Function):
    """The training call of LocalTensorfs.forward for one field (local_tensorfs.py:397-499 with is_train) as ONE
    autograd node.  Forward: lrf_render generates the rays from the ids and cameras (finalize = 0), then
    lrf_exposure_clamp.  Backward: lrf_render_backward_batch -- the field's gradients as _RenderFn's, plus those of
    cam2world [V,3,4], the intrinsics [3] = (focal, cx, cy), the exposure [V,3,3] and world2rf [3], with
    grad_directions joining the intrinsics' gradient.  -> (rgb, depth, directions, ij); ij is not differentiable.

    `sources` are the leaves the camera inputs were built from (poses, exposure, intrinsics): like the field's
    parameters, an in-place change to one of them between forward and backward raises."""

    @staticmethod
    def forward(ctx, rf, z, bg, ray_ids, W, H, fov360, sources, cam2world, intr, exposure, w2rf, *params):
        dev, n = ray_ids.device, ray_ids.shape[0]
        cams = [t.detach().to(dev, torch.float32).contiguous() if t is not None else None
                for t in (cam2world, intr, exposure, w2rf)]
        c2w, it, E, w2 = cams
        rgb_lin = torch.empty(n, 3, dtype=torch.float32, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(n, dtype=torch.float32, device=dev)
        dirs = torch.empty(n, 3, dtype=torch.float32, device=dev)
        ij = torch.empty(n, 2, dtype=torch.int64, device=dev)
        lib = _lib.lib()
        with torch.cuda.device(dev):
            stream = _stream(dev)
            fs, prep = rf.field_and_prepared(z, fp32=True)
            b = _train_batch(ray_ids, W, H, fov360, c2w, it, None, w2, bg)
            o = _lib.LrfOutputs()
            o.rgb, o.depth, o.directions, o.ij = rgb_lin.data_ptr(), depth.data_ptr(), dirs.data_ptr(), ij.data_ptr()
            _lib.check(lib.lrf_render(C.byref(fs), _ptr(prep), C.byref(b), C.byref(o), stream))
            _lib.check(lib.lrf_exposure_clamp(_ptr(rgb_lin), _ptr(E), n, c2w.shape[0], _ptr(rgb), stream))
        ctx.rf, ctx.bg, ctx.W, ctx.H, ctx.fov360 = rf, bg, W, H, fov360
        ctx.seen = _field_state(rf, params)
        ctx.sources = tuple(sources)
        ctx.seen_cams = tuple((t.data_ptr(), t._version) for t in ctx.sources)
        ctx.has_exposure = E is not None
        ctx.save_for_backward(ray_ids, z, c2w, it, E, w2, rgb_lin)
        ctx.mark_non_differentiable(ij)
        return rgb, depth, dirs, ij

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_dirs, g_ij):
        ray_ids, z, c2w, it, E, w2, rgb_lin = ctx.saved_tensors
        rf, dev, n, V = ctx.rf, ray_ids.device, ray_ids.shape[0], c2w.shape[0]
        _check_field_state(rf, ctx.seen)
        if tuple((t.data_ptr(), t._version) for t in ctx.sources) != ctx.seen_cams:
            raise RuntimeError("localrf_b200: a pose, exposure or intrinsics parameter was modified between the "
                               "fused training forward and its backward")
        f32 = lambda g: g.detach().to(torch.float32).contiguous()
        g_rgb = torch.zeros(n, 3, device=dev) if g_rgb is None else f32(g_rgb)
        g_depth = torch.zeros(n, device=dev) if g_depth is None else f32(g_depth)
        g_dirs = None if g_dirs is None else f32(g_dirs)
        need = ctx.needs_input_grad
        d_c2w = torch.empty(V, 3, 4, device=dev) if need[8] else None
        d_intr = torch.empty(3, device=dev) if need[9] else None
        d_expo = torch.empty(V, 3, 3, device=dev) if ctx.has_exposure and need[10] else None
        d_w2 = torch.empty(3, device=dev) if need[11] else None
        bufs, g = _field_grad_buffers(rf, dev)
        cg = _lib.LrfCameraGrads()
        cg.d_cam2world, cg.d_intrinsics = _ptr(d_c2w), _ptr(d_intr)
        cg.d_exposure, cg.d_world2rf = _ptr(d_expo), _ptr(d_w2)
        lib = _lib.lib()
        with torch.cuda.device(dev):
            fs, _ = rf.field_and_prepared(z, fp32=True)
            bp = rf._prepared_backward()
            b = _train_batch(ray_ids, ctx.W, ctx.H, ctx.fov360, c2w, it, E, w2, ctx.bg)
            scratch = torch.empty(lib.lrf_backward_batch_scratch_bytes(n, z.numel(), V), dtype=torch.uint8,
                                  device=dev)
            _lib.check(lib.lrf_render_backward_batch(C.byref(fs), _ptr(bp), C.byref(b), _ptr(rgb_lin), _ptr(g_rgb),
                                                     _ptr(g_depth), _ptr(g_dirs), C.byref(g), C.byref(cg),
                                                     _ptr(scratch), scratch.numel(), _stream(dev)))
        return (None,) * 8 + (d_c2w, d_intr, d_expo, d_w2) + _field_grads(rf, bufs)


class LocalTensorfs(torch.nn.Module):
    """Self-calibrating sequence of local radiance fields."""

    def __init__(self, fov, n_init_frames, n_overlap, WH, n_iters_per_frame, n_iters_reg,
                 lr_R_init, lr_t_init, lr_i_init, lr_exposure_init, rf_lr_init, rf_lr_basis,
                 lr_decay_target_ratio, N_voxel_list, update_AlphaMask_list, camera_prior, device,
                 lr_upsample_reset, **tensorf_args):
        super().__init__()
        # hyper-parameters, under the attribute names the reference's callers read
        # (local_tensorfs.py:61-82); the *_per_frame_* copies feed the per-field schedule rescaling
        self.W, self.H = WH
        for name, value in dict(
                fov=fov, n_init_frames=n_init_frames, n_overlap=n_overlap,
                n_iters_per_frame=n_iters_per_frame, n_iters_reg_per_frame=n_iters_reg,
                lr_R_init=lr_R_init, lr_t_init=lr_t_init, lr_i_init=lr_i_init,
                lr_exposure_init=lr_exposure_init, rf_lr_init=rf_lr_init, rf_lr_basis=rf_lr_basis,
                lr_decay_target_ratio=lr_decay_target_ratio, N_voxel_per_frame_list=N_voxel_list,
                update_AlphaMask_per_frame_list=update_AlphaMask_list, camera_prior=camera_prior,
                tensorf_args=tensorf_args, lr_upsample_reset=lr_upsample_reset,
                device=torch.device(device)).items():
            setattr(self, name, value)
        # schedule state of the field being optimised (rescaled in optimizer_step at iteration 1)
        self.is_refining, self.regularize, self.lr_factor = False, True, 1
        self.n_iters, self.n_iters_reg = n_iters_per_frame, n_iters_reg
        self.N_voxel_list, self.update_AlphaMask_list = N_voxel_list, update_AlphaMask_list

        # per-frame pose / exposure parameters, one optimiser each (local_tensorfs.py:85-92)
        self.r_c2w = torch.nn.ParameterList()
        self.t_c2w = torch.nn.ParameterList()
        self.exposure = torch.nn.ParameterList()
        self.r_optimizers, self.t_optimizers, self.exp_optimizers = [], [], []
        self.pose_linked_rf = []
        self.blending_weights = torch.nn.Parameter(
            torch.ones([1, 1], device=self.device), requires_grad=False)
        for _ in range(n_init_frames):
            self.append_frame()

        if self.camera_prior is not None:
            focal = self.camera_prior["transforms"]["fl_x"] * self.W / self.camera_prior["transforms"]["w"]
        else:
            focal = self.W / math.tan(fov * math.pi / 180 / 2) / 2
        self.init_focal = torch.nn.Parameter(torch.Tensor([focal]).to(self.device))
        self.focal_offset = torch.nn.Parameter(torch.ones(1, device=device))
        self.center_rel = torch.nn.Parameter(0.5 * torch.ones(2, device=device))
        if lr_i_init > 0:
            self.intrinsic_optimizer = torch.optim.Adam(
                [self.focal_offset, self.center_rel], betas=(0.9, 0.99), lr=self.lr_i_init)

        # radiance fields
        self.dp_group = None      # set to a process group (or True = WORLD) for data-parallel training
        self.tensorfs = torch.nn.ParameterList()
        self.rf_iter = []
        self.world2rf = torch.nn.ParameterList()
        self.append_rf()

    # ---------------------------------------------------------------------------------------------
    # progressive-schedule bookkeeping (host side; local_tensorfs.py:116-290)
    # ---------------------------------------------------------------------------------------------
    def append_rf(self, n_added_frames=1):
        """Opens a new field centred at the latest camera and cross-fades the blending rows of the
        last `n_overlap` frames from the previous field to the new one (:116-146)."""
        self.is_refining = False
        if len(self.tensorfs) > 0:
            n_ov = min(n_added_frames, self.n_overlap, self.blending_weights.shape[0] - 1)
            ramp = 1 / n_ov + torch.arange(0, 1, 1 / n_ov)
            bw = self.blending_weights.detach().clone()
            bw[-n_ov:, -1] = (1 - ramp).to(bw)
            new_col = torch.zeros_like(bw[:, :1])
            new_col[-n_ov:, 0] = ramp.to(bw)
            self.blending_weights = torch.nn.Parameter(torch.cat([bw, new_col], dim=1),
                                                       requires_grad=False)
            world2rf = -self.t_c2w[-1].clone().detach()
            # (the reference parks the previous field on the CPU here; it stays resident)
        else:
            world2rf = torch.zeros(3, device=self.device)
        self.tensorfs.append(TensorVMSplit(device=self.device, **self.tensorf_args))
        if self.__dict__.get("grid_storage", "fp32") != "fp32":
            self.tensorfs[-1].set_grid_storage(self.grid_storage)
        self.world2rf.append(world2rf.clone().detach())
        self.rf_iter.append(0)
        groups = self.tensorfs[-1].get_optparam_groups(self.rf_lr_init, self.rf_lr_basis)
        self.rf_optimizer = torch.optim.Adam(groups, betas=(0.9, 0.99))

    def set_grid_storage(self, kind="fp32"):
        """Inference storage type of every field's grids (TensorBase.set_grid_storage): "fp32" or "bf16"
        (eval renders gather bfloat16 copies: half the bytes per texel; training is unaffected).  Fields
        appended later inherit the setting."""
        for rf in self.tensorfs:
            rf.set_grid_storage(kind)
        self.__dict__["grid_storage"] = kind
        return self

    def append_frame(self):
        """Adds one frame's pose / exposure parameters, initialised from the previous frame
        (:148-177)."""
        if len(self.r_c2w) == 0:
            self.r_c2w.append(torch.eye(3, 2, device=self.device))
            self.t_c2w.append(torch.zeros(3, device=self.device))
            self.pose_linked_rf.append(0)
        else:
            prev_r = self.r_c2w[-1].clone().detach()[None]
            self.r_c2w.append(mtx_to_sixD(sixD_to_mtx(prev_r))[0])
            self.t_c2w.append(self.t_c2w[-1].clone().detach())
            self.blending_weights = torch.nn.Parameter(
                torch.cat([self.blending_weights, self.blending_weights[-1:, :]], dim=0),
                requires_grad=False)
            self.pose_linked_rf.append(int(torch.nonzero(self.blending_weights[-1, :])[0]))
        self.exposure.append(torch.eye(3, 3, device=self.device))

        if self.camera_prior is not None:
            idx = len(self.r_c2w) - 1
            rel_pose = self.camera_prior["rel_poses"][idx]
            last_r = sixD_to_mtx(self.r_c2w[-1].clone().detach()[None])[0]
            self.r_c2w[-1] = last_r @ rel_pose[:3, :3]
            self.t_c2w[-1].data += last_r @ rel_pose[:3, 3]

        adam = lambda p, lr: torch.optim.Adam([p], betas=(0.9, 0.99), lr=lr)
        self.r_optimizers.append(adam(self.r_c2w[-1], self.lr_R_init))
        self.t_optimizers.append(adam(self.t_c2w[-1], self.lr_t_init))
        self.exp_optimizers.append(adam(self.exposure[-1], self.lr_exposure_init))

    def _live_pose_ids(self):
        """Frames whose pose is still optimised: linked to the newest field, within its budget."""
        newest = len(self.rf_iter) - 1
        if self.rf_iter[-1] >= self.n_iters:
            return []
        return [i for i, rf in enumerate(self.pose_linked_rf) if rf == newest]

    def optimizer_step_poses_only(self, loss):
        live = self._live_pose_ids()
        stepped = [o for i in live for o in (self.r_optimizers[i], self.t_optimizers[i])]
        zero_grad(stepped)
        loss.backward()
        adam_step(stepped)

    def optimizer_step(self, loss, optimize_poses):
        """One optimisation step + the schedule events it triggers (:193-290)."""
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

        stepped = [self.rf_optimizer]                       # every optimiser this step updates
        for i in self._live_pose_ids():
            if optimize_poses:
                decay(self.r_optimizers[i]); decay(self.t_optimizers[i])
                stepped += [self.r_optimizers[i], self.t_optimizers[i]]
            if self.lr_exposure_init > 0:
                decay(self.exp_optimizers[i])
                stepped.append(self.exp_optimizers[i])
        if self.lr_i_init > 0 and self.blending_weights.shape[1] == 1 and self.is_refining:
            decay(self.intrinsic_optimizer)
            stepped.append(self.intrinsic_optimizer)
        zero_grad(stepped)

        loss.backward()
        if getattr(self, "dp_group", None) is not None:     # data-parallel training: average the step's
            from .dist import allreduce_gradients            # gradients over the ranks before any update
            allreduce_gradients(self, None if self.dp_group is True else self.dp_group)

        # One launch updates the field, the live frames' poses and exposures and the intrinsics.  The reference
        # steps the pose, exposure and intrinsics optimisers after the upsample / alpha-mask events below; doing
        # it here gives the same result, because those events read only the field's tensors.
        adam_step(stepped)
        if self.is_refining:
            decay(self.rf_optimizer)

        if self.rf_iter[-1] in self.N_voxel_list:          # raise the grid resolution
            reso = N_to_reso(self.N_voxel_list[self.rf_iter[-1]], self.tensorfs[-1].aabb)
            self.tensorfs[-1].upsample_volume_grid(reso)
            if self.lr_upsample_reset:
                print("reset lr to initial")
                groups = self.tensorfs[-1].get_optparam_groups(self.rf_lr_init, self.rf_lr_basis)
                self.rf_optimizer = torch.optim.Adam(groups, betas=(0.9, 0.99))
        if self.rf_iter[-1] in self.update_AlphaMask_list:  # rebuild the occupancy mask
            self.tensorfs[-1].updateAlphaMask(tuple((self.tensorfs[-1].gridSize / 2).int()))

        if self.is_refining:
            self.rf_iter[-1] += 1
        return self.rf_iter[-1] >= self.n_iters - 1       # can_add_rf

    # ---------------------------------------------------------------------------------------------
    def get_cam2world(self, view_ids=None, starting_id=0):
        """[V,3,4] camera-to-world matrices from the 6-D rotations and translations (:292-299)."""
        if view_ids is not None:
            ids = view_ids.tolist() if torch.is_tensor(view_ids) else list(view_ids)
            r = torch.stack([self.r_c2w[i] for i in ids], dim=0)
            t = torch.stack([self.t_c2w[i] for i in ids], dim=0)
        else:
            r = torch.stack(list(self.r_c2w[starting_id:]), dim=0)
            t = torch.stack(list(self.t_c2w[starting_id:]), dim=0)
        return torch.cat([sixD_to_mtx(r), t[..., None]], dim=-1)

    _CKPT_FIELDS = ("fov", "n_init_frames", "n_overlap", "n_iters_per_frame", "lr_R_init", "lr_t_init",
                    "lr_i_init", "lr_exposure_init", "rf_lr_init", "rf_lr_basis",
                    "lr_decay_target_ratio", "lr_upsample_reset")

    def get_kwargs(self):
        """Constructor kwargs stored next to the state_dict in a checkpoint (:301-324)."""
        kwargs = {name: getattr(self, name) for name in self._CKPT_FIELDS}
        kwargs.update(camera_prior=None, WH=(self.W, self.H), n_iters_reg=self.n_iters_reg_per_frame,
                      N_voxel_list=self.N_voxel_per_frame_list,
                      update_AlphaMask_list=self.update_AlphaMask_per_frame_list)
        kwargs.update(self.tensorfs[0].get_kwargs())
        return kwargs

    def save(self, path):
        torch.save({"kwargs": self.get_kwargs(), "state_dict": self.state_dict()}, path)

    def load(self, state_dict):
        """Rebuilds the frame / field structure from the key names, then loads (:331-356)."""
        n_frames = 0
        for key in state_dict:
            if re.fullmatch(r"r_c2w.[0-9]*", key):
                n_frames += 1
            if re.fullmatch(r"tensorfs.[1-9][0-9]*.density_plane.0", key):
                plane0 = state_dict[key]
                line0 = state_dict[key[: -len("density_plane.0")] + "density_line.0"]
                # plane 0 is [1,C,G_y,G_x], line 0 is [1,C,G_z,1].  (The reference reads x and y
                # swapped here, which only works for G_x == G_y; the intended order is used.)
                self.tensorf_args["gridSize"] = [plane0.shape[3], plane0.shape[2], line0.shape[2]]
                self.append_rf()
        for i, rf in enumerate(self.tensorfs):
            if f"tensorfs.{i}.alphaMask.aabb" in state_dict:
                vol = state_dict[f"tensorfs.{i}.alphaMask.alpha_volume"].to(self.device)
                aabb = state_dict[f"tensorfs.{i}.alphaMask.aabb"].to(self.device)
                rf.alphaMask = AlphaGridMask(self.device, aabb, vol)
        for _ in range(n_frames - len(self.r_c2w)):
            self.append_frame()
        self.blending_weights = torch.nn.Parameter(
            torch.ones_like(state_dict["blending_weights"]), requires_grad=False)
        self.load_state_dict(state_dict)

    def get_dist_to_last_rf(self):
        return torch.norm(self.t_c2w[-1] + self.world2rf[-1])

    def get_reg_loss(self, tvreg, TV_weight_density, TV_weight_app, L1_weight_inital):
        tv_loss, l1_loss = 0, 0
        if self.rf_iter[-1] < self.n_iters:
            anneal = self.lr_factor ** self.rf_iter[-1]
            if TV_weight_density > 0:
                tv_loss += self.tensorfs[-1].TV_loss_density(tvreg).mean() * (TV_weight_density * anneal)
            if TV_weight_app > 0:
                tv_loss += self.tensorfs[-1].TV_loss_app(tvreg).mean() * (TV_weight_app * anneal)
            if L1_weight_inital > 0:
                l1_loss += self.tensorfs[-1].density_L1() * L1_weight_inital
        return tv_loss, l1_loss

    def focal(self, W):
        return self.init_focal * self.focal_offset * W / self.W

    def center(self, W, H):
        return torch.Tensor([W, H]).to(self.center_rel) * self.center_rel

    # ---------------------------------------------------------------------------------------------
    # the hot path (local_tensorfs.py:382-499)
    # ---------------------------------------------------------------------------------------------
    def _intrinsics(self, W, H):
        """[focal(W), cx, cy]: center(W, H) as the same fp32 products, without its host-to-device copy."""
        return torch.cat([self.focal(W).reshape(1), self.center_rel[0:1] * W, self.center_rel[1:2] * H])

    def _exposure_for(self, ids, test_id, dev):
        """Per-view 3x3 exposure [V,3,3], fp32 on `dev`, of the host list of view ids: the stacked parameters (with
        their graph); held-out frames (`test_id`) average their neighbours, detached, with the reference's edge rules
        (:481-493)."""
        if not test_id:
            return torch.stack([self.exposure[i] for i in ids]).to(dev, torch.float32)
        n = len(self.exposure)
        mats = []
        for v in ids:
            lo = max(v - 1, 0)
            if lo == v:
                lo = 1
            hi = min(v + 1, n - 1)
            if lo == v:                     # the reference re-tests the rewritten lower index
                hi = n - 2
            mats.append((self.exposure[lo].detach() + self.exposure[hi].detach()) / 2)
        return torch.stack(mats).to(dev, torch.float32)

    def _forward_autograd(self, ray_ids, view_ids, ids, W, H, white_bg, is_train, cam2world,
                          world2rf, blend, active, chunk, test_id, floater_thresh):
        """Composed path (local_tensorfs.py:397-499 with torch ops around the CUDA lookups): rays are
        generated with torch ops so gradients reach poses and intrinsics, each active field renders
        through TensorBase.forward (composed when autograd records or the field uses positional
        encodings), blend / exposure / clamp are torch ops.  Chunked like the reference, because
        this path materialises per-sample tensors."""
        from .ray_utils import get_ray_directions_360, get_ray_directions_lean, get_rays_lean
        dev = ray_ids.device
        n, n_views = ray_ids.shape[0], len(ids)
        i, j = ids2pixel(W, H, ray_ids)
        ij = torch.stack([i, j], dim=-1)
        if self.fov == 360:
            directions = get_ray_directions_360(i, j, W, H)
        else:
            directions = get_ray_directions_lean(i, j, self.focal(W), self.center(W, H))
        if cam2world is None:
            cam2world = self.get_cam2world(ids)
        per_view = n // n_views
        outs_rgb, outs_depth = [], []
        for lo, hi, _, _ in _chunks(n, n_views, max(chunk // len(active), 1)):
            rgb_c = torch.zeros(hi - lo, 3, device=dev)
            depth_c = torch.zeros(hi - lo, device=dev)
            for k in active:
                cam2rf = cam2world.clone()
                cam2rf[:, :3, 3] = cam2rf[:, :3, 3] + world2rf[k]
                cam2rf = cam2rf.repeat_interleave(per_view, dim=0)[lo:hi]
                rays_o, rays_d = get_rays_lean(directions[lo:hi], cam2rf)
                rgb_k, depth_k = self.tensorfs[k](torch.cat([rays_o, rays_d], -1), is_train=is_train,
                                                  white_bg=white_bg, N_samples=-1,
                                                  refine=self.is_refining,
                                                  floater_thresh=floater_thresh)
                if blend is None:
                    w = 1.0
                    rgb_c, depth_c = rgb_c + rgb_k, depth_c + depth_k
                else:
                    w = blend.repeat_interleave(per_view, dim=0)[lo:hi, k]
                    rgb_c, depth_c = rgb_c + rgb_k * w[..., None], depth_c + depth_k * w
            outs_rgb.append(rgb_c); outs_depth.append(depth_c)
        rgbs = torch.cat(outs_rgb); depth_maps = torch.cat(outs_depth)
        if self.lr_exposure_init > 0:
            exposure = self._exposure_for(ids, test_id, dev).repeat_interleave(per_view, dim=0)
            rgbs = torch.bmm(exposure, rgbs[..., None])[..., 0]
        return rgbs.clamp(0, 1), depth_maps, directions, ij

    def _forward_train(self, ray_ids, ids, W, H, white_bg, cam2world, world2rf, k, chunk, test_id):
        """The training call under autograd for a field _RenderFn covers: one _TrainRenderFn node per chunk (each
        with its own distance-table draw, then its background coin, in the composed path's RNG order)."""
        dev = ray_ids.device
        rf = self.tensorfs[k]
        sources = [self.init_focal, self.focal_offset, self.center_rel]
        if cam2world is None:
            cam2world = self.get_cam2world(ids)
            sources += [self.r_c2w[i] for i in ids] + [self.t_c2w[i] for i in ids]
        intr = self._intrinsics(W, H)
        exposure = None
        if self.lr_exposure_init > 0:
            exposure = self._exposure_for(ids, test_id, dev)
            sources += list(self.exposure) if test_id else [self.exposure[v] for v in ids]
        w2 = world2rf[k]
        sources.append(w2)
        rays_i, _ = _ray_ids(ray_ids)
        params = rf._grad_params()
        outs = []
        for lo, hi, v_lo, v_hi in _chunks(ray_ids.shape[0], len(ids), chunk):
            z = rf.sample_table(True, -1, dev)
            bg = bool(white_bg) or bool(torch.rand((1,)) < 0.5)     # tensorBase.py:633, after the table's jitter
            outs.append(_TrainRenderFn.apply(rf, z, bg, rays_i[lo:hi], W, H, self.fov == 360, sources,
                                             cam2world[v_lo:v_hi], intr,
                                             None if exposure is None else exposure[v_lo:v_hi], w2, *params))
        if len(outs) == 1:
            return outs[0]
        return tuple(torch.cat([o[i] for o in outs]) for i in range(4))

    def _train_node_covers(self, k, floater_thresh):
        """Whether a training call of field k runs as one _TrainRenderFn node: the fields _RenderFn covers
        (pe = 0, no floater filter) unless LRF_TRAIN_PATH=composed selects the torch-op path."""
        rf = self.tensorfs[k]
        return (rf.fused_supported() and rf.fea_pe == 0 and rf.view_pe == 0 and floater_thresh == 0
                and os.environ.get("LRF_TRAIN_PATH", "fused") != "composed")

    def _blend_host(self):
        bw = self.blending_weights
        return _memo(self, "bw_host", _key((bw,)), lambda _: bw.detach().cpu(), (bw,))

    def forward(self, ray_ids, view_ids, W, H, white_bg=True, is_train=True, cam2world=None,
                world2rf=None, blending_weights=None, chunk=16384, test_id=False,
                floater_thresh=0, stats=None, exchange=None, out=None):
        """-> (rgbs [N,3], depth_maps [N], directions [N,3], ij [N,2]) like the reference.

        Extensions (all optional, defaults = the reference's behaviour):
        `ray_ids` may be a PINNED host tensor: the kernel reads the ids over PCIe itself (no staging
        copy).  `out=(rgb [N,3], depth [N])` preallocated float32 outputs, on the device or in pinned
        host memory -- in the latter case finished pixels are stored straight into host memory by the
        kernel and only a stream synchronisation is left to the caller.
        `exchange=(PixelExchange, ray_lo)` (multi-GPU eval, dist.render_sharded): the kernel also
        stores every finished pixel into all peers' gathered buffers at row ray_lo + r and the step
        barrier is enqueued after the last launch; rgbs / depth_maps are then views of an interleaved
        [N,4] buffer."""
        if ray_ids.is_cuda:
            dev = ray_ids.device
        else:
            _uva_pointer(ray_ids)                       # raises unless pinned
            dev = self.blending_weights.device
            if dev.type != "cuda":
                raise RuntimeError("localrf_b200: the scene model is on the CPU; the render path runs "
                                   "only on a CUDA device (there is no CPU fallback)")
        n = ray_ids.shape[0]
        if n == 0:                                        # an empty batch / shard: nothing to launch
            if exchange is not None:
                exchange[0].skip_step(_stream(dev))       # ... but the peers still need this rank's step flag
            return (torch.empty(0, 3, device=dev), torch.empty(0, device=dev), torch.empty(0, 3, device=dev),
                    torch.empty(0, 2, dtype=torch.int64, device=dev))
        key = plan = None
        if not is_train and not torch.is_grad_enabled():
            # eval: the plan of an identical earlier call serves this one while its guards hold
            vkey = (id(view_ids), view_ids._version) if torch.is_tensor(view_ids) else tuple(view_ids)
            key = (vkey, n, W, H, bool(white_bg), bool(test_id), float(floater_thresh),
                   None if cam2world is None else (id(cam2world), cam2world._version),
                   None if world2rf is None else id(world2rf),
                   None if blending_weights is None else (id(blending_weights), blending_weights._version),
                   id(self.blending_weights), len(self.tensorfs), exchange is not None, bool(self.is_refining), dev)
            plan = self.__dict__.setdefault("_plans", {}).get(key)
            if plan is not None and not plan.valid():
                plan = None
        if plan is None:
            # (not memoised: a new tensor can reuse a freed tensor's id and storage)
            ids = view_ids.tolist() if torch.is_tensor(view_ids) else [int(v) for v in view_ids]
            n_views = len(ids)
            if n_views == 0 or n % n_views != 0:
                raise ValueError("ray_ids must hold the same number of rays for every view")
            n_fields = len(self.tensorfs)

            # -- which fields render, with which per-view weights (:403-418) ------------------------
            blend = None                                   # device [V, n_fields] or None (= weight 1)
            if is_train:                                   # one field trains at a time (:411-416)
                active = [n_fields - 1]
            elif blending_weights is None:
                rows = self._blend_host()[ids]
                active = torch.nonzero(rows.sum(dim=0))[:, 0].tolist()
                bw = self.blending_weights
                blend = bw.detach()[ids[0]:ids[0] + 1] if n_views == 1 else bw.detach()[view_ids]
                blend = blend.to(dev, torch.float32).contiguous()
            else:
                blend = blending_weights.detach().to(dev, torch.float32).contiguous()
                active = torch.nonzero(blend.sum(dim=0))[:, 0].tolist()
            if len(active) == 0:
                if exchange is not None:
                    # (before anything is enqueued: the exchange's step count does not advance; ranks sharding
                    # one view hold the same blending row, so they all raise at this step)
                    raise NotImplementedError("exchange= needs a field that renders the batch's views")
                print("****** No valid RF")
                i, j = ids2pixel(W, H, ray_ids)
                ones = torch.ones_like(ray_ids).float()
                if out is None:
                    return torch.ones([n, 3], device=dev), ones, torch.zeros(n, 3, device=dev), torch.stack([i, j], -1)
                rgbs, depth = self._alloc_outputs(n, dev, None, out)[1:3]
                with torch.cuda.device(dev):            # in stream order, like the kernel's stores (out may be pinned)
                    rgbs.copy_(torch.ones(n, 3, device=dev), non_blocking=True)
                    depth.copy_(torch.ones(n, device=dev), non_blocking=True)
                return rgbs, depth, torch.zeros(n, 3, device=dev), torch.stack([i, j], -1)

            if world2rf is None:
                world2rf = self.world2rf
            if torch.is_grad_enabled():
                tracked = [self.init_focal, self.focal_offset, self.center_rel]
                tracked += [cam2world] if cam2world is not None else \
                    [self.r_c2w[i] for i in ids] + [self.t_c2w[i] for i in ids]
                tracked += [self.exposure[i] for i in ids] if self.lr_exposure_init > 0 else []
                for k in active:
                    tracked += list(self.tensorfs[k].parameters())
                needs_composed = any(t is not None and t.requires_grad for t in tracked)
            else:
                needs_composed = False
            if needs_composed or not all(self.tensorfs[k].fused_supported() for k in active):
                if exchange is not None or out is not None:
                    raise NotImplementedError("exchange= / out= are served by the fused eval path only")
                if not ray_ids.is_cuda:
                    ray_ids = ray_ids.to(dev)
                if needs_composed and is_train and self._train_node_covers(active[0], floater_thresh):
                    return self._forward_train(ray_ids, ids, W, H, white_bg, cam2world, world2rf, active[0], chunk,
                                               test_id)
                return self._forward_autograd(ray_ids, view_ids, ids, W, H, white_bg, is_train,
                                              cam2world, world2rf, blend, active, chunk, test_id,
                                              floater_thresh)
            if exchange is not None and is_train:
                raise ValueError("the fused pixel exchange serves eval batches (is_train=False)")

        rays_i, ids_ptr = _ray_ids(ray_ids)               # (rays_i holds the ids until the launches are enqueued)
        outs = self._alloc_outputs(n, dev, exchange, out)
        if plan is None:
            plan = self._resolve(ids, n, W, H, white_bg, is_train, cam2world, world2rf, blending_weights, blend,
                                 active, chunk, test_id, floater_thresh, dev)
            if key is not None:
                # the key holds ids of caller objects: keep them alive so the ids cannot be recycled
                plan.key_refs = (view_ids, cam2world, world2rf, blending_weights)
                plans = self.__dict__["_plans"]
                if len(plans) >= 256:
                    plans.clear()
                plans[key] = plan
        return self._run(plan, ids_ptr, outs, stats, exchange)

    def _alloc_outputs(self, n, dev, exchange, out):
        """(pix or None, rgbs, depth, directions, ij) -- fresh tensors owned by the caller."""
        pix = None
        if exchange is not None:
            pix = torch.empty(n, 4, dtype=torch.float32, device=dev)
            rgbs, depth = pix[:, :3], pix[:, 3]
        elif out is not None:
            rgbs, depth = out
            for t, shape in ((rgbs, (n, 3)), (depth, (n,))):
                if t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous():
                    raise ValueError("out=(rgb [N,3], depth [N]) must be contiguous float32 tensors")
                _uva_pointer(t)
        else:
            rgbs = torch.empty(n, 3, dtype=torch.float32, device=dev)
            depth = torch.empty(n, dtype=torch.float32, device=dev)
        directions = torch.empty(n, 3, dtype=torch.float32, device=dev)
        ij = torch.empty(n, 2, dtype=torch.int64, device=dev)
        return pix, rgbs, depth, directions, ij

    def _resolve(self, ids, n, W, H, white_bg, is_train, cam2world, world2rf, blending_weights, blend, active,
                 chunk, test_id, floater_thresh, dev):
        """The _LaunchPlan of a fused call: the device copies of the cameras, intrinsics and exposure (memoised on
        parameter versions), then per chunk and active field its distance table, background coin and LrfBatch.  Train
        mode draws fresh jitter per chunk like the reference, in the composed path's RNG order; eval has no
        randomness, so the whole batch is one launch per field."""
        guards = []
        P = self._parameters
        if blending_weights is None and not is_train:
            guards.append((P, "blending_weights", self.blending_weights, self.blending_weights._version))
        if cam2world is None:
            src = [self.r_c2w[i] for i in ids] + [self.t_c2w[i] for i in ids]
            cam2world = _memo(self, "c2w", (tuple(ids), _key(src), str(dev)),
                              lambda _: self.get_cam2world(ids).detach().to(dev, torch.float32).contiguous(), src)
            for i in set(ids):     # (guards index the lists' _parameters dicts: ~10x cheaper than __getitem__)
                guards.append((self.r_c2w._parameters, str(i), self.r_c2w[i], self.r_c2w[i]._version))
                guards.append((self.t_c2w._parameters, str(i), self.t_c2w[i], self.t_c2w[i]._version))
        else:
            cam2world = cam2world.detach().to(dev, torch.float32).contiguous()
        src = [self.init_focal, self.focal_offset, self.center_rel]
        intr = _memo(self, "intr", (W, H, self.W, _key(src), str(dev)),
                     lambda _: self._intrinsics(W, H).detach().to(dev, torch.float32).contiguous(), src)
        for name in ("init_focal", "focal_offset", "center_rel"):
            guards.append((P, name, P[name], P[name]._version))
        exposure = None
        if self.lr_exposure_init > 0:
            n_e = len(self.exposure)
            used = sorted(set(ids + ([max(v - 1, 0) for v in ids] + [min(v + 1, n_e - 1) for v in ids]
                                     + [min(1, n_e - 1), max(n_e - 2, 0)] if test_id else [])))
            src = [self.exposure[i] for i in used]
            exposure = _memo(self, "expo", (tuple(ids), bool(test_id), n_e, _key(src), str(dev)),
                             lambda _: self._exposure_for(ids, test_id, dev).detach(), src)
            for i, t in zip(used, src):
                guards.append((self.exposure._parameters, str(i), t, t._version))

        plan = _LaunchPlan()
        plan.guards, plan.launches, plan.dev, plan.key_refs = guards, [], dev, None
        plan.keep = [cam2world, intr, exposure, blend]
        fov360 = self.fov == 360
        for lo, hi, v_lo, v_hi in _chunks(n, len(ids), max(chunk // len(active), 1) if is_train else n):
            for pos, k in enumerate(active):
                rf = self.tensorfs[k]
                if rf.basis_mat.weight.device != dev:
                    rf.to(dev)
                z = rf.sample_table(is_train, -1, dev)
                w2 = world2rf[k]
                w2rf = w2.detach() if (w2.device == dev and w2.dtype == torch.float32 and w2.is_contiguous()) else \
                    w2.detach().to(dev, torch.float32).contiguous()
                last = pos == len(active) - 1
                b = _ray_batch(None, hi - lo, W, H, fov360, intr, cam2world, w2rf, v_lo, v_hi, exposure, blend, k,
                               accumulate=int(pos > 0), finalize=int(last),
                               white_bg=int(bool(white_bg) or bool(is_train and torch.rand((1,)) < 0.5)),
                               floater_thresh=float(floater_thresh),
                               refine=int(bool(self.is_refining)))        # local_tensorfs.py:463
                plan.launches.append((rf, z, b, lo, last))
                plan.keep.append(w2rf)
                guards.append((self.tensorfs._modules, str(k), rf, None))
                if isinstance(world2rf, torch.nn.ParameterList):
                    guards.append((world2rf._parameters, str(k), w2, w2._version))
                else:
                    guards.append((world2rf, k, w2, w2._version))
                guards.append((rf.__dict__, "nSamples", rf.nSamples, "eq"))
        return plan

    def _run(self, plan, ids_ptr, outs, stats, exchange):
        """Enqueues the plan's launches on the ids at `ids_ptr` into `outs` (_alloc_outputs).  With an exchange the
        last launch of a chunk also stores every finished pixel into the peers' buffers (exchange calls are eval
        calls: one chunk)."""
        pix, rgbs, depth, directions, ij = outs
        o = _lib.LrfOutputs()
        if stats is not None:
            o.stats = stats.data_ptr()
        if pix is not None:
            p_pix = pix.data_ptr()
        else:
            p_rgb, p_depth = rgbs.data_ptr(), depth.data_ptr()
        p_dirs, p_ij = directions.data_ptr(), ij.data_ptr()
        lib = _lib.lib()
        with torch.cuda.device(plan.dev):
            stream = _stream(plan.dev)
            for rf, z, b, lo, last in plan.launches:
                fs, prep = rf.field_and_prepared(z)
                b.ray_ids = ids_ptr + 8 * lo
                if pix is not None:
                    o.pix = p_pix + 16 * lo
                    if last:
                        exchange[0].fill_outputs(o, exchange[1] + lo)
                else:
                    o.rgb, o.depth = p_rgb + 12 * lo, p_depth + 4 * lo
                o.directions, o.ij = p_dirs + 12 * lo, p_ij + 16 * lo
                _lib.check(lib.lrf_render(C.byref(fs), _ptr(prep), C.byref(b), C.byref(o), stream))
            if exchange is not None:
                exchange[0].close_step(stream)
        return rgbs, depth, directions, ij

    def _eval_plan(self, view, n, W, H, test_id, dev):
        """The (uncached) plan of an eval forward of `n` rays of one view, with forward's defaults (white background,
        floater_thresh = 0), or None when no field renders the view."""
        active = torch.nonzero(self._blend_host()[view])[:, 0].tolist()
        if not active:
            return None
        blend = self.blending_weights.detach()[view:view + 1].to(dev, torch.float32).contiguous()
        return self._resolve([view], n, W, H, True, False, None, self.world2rf, None, blend, active, n, test_id, 0, dev)

    def _run_weights(self, plan, ids_ptr, outs, weights, acc):
        """_run for a one-chunk eval plan without exchange, where every launch also writes its per-sample weights into
        `weights` (fp32, at least n x S of every field) and lrf_ray_opacity folds them, with the launch's blend, into
        the blended opacity `acc` [n]."""
        _, rgbs, depth, directions, ij = outs
        o = _lib.LrfOutputs(rgb=rgbs.data_ptr(), depth=depth.data_ptr(), weights=weights.data_ptr(),
                            directions=directions.data_ptr(), ij=ij.data_ptr())
        lib = _lib.lib()
        with torch.cuda.device(plan.dev):
            stream = _stream(plan.dev)
            for pos, (rf, z, b, lo, last) in enumerate(plan.launches):
                fs, prep = rf.field_and_prepared(z)
                if b.n_rays * fs.n_samples > weights.numel():
                    raise ValueError("localrf_b200: the weights buffer is smaller than n_rays x n_samples")
                b.ray_ids = ids_ptr
                _lib.check(lib.lrf_render(C.byref(fs), _ptr(prep), C.byref(b), C.byref(o), stream))
                _lib.check(lib.lrf_ray_opacity(o.weights, b.n_rays, fs.n_samples, b.n_views, b.blend, b.blend_stride,
                                               int(pos > 0), acc.data_ptr(), stream))
        return rgbs, depth, directions, ij
