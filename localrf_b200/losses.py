"""Supervision losses of a training step on the device: the block train.py:369-423 computes every iteration.

    rgb, flow, depth = supervision_losses(rgb_map, rgb_train, loss_weights, view_ids=..., ...)

  * rgb    mean(0.25 * |rgb_map - rgb_train| * w / mean(w))                                    (:369-371)
  * flow   the optical-flow reprojection residual (get_fwd_bwd_cam2cams, get_pred_flow, pts2px,
           utils/utils.py:15-48), zeroed per view above its 0.9 quantile, mean * flow_weight        (:385-410)
  * depth  the scale- and shift-invariant inverse-depth residual (compute_depth_loss, utils/utils.py:50-59),
           zeroed per view above its 0.8 quantile, mean * depth_weight                              (:413-423)

Two kernels forward (lrf_supervision_losses) and two backward, behind one torch.autograd.Function, where the
block as torch ops launches about 370 kernels per iteration.  Nothing here synchronises the host (the torch
block does not either: its boolean-mask assignments with a scalar value run as masked_fill_), and the results
are bitwise repeatable.  There is no CPU fallback.
"""
import ctypes as C

import torch

from . import _lib
from .tensorf import _ptr, _stream

MAX_RAYS_PER_VIEW = 4096


def _flat(t, n, width, name, dtype=torch.float32):
    """t as a contiguous [n] / [n, width] tensor of `dtype` (any view-major shape with n * width elements)."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if t.numel() != n * width:
        raise ValueError(f"{name} has {t.numel()} elements, expected {n} x {width}")
    return t.reshape((n, width) if width > 1 else (n,)).contiguous()


def _scalar_param(t, numel, name, dev):
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(t, dtype=torch.float32).to(dev)
    if t.dtype != torch.float32 or t.numel() != numel:
        raise ValueError(f"{name} must be a float32 tensor of {numel} element(s)")
    return t


class _Config:
    """The non-differentiable inputs and the filled LrfLossBatch of one call (keeps every tensor alive)."""

    def __init__(self, batch, keep, dev):
        self.batch, self.keep, self.dev = batch, keep, dev


class _SupervisionLosses(torch.autograd.Function):
    """Every tensor the kernels read -- the differentiable inputs, the data in cfg.keep and the scratch holding the
    forward's decisions -- is saved for backward, so an in-place change between forward and backward raises
    instead of giving wrong gradients."""

    @staticmethod
    def forward(ctx, cfg, rgb_map, depth_map, directions, cam2world, focal, center):
        b = cfg.batch
        for name, t in (("rgb_map", rgb_map), ("depth_map", depth_map), ("directions", directions),
                        ("cam2world", cam2world), ("focal", focal), ("center", center)):
            setattr(b, name, _ptr(t).value if t is not None else None)
        L = _lib.lib()
        nbytes = int(L.lrf_supervision_scratch_bytes(b.n_rays, b.n_views, b.n_cams))
        scratch = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=cfg.dev)
        out = torch.empty(3, dtype=torch.float32, device=cfg.dev)
        with torch.cuda.device(cfg.dev):
            _lib.check(L.lrf_supervision_losses(C.byref(b), _ptr(out), _ptr(scratch), nbytes, _stream(cfg.dev)))
        ctx.cfg, ctx.nbytes = cfg, nbytes
        ctx.save_for_backward(rgb_map, depth_map, directions, cam2world, focal, center, scratch,
                              *cfg.keep.values())
        ctx.mark_non_differentiable(scratch)
        return out, scratch

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out, _grad_scratch):
        cfg, dev = ctx.cfg, ctx.cfg.dev
        b = cfg.batch
        need = ctx.needs_input_grad[1:]
        rgb_map, depth_map, directions, cam2world, focal, center, scratch = ctx.saved_tensors[:7]
        mk = lambda t, want: torch.empty_like(t) if (want and t is not None) else None
        flow = bool(b.use_flow)
        grads = [mk(rgb_map, need[0]), mk(depth_map, need[1]), mk(directions, need[2] and flow),
                 mk(cam2world, need[3] and flow), mk(focal, need[4] and flow), mk(center, need[5] and flow)]
        g = _lib.LrfLossGrads()
        g.d_rgb, g.d_depth, g.d_directions, g.d_cam2world, g.d_focal, g.d_center = (
            _ptr(t).value if t is not None else None for t in grads)
        gl = grad_out.to(torch.float32).contiguous()
        L = _lib.lib()
        with torch.cuda.device(dev):
            _lib.check(L.lrf_supervision_losses_backward(C.byref(b), _ptr(gl), C.byref(g), _ptr(scratch),
                                                         ctx.nbytes, _stream(dev)))
        return (None, *grads)


def supervision_losses(rgb_map, rgb_train, loss_weights, *, view_ids=None, depth_map=None, directions=None,
                       ij=None, cam2world=None, starting_id=0, focal=None, center=None, fwd_flow=None,
                       fwd_mask=None, bwd_flow=None, bwd_mask=None, flow_weight=0.0, invdepths=None,
                       depth_weight=0.0, return_arrays=False):
    """The supervision losses of train.py:369-423 on the device -> (rgb_loss, flow_loss, depth_loss), 0-d fp32
    tensors on rgb_map's device, differentiable with respect to rgb_map, depth_map, directions, cam2world, focal
    and center.  A term whose weight is 0 is not computed and comes back as None.

    The batch is view-major, as LocalTensorfs.forward returns it: N = V x R rays, rays v*R .. v*R+R-1 from view
    v (R <= 4096).  rgb_map / rgb_train [N,3]; loss_weights [N,1] or [N]; view_ids int64 [V] (absolute frame ids);
    depth_map [N]; directions [N,3]; ij int64 [N,2] (column, row); cam2world [n_cams,3,4] =
    get_cam2world(starting_id=starting_id); focal [1] and center [2] tensors (LocalTensorfs.focal(W) / .center(W,
    H); they are read on the device); fwd_flow / bwd_flow [N,2] and fwd_mask / bwd_mask [N] (or their [V,R,...]
    shapes); invdepths [N].  flow_weight = loss_flow_weight_inital * reg_loss_weight / ((W + H) / 2) and
    depth_weight = loss_depth_weight_inital * reg_loss_weight, folded by the caller.

    Reproduced as the reference computes them: the forward mask is zeroed for every view whose ABSOLUTE id equals
    len(cam2world) - 1; the first camera's backward flow uses the clamped (identity) cam2cam; the medians are
    torch.median's lower medians; the cuts are `> torch.quantile(...)`, bit for bit.  A view whose camera id
    view_ids[v] - starting_id is outside [0, len(cam2world)) makes the flow loss NaN (the ids are not read on the
    host, which would synchronise).  R = 1 makes the depth loss NaN, as in the reference.

    return_arrays=True adds a dict: the pre-cut residuals "flow" / "depth" [V,R], the thresholds "flow_tau" /
    "depth_tau" [V] and "depth_median_index" int32 [V,2] (ray index within the view of the x and g medians)."""
    if not isinstance(rgb_map, torch.Tensor) or not rgb_map.is_cuda:
        raise RuntimeError("localrf_b200.supervision_losses runs on a CUDA device (there is no CPU fallback)")
    dev = rgb_map.device
    N = rgb_map.shape[0]
    use_flow, use_depth = float(flow_weight) != 0.0, float(depth_weight) != 0.0
    if view_ids is not None:
        if not isinstance(view_ids, torch.Tensor):
            raise TypeError("view_ids must be an int64 tensor on the batch's device")
        V = int(view_ids.shape[0])
    elif use_flow or use_depth:
        raise ValueError("the flow and depth terms need view_ids")
    else:                                        # rgb only: any split into views of <= 4096 rays
        V = next(v for v in range(max(1, -(-N // MAX_RAYS_PER_VIEW)), N + 1) if N % v == 0)
    if V < 1 or N % V:
        raise ValueError(f"{N} rays do not split into {V} views of equal size")

    tensors = {}
    rgb_map = _flat(rgb_map, N, 3, "rgb_map")
    tensors["rgb_train"] = _flat(rgb_train, N, 3, "rgb_train")
    tensors["loss_weights"] = _flat(loss_weights, N, 1, "loss_weights")
    n_cams = 1
    if use_flow or use_depth:
        if depth_map is None:
            raise ValueError("the flow and depth terms need depth_map")
        depth_map = _flat(depth_map, N, 1, "depth_map")
    else:
        depth_map = None
    if use_flow:
        for name, t in (("directions", directions), ("ij", ij), ("cam2world", cam2world), ("focal", focal),
                        ("center", center), ("fwd_flow", fwd_flow), ("fwd_mask", fwd_mask),
                        ("bwd_flow", bwd_flow), ("bwd_mask", bwd_mask)):
            if t is None:
                raise ValueError(f"the flow term needs {name}")
        if view_ids.dtype != torch.int64:
            raise TypeError("view_ids must be int64")
        tensors["view_ids"] = view_ids.contiguous()
        directions = _flat(directions, N, 3, "directions")
        tensors["ij"] = _flat(ij, N, 2, "ij", torch.int64)
        if cam2world.dim() != 3 or tuple(cam2world.shape[1:]) != (3, 4) or cam2world.dtype != torch.float32:
            raise ValueError("cam2world must be float32 [n_cams,3,4]")
        n_cams = int(cam2world.shape[0])
        if n_cams < 1:
            raise ValueError("cam2world is empty")
        cam2world = cam2world.contiguous()
        focal = _scalar_param(focal, 1, "focal", dev).reshape(1).contiguous()
        center = _scalar_param(center, 2, "center", dev).reshape(2).contiguous()
        for name, t, w in (("fwd_flow", fwd_flow, 2), ("bwd_flow", bwd_flow, 2), ("fwd_mask", fwd_mask, 1),
                           ("bwd_mask", bwd_mask, 1)):
            tensors[name] = _flat(t, N, w, name)
    else:
        directions = cam2world = focal = center = None
    if use_depth:
        if invdepths is None:
            raise ValueError("the depth term needs invdepths")
        tensors["invdepths"] = _flat(invdepths, N, 1, "invdepths")
    devs = {t.device for t in list(tensors.values()) + [x for x in (rgb_map, depth_map, directions, cam2world,
                                                                     focal, center) if x is not None]}
    if devs != {dev}:
        raise ValueError(f"all tensors must be on {dev}, got {sorted(map(str, devs))}")

    b = _lib.LrfLossBatch()
    b.n_rays, b.n_views, b.n_cams, b.starting_id = N, V, n_cams, int(starting_id)
    b.use_flow, b.use_depth = int(use_flow), int(use_depth)
    b.flow_weight, b.depth_weight = float(flow_weight), float(depth_weight)
    for name, t in tensors.items():
        setattr(b, name, _ptr(t).value)
    cfg = _Config(b, tensors, dev)
    out, scratch = _SupervisionLosses.apply(cfg, rgb_map, depth_map, directions, cam2world, focal, center)
    rgb, flow, depth = out.unbind(0)
    res = (rgb, flow if use_flow else None, depth if use_depth else None)
    if not return_arrays:
        return res
    R = N // V
    f32 = scratch[: 8 * N + 8 * V].view(torch.float32)
    arrays = {"flow": f32[:N].view(V, R), "depth": f32[N:2 * N].view(V, R), "flow_tau": f32[2 * N:2 * N + V],
              "depth_tau": f32[2 * N + V:2 * N + 2 * V],
              "depth_median_index": scratch[8 * N + 8 * V: 8 * N + 16 * V].view(torch.int32).view(V, 2)}
    return res + (arrays,)
