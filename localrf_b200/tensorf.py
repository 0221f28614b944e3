"""Host-side mirror of the reference's radiance-field modules, backed by the fused CUDA kernel.

Mirrors (same class names, constructor kwargs, attributes, `state_dict` keys and method
signatures, SURVEY.md §8b):

    AlphaGridMask             models/tensorBase.py:38-62
    MLPRender_Fea_late_view   models/tensorBase.py:97-135      (parameter container only)
    TensorBase                models/tensorBase.py:231-636
    TensorVMSplit             models/tensoRF.py:10-277

`forward`, `compute_densityfeature` and `compute_appfeature` run through the C ABI
(include/localrf_b200.h); there is no PyTorch or CPU fallback for them.  The remaining methods are
host-side bookkeeping off the per-batch path (grid upsampling, alpha-mask rebuild, regularisers,
optimiser groups) and are written with stock torch ops.

Device layout: plane/line parameters keep the reference's logical shapes
([1,C,H,W] / [1,C,L,1]) and names, but are allocated in torch.channels_last memory format, i.e.
physically [H][W][C] / [L][C] -- one texel's components are one 32-byte (density) or 96-byte
(appearance) contiguous run, which is what the kernel gathers.
"""
import ctypes as C
import operator
import os

import torch
import torch.nn.functional as F

from . import _lib

MAT_MODE = ((0, 1), (0, 2), (1, 2))   # models/tensorBase.py:274
VEC_MODE = (2, 1, 0)                  # models/tensorBase.py:275

# The field's 19 tensors in _grad_params order: (LrfField slot, index in the slot's array of three or None, module
# attribute).  TensorBase._tensors reads them in this order; the gradient of slot s is LrfGradients.d_<s>, except
# that basis and w1 share d_w1b (the kernels read their product w1 @ basis).
_FIELD_TENSORS = (
    *((slot, i, f"{attr}.{i}") for slot, attr in (("dplane", "density_plane"), ("dline", "density_line"),
                                                  ("aplane", "app_plane"), ("aline", "app_line")) for i in range(3)),
    ("basis", None, "basis_mat.weight"), ("w1", None, "renderModule.mlp.0.weight"),
    ("b1", None, "renderModule.mlp.0.bias"), ("w2", None, "renderModule.mlp.2.weight"),
    ("b2", None, "renderModule.mlp.2.bias"), ("w3", None, "renderModule.mlp_view.0.weight"),
    ("b3", None, "renderModule.mlp_view.0.bias"))

# _memo slots of a field's LrfFields, [bf16][without a distance table]
_FIELD_SLOTS = (("field", "field without table"), ("field16", "field16 without table"))

_data_ptr, _version = torch.Tensor.data_ptr, operator.attrgetter("_version")


def _key(tensors):
    """Memo key of tensors: their addresses and version counters (an in-place update bumps the counter)."""
    return tuple(map(_data_ptr, tensors)), tuple(map(_version, tensors))


def _memo(owner, slot, key, build, refs=()):
    """The object `owner` derives under `slot`: build(previous object or None) when the slot is empty or was built
    under another key.  The entry holds `refs` (the tensors the key was made from), so none of them can be freed
    and its address reused by another tensor while the entry exists."""
    memo = owner.__dict__.setdefault("_memo", {})
    hit = memo.get(slot)
    if hit is None or hit[0] != key:
        hit = memo[slot] = (key, build(None if hit is None else hit[1]), refs)
    return hit[1]


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _cl(t):
    """channels_last view/copy of a [1,C,H,W] tensor."""
    return t.contiguous(memory_format=torch.channels_last)


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(
            f"localrf_b200: {what} is on {t.device}; the render path runs only on a CUDA device "
            "(there is no CPU fallback)")


def _grid_grads(grids):
    """Zeroed gradient buffers of three planes and three lines, laid out like them (channel-last), and the two
    `void* [3]` arrays of their addresses -> (buffers, planes, lines)."""
    bufs = [torch.zeros_like(t, memory_format=torch.channels_last) for t in grids]
    return (bufs, (C.c_void_p * 3)(*[t.data_ptr() for t in bufs[:3]]),
            (C.c_void_p * 3)(*[t.data_ptr() for t in bufs[3:]]))


class _VMLookup(torch.autograd.Function):
    """Differentiable VM lookups of the training path: forward and backward are CUDA kernels behind
    the C ABI (lrf_density_feature / lrf_app_products and their *_backward); gradients reach the
    channel-last planes and lines by atomic adds and the sample coordinates by the bilinear
    derivative (zero where grid_sample's border padding clips)."""

    @staticmethod
    def forward(ctx, module, kind, xyz, *grids):
        ctx.module, ctx.kind = module, kind
        xyz = xyz.detach().reshape(-1, 3).to(torch.float32).contiguous()
        ctx.save_for_backward(xyz)
        if kind == "density":
            return module._feature_call_raw(xyz, "lrf_density_feature", 1)
        return module._feature_call_raw(xyz, "lrf_app_products", 3 * module.app_n_comp[0])

    @staticmethod
    def backward(ctx, grad_out):
        (xyz,) = ctx.saved_tensors
        m, dev = ctx.module, xyz.device
        grids = m._tensors()[0]
        d_grids, planes, lines = _grid_grads(grids[:6] if ctx.kind == "density" else grids[6:])
        d_xyz = torch.empty_like(xyz) if ctx.needs_input_grad[2] else None
        g = grad_out.detach().to(torch.float32).contiguous()
        fn = getattr(_lib.lib(), "lrf_density_feature_backward" if ctx.kind == "density"
                     else "lrf_app_products_backward")
        with torch.cuda.device(dev):
            _lib.check(fn(C.byref(m._field()), _ptr(xyz), _ptr(g), xyz.shape[0], planes, lines, _ptr(d_xyz),
                          _stream(dev)))
        return (None, None, d_xyz, *d_grids)


def _field_state(m, params):
    """What a fused backward recomputes from: the parameters' storage and versions, the grid size and the alpha
    mask.  The backward compares it with the forward's to catch in-place updates in between."""
    am = m.alphaMask
    return _key(params), tuple(m._grid_host), None if am is None else _key((am.alpha_volume,))


def _check_field_state(m, seen):
    if _field_state(m, m._grad_params()) != seen:
        raise RuntimeError("localrf_b200: a parameter (or the grid size / alpha mask) of the field was "
                           "modified between the fused forward and its backward; the backward "
                           "recomputes from the live parameters and would return gradients of a "
                           "different model")


def _field_grad_buffers(m, dev):
    """Zeroed gradient buffers laid out like the field's tensors, in _FIELD_TENSORS order with one d_w1b =
    d(w1 @ basis) in place of basis and w1, and the LrfGradients struct pointing at them (d_rays left NULL)
    -> ((d_dplane, d_dline, d_aplane, d_aline: lists of three), d_w1b, d_b1, d_w2, d_b2, d_w3, d_b3), struct."""
    grids, mlp = m._tensors()
    g = _lib.LrfGradients()
    bufs = []
    for k in (0, 6):                                   # the density, then the appearance planes and lines
        d_grids, planes, lines = _grid_grads(grids[k:k + 6])
        setattr(g, "d_" + _FIELD_TENSORS[k][0], planes)
        setattr(g, "d_" + _FIELD_TENSORS[k + 3][0], lines)
        bufs += [d_grids[:3], d_grids[3:]]
    basis, w1 = mlp[:2]
    bufs += [torch.zeros(w1.shape[0], basis.shape[1], device=dev)] + [torch.zeros_like(t) for t in mlp[2:]]
    for (slot, _, _), t in zip(_FIELD_TENSORS[13:], bufs[4:]):
        setattr(g, "d_w1b" if slot == "w1" else "d_" + slot, t.data_ptr())
    return tuple(bufs), g


def _field_grads(m, bufs):
    """The buffers of _field_grad_buffers as gradients in _grad_params order: d_w1b, the gradient of the product
    w1 @ basis the kernels read, is unfolded into those of basis and w1."""
    basis, w1 = (t.detach() for t in m._tensors()[1][:2])
    d_w1b = bufs[4]
    return (*(t for d_grids in bufs[:4] for t in d_grids), w1.t() @ d_w1b, d_w1b @ basis.t(), *bufs[5:])


class _RenderFn(torch.autograd.Function):
    """TensorBase.forward as ONE autograd node: the forward is the fused render kernel (lrf_render),
    the backward is lrf_render_backward (march again -> MLP backward over the shaded samples ->
    density branch), so a training step never materialises per-sample tensors in torch.  Gradients
    reach the planes, lines, basis, MLP and the rays (hence poses / intrinsics upstream)."""

    @staticmethod
    def forward(ctx, module, z, white_bg, rays, *params):
        rays_c = rays.detach().to(torch.float32).contiguous()
        rgb, depth = module._render_fused(rays_c, z, white_bg, 0.0, False, None, fp32=True)
        ctx.module, ctx.white_bg = module, white_bg
        # the backward re-reads the module's live parameters (nothing per-sample is saved): remember
        # what the forward saw, so an in-place update / upsample / mask rebuild in between raises like
        # torch's own version-counter check would instead of producing gradients of a different model
        ctx.seen = _field_state(module, params)
        ctx.save_for_backward(rays_c, z)
        return rgb, depth

    @staticmethod
    def backward(ctx, g_rgb, g_depth):
        rays, z = ctx.saved_tensors
        m, dev, n = ctx.module, rays.device, rays.shape[0]
        _check_field_state(m, ctx.seen)
        g_rgb = torch.zeros(n, 3, device=dev) if g_rgb is None else g_rgb.detach().to(torch.float32).contiguous()
        g_depth = torch.zeros(n, device=dev) if g_depth is None else g_depth.detach().to(torch.float32).contiguous()
        bufs, g = _field_grad_buffers(m, dev)
        d_rays = torch.empty_like(rays)
        g.d_rays = d_rays.data_ptr()
        lib = _lib.lib()
        with torch.cuda.device(dev):
            fs, _ = m.field_and_prepared(z, fp32=True)
            bp = m._prepared_backward()
            need = lib.lrf_backward_scratch_bytes(n, z.numel())
            # per call, from torch's caching allocator (stream-ordered reuse): backwards of the same module on
            # different streams never share a scratch block
            scratch = torch.empty(need, dtype=torch.uint8, device=dev)
            _lib.check(lib.lrf_render_backward(C.byref(fs), _ptr(bp), _ptr(rays), n, int(ctx.white_bg),
                                               _ptr(g_rgb), _ptr(g_depth), C.byref(g), _ptr(scratch),
                                               scratch.numel(), _stream(dev)))
        return (None, None, None, d_rays, *_field_grads(m, bufs))


class _DensityL1Fn(torch.autograd.Function):
    """density_L1 (tensoRF.py:83-92) as two streaming kernels: nothing of size G^3 is materialised
    (the reference's bmm intermediate is 8*G^3 floats: 8.4 GB at 640^3)."""

    @staticmethod
    def forward(ctx, module, *grids):
        dev = grids[0].device
        acc = torch.zeros(1, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().lrf_density_l1(C.byref(module._field()), _ptr(acc), _stream(dev)))
        ctx.module = module
        n = 1
        for g in module._grid_host:
            n *= g
        return (acc / n).to(torch.float32)[0]

    @staticmethod
    def backward(ctx, g):
        m = ctx.module
        grids = m._tensors()[0][:6]
        dev = grids[0].device
        d_grids, planes, lines = _grid_grads(grids)
        gg = g.detach().to(torch.float32).reshape(1).contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().lrf_density_l1_backward(C.byref(m._field()), _ptr(gg), planes, lines,
                                                          _stream(dev)))
        return (None, *d_grids)


class _TVFn(torch.autograd.Function):
    """sum_i coef_plane * TVLoss(plane_i) + coef_line * TVLoss(line_i) (tensoRF.py:94-110 with
    utils/utils.py:293-312) on the channel-last tensors: one reduction kernel per tensor forward, one
    stencil kernel per tensor backward -- no transposed / shifted copies."""

    @staticmethod
    def _geom(t):
        c, h, w = t.shape[1], t.shape[2], t.shape[3]
        kh = 1.0 / (c * (h - 1) * w) if h > 1 else 0.0          # 1 / numel of the H-difference tensor
        kw = 1.0 / (c * h * (w - 1)) if w > 1 else 0.0
        return c, h, w, kh, kw

    @staticmethod
    def forward(ctx, weight, coefs, *tensors):
        dev = tensors[0].device
        sums = torch.zeros(len(tensors), 2, dtype=torch.float64, device=dev)
        lib = _lib.lib()
        scale = []
        with torch.cuda.device(dev):
            st = _stream(dev)
            for i, t in enumerate(tensors):
                c, h, w, kh, kw = _TVFn._geom(t)
                _lib.check(lib.lrf_tv_sums(_ptr(t.detach()), h, w, c, C.c_void_p(sums.data_ptr() + 16 * i), st))
                scale.append([2.0 * weight * coefs[i] * kh, 2.0 * weight * coefs[i] * kw])
        ctx.scale = scale
        ctx.save_for_backward(*tensors)
        return (sums * torch.tensor(scale, dtype=torch.float64, device=dev)).sum().to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        tensors = ctx.saved_tensors
        dev = tensors[0].device
        gg = g.detach().to(torch.float32).reshape(1).contiguous()
        grads = []
        lib = _lib.lib()
        with torch.cuda.device(dev):
            st = _stream(dev)
            for (kh, kw), t in zip(ctx.scale, tensors):
                d = torch.zeros_like(t, memory_format=torch.channels_last)
                c, h, w = t.shape[1], t.shape[2], t.shape[3]
                _lib.check(lib.lrf_tv_sums_backward(_ptr(t.detach()), h, w, c, _ptr(gg), kh, kw, _ptr(d), st))
                grads.append(d)
        return (None, None, *grads)


def _cl_empty(c, h, w, device):
    """uninitialised [1,c,h,w] float32 tensor whose memory is [h][w][c] (channels_last strides, also for
    the degenerate w == 1 of the line tensors)."""
    return torch.empty(1, h, w, c, dtype=torch.float32, device=device).permute(0, 3, 1, 2)


class AlphaGridMask(torch.nn.Module):
    """models/tensorBase.py:38-62 -- binary occupancy volume, trilinearly sampled."""

    def __init__(self, device, aabb, alpha_volume):
        super().__init__()
        self.device = device
        self.aabb = torch.nn.Parameter(aabb.to(device), requires_grad=False)
        self.aabbSize = self.aabb[1] - self.aabb[0]
        self.invgridSize = torch.nn.Parameter(1.0 / self.aabbSize * 2, requires_grad=False)
        vol = alpha_volume.view(1, 1, *alpha_volume.shape[-3:])
        self.alpha_volume = torch.nn.Parameter(vol.to(device), requires_grad=False)
        d, h, w = vol.shape[-3:]
        self.gridSize = torch.LongTensor([w, h, d]).to(device)

    def normalize_coord(self, xyz_sampled):
        return (xyz_sampled - self.aabb[0]) * self.invgridSize - 1

    def sample_alpha(self, xyz_sampled):
        # off the per-batch path (used by compute_alpha / filtering); the render kernel has its
        # own fused lookup
        grid = self.normalize_coord(xyz_sampled).view(1, -1, 1, 1, 3)
        return F.grid_sample(self.alpha_volume, grid, align_corners=True).view(-1)

    def to(self, device):
        self.device = torch.device(device)
        return super().to(device)


class MLPRender_Fea_late_view(torch.nn.Module):
    """models/tensorBase.py:97-135 -- holds mlp[0], mlp[2], mlp_view[0] (same state_dict keys).

    Inside TensorBase.forward the MLP is evaluated by the fused kernel; calling this module
    directly evaluates it with torch ops (used by tests and by code that shades points itself).
    """

    def __init__(self, inChanel, viewpe=6, feape=6, featureC=128):
        super().__init__()
        self.in_mlpC = inChanel * (1 + 2 * feape)
        self.in_view = 3 * (1 + 2 * viewpe)
        self.viewpe, self.feape = viewpe, feape
        self.mlp = torch.nn.Sequential(
            torch.nn.Linear(self.in_mlpC, featureC), torch.nn.ReLU(inplace=True),
            torch.nn.Linear(featureC, featureC), torch.nn.ReLU(inplace=True))
        self.mlp_view = torch.nn.Sequential(torch.nn.Linear(featureC + self.in_view, 3))
        torch.nn.init.constant_(self.mlp_view[-1].bias, 0)

    @staticmethod
    def _pe(x, n_freq):
        bands = 2.0 ** torch.arange(n_freq, device=x.device, dtype=torch.float32)
        ang = (x[..., None] * bands).reshape(*x.shape[:-1], -1)
        return torch.cat([ang.sin(), ang.cos()], dim=-1)

    def forward(self, pts, viewdirs, features, refine):
        x = features
        if self.feape > 0:
            extra = self._pe(features, self.feape) if refine else \
                features.new_zeros(features.shape[0], self.in_mlpC - features.shape[-1])
            x = torch.cat([features, extra], dim=-1)
        v = viewdirs if self.viewpe == 0 else torch.cat([viewdirs, self._pe(viewdirs, self.viewpe)], -1)
        return torch.sigmoid(self.mlp_view(torch.cat([self.mlp(x), v], dim=-1)))


class TensorBase(torch.nn.Module):
    """models/tensorBase.py:231-636."""

    def __init__(self, device, aabb, gridSize, density_n_comp=8, appearance_n_comp=24, app_dim=27,
                 shadingMode="MLP_PE", alphaMask=None, near_far=[2.0, 6.0], density_shift=-10,
                 alphaMask_thres=0.001, distance_scale=25, rayMarch_weight_thres=0.001, pos_pe=6,
                 view_pe=6, fea_pe=6, featureC=128, step_ratio=2.0, fea2denseAct="softplus"):
        super().__init__()
        self.density_n_comp = list(density_n_comp)
        self.app_n_comp = list(appearance_n_comp)
        self.app_dim = app_dim
        self.aabb = torch.nn.Parameter(aabb, requires_grad=False)
        self.alphaMask = alphaMask
        self.device = device
        self.density_shift = density_shift
        self.alphaMask_thres = alphaMask_thres
        self.distance_scale = distance_scale
        self.rayMarch_weight_thres = rayMarch_weight_thres
        self.fea2denseAct = fea2denseAct
        self.near_far = list(near_far)
        self.step_ratio = step_ratio
        self.matMode = [list(m) for m in MAT_MODE]
        self.vecMode = list(VEC_MODE)
        self.comp_w = [1, 1, 1]
        self.update_stepSize(list(gridSize))
        self.init_svd_volume(gridSize, device)
        self.shadingMode, self.pos_pe, self.view_pe, self.fea_pe, self.featureC = (
            shadingMode, pos_pe, view_pe, fea_pe, featureC)
        self.init_render_func(shadingMode, pos_pe, view_pe, fea_pe, featureC, device)
        self.last_weights = None     # set by forward(..., return_weights=True)
        self.grid_storage = "fp32"   # see set_grid_storage()

    # -- construction helpers ---------------------------------------------------------------------
    def init_render_func(self, shadingMode, pos_pe, view_pe, fea_pe, featureC, device):
        # Only "MLP_Fea_late_view" accepts the 4-argument renderModule call of
        # TensorBase.forward (tensorBase.py:627-629); the other modes are dead options there.
        if shadingMode != "MLP_Fea_late_view":
            raise NotImplementedError(
                f"shadingMode={shadingMode!r}: only 'MLP_Fea_late_view' is usable on the "
                "reference's render path (tensorBase.py:627-629) and built here")
        self.renderModule = MLPRender_Fea_late_view(self.app_dim, view_pe, fea_pe, featureC).to(device)

    def update_stepSize(self, gridSize):
        """tensorBase.py:317-328 -- derives stepSize / nSamples from the grid resolution."""
        self.aabbSize = self.aabb[1] - self.aabb[0]
        self.invaabbSize = torch.nn.Parameter(2.0 / self.aabbSize, requires_grad=False)
        self.gridSize = torch.LongTensor(list(gridSize)).to(self.device)
        self._grid_host = [int(g) for g in gridSize]
        self.units = self.aabbSize / (self.gridSize - 1)
        self.stepSize = torch.mean(self.units) * self.step_ratio
        self.aabbDiag = torch.sqrt(torch.sum(torch.square(self.aabbSize)))
        self.nSamples = int((self.aabbDiag / self.stepSize).item()) + 1

    def init_svd_volume(self, res, device):
        raise NotImplementedError

    def normalize_coord(self, xyz_sampled):
        return (xyz_sampled - self.aabb[0]) * self.invaabbSize - 1

    def get_kwargs(self):
        return {
            "aabb": self.aabb, "gridSize": self.gridSize.tolist(),
            "density_n_comp": self.density_n_comp, "appearance_n_comp": self.app_n_comp,
            "app_dim": self.app_dim, "density_shift": self.density_shift,
            "alphaMask_thres": self.alphaMask_thres, "distance_scale": self.distance_scale,
            "rayMarch_weight_thres": self.rayMarch_weight_thres, "fea2denseAct": self.fea2denseAct,
            "near_far": self.near_far, "step_ratio": self.step_ratio,
            "shadingMode": self.shadingMode, "pos_pe": self.pos_pe, "view_pe": self.view_pe,
            "fea_pe": self.fea_pe, "featureC": self.featureC,
        }

    def to(self, device):
        self.device = torch.device(device)
        self.stepSize = self.stepSize.to(device)
        if self.alphaMask is not None:
            self.alphaMask = self.alphaMask.to(device)
        self.__dict__.pop("_memo", None)
        return super().to(device)

    # -- the per-batch distance table (tensorBase.py:419-437) -------------------------------------
    def sample_table(self, is_train=False, N_samples=-1, device=None):
        """z_vals of sample_ray_contracted: identical for every ray of the batch ([S] tensor).

        Train mode draws the two jitter tensors with torch.rand_like in the reference's order so a
        seeded run consumes the RNG stream exactly like the reference does.
        """
        device = device if device is not None else self.aabb.device
        n = (N_samples if N_samples > 0 else self.nSamples) // 6
        if not is_train:   # deterministic: build once per (n, device)
            return _memo(self, "z", (n, str(device)), lambda _: self._build_table(n, device, False))
        return self._build_table(n, device, True)

    @staticmethod
    def _build_table(n, device, is_train):
        t = torch.linspace(0.0, n - 1, n, device=device)[None] / n
        near_t = t.clone()
        if is_train:
            near_t += torch.rand_like(t) / n
            t += torch.rand_like(t) / n
        far_t = 1.0 / (1.0 * (1.0 - t) + 1.0 / 1e3 * t)
        z = torch.cat([near_t, far_t], dim=1)
        z += 1e-1
        return z.reshape(-1).contiguous()

    def feature2density(self, density_features):
        if self.fea2denseAct == "softplus":
            return F.softplus(density_features + self.density_shift)
        if self.fea2denseAct == "relu":
            return F.relu(density_features)
        raise ValueError(self.fea2denseAct)

    # -- C-ABI marshalling ------------------------------------------------------------------------
    def set_grid_storage(self, kind="fp32"):
        """Storage type the INFERENCE kernels read the plane / line grids from.

        "fp32" (default): the parameters themselves.  "bf16": bfloat16 copies in the same channel-last
        layout (LrfField.grid_dtype = LRF_GRID_BF16) -- a density texel is one 16-byte load, an appearance
        texel three, i.e. half the gather bytes and half the load instructions.  The copies are made by
        lrf_pack_bf16 (round to nearest even) and refreshed whenever a parameter changes; arithmetic stays
        fp32, so the render equals the fp32 render of the bf16-rounded parameters (exactly so for a field
        whose grids are bf16-representable, e.g. a checkpoint stored in bf16).  The parameters, `state_dict`
        and everything that records autograd (training) are untouched: they keep reading fp32."""
        if kind not in ("fp32", "bf16"):
            raise ValueError("grid storage must be 'fp32' or 'bf16'")
        if kind == "bf16" and (self.fea_pe or self.view_pe):
            raise NotImplementedError("localrf_b200: bf16 grid storage is built for fields without positional encodings")
        self.grid_storage = kind
        self.__dict__.pop("_memo", None)
        return self

    def _tensors(self):
        """(grids, mlp): the field's tensors as two tuples in _FIELD_TENSORS order.  Read through the modules'
        _parameters / _modules dicts: ParameterList / Sequential indexing costs ~1 us per access, and this runs on
        every render call."""
        mods = self._modules
        rm = mods["renderModule"]._modules
        l0, l2, l3 = rm["mlp"]._modules["0"]._parameters, rm["mlp"]._modules["2"]._parameters, \
            rm["mlp_view"]._modules["0"]._parameters
        return ((*mods["density_plane"]._parameters.values(), *mods["density_line"]._parameters.values(),
                 *mods["app_plane"]._parameters.values(), *mods["app_line"]._parameters.values()),
                (mods["basis_mat"]._parameters["weight"], l0["weight"], l0["bias"], l2["weight"], l2["bias"],
                 l3["weight"], l3["bias"]))

    def _grids16(self, grids):
        """bfloat16 copies of the twelve grids (memory [H][W][C] / [L][C]), rebuilt when a grid is replaced or
        updated in place."""
        def build(_):
            lib = _lib.lib()
            out = []
            for p in grids:
                dst = torch.empty(p.numel(), dtype=torch.bfloat16, device=p.device)
                with torch.cuda.device(p.device):
                    _lib.check(lib.lrf_pack_bf16(_ptr(p.detach()), _ptr(dst), p.numel(), _stream(p.device)))
                out.append(dst)
            return tuple(out)
        return _memo(self, "grids16", _key(grids), build, grids)

    def _field(self, z=None, bf16=False, prepared=False):
        """This field's LrfField, memoised: rebuilt when a tensor it points at or copies from is replaced or
        updated in place, or a scalar it holds changes.  `bf16`: the grids are their bfloat16 copies.  Without `z`
        the table is NULL, for the entry points that read no table.  With `prepared`: (struct, forward prepared
        block), the block rebuilt in place when the MLP / basis weights change."""
        grids, mlp = self._tensors()
        am = self.alphaMask
        src = mlp + grids + (self._parameters["aabb"],) + (() if z is None else (z,)) + \
            (() if am is None else (am._parameters["alpha_volume"], am._parameters["aabb"]))
        k = _key(src)
        key = (k, None if z is None else z.numel(), tuple(self._grid_host), float(self.density_shift),
               float(self.distance_scale), float(self.rayMarch_weight_thres), self.fea2denseAct)
        fs = _memo(self, _FIELD_SLOTS[bf16][z is None], key, lambda _: self._field_struct(z, grid16=bf16), src)[0]
        if not prepared:
            return fs
        n = len(mlp)                   # src starts with the MLP tensors: the head of k is _key(mlp)
        return fs, _memo(self, "prepared", (k[0][:n], k[1][:n]), lambda block: self.prepare(fs, block), mlp)

    def _field_struct(self, z=None, need_mlp=True, grid16=False):
        """A new LrfField of this field and the bfloat16 copies it points at, if any -> (struct, copies).  The
        builder of _field's memo, which is where callers take their struct from.  `need_mlp=False` leaves the MLP
        pointers other than basis NULL, for the entry points that run no MLP."""
        grids, mlp = self._tensors()
        s = _lib.LrfField()
        g = self._grid_host
        aabb = self._host_copy("aabb", self.aabb)
        for i in range(3):
            s.grid[i] = int(g[i])
        for i in range(6):
            s.aabb[i] = aabb[i]
        if len(set(self.density_n_comp)) != 1 or len(set(self.app_n_comp)) != 1:
            raise NotImplementedError("per-plane component counts must be equal")
        s.n_dcomp, s.n_acomp = self.density_n_comp[0], self.app_n_comp[0]
        for (slot, i, _), p in zip(_FIELD_TENSORS, grids):
            _require_cuda(p, f"{slot}[{i}]")
            if p.dtype != torch.float32:
                raise TypeError(f"{slot}[{i}] must be float32, got {p.dtype}")
            if not p.is_contiguous(memory_format=torch.channels_last):
                # a parameter swapped in from outside in NCHW layout: re-lay it out IN PLACE, once,
                # so the struct always points at the live storage the optimiser updates (a
                # temporary copy would go stale on the next in-place update)
                p.data = _cl(p.data)
            getattr(s, slot)[i] = p.data_ptr()
        s.app_dim = self.app_dim
        s.featureC = self.featureC
        s.fea_pe, s.view_pe = self.fea_pe, self.view_pe
        for (slot, _, _), t in zip(_FIELD_TENSORS[12:], mlp if need_mlp else ()):
            _require_cuda(t, slot)
            if t.dtype != torch.float32:
                raise TypeError(f"{slot} must be float32, got {t.dtype}")
            if not t.is_contiguous():
                t.data = t.data.contiguous()       # in place, for the same reason as above
            setattr(s, slot, t.data_ptr())
        if not need_mlp:
            s.basis = mlp[0].detach().data_ptr()
        if self.alphaMask is not None:
            vol = self.alphaMask.alpha_volume
            _require_cuda(vol, "alphaMask.alpha_volume")
            if vol.dtype != torch.float32 or not vol.is_contiguous():
                vol.data = vol.data.to(torch.float32).contiguous()     # the kernel reads fp32 [D][H][W]
            s.alpha_vol = vol.data_ptr()
            for i in range(3):
                s.alpha_dims[i] = vol.shape[-3 + i]
            ab = self._host_copy("alpha_aabb", self.alphaMask.aabb)
            for i in range(6):
                s.alpha_aabb[i] = ab[i]
        s.density_shift = float(self.density_shift)
        s.distance_scale = float(self.distance_scale)
        s.weight_thres = float(self.rayMarch_weight_thres)
        s.act = {"softplus": 0, "relu": 1}[self.fea2denseAct]
        if z is not None:
            s.z_vals = z.data_ptr()
            s.n_samples = z.numel()
        copies = ()
        if grid16:
            # (after the loop above: the fp32 parameters are channel-last by now, so the copies are too)
            copies = self._grids16(grids)
            for (slot, i, _), t in zip(_FIELD_TENSORS, copies):
                getattr(s, slot)[i] = t.data_ptr()
            s.grid_dtype = _lib.GRID_BF16
        return s, copies

    def _host_copy(self, slot, t):
        """Host list of a small device tensor (an aabb), memoised: the per-call path does no device-to-host
        synchronisation."""
        return _memo(self, slot, _key((t,)), lambda _: t.detach().reshape(-1).tolist(), (t,))

    def field_and_prepared(self, z, fp32=False):
        """(LrfField struct, prepared block) for this field, memoised (_field): rebuilt every optimiser step
        while training, never inside an eval loop.  With grid_storage == "bf16" the struct points at the bfloat16
        copies of the grids unless `fp32` is set (the autograd node: forward and backward read the live fp32
        parameters)."""
        return self._field(z, self.grid_storage == "bf16" and not fp32, prepared=True)

    def prepare(self, field_struct, block=None):
        """Fills the folded / re-laid-out MLP block the kernel stages into shared memory (for a field with
        positional encodings: the separate basis / layer-1 operand images, 1024-byte aligned for TMA) -> the
        block: `block` rewritten in place when it has the size and device, else a new one."""
        dev = self.basis_mat.weight.device
        n = _lib.lib().lrf_prepared_bytes_for(C.byref(field_struct))
        if n == 0:
            raise NotImplementedError("localrf_b200: fea_pe / view_pe above 8 are not built")
        if block is None or block.device != dev or block.numel() != n:
            raw = torch.empty(n + 1024, dtype=torch.uint8, device=dev)
            off = (-raw.data_ptr()) % 1024
            block = raw[off:off + n]
        _lib.check(_lib.lib().lrf_field_prepare(C.byref(field_struct), _ptr(block), _stream(dev)))
        return block

    def shade_products(self, products, viewdirs):
        """basis_mat + renderModule on explicit plane x line products [M,72] and normalised view
        directions [M,3] -> rgb [M,3]; the tensor-core MLP of the render kernel on its own."""
        _require_cuda(products, "products")
        if self.fea_pe or self.view_pe:
            raise NotImplementedError("localrf_b200: the stand-alone MLP entry (lrf_mlp_forward) covers pe = 0")
        dev = products.device
        x = products.detach().to(torch.float32).contiguous()
        v = viewdirs.detach().to(dev, torch.float32).contiguous()
        out = torch.empty(x.shape[0], 3, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _, prep = self.field_and_prepared(None, fp32=True)
            _lib.check(_lib.lib().lrf_mlp_forward(_ptr(prep), _ptr(x), _ptr(v), x.shape[0],
                                                  _ptr(out), _stream(dev)))
        return out

    # -- the hot path ------------------------------------------------------------------------------
    def forward(self, rays_chunk, white_bg=True, is_train=False, N_samples=-1, refine=True,
                floater_thresh=0, return_weights=False, stats=None, z_vals=None):
        """tensorBase.py:567-636 -> (rgb_map [N,3], depth_map [N]).

        `return_weights=True` additionally stores the final per-sample weights [N,S] in
        `self.last_weights` (the default return arity is the reference's).  `z_vals` overrides the
        distance table (parity tests feed the reference's own jittered table).
        """
        _require_cuda(rays_chunk, "rays_chunk")
        wants_grad = self._wants_grad(rays_chunk, *self.parameters())
        fused_grad = (wants_grad and floater_thresh == 0 and not return_weights and stats is None
                      and rays_chunk.dim() == 2 and rays_chunk.shape[1] == 6
                      and self.fea_pe == 0 and self.view_pe == 0       # the fused backward covers pe = 0
                      and os.environ.get("LRF_TRAIN_PATH", "fused") != "composed")
        if not self.fused_supported() or (wants_grad and not fused_grad):
            return self._forward_autograd(rays_chunk, white_bg, is_train, N_samples, refine,
                                          floater_thresh, return_weights, z_vals)
        dev = rays_chunk.device
        if rays_chunk.dtype != torch.float32 or rays_chunk.dim() != 2 or rays_chunk.shape[1] < 6:
            raise ValueError("rays_chunk must be a float32 [N, 6] tensor")
        if z_vals is None:
            z = self.sample_table(is_train, N_samples, dev)
        else:
            z = z_vals.detach().to(dev, torch.float32).reshape(-1).contiguous()
        # tensorBase.py:633 -- the coin is only tossed when white_bg is False and is_train
        bg = bool(white_bg) or bool(is_train and torch.rand((1,)) < 0.5)
        if wants_grad:
            self.last_weights = None
            return _RenderFn.apply(self, z, bg, rays_chunk, *self._grad_params())
        rays = rays_chunk.detach()[:, :6].contiguous()
        return self._render_fused(rays, z, bg, floater_thresh, return_weights, stats, refine)

    def _grad_params(self):
        """Parameters in the order _RenderFn.backward returns their gradients."""
        grids, mlp = self._tensors()
        return grids + mlp

    def _prepared_backward(self):
        """Folded / transposed MLP block of lrf_render_backward, rebuilt in place when the MLP / basis weights
        change."""
        mlp = self._tensors()[1]

        def build(block):
            dev, lib = mlp[0].device, _lib.lib()
            if block is None or block.device != dev:
                block = torch.empty(lib.lrf_prepared_backward_bytes(), dtype=torch.uint8, device=dev)
            _lib.check(lib.lrf_field_prepare_backward(C.byref(self._field()), _ptr(block), _stream(dev)))
            return block
        return _memo(self, "prepared_backward", _key(mlp), build, mlp)

    def _render_fused(self, rays, z, bg, floater_thresh, return_weights, stats, refine=True, fp32=False):
        """One lrf_render launch on explicit rays [n,6] (contiguous fp32) -> (rgb [n,3], depth [n])."""
        dev, n = rays.device, rays.shape[0]
        with torch.cuda.device(dev):
            fs, prep = self.field_and_prepared(z, fp32=fp32)
            rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
            depth = torch.empty(n, dtype=torch.float32, device=dev)
            weights = torch.empty(n, z.numel(), dtype=torch.float32, device=dev) if return_weights else None
            b = _lib.LrfBatch(n_rays=n, rays=rays.data_ptr(), n_views=1, white_bg=int(bg),
                              floater_thresh=float(floater_thresh), refine=int(bool(refine)))
            o = _lib.LrfOutputs(rgb=rgb.data_ptr(), depth=depth.data_ptr(),
                                weights=None if weights is None else weights.data_ptr(),
                                stats=None if stats is None else stats.data_ptr())
            _lib.check(_lib.lib().lrf_render(C.byref(fs), _ptr(prep), C.byref(b), C.byref(o),
                                             _stream(dev)))
        self.last_weights = weights
        return rgb, depth

    def fused_supported(self):
        """Configurations the fused forward kernel covers: the reference defaults (pe = 0: basis folded
        into layer 1) and positional encodings up to 8 frequencies (a second instantiation of the kernel:
        basis as its own tensor-core product, encoded input built in registers, layer-1 weights streamed).
        The fused BACKWARD covers pe = 0; fields with encodings train through the composed path."""
        return self.app_dim == 27 and self.featureC == 128 and 0 <= self.fea_pe <= 8 and 0 <= self.view_pe <= 8

    def _forward_autograd(self, rays_chunk, white_bg, is_train, N_samples, refine, floater_thresh,
                          return_weights, z_vals):
        """The composed path: the same algorithm as the fused kernel, built from the two
        differentiable CUDA lookups (`_VMLookup`: density feature, appearance products) and torch ops
        for the cheap per-sample arithmetic and the dense MLP; differentiable end to end.  Used for
        configurations the fused kernels do not cover (positional encodings; floater filter or
        `return_weights` while autograd records) and, with LRF_TRAIN_PATH=composed, as the independent
        implementation the fused backward is compared with.  tensorBase.py:567-636."""
        from .ray_utils import contract
        dev = rays_chunk.device
        rays_o, d = rays_chunk[:, :3], rays_chunk[:, 3:6]
        norm = torch.norm(d, dim=-1, keepdim=True)
        viewdirs = d / norm
        z = self.sample_table(is_train, N_samples, dev) if z_vals is None else \
            z_vals.detach().to(dev, torch.float32).reshape(-1)
        z = z[None]                                                     # [1,S] like the reference
        xyz = contract(rays_o[:, None, :] + viewdirs[:, None, :] * z[..., None])
        n, S = xyz.shape[0], z.shape[1]
        dists = torch.cat([z[:, 1:] - z[:, :-1], torch.zeros_like(z[:, :1])], dim=-1)
        valid = torch.ones(n, S, dtype=torch.bool, device=dev)
        if self.alphaMask is not None:
            with torch.no_grad():
                valid &= (self.alphaMask.sample_alpha(xyz.reshape(-1, 3)) > 0).view(n, S)
        valid[:, -1] = False
        xyzn = self.normalize_coord(xyz)
        sigma = torch.zeros(n, S, device=dev)
        if valid.any():
            sigma = sigma.masked_scatter(valid, self.feature2density(
                self.compute_densityfeature(xyzn[valid])))
        alpha = 1.0 - torch.exp(-sigma * dists * self.distance_scale)

        def weights_of(a):
            a = torch.cat([a[:, :-1], torch.ones_like(a[:, :1])], dim=-1)      # alpha[:, -1] = 1
            T = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1.0 - a + 1e-10], -1), -1)
            return a * T[:, :-1]

        weight = weights_of(alpha)
        acc_map = weight.sum(-1)
        depth_map = (weight * z).sum(-1) / norm[..., 0]
        if floater_thresh > 0:
            ks = torch.arange(S, device=dev)[None]
            idx_map = (weight * ks).sum(-1, keepdim=True)
            alpha = torch.where(ks < idx_map * floater_thresh, torch.zeros_like(alpha), alpha)
            weight = weights_of(alpha)
        app_mask = weight > self.rayMarch_weight_thres
        rgb = torch.zeros(n, S, 3, device=dev)
        if app_mask.any():
            feats = self.compute_appfeature(xyzn[app_mask])
            vd = viewdirs[:, None, :].expand(n, S, 3)[app_mask].clone().detach()
            rgb = rgb.masked_scatter(app_mask[..., None].expand(n, S, 3),
                                     self.renderModule(None, vd, feats, refine))
        rgb_map = (weight[..., None] * rgb).sum(-2)
        if white_bg or (is_train and torch.rand((1,)) < 0.5):
            rgb_map = rgb_map + (1.0 - acc_map[..., None])
        self.last_weights = weight.detach() if return_weights else None
        return rgb_map, depth_map

    # -- off-path methods of the reference (host bookkeeping, stock torch) ------------------------
    def compute_alpha(self, xyz_locs, length=1):
        """tensorBase.py:538-558."""
        if self.alphaMask is not None:
            keep = self.alphaMask.sample_alpha(xyz_locs) > 0
        else:
            keep = torch.ones_like(xyz_locs[:, 0], dtype=torch.bool)
        sigma = torch.zeros(xyz_locs.shape[:-1], device=xyz_locs.device)
        if keep.any():
            feat = self.compute_densityfeature(self.normalize_coord(xyz_locs[keep]))
            sigma[keep] = self.feature2density(feat)
        return 1 - torch.exp(-sigma * length).view(xyz_locs.shape[:-1])

    def _alpha_lattice(self, gridSize, want_mask):
        """One lrf_alpha_mask_build call: dense alpha [gx,gy,gz] (+ the pooled / thresholded mask
        [gz,gy,gx] and the number of kept voxels)."""
        dims = [int(g) for g in gridSize]
        dev = self.aabb.device
        _require_cuda(self.aabb, "aabb")
        alpha = torch.empty(dims, dtype=torch.float32, device=dev)
        mask = torch.empty(dims[::-1], dtype=torch.float32, device=dev) if want_mask else None
        kept = torch.zeros(1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().lrf_alpha_mask_build(
                C.byref(self._field()), (C.c_int32 * 3)(*dims), float(self.stepSize), float(self.alphaMask_thres),
                _ptr(alpha), _ptr(mask), _ptr(kept), _stream(dev)))
        return alpha, mask, kept

    @torch.no_grad()
    def getDenseAlpha(self, gridSize=None):
        """tensorBase.py:501-515 -- alpha on a dense lattice of the aabb: one kernel launch."""
        gridSize = self._grid_host if gridSize is None else gridSize
        return self._alpha_lattice(gridSize, False)[0]

    @torch.no_grad()
    def updateAlphaMask(self, gridSize=(200, 200, 200)):
        """tensorBase.py:517-536 -- rebuilt ON THE DEVICE by two kernels (lattice density + 3x3x3
        max-pool / threshold); the reference moves the model to the CPU and loops over slabs."""
        gridSize = tuple(int(g) for g in gridSize)
        _, mask, kept = self._alpha_lattice(gridSize, True)
        self.alphaMask = AlphaGridMask(self.aabb.device, self.aabb.detach(), mask)
        total = gridSize[0] * gridSize[1] * gridSize[2]
        print(f"alpha rest %%%f" % (float(kept) / total * 100))

    # -- sample_ray (tensorBase.py:396-417): the ray-AABB sampler (not on LocalTensorfs' render path,
    #    which samples contracted space; kept as the utility north_star names) -----------------------
    def sample_ray(self, rays_o, rays_d, is_train=True, N_samples=-1):
        """-> (rays_pts [N,S,3], interpx [N,S], inside-the-aabb mask [N,S]) like the reference."""
        _require_cuda(rays_o, "rays_o")
        dev = rays_o.device
        S = int(N_samples if N_samples > 0 else self.nSamples)
        rays = torch.cat([rays_o.detach().reshape(-1, 3), rays_d.detach().reshape(-1, 3)], -1) \
            .to(torch.float32).contiguous()
        n = rays.shape[0]
        jitter = torch.rand(n, 1).to(dev).reshape(-1).contiguous() if is_train else None   # CPU draw, as :404-406
        pts = torch.empty(n, S, 3, dtype=torch.float32, device=dev)
        z = torch.empty(n, S, dtype=torch.float32, device=dev)
        inside = torch.empty(n, S, dtype=torch.uint8, device=dev)
        aabb = self._host_copy("aabb", self.aabb)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().lrf_sample_ray(
                _ptr(rays), _ptr(jitter), n, S, (C.c_float * 6)(*aabb), float(self.near_far[0]),
                float(self.near_far[1]), float(self.stepSize), _ptr(pts), _ptr(z), _ptr(inside), _stream(dev)))
        return pts, z, inside.bool()


class TensorVMSplit(TensorBase):
    """models/tensoRF.py:10-277 -- vector-matrix decomposed density / appearance grids."""

    def __init__(self, device, aabb, gridSize, **kargs):
        super().__init__(device, aabb, gridSize, **kargs)

    def init_svd_volume(self, res, device):
        self.density_plane, self.density_line = self.init_one_svd(self.density_n_comp, res, 0.1, device)
        self.app_plane, self.app_line = self.init_one_svd(self.app_n_comp, res, 0.1, device)
        self.basis_mat = torch.nn.Linear(sum(self.app_n_comp), self.app_dim, bias=False).to(device)

    def init_one_svd(self, n_component, gridSize, scale, device):
        """tensoRF.py:29-50; same shapes and init draws, channels_last storage."""
        planes, lines = [], []
        for i, (vec_id, (m0, m1)) in enumerate(zip(self.vecMode, self.matMode)):
            # the reference draws plane then line for each i, on the CPU generator
            p = scale * torch.randn((1, n_component[i], gridSize[m1], gridSize[m0]))
            l = scale * torch.randn((1, n_component[i], gridSize[vec_id], 1))
            planes.append(torch.nn.Parameter(_cl(p.to(device))))
            lines.append(torch.nn.Parameter(_cl(l.to(device))))
        return torch.nn.ParameterList(planes), torch.nn.ParameterList(lines)

    def get_optparam_groups(self, lr_init_spatialxyz=0.02, lr_init_network=0.001):
        groups = [{"params": p, "lr": lr_init_spatialxyz}
                  for p in (self.density_line, self.density_plane, self.app_line, self.app_plane)]
        groups.append({"params": self.basis_mat.parameters(), "lr": lr_init_network})
        if isinstance(self.renderModule, torch.nn.Module):
            groups.append({"params": self.renderModule.parameters(), "lr": lr_init_network})
        return groups

    # -- feature lookups through the C ABI ---------------------------------------------------------
    def _feature_call_raw(self, xyz_sampled, fn_name, width):
        _require_cuda(xyz_sampled, "xyz_sampled")
        dev = xyz_sampled.device
        xyz = xyz_sampled.detach().reshape(-1, 3).to(torch.float32).contiguous()
        m = xyz.shape[0]
        out = torch.empty((m,) if width == 1 else (m, width), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(getattr(_lib.lib(), fn_name)(C.byref(self._field()), _ptr(xyz), m, _ptr(out), _stream(dev)))
        return out

    @staticmethod
    def _wants_grad(*tensors):
        return torch.is_grad_enabled() and any(t.requires_grad for t in tensors)

    def compute_densityfeature(self, xyz_sampled):
        """tensoRF.py:112-151: [M,3] normalised coords -> [M] (differentiable)."""
        grids = list(self.density_plane) + list(self.density_line)
        if self._wants_grad(xyz_sampled, *grids):
            return _VMLookup.apply(self, "density", xyz_sampled, *grids)
        return self._feature_call_raw(xyz_sampled, "lrf_density_feature", 1)

    def compute_appfeature(self, xyz_sampled):
        """tensoRF.py:153-196: [M,3] normalised coords -> [M, app_dim] (differentiable)."""
        grids = list(self.app_plane) + list(self.app_line)
        if self._wants_grad(xyz_sampled, self.basis_mat.weight, *grids):
            return self.basis_mat(_VMLookup.apply(self, "app", xyz_sampled, *grids))
        return self._feature_call_raw(xyz_sampled, "lrf_app_feature", self.app_dim)

    # -- regularisers (tensoRF.py:66-110), stock torch ---------------------------------------------
    def vectorDiffs(self, vector_comps):
        total = 0
        for v in vector_comps:
            n_comp, n_size = v.shape[1:-1]
            m = v.reshape(n_comp, n_size)
            gram = m @ m.t()
            off_diag = gram.reshape(-1)[1:].view(n_comp - 1, n_comp + 1)[..., :-1]
            total = total + off_diag.abs().mean()
        return total

    def vector_comp_diffs(self):
        return self.vectorDiffs(self.density_line) + self.vectorDiffs(self.app_line)

    def density_L1(self):
        """tensoRF.py:83-92 -- streamed over the G^3 flat indices (differentiable, no dense intermediate)."""
        _require_cuda(self.density_plane[0], "density_plane")
        return _DensityL1Fn.apply(self, *self.density_plane, *self.density_line)

    def _tv(self, planes, lines, reg):
        if type(reg).__name__ == "TVLoss" and hasattr(reg, "TVLoss_weight") and planes[0].is_cuda:
            coefs = [1e-2] * len(planes) + [1e-3] * len(lines)
            return _TVFn.apply(float(reg.TVLoss_weight), coefs, *planes, *lines)
        total = 0                                   # any other callable: the reference's formulation
        for p, l in zip(planes, lines):
            total = total + reg(p.transpose(0, 1)) * 1e-2 + reg(l.transpose(0, 1)) * 1e-3
        return total

    def TV_loss_density(self, reg):
        return self._tv(self.density_plane, self.density_line, reg)

    def TV_loss_app(self, reg):
        return self._tv(self.app_plane, self.app_line, reg)

    # -- resolution schedule (tensoRF.py:198-233) --------------------------------------------------
    @torch.no_grad()
    def up_sampling_VM(self, plane_coef, line_coef, res_target):
        """tensoRF.py:198-221 -- bilinear / align_corners=True resize, written channel-last directly by
        lrf_upsample (CPU tensors, e.g. in host-only tests, go through F.interpolate)."""
        lib = None
        for i, (vec_id, (m0, m1)) in enumerate(zip(self.vecMode, self.matMode)):
            for coef, (h2, w2) in ((plane_coef, (int(res_target[m1]), int(res_target[m0]))),
                                   (line_coef, (int(res_target[vec_id]), 1))):
                src = coef[i].detach()
                if not src.is_cuda:
                    coef[i] = torch.nn.Parameter(_cl(F.interpolate(src, size=(h2, w2), mode="bilinear",
                                                                   align_corners=True)))
                    continue
                if not src.is_contiguous(memory_format=torch.channels_last) or src.shape[3] == 1:
                    src = src.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)    # memory [H][W][C]
                c, h, w = src.shape[1], src.shape[2], src.shape[3]
                dst = _cl_empty(c, h2, w2, src.device)
                lib = lib or _lib.lib()
                with torch.cuda.device(src.device):
                    _lib.check(lib.lrf_upsample(_ptr(src), h, w, _ptr(dst), h2, w2, c, _stream(src.device)))
                coef[i] = torch.nn.Parameter(dst)
        return plane_coef, line_coef

    @torch.no_grad()
    def upsample_volume_grid(self, res_target):
        self.app_plane, self.app_line = self.up_sampling_VM(self.app_plane, self.app_line, res_target)
        self.density_plane, self.density_line = self.up_sampling_VM(
            self.density_plane, self.density_line, res_target)
        self.update_stepSize(res_target)
        print(f"upsamping to {res_target}")
