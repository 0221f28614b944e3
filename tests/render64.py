"""float64 restatement of the training call, differentiated by torch autograd, with each ray's decision margins.

What is restated:
  - TensorBase.forward (models/tensorBase.py:567-636): sample points o + (d / |d|) z, contract (utils/ray_utils.py:
    9-12), the alpha mask (trilinear, zero padding) on the contracted points, normalise_coord, the VM lookups with
    F.grid_sample(align_corners=True, padding_mode="border") (tensoRF.py:112-196), softplus(f + shift) or relu(f),
    alpha = 1 - exp(-sigma dist scale) with alpha[:, -1] = 1, T = cumprod(1 - alpha + 1e-10), w = alpha T, depth =
    sum(w z) / |d|, the floater filter (tensorBase.py:617-620: idx = sum_k w_k k, alpha[k < idx thresh] = 0, the
    weights again; acc and depth keep the pre-filter weights), the shading switch w > rayMarch_weight_thres,
    MLPRender_Fea_late_view (viewdirs detached) with positional encodings fea_pe / view_pe 0..8 (the 27 features, then
    sin (d-major, f-minor), then cos; zeros for the feature encoding when `refine` is 0) and sigmoid, and the white
    background (the pre-filter acc).  field_forward's extras also give what the render kernel's early termination
    leaves: the samples before the end of the 32-sample block in which T first falls below 1e-10 (`k_end`), the
    valid samples marched and the samples shaded there (`n_march`, `n_shade`, what its `stats` counts).
  - The camera side of LocalTensorfs.forward (local_tensorfs.py:397-499): pixel directions (lean or 360), rays (t +
    world2rf, R dir), per-view blend and accumulation over several fields (render_views), exposure E x and clamp(0,
    1), whose backward passes the gradient at both bounds.

Every hard switch of that function is evaluated on the float64 values, and for each ray `margins` gives how close its
float64 forward comes to each switch.  Where an fp32 implementation's error in the switched quantity grows along the
computation, the margin is in units of a propagated bound on that error (EPS = 2^-24, one fp32 rounding):
  thres     |w - rayMarch_weight_thres| / w_err.  The density feature f carries 32 EPS |f|_1 (|f|_1: the sum of the
            absolute values of every term of its lookups and sum) plus the position error of the sample (p = o + vd z
            carries 4 EPS (|o| + |z|), scaled by the contraction) times the feature's slope; sigma, x = sigma dist
            scale and alpha = 1 - exp(-x) add a few roundings each and carry f's error; T_k = prod_{j < k} ((1 -
            alpha_j) + 1e-10) accumulates each factor's relative error along the ray, so w_err = T dalpha + w relT
            (per sample in `w_err`; plus 2^-126, fp32's subnormal range).  alpha = 0 exactly (sigma = 0) gives w = 0 on both sides: no margin.  With a
            threshold of 0, a T below 2^-100 has margin 0 (fp32's T underflows to 0 where float64's does not);
  relu_f    |f| / f's error bound, act = relu;  softplus  |f + shift - 20| / (f's error bound + 20 EPS);
  mlp       each of the 2 x featureC MLP pre-activations against 0 on each shaded sample, over its error: 8 EPS of
            the layer-1 sum of |terms| (folded W1 basis on the 72 products; a sum of independently rounded terms
            grows as the square root of its length) plus the position error through the products' slope; 8 EPS of
            layer 2's plus layer 1's error through |W2|.  With positional encodings the 27 features are their own
            sum (8 EPS of it plus the slope), and their error reaches layer 1 through the encoding: 2^f times it in
            sin / cos of frequency f, plus 4 EPS for sin / cos themselves;
  floater   |idx thresh - k| for the integer k nearest to idx thresh (the floater cut), over a bound on the fp32 idx
            times thresh: sum_k w_err_k k, plus the rounding of a per-lane sequential sum of ceil(S / 32) terms and a
            5-level warp tree (ceil(S / 32) + 6 EPS of sum_k w_k k), plus the product's rounding.  inf where the
            filter is off, k is the last sample (its alpha is 1 either way) or alpha_k = 0 (the cut changes nothing).
            With the filter, `thres` is measured on the filtered weights, whose product restarts at 1 and carries
            only the errors of the alphas it keeps;
and in units of EPS times the quantity's size where the rounding does not accumulate:
  contract  max|p| - 1 (p = o + vd z carries (|o| + |z|) EPS), and, where the point is contracted, the gap between
            the largest and second-largest |p_a| (the contraction's argmax, which routes the norm's gradient);
  mask      the alpha-mask value against 0 (its fp32 value is a sum of non-negative terms: only an exact 0 in one
            implementation and not the other flips it, which happens at a mask-cell boundary: the margin is the
            distance of the mask-lattice coordinate to the nearest integer, in units of (dim) EPS).
Not a decision of the colour, but of what the kernel counts (`term`): |T_b - 1e-10| over T_b's propagated error,
for the transmittance T_b at the end of each 32-sample block up to the one where the march stops (the kernel's
early termination; inf with the floater filter, which marches every sample).
The texel floors (`texel`): the distance of every un-clipped pixel coordinate ((q + 1) / 2) (size - 1) of the twelve
lookups to the nearest integer in [0, size - 1] (unit: size EPS).  floor() chooses the cell, and the clip at 0 and
size - 1 zeroes the position gradient, so only the position gradients (d_rays and what the cameras derive from it)
jump there; the parameter gradients are continuous.

Runs on CPU or CUDA; rays are processed in chunks of about CHUNK_SAMPLES samples so that the autograd graph stays at
a few hundred MB.  Nothing here reads the reference project."""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

EPS = 2.0 ** -24
CHUNK_SAMPLES = 1 << 18
MAT0, MAT1, VEC = (0, 0, 1), (1, 2, 2), (2, 1, 0)
GRID_KEYS = [f"{n}.{i}" for n in ("density_plane", "density_line", "app_plane", "app_line") for i in range(3)]
MLP_KEYS = ["basis_mat.weight", "renderModule.mlp.0.weight", "renderModule.mlp.0.bias", "renderModule.mlp.2.weight",
            "renderModule.mlp.2.bias", "renderModule.mlp_view.0.weight", "renderModule.mlp_view.0.bias"]
PARAM_KEYS = GRID_KEYS + MLP_KEYS
MARGIN_KEYS = ("thres", "contract", "mask", "relu_f", "softplus", "mlp", "floater")
BOUND_KEYS = ("thres", "relu_f", "softplus", "mlp", "floater")     # margins in units of a propagated error bound
T_TERM = float(np.float32(1e-10))                       # the render kernel's early-termination transmittance (fp32)


class Field64:
    """A field's parameters as float64 leaves in the reference layout ([1, C, H, W] planes, [1, C, L, 1] lines)."""

    def __init__(self, fd, device="cpu"):
        t = lambda k: torch.as_tensor(np.asarray(fd[k]) if not torch.is_tensor(fd[k]) else fd[k].detach().cpu()
                                      ).to(device=device, dtype=torch.float64)
        self.p = {k: t(k).requires_grad_(True) for k in PARAM_KEYS}
        self.aabb = t("aabb").reshape(2, 3)
        self.grid = [int(self.p["density_plane.0"].shape[3]), int(self.p["density_plane.0"].shape[2]),
                     int(self.p["density_plane.1"].shape[2])]
        self.alpha_vol = t("alphaMask.alpha_volume") if fd.get("alphaMask.alpha_volume") is not None else None
        if self.alpha_vol is not None:
            self.alpha_vol = self.alpha_vol.reshape(1, 1, *self.alpha_vol.shape[-3:])
        self.alpha_aabb = t("alphaMask.aabb").reshape(2, 3) if self.alpha_vol is not None else None
        self.shift = float(fd.get("density_shift", -10.0))
        self.scale = float(fd.get("distance_scale", 25.0))
        self.thres = float(fd.get("rayMarch_weight_thres", 1e-3))
        self.act = str(fd.get("fea2denseAct", "softplus"))
        self.fea_pe = int(fd.get("fea_pe", 0))
        self.view_pe = int(fd.get("view_pe", 0))
        self.device = device

    @staticmethod
    def from_module(m, device="cpu", thres=None):
        """From a (product) TensorVMSplit: its state dict and scalars."""
        fd = {k: v for k, v in m.state_dict().items()}
        fd["density_shift"] = float(m.density_shift)
        fd["distance_scale"] = float(m.distance_scale)
        fd["rayMarch_weight_thres"] = float(m.rayMarch_weight_thres if thres is None else thres)
        fd["fea2denseAct"] = m.fea2denseAct
        fd["fea_pe"], fd["view_pe"] = int(m.fea_pe), int(m.view_pe)
        if m.alphaMask is None:
            fd.pop("alphaMask.alpha_volume", None)
        return Field64(fd, device)


def random_field(grid=(9, 11, 13), act="softplus", shift=-2.0, thres=1e-3, seed=0, mask=None, aabb=2.0,
                 safe_mlp=False, coarse=None, fea_pe=0, view_pe=0):
    """A field dict (reference layout, float64 numpy, with the scalars module_from_golden reads) with random grids:
    density features of spread ~1.5, so softplus(f + shift) spans several decades.  `mask`: an alpha volume
    [1, 1, D, H, W] over the same aabb.  safe_mlp: both hidden layers' units biased +-1 alternately with weights
    small enough that no pre-activation comes near 0 (check it with the `mlp` margin); the MLP is then smooth on
    every sample, at any number of samples.  coarse: draw the grids at that resolution per axis and upsample them
    bilinearly (align_corners, as up_sampling_VM does) to `grid` -- a field as training leaves it after an upsample,
    whose slope per unit length does not grow with the grid size.  fea_pe / view_pe: the MLP's positional
    encodings (layer 1 then reads 27 (1 + 2 fea_pe) inputs, the view layer 128 + 3 (1 + 2 view_pe))."""
    rng = np.random.default_rng(seed)
    gx, gy, gz = grid
    hw, L = [(gy, gx), (gz, gx), (gz, gy)], [gz, gy, gx]
    fd = {"aabb": np.array([[-aabb] * 3, [aabb] * 3])}

    def draw(scale, c, shape):
        if coarse is None:
            return scale * rng.standard_normal((1, c, *shape))
        small = scale * rng.standard_normal((1, c, *[min(coarse, v) for v in shape]))
        return Fn.interpolate(torch.from_numpy(small), size=shape, mode="bilinear", align_corners=True).numpy()

    for i in range(3):
        fd[f"density_plane.{i}"] = draw(0.3, 8, hw[i])
        fd[f"density_line.{i}"] = draw(1.0, 8, (L[i], 1))
        fd[f"app_plane.{i}"] = draw(0.3, 24, hw[i])
        fd[f"app_line.{i}"] = draw(1.0, 24, (L[i], 1))
    fd["basis_mat.weight"] = 0.2 * rng.standard_normal((27, 72))
    n_in, n_view = 27 * (1 + 2 * fea_pe), 3 * (1 + 2 * view_pe)
    fd["renderModule.mlp.0.weight"] = 0.2 * rng.standard_normal((128, n_in)) / math.sqrt(1 + 2 * fea_pe)
    fd["renderModule.mlp.0.bias"] = 0.1 * rng.standard_normal(128)
    fd["renderModule.mlp.2.weight"] = 0.1 * rng.standard_normal((128, 128))
    fd["renderModule.mlp.2.bias"] = 0.1 * rng.standard_normal(128)
    fd["renderModule.mlp_view.0.weight"] = 0.3 * rng.standard_normal((3, 128 + n_view))
    fd["renderModule.mlp_view.0.bias"] = 0.1 * rng.standard_normal(3)
    if safe_mlp:
        sign = np.where(np.arange(128) % 2 == 0, 1.0, -1.0)
        fd["renderModule.mlp.0.weight"] *= 0.05
        fd["renderModule.mlp.0.bias"] = sign
        fd["renderModule.mlp.2.weight"] *= 0.05
        fd["renderModule.mlp.2.bias"] = sign.copy()        # its own array: Field64's two leaves would share storage
        fd["renderModule.mlp_view.0.weight"] *= 0.2         # keeps the sigmoid away from saturation
    scal = dict(density_shift=shift, distance_scale=25.0, rayMarch_weight_thres=thres, fea2denseAct=act,
                fea_pe=fea_pe, view_pe=view_pe, featureC=128, app_dim=27, step_ratio=0.5, gridSize=list(grid))
    fd.update({k: np.asarray(v) for k, v in scal.items()})
    if mask is not None:
        fd["alphaMask.alpha_volume"] = np.asarray(mask, np.float64)
        fd["alphaMask.aabb"] = fd["aabb"].copy()
    return fd


def _lookup(plane, line, q, i):
    """Plane i x line i at normalised points q [M, 3] -> products [M, C], their |.|, and the 3 un-clipped pixel
    coordinates with their sizes."""
    xp = torch.stack([q[:, MAT0[i]], q[:, MAT1[i]]], -1).view(1, -1, 1, 2)
    xl = torch.stack([torch.zeros_like(q[:, VEC[i]]), q[:, VEC[i]]], -1).view(1, -1, 1, 2)
    P = Fn.grid_sample(plane, xp, mode="bilinear", padding_mode="border", align_corners=True)[0, :, :, 0].t()
    Lc = Fn.grid_sample(line, xl, mode="bilinear", padding_mode="border", align_corners=True)[0, :, :, 0].t()
    return P * Lc


def ztable(S, far=True):
    """S increasing distances (fp32): S // 2 uniform steps from 0.1 to 1.1, then inverse-depth steps to 1000 (the
    shape of sample_ray_contracted's table); far = False: uniform to 4.1; a number: uniform to that distance."""
    if far is not True or S < 4:
        top = 1.1 if far is True else 4.1 if far is False else float(far)
        return torch.linspace(0.1, top, S, dtype=torch.float32)
    n1 = S // 2
    t = torch.arange(S - n1, dtype=torch.float64) / (S - n1)
    return torch.cat([0.1 + torch.arange(n1, dtype=torch.float64) / n1,
                      0.1 + 1.0 / (1.0 * (1 - t) + 1e-3 * t)]).float()


def make_rays(n, seed, spread=2.5):
    """fp32 rays [n, 6]: origins in [-spread, spread]^3 (outside the aabb of +-2 for some), |d| in [0.5, 2]."""
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g) * 2 - 1) * spread
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True) * (0.5 + 1.5 * torch.rand(n, 1, generator=g))
    return torch.cat([o, d], -1).contiguous()


def _abs_sum(keys, q, F):
    """sum over the components of |bilinear|(|plane|) x |linear|(|line|): the sum of the absolute values of every
    term a lookup's fp32 arithmetic adds, per point [M, C] (bilinear weights are >= 0)."""
    return [_lookup(F.p[a].detach().abs(), F.p[b].detach().abs(), q, i) for i, (a, b) in enumerate(keys)]


def _slope(fn, q, dq):
    """sum_a |d fn / d q_a| dq_a per point (fn: [M, 3] -> [M, K]) from one-sided differences on both sides, the
    larger taken (a step may cross into the neighbouring cell, whose slope then counts too)."""
    h = 1e-7
    f0 = fn(q)
    out = torch.zeros_like(f0)
    for a in range(3):
        e = torch.zeros_like(q)
        e[:, a] = h
        sl = torch.maximum((fn(q + e) - f0).abs(), (f0 - fn(q - e)).abs()) / h
        out = out + sl * dq[:, a:a + 1]
    return out


def _texel_margin(q, grid):
    """[M] smallest distance of the 3 un-clipped pixel coordinates (one per axis, shared by the plane and the line
    lookups along it) to an integer in [0, size - 1]."""
    out = torch.full(q.shape[:1], math.inf, dtype=q.dtype, device=q.device)
    for a in range(3):
        size = grid[a]
        x = (q[:, a] + 1) / 2 * (size - 1)
        k = torch.clamp(torch.round(x), 0, size - 1)
        out = torch.minimum(out, (x - k).abs() / (EPS * max(size, 2) * 4))
    return out


def _mask_value(F, p):
    """AlphaGridMask.sample_alpha at contracted points p [M, 3] -> (value [M], lattice margin [M])."""
    lo, hi = F.alpha_aabb[0], F.alpha_aabb[1]
    qn = (p - lo) * (2.0 / (hi - lo)) - 1
    v = Fn.grid_sample(F.alpha_vol, qn.view(1, -1, 1, 1, 3), mode="bilinear", padding_mode="zeros",
                       align_corners=True).reshape(-1)
    D, H, W = F.alpha_vol.shape[-3:]
    marg = torch.full_like(v, math.inf)
    for a, size in enumerate((W, H, D)):
        x = (qn[:, a] + 1) / 2 * (size - 1)
        marg = torch.minimum(marg, (x - torch.round(x)).abs() / (EPS * max(size, 2) * 4))
    return v, marg


def _pe(x, n_freq):
    """[sin(x_d 2^f), cos(x_d 2^f)] with d-major, f-minor order (tensorBase.py:14-21)."""
    bands = 2.0 ** torch.arange(n_freq, dtype=x.dtype, device=x.device)
    ang = (x[..., None] * bands).reshape(*x.shape[:-1], -1)
    return torch.cat([ang.sin(), ang.cos()], -1)


def _mlp(F, feats, vd, want_margin, qa=None, dqa=None, refine=True):
    """MLPRender_Fea_late_view on products feats [M, 72] -> rgb [M, 3], per-sample MLP margin [M] (in units of the
    pre-activations' fp32 error bound; qa / dqa: the shaded points and their position error).  fea_pe / view_pe:
    the 27 features, then sin, then cos of each feature times 2^f (zeros when refine is off); the view term
    likewise (always encoded)."""
    p = F.p
    x = feats @ p["basis_mat.weight"].t()
    enc = x
    if F.fea_pe:
        enc = torch.cat([x, _pe(x, F.fea_pe) if refine else x.new_zeros(x.shape[0], 2 * x.shape[1] * F.fea_pe)], -1)
    w1, b1, w2, b2 = p["renderModule.mlp.0.weight"], p["renderModule.mlp.0.bias"], p["renderModule.mlp.2.weight"], \
        p["renderModule.mlp.2.bias"]
    a1 = enc @ w1.t() + b1
    h1 = torch.relu(a1)
    a2 = h1 @ w2.t() + b2
    h2 = torch.relu(a2)
    v = vd if not F.view_pe else torch.cat([vd, _pe(vd, F.view_pe)], -1)
    s = torch.cat([h2, v], -1) @ p["renderModule.mlp_view.0.weight"].t() + p["renderModule.mlp_view.0.bias"]
    marg = None
    if want_margin:
        with torch.no_grad():
            # the kernels fold W1 @ basis into one 72-term product; the rounding of a long fp32 sum of independently
            # rounded terms grows as its square root (8 EPS of the sum of |terms| covers 72 and 128 terms), plus the
            # position error through the features' slope; layer 2: plus layer 1's error through |W2| on the units
            # that are on.  The tensor-core path's 16-bit products need a 2^8 larger margin (the tests' bound).
            keys = [(f"app_plane.{i}", f"app_line.{i}") for i in range(3)]
            fabs = torch.cat(_abs_sum(keys, qa, F), -1)
            prods = lambda qq: torch.cat([_lookup(p[a].detach(), p[b].detach(), qq, i)
                                          for i, (a, b) in enumerate(keys)], -1)
            w1d = w1.detach()
            if not (F.fea_pe or F.view_pe):
                w1b = w1d @ p["basis_mat.weight"].detach()
                e1 = 8 * EPS * (fabs @ w1b.abs().t() + b1.abs()) + _slope(lambda qq: prods(qq) @ w1b.t(), qa, dqa)
            else:
                # the 27 features are a sum of their own (layer 0); their error reaches layer 1 through the encoding:
                # 2^f times it in sin / cos of frequency f (x 2^f is exact), plus 4 EPS for sin / cos themselves
                basis = p["basis_mat.weight"].detach()
                e0 = 8 * EPS * (fabs @ basis.abs().t()) + _slope(lambda qq: prods(qq) @ basis.t(), qa, dqa)
                e_enc = e0
                if F.fea_pe:
                    bands = 2.0 ** torch.arange(F.fea_pe, dtype=e0.dtype, device=e0.device)
                    e_f = (e0[..., None] * bands).reshape(e0.shape[0], -1) + 4 * EPS
                    e_enc = torch.cat([e0, e_f, e_f] if refine else [e0, torch.zeros_like(e_f), torch.zeros_like(e_f)],
                                      -1)
                e1 = 8 * EPS * (enc.detach().abs() @ w1d.abs().t() + b1.abs()) + e_enc @ w1d.abs().t()
            e2 = 8 * EPS * (h1.abs() @ w2.abs().t() + b2.abs()) + (e1 * (a1 > 0)) @ w2.abs().t()
            marg = torch.minimum((a1.abs() / e1).amin(-1), (a2.abs() / e2).amin(-1))
    return torch.sigmoid(s), marg


def field_forward(F, rays, z, white_bg, want_margins=False, floater=0.0, refine=True):
    """TensorBase.forward on rays [n, 6] (float64, may require grad) with the distance table z [S] ->
    (rgb [n, 3], depth [n], extras dict: w [n, S] (after the floater filter) and, with want_margins, the margins,
    `texel` [n], `term` [n], and the early termination's `k_end`, `n_march` and `n_shade` [n])."""
    n, S = rays.shape[0], z.shape[0]
    dev, f64 = rays.device, torch.float64
    o, d = rays[:, :3], rays[:, 3:]
    nrm = d.norm(dim=-1, keepdim=True)
    vd = d / nrm
    zz = z.to(dev, f64)
    p = o[:, None, :] + vd[:, None, :] * zz[None, :, None]                       # [n, S, 3]
    amax = p.abs().amax(-1, keepdim=True).clamp_min(1e-6)
    pc = torch.where(amax <= 1, p, ((2 * amax - 1) / amax ** 2) * p)
    valid = torch.ones(n, S, dtype=torch.bool, device=dev)
    mk = {}
    if F.alpha_vol is not None:
        with torch.no_grad():
            mv, mlat = _mask_value(F, pc.detach().reshape(-1, 3))
        mv, mlat = mv.view(n, S), mlat.view(n, S)
        valid &= mv > 0
        mk["mask"] = torch.where(mv > 0, mv / EPS, mlat)
    valid[:, -1] = False
    aabb = F.aabb.to(dev)
    ainv = 2.0 / (aabb[1] - aabb[0])
    q = (pc - aabb[0]) * ainv - 1
    qv = q[valid]
    dq = None
    if want_margins:
        with torch.no_grad():
            # p = o + vd z carries 4 EPS (|o| + |z|); the contraction scales an error by at most 2 / max|p| beyond 1
            am_ = amax.detach()
            jac = torch.where(am_ <= 1, torch.ones_like(am_), 2 / am_)
            dpc = 4 * EPS * ((o.detach().abs().amax(-1)[:, None, None] + zz.abs()[None, :, None]) * jac
                             + pc.detach().abs().amax(-1, keepdim=True))
            dq = dpc * ainv + 2 * EPS * (q.detach().abs() + 1)
    fe = torch.zeros(n, S, dtype=f64, device=dev)
    if qv.shape[0]:
        prods = [_lookup(F.p[f"density_plane.{i}"], F.p[f"density_line.{i}"], qv, i) for i in range(3)]
        fe = fe.index_put((valid,), sum(pr.sum(-1) for pr in prods))
    if F.act == "softplus":
        sig = Fn.softplus(fe + F.shift)
    else:
        sig = torch.relu(fe)
    sig = torch.where(valid, sig, torch.zeros_like(sig))
    dist = torch.cat([zz[1:] - zz[:-1], zz.new_zeros(1)])
    alpha = 1.0 - torch.exp(-sig * dist[None] * F.scale)
    alpha = torch.cat([alpha[:, :-1], torch.ones_like(alpha[:, -1:])], -1)       # alpha[:, -1] = 1
    T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    w = alpha * T
    acc = w.sum(-1)
    depth = (w * zz[None]).sum(-1) / nrm[:, 0]
    wf, af, Tf = w, alpha, T
    if floater > 0:                         # tensorBase.py:617-620; acc and depth keep the pre-filter weights
        ks = torch.arange(S, dtype=f64, device=dev)
        idx = (w * ks).sum(-1, keepdim=True)
        af = torch.where(ks[None] < idx * floater, torch.zeros_like(alpha), alpha)
        af = torch.cat([af[:, :-1], torch.ones_like(af[:, -1:])], -1)
        Tf = torch.cumprod(torch.cat([torch.ones_like(af[:, :1]), 1.0 - af + 1e-10], -1), -1)[:, :-1]
        wf = af * Tf
    app = wf > F.thres
    rgb_s = torch.zeros(n, S, 3, dtype=f64, device=dev)
    mlp_m = torch.full((n, S), math.inf, dtype=f64, device=dev)
    if app.any():
        qa = q[app]
        feats = torch.cat([_lookup(F.p[f"app_plane.{i}"], F.p[f"app_line.{i}"], qa, i) for i in range(3)], -1)
        vda = vd[:, None, :].expand(n, S, 3)[app].detach()
        col, mm = _mlp(F, feats, vda, want_margins, qa.detach(), dq[app] if want_margins else None, refine)
        rgb_s = rgb_s.index_put((app,), col)
        if want_margins:
            mlp_m[app] = mm
    rgb = (wf[..., None] * rgb_s).sum(-2)
    if white_bg:
        rgb = rgb + (1.0 - acc)[:, None]
    ex = {"w": wf.detach()}
    if not want_margins:
        return rgb, depth, ex
    with torch.no_grad():
        inf = torch.full((n, S), math.inf, dtype=f64, device=dev)
        pa = p.detach().abs()
        pscale = (o.detach().abs().amax(-1, keepdim=True) + zz[None].abs()) * EPS      # [n, S]
        am = amax.detach()[..., 0]
        top2 = pa.topk(2, dim=-1).values
        mk["contract"] = torch.minimum((am - 1).abs() / pscale,
                                       torch.where(am > 1, (top2[..., 0] - top2[..., 1]) / pscale, inf))
        x = (fe.detach() + F.shift)
        dsig = torch.sigmoid(x) if F.act == "softplus" else (fe.detach() > 0).to(f64)
        a, Td, wd, sg = alpha.detach(), T.detach(), w.detach(), sig.detach()
        # the density feature: 8 roundings per product and a 24-term sum (32 EPS of the sum of |terms|), plus the
        # position error through the feature's slope
        df = torch.zeros(n, S, dtype=f64, device=dev)
        if qv.shape[0]:
            keys = [(f"density_plane.{i}", f"density_line.{i}") for i in range(3)]
            fsum = lambda qq: sum(_lookup(F.p[a_].detach(), F.p[b_].detach(), qq, i).sum(-1, keepdim=True)
                                  for i, (a_, b_) in enumerate(keys))
            df[valid] = 32 * EPS * sum(t.sum(-1) for t in _abs_sum(keys, qv.detach(), F)) \
                + _slope(fsum, qv.detach(), dq[valid])[:, 0]
        # sigma, x = sigma dist scale, alpha = 1 - exp(-x): a few roundings each, and the inherited error
        dx = (dsig * df + 4 * EPS * sg) * dist[None] * F.scale + 4 * EPS * sg * dist[None] * F.scale
        last = torch.zeros(n, S, dtype=torch.bool, device=dev)
        last[:, -1] = True
        dalpha = torch.where(valid & ~last, (1 - a) * (dx + 4 * EPS) + EPS, torch.zeros_like(a))
        # T_k = prod_{j < k} ((1 - alpha_j) + 1e-10): each factor's relative error (its alpha's error over the
        # factor, and 3 roundings) accumulates along the ray; w = alpha T
        fac = (1 - a) + 1e-10
        rel = dalpha / fac + 3 * EPS
        relT = torch.cumsum(rel, -1) - rel
        # below 2^-126 fp32 is subnormal: its rounding there is absolute (and products flush to 0)
        ex["w_err"] = Td * dalpha + wd * (relT + EPS) + 2.0 ** -126
        ks = torch.arange(S, dtype=f64, device=dev)
        ta, tT, tw, terr = a, Td, wd, ex["w_err"]
        if floater > 0:
            # the cut k < idx thresh against the nearest integer; idx = sum_k w_k k carries each weight's error times
            # k and the rounding of the kernel's sum (per lane ceil(S / 32) terms in sequence, then a warp tree)
            idx = (wd * ks).sum(-1)
            lim = idx * floater
            kr = torch.round(lim)
            idx_err = (ex["w_err"] * ks).sum(-1) + ((S + 31) // 32 + 6) * EPS * idx
            fm = (lim - kr).abs() / (idx_err * floater + EPS * lim + 1e-300)
            a_at = a.gather(1, kr.long().clamp(0, S - 1)[:, None])[:, 0]
            mk["floater"] = torch.where((kr >= S - 1) | (a_at == 0), torch.full_like(fm, math.inf), fm)[:, None]
            # the filtered product restarts at 1 and carries the errors of the alphas it keeps
            ta, tT, tw = af.detach(), Tf.detach(), wf.detach()
            daf = torch.where(ta == a, dalpha, torch.zeros_like(dalpha))
            relf = daf / ((1 - ta) + 1e-10) + 3 * EPS
            terr = tT * daf + tw * (torch.cumsum(relf, -1) - relf + EPS) + 2.0 ** -126
            ex["w_err"] = terr
        mk["thres"] = (tw - F.thres).abs() / terr
        if F.thres <= 0:      # an fp32 T below ~2^-126 is 0, and its w then fails w > 0 where float64's passes
            mk["thres"] = torch.where(tT < 2.0 ** -100, torch.zeros_like(tw), mk["thres"])
        mk["thres"] = torch.where(ta == 0, inf, mk["thres"])    # sigma exactly 0 (or cut): w = 0 on both sides
        # early termination (floater 0): the march stops after the 32-sample block whose end leaves T < 1e-10
        nb = (S + 31) // 32
        ends = torch.clamp(torch.arange(nb, device=dev) * 32 + 31, max=S - 1)
        Tb = torch.cumprod(fac, -1)[:, ends]
        eb = torch.cumsum(rel, -1)[:, ends]
        hit = Tb < T_TERM                  # (an empty ray's last factor, (1 + 1e-10)^S 1e-10, can end above 1e-10f)
        b_term = torch.where(hit.any(-1), hit.to(torch.int64).argmax(-1), nb - 1)
        tm = (Tb - T_TERM).abs() / (Tb * eb + T_TERM * EPS)
        reached = torch.arange(nb, device=dev)[None] <= b_term[:, None]
        tm = torch.where(reached & (torch.arange(nb, device=dev)[None] < nb - 1), tm, torch.full_like(tm, math.inf))
        k_end = torch.clamp((b_term + 1) * 32, max=S)
        if floater > 0:                                         # the filter marches every sample
            k_end, tm = torch.full_like(k_end, S), torch.full_like(tm, math.inf)
        before = ks[None] < k_end[:, None]
        ex["k_end"] = k_end
        ex["term"] = tm.amin(-1)
        ex["n_march"] = (valid & before).sum(-1)
        ex["n_shade"] = (app & before).sum(-1)
        if F.act == "softplus":
            mk["softplus"] = torch.where(valid, (x - 20).abs() / (df + 20 * EPS), inf)
        else:
            mk["relu_f"] = torch.where(valid, fe.detach().abs() / df.clamp_min(1e-300), inf)
        mk["mlp"] = mlp_m
        tex = torch.full((n, S), math.inf, dtype=f64, device=dev)
        # texel floors matter where a lookup's position gradient is used: valid samples (density) and shaded ones
        used = valid | app
        tq = _texel_margin(q.detach()[used], F.grid)
        tex[used] = tq
        ex["texel"] = tex.amin(-1)
        for key in MARGIN_KEYS:
            ex[key] = mk[key].amin(-1) if key in mk else torch.full((n,), math.inf, dtype=f64, device=dev)
        ex["n_app"] = app.sum(-1)
    return rgb, depth, ex


def field_backward(F, rays, z, white_bg, g_rgb, g_depth, want_margins=True, chunk_samples=CHUNK_SAMPLES,
                   floater=0.0, refine=True):
    """Chunked forward + autograd: -> (grads dict keyed like PARAM_KEYS plus "rays" [n, 6], forward dict with
    rgb, depth, w and the per-ray margins).  Cotangents may be zero on any ray: that ray then adds exactly nothing.
    floater / refine as in field_forward (the floater cut is a hard switch: no gradient flows through idx)."""
    dev = F.device
    rays = torch.as_tensor(rays).to(dev, torch.float64)
    g_rgb = torch.as_tensor(g_rgb).to(dev, torch.float64)
    g_depth = torch.as_tensor(g_depth).to(dev, torch.float64)
    z = torch.as_tensor(z).to(dev, torch.float64)
    n, S = rays.shape[0], z.shape[0]
    step = max(1, chunk_samples // S)
    grads = {k: torch.zeros_like(v) for k, v in F.p.items()}
    d_rays = torch.zeros(n, 6, dtype=torch.float64, device=dev)
    fwd = {}
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        rc = rays[r0:r1].clone().requires_grad_(True)
        rgb, depth, ex = field_forward(F, rc, z, white_bg, want_margins, floater, refine)
        loss = (rgb * g_rgb[r0:r1]).sum() + (depth * g_depth[r0:r1]).sum()
        keys = list(F.p)
        gs = torch.autograd.grad(loss, [rc] + [F.p[k] for k in keys], allow_unused=True)
        d_rays[r0:r1] = gs[0]
        for k, g in zip(keys, gs[1:]):
            if g is not None:
                grads[k] += g
        ex["rgb"], ex["depth"] = rgb.detach(), depth.detach()
        for k, v in ex.items():
            fwd.setdefault(k, []).append(v)
    grads["rays"] = d_rays
    return grads, {k: torch.cat(v) for k, v in fwd.items()}


def forward_chunked(F, rays, z, white_bg, floater=0.0, refine=True, chunk_samples=CHUNK_SAMPLES):
    """field_forward with margins, without autograd, in chunks of rays -> dict: rgb, depth, w and the extras."""
    dev = F.device
    rays = torch.as_tensor(rays).to(dev, torch.float64)
    z = torch.as_tensor(z).to(dev, torch.float64)
    step = max(1, chunk_samples // z.shape[0])
    out = {}
    with torch.no_grad():
        for r0 in range(0, rays.shape[0], step):
            rgb, depth, ex = field_forward(F, rays[r0:r0 + step], z, white_bg, True, floater, refine)
            ex["rgb"], ex["depth"] = rgb, depth
            for k, v in ex.items():
                out.setdefault(k, []).append(v)
    return {k: torch.cat(v) for k, v in out.items()}


def clear(fwd, bound=2.0, margin=64.0, mlp_bound=None):
    """Per ray: True where every decision margin clears its bound -- `bound` for the margins in units of a propagated
    error bound (BOUND_KEYS; `mlp_bound` for the MLP when given), `margin` for the others (EPS units)."""
    ok = torch.ones_like(fwd["thres"], dtype=torch.bool)
    for k in MARGIN_KEYS:
        b = (mlp_bound if mlp_bound is not None and k == "mlp" else bound) if k in BOUND_KEYS else margin
        ok &= fwd[k] >= b
    return ok


def min_margin(fwd, keys=MARGIN_KEYS):
    """Per ray, the smallest of the given margins."""
    return torch.stack([fwd[k] for k in keys]).amin(0)


# ---- the camera side -------------------------------------------------------------------------------------------
def directions(ray_ids, W, H, intr, fov360):
    """Camera-space directions [n, 3] (get_ray_directions_lean / _360); intr = (focal, cx, cy) float64 tensor."""
    ids = ray_ids.to(torch.int64)
    i = (ids % W).to(intr.dtype) + 0.5
    j = ((ids // W) % H).to(intr.dtype) + 0.5
    if fov360:
        phi = j * math.pi / H - math.pi / 2
        theta = i * 2 * math.pi / W + math.pi
        return torch.stack([torch.cos(phi) * torch.sin(theta), torch.sin(phi), torch.cos(phi) * torch.cos(theta)], -1)
    return torch.stack([(i - intr[1]) / intr[0], -(j - intr[2]) / intr[0], -torch.ones_like(i)], -1)


def render_views(fields, z, ray_ids, W, H, fov360, intr, c2w, w2rf, blend, E, white_bg, floater=0.0, refine=True,
                 finalize=True):
    """The eval call of LocalTensorfs.forward in float64 (local_tensorfs.py:397-499): each ray's camera-space
    direction and pixel from its id, its view r // (n / V), then for every field f the rays t_v + world2rf_f and
    R_v dir, rendered and blended: rgb = sum_f blend[v, f] rgb_f (likewise depth); with `finalize`, clamp(E_v rgb, 0,
    1) (E None: clamp only).  fields: Field64 list; w2rf: one [3] per field (or None); blend [V, n_fields] or None
    (weight 1).  -> dict: rgb, depth, dirs [n, 3], ij [n, 2], per-field forward dicts `fwd` (forward_chunked), and
    every margin and count of forward_chunked combined over the fields (smallest margin, summed counts)."""
    dev, f64 = fields[0].device, torch.float64
    T = lambda a: torch.as_tensor(a).to(dev, f64)
    ray_ids = torch.as_tensor(ray_ids).to(dev)
    n, V = ray_ids.shape[0], c2w.shape[0]
    view = torch.arange(n, device=dev) // (n // V)
    c2w, intr = T(c2w), T(intr)
    dirs = directions(ray_ids, W, H, intr, fov360)
    rays_d = (c2w[view, :, :3] @ dirs[:, :, None])[..., 0]
    rgb = torch.zeros(n, 3, dtype=f64, device=dev)
    depth = torch.zeros(n, dtype=f64, device=dev)
    out = {"fwd": []}
    for f, F in enumerate(fields):
        o = c2w[view, :, 3] + (T(w2rf[f]) if w2rf is not None and w2rf[f] is not None else 0.0)
        fw = forward_chunked(F, torch.cat([o, rays_d], -1), z, white_bg, floater, refine)
        b = T(blend)[view, f] if blend is not None else torch.ones(n, dtype=f64, device=dev)
        rgb = rgb + b[:, None] * fw["rgb"]
        depth = depth + b * fw["depth"]
        out["fwd"].append(fw)
        for k in MARGIN_KEYS + ("texel", "term"):
            out[k] = torch.minimum(out[k], fw[k]) if k in out else fw[k]
        for k in ("n_march", "n_shade"):
            out[k] = out[k] + fw[k] if k in out else fw[k]
    if finalize:
        if E is not None:
            rgb = torch.einsum("nab,nb->na", T(E)[view], rgb)
        rgb = rgb.clamp(0, 1)
    ids = ray_ids.to(torch.int64)
    out.update(rgb=rgb, depth=depth, dirs=dirs, ij=torch.stack([ids % W, (ids // W) % H], -1))
    return out


def train_backward(F, z, ray_ids, W, H, fov360, intr, c2w, w2rf, E, x, white_bg, g_rgb, g_depth, g_dirs,
                   chunk_samples=CHUNK_SAMPLES):
    """The training call's gradients in float64: rays from the cameras, the field, rgb = clamp(E_v x, 0, 1) with the
    forward's pre-exposure colour x given (its gradient reaches the field as E^T g'), depth, directions.  E may be
    None (identity).  -> (grads dict: the field's as field_backward plus d_cam2world [V, 3, 4], d_intrinsics [3],
    d_exposure [V, 3, 3], d_world2rf [3]; forward dict with the field's margins, `clamp` = the per-ray distance of
    E x to 0 and 1 in units of its rounding (inf where it is exactly 0 or 1: both sides then agree), and the
    generated rays)."""
    dev, f64 = F.device, torch.float64
    T = lambda a: torch.as_tensor(a).to(dev, f64)
    ray_ids = torch.as_tensor(ray_ids).to(dev)
    n, V = ray_ids.shape[0], c2w.shape[0]
    view = torch.arange(n, device=dev) // (n // V)
    c2w = T(c2w).requires_grad_(True)
    intr = T(intr).requires_grad_(True)
    w2rf = T(w2rf).requires_grad_(True)
    Ev = T(E).requires_grad_(True) if E is not None else torch.eye(3, dtype=f64, device=dev).expand(V, 3, 3)
    x, g_rgb, g_depth = T(x), T(g_rgb), T(g_depth)
    g_dirs = T(g_dirs) if g_dirs is not None else torch.zeros(n, 3, dtype=f64, device=dev)
    dirs = directions(ray_ids, W, H, intr, fov360)
    R = c2w[view, :, :3]
    rays_o = c2w[view, :, 3] + w2rf
    rays_d = (R @ dirs[:, :, None])[..., 0]
    rays = torch.cat([rays_o, rays_d], -1)
    # the field part through rays (chunked), then the camera graph once with the rays' gradient
    with torch.no_grad():
        y = torch.einsum("nab,nb->na", Ev[view], x)
        gp = g_rgb * ((y >= 0) & (y <= 1))
        g_lin = torch.einsum("nab,na->nb", Ev[view], gp)
        ysc = torch.einsum("nab,nb->na", Ev[view].abs(), x.abs())
        clamp = torch.minimum(y.abs(), (y - 1).abs()) / (EPS * ysc.clamp_min(1e-300))
        clamp = torch.where((y == 0) | (y == 1), torch.full_like(clamp, math.inf), clamp).amin(-1)
    grads, fwd = field_backward(F, rays.detach(), z, white_bg, g_lin, g_depth, chunk_samples=chunk_samples)
    loss = (rays * grads["rays"]).sum() + (dirs * g_dirs).sum()
    yx = torch.einsum("nab,nb->na", Ev[view], x)
    loss = loss + (torch.clamp(yx, 0, 1) * g_rgb).sum()
    leaves = [c2w, intr, w2rf] + ([Ev] if E is not None else [])
    gs = torch.autograd.grad(loss, leaves, allow_unused=True)
    grads["d_cam2world"], grads["d_intrinsics"], grads["d_world2rf"] = (
        g if g is not None else torch.zeros_like(l) for g, l in zip(gs[:3], leaves[:3]))
    if E is not None:
        grads["d_exposure"] = gs[3]
    else:                                                   # the gradient at the identity: sum over a view of g' x^T
        grads["d_exposure"] = torch.zeros(V, 3, 3, dtype=f64, device=dev).index_add_(0, view, gp[:, :, None] * x[:, None, :])
    fwd["clamp"] = clamp
    fwd["rays"] = rays.detach()
    fwd["dirs"] = dirs.detach()
    return grads, fwd
