"""Float64 torch restatement of the supervision losses of train.py:369-423 (the rgb, flow-reprojection and
mono-depth terms), written from the formulas, and the fp32 selection formulas the kernels use.

    losses_f64(case)            -> (losses [3] float64, {name: gradient}) for a dict of inputs
    losses_f64(case, decisions=decisions_of(arrays))
                                -> the same with the kernel's cuts and medians (the arithmetic stays float64)
    quantile_fp32(rows, q)      -> torch.quantile(rows, q, dim=1) in fp32, restated (numpy)
    lower_median(rows)          -> (values, indices) of torch.median(rows, dim=1), ties to the lowest index
    torch_block(kw)             -> the three losses as the reference's train.py computes them, in torch ops on
                                   the inputs' device and dtype (the baseline of tools/loss_time.py)
"""
import numpy as np
import torch

GRAD_NAMES = ("rgb_map", "depth_map", "directions", "cam2world", "focal", "center")


def _fma32(a, b, c):
    """fp32 fused multiply-add (the float64 product of two fp32 values is exact; one rounding of the sum)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def quantile_fp32(rows, q):
    """Linear-interpolation quantile of each row as torch computes it in fp32: rank fp32(q) * (R - 1) rounded to
    fp32, neighbours floor / ceil of the rank, and ATen's lerp (weight < 0.5: a + w (b - a), else
    b - (b - a)(1 - w), each fused).  A row with a NaN gives NaN."""
    rows = np.asarray(rows, dtype=np.float32)
    s = np.sort(rows, axis=1)
    R = s.shape[1]
    r = np.float32(np.float32(q) * np.float32(R - 1))
    lo, hi = int(np.floor(r)), int(np.ceil(r))
    w = np.float32(r - np.float32(lo))
    a, b = s[:, lo], s[:, hi]
    diff = (b - a).astype(np.float32)
    if abs(w) < 0.5:
        out = _fma32(np.full_like(a, w), diff, a)
    else:
        out = _fma32(-diff, np.full_like(a, np.float32(1) - w), b)
    return np.where(np.isnan(rows).any(axis=1), np.float32(np.nan), out)


def lower_median(rows):
    """sorted[(R - 1) // 2] of each row and the lowest index holding that value."""
    rows = np.asarray(rows)
    k = (rows.shape[1] - 1) // 2
    vals = np.sort(rows, axis=1)[:, k]
    idx = np.argmax(rows == vals[:, None], axis=1)
    return vals, idx


def _quantile_f64(x, q):
    """The same interpolation on float64 rows, with torch's fp32 rank and weight."""
    R = x.shape[1]
    r = np.float32(np.float32(q) * np.float32(R - 1))
    lo, hi = int(np.floor(r)), int(np.ceil(r))
    w = float(np.float32(r - np.float32(lo)))
    s = torch.sort(x, dim=1).values
    return s[:, lo] + w * (s[:, hi] - s[:, lo])


def _median_index(x):
    k = (x.shape[1] - 1) // 2
    return torch.sort(x, dim=1, stable=True).indices[:, k]


def losses_f64(c, flow_weight=None, depth_weight=None, return_arrays=False, decisions=None):
    """c: dict of the inputs (numpy or tensors, as stored in tests/golden/train_losses.npz).  Gradients of
    L_rgb + L_flow + L_depth with respect to GRAD_NAMES, in float64.

    decisions: None (the selections are made here, in float64), or a dict of the hard decisions to use instead:
    "flow_cut" and "depth_cut" (bool [V,R], the rays zeroed above the thresholds) and "median_x" / "median_g"
    (int [V], the ray within each view whose 1 / clamp(depth) and invdepths are the medians).  The kernels'
    return_arrays=True output gives all four (decisions_of); return_arrays=True here returns this call's own
    under "decisions".  Everything else stays float64: at ties or within rounding of a threshold the float64
    selections may differ from fp32 ones, and this keeps the arithmetic comparable there."""
    t = lambda k, dt=torch.float64: torch.as_tensor(np.asarray(c[k])).to(dt)
    p = {k: t(k).clone().requires_grad_() for k in GRAD_NAMES}
    view_ids = t("view_ids", torch.int64)
    V = view_ids.shape[0]
    n_cams = p["cam2world"].shape[0]
    fw = float(c["flow_weight"] if flow_weight is None else flow_weight)
    dw = float(c["depth_weight"] if depth_weight is None else depth_weight)
    w = t("loss_weights").reshape(-1, 1)

    rgb = (0.25 * torch.abs(p["rgb_map"] - t("rgb_train")) * w / w.mean()).mean()

    # flow: q = Rcc p + tcc with Rcc = Rk^T Rrel, tcc = Rk^T (trel - tk), k = clamp(rel +- 1)
    depth = p["depth_map"].reshape(V, -1)
    pts = p["directions"].reshape(V, -1, 3) * depth[..., None]
    ij = t("ij").reshape(V, -1, 2)
    rel = view_ids - int(c["starting_id"])
    Rm, tv = p["cam2world"][..., :3], p["cam2world"][..., 3]
    f, cx, cy = p["focal"].reshape(()), p["center"].reshape(-1)[0], p["center"].reshape(-1)[1]
    e = 0
    for off, flow_key, mask in ((-1, "bwd_flow", t("bwd_mask").reshape(V, -1)),
                                (1, "fwd_flow", t("fwd_mask").reshape(V, -1) * (view_ids != n_cams - 1)[:, None])):
        k = torch.clamp(rel + off, 0, n_cams - 1)
        Rk, Rr = Rm[k], Rm[rel]
        Rcc = Rk.transpose(1, 2) @ Rr
        tcc = (Rk.transpose(1, 2) @ (tv[rel] - tv[k])[..., None])[..., 0]
        q = torch.einsum("vij,vrj->vri", Rcc, pts) + tcc[:, None, :]
        z = torch.clamp(-q[..., 2], min=1e-6)
        u = q[..., 0] / z * f + cx - 0.5 - ij[..., 0]
        v = -q[..., 1] / z * f + cy - 0.5 - ij[..., 1]
        fl = t(flow_key).reshape(V, -1, 2)
        e = e + (torch.abs(u - fl[..., 0]) + torch.abs(v - fl[..., 1])) * mask
    given = {} if decisions is None else decisions
    own = {}
    pick = lambda k, dt: torch.as_tensor(given[k]).cpu().to(dt) if given.get(k) is not None else own[k]
    tau_f = _quantile_f64(e.detach(), 0.9)
    own["flow_cut"] = e.detach() > tau_f[:, None]
    flow = torch.where(pick("flow_cut", torch.bool), 0, e).mean() * fw

    # depth: lower medians, mean absolute deviations
    def norm(x, key):
        own[key] = _median_index(x.detach())
        m = torch.gather(x, 1, pick(key, torch.int64)[:, None])
        return (x - m) / torch.abs(x - m).mean(dim=1, keepdim=True)
    d = (norm(1 / torch.clamp(depth, min=1e-6), "median_x") - norm(t("invdepths").reshape(V, -1), "median_g")) ** 2
    tau_d = _quantile_f64(d.detach(), 0.8)
    own["depth_cut"] = d.detach() > tau_d[:, None]
    dl = torch.where(pick("depth_cut", torch.bool), 0, d).mean() * dw

    (rgb + flow + dl).backward()
    losses = torch.stack([rgb, flow, dl]).detach()
    grads = {k: p[k].grad for k in GRAD_NAMES}
    if return_arrays:
        return losses, grads, {"flow": e.detach(), "depth": d.detach(), "flow_tau": tau_f, "depth_tau": tau_d,
                               "decisions": own}
    return losses, grads


def decisions_of(arr, flow=True, depth=True):
    """The hard decisions in supervision_losses(..., return_arrays=True)'s arrays, as losses_f64 takes them: the
    cuts are the kernel's rows above the kernel's thresholds.  A term the call did not compute (flow / depth
    False) leaves its parts out, and losses_f64 makes those selections itself."""
    out = {}
    if flow:
        out["flow_cut"] = (arr["flow"] > arr["flow_tau"][:, None]).cpu()
    if depth:
        idx = arr["depth_median_index"].long().cpu()
        out.update(depth_cut=(arr["depth"] > arr["depth_tau"][:, None]).cpu(), median_x=idx[:, 0],
                   median_g=idx[:, 1])
    return out


def torch_block(kw):
    """train.py:369-423 restated in torch, as the reference runs it on the device."""
    V = kw["view_ids"].shape[0]
    w = kw["loss_weights"]
    rgb = (0.25 * (torch.abs(kw["rgb_map"] - kw["rgb_train"]) * w) / w.mean()).mean()
    d = kw["depth_map"].view(V, -1)
    c2w = kw["cam2world"]
    fm = kw["fwd_mask"].view(V, -1).clone()
    fm[kw["view_ids"] == len(c2w) - 1] = 0
    e = torch.zeros_like(d)
    pts = kw["directions"].view(V, -1, 3) * d[..., None]
    rel = kw["view_ids"] - kw["starting_id"]
    for off, fl, m in ((-1, kw["bwd_flow"], kw["bwd_mask"].view(V, -1)), (1, kw["fwd_flow"], fm)):
        k = torch.clamp(rel + off, 0, len(c2w) - 1)
        Rk = c2w[k, :, :3].transpose(1, 2)
        q = pts @ (Rk @ c2w[rel, :, :3]).transpose(1, 2) + (Rk @ (c2w[rel, :, 3:] - c2w[k, :, 3:]))[:, None, :, 0]
        z = torch.clip(-q[..., 2], min=1e-6)
        u = q[..., 0] / z * kw["focal"] + kw["center"][0] - 0.5 - kw["ij"].view(V, -1, 2)[..., 0]
        v = -q[..., 1] / z * kw["focal"] + kw["center"][1] - 0.5 - kw["ij"].view(V, -1, 2)[..., 1]
        f = fl.view(V, -1, 2)
        e = e + (torch.abs(u - f[..., 0]) + torch.abs(v - f[..., 1])) * m
    e[e > torch.quantile(e, 0.9, dim=1)[..., None]] = 0
    x = 1 / d.clamp(1e-6)
    xn = (x - x.median(1, keepdim=True).values) / (x - x.median(1, keepdim=True).values).abs().mean(1, keepdim=True)
    g = kw["invdepths"].view(V, -1)
    gn = (g - g.median(1, keepdim=True).values) / (g - g.median(1, keepdim=True).values).abs().mean(1, keepdim=True)
    dd = (xn - gn) ** 2
    dd[dd > torch.quantile(dd, 0.8, dim=1)[..., None]] = 0
    return rgb, e.mean() * kw["flow_weight"], dd.mean() * kw["depth_weight"]
