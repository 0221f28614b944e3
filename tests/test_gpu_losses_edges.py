"""-m gpu: the supervision losses (localrf_b200.supervision_losses, lrf_losses.cu) at the shapes and values where
a sort-and-select kernel goes wrong: several views of more than 256 rays, non-power-of-two rays per view (padded
sort keys), more than 256 views (the final kernels' second stride), ties, clamped depths, infinities and NaNs of
either sign, and the edge cameras.

Every case checks:
  * the decisions exactly, on the device: flow_tau / depth_tau are torch.quantile over the kernel's own rows as
    int32 bit patterns, the cut sets are `rows > torch.quantile(...)`, and the medians are torch.median's values
    at the lowest ray index holding them;
  * the arithmetic against the float64 restatement fed the kernel's decisions (losses_f64(decisions=...)): each
    loss within 1e-6 of its value, each gradient within 1e-5 of the tensor's max |gradient| (one exception, at
    R = 2, is measured and explained in test_shapes);
  * where nothing ties, each loss within 1e-5 of the reference's block as torch ops on the device (O.torch_block).
    At ties CUDA torch.median does not promise which tied ray it returns, so gradients are never compared with
    torch's autograd here.
With non-finite inputs each loss is NaN, infinite or finite exactly where torch_block's is, and the finite ones
meet the bars above (gradients are compared when every computed loss is finite).
"""
import numpy as np
import pytest
import torch

import losses_oracle as O

pytestmark = pytest.mark.gpu

FW, DW = 1.0 / 750.0, 0.1                       # loss_flow_weight_inital / ((960 + 540) / 2), depth weight
FLOW_NAMES = ("directions", "cam2world", "focal", "center")


def batch(seed, V, R, n_frames=40, starting_id=12, view_ids=None):
    """test_gpu_losses.training_batch for any V, R and camera count, on the CPU: cam2world [n_frames -
    starting_id, 3, 4] from 6-D rotations as LocalTensorfs.get_cam2world builds it.  Without view_ids, view 0
    is at starting_id and view 1 at the absolute id n_cams - 1 (whose forward mask the reference zeroes)."""
    from localrf_b200.utils import sixD_to_mtx
    g = torch.Generator().manual_seed(seed)
    N, n_cams = V * R, n_frames - starting_id
    r = torch.eye(3, 2) + 0.02 * torch.randn(n_cams, 3, 2, generator=g)
    t = 0.02 * torch.randn(n_cams, 3, generator=g)
    t[:, 2] -= 0.1 * torch.arange(starting_id, n_frames)
    if view_ids is None:
        view_ids = torch.randint(starting_id, n_frames, (V,), generator=g)
        view_ids[0] = starting_id
        if V > 1 and n_cams - 1 >= starting_id:
            view_ids[1] = n_cams - 1
    kw = {
        "rgb_map": torch.rand(N, 3, generator=g), "rgb_train": torch.rand(N, 3, generator=g),
        "loss_weights": 0.2 + torch.rand(N, 1, generator=g), "view_ids": torch.as_tensor(view_ids),
        "depth_map": 0.5 + 4.5 * torch.rand(N, generator=g),
        "directions": torch.cat([torch.rand(N, 2, generator=g) - 0.5, -torch.ones(N, 1)], 1),
        "ij": torch.stack([torch.randint(0, 960, (N,), generator=g), torch.randint(0, 540, (N,), generator=g)], 1),
        "focal": torch.tensor([500.0]), "center": torch.tensor([480.0, 270.0]),
        "fwd_flow": 3 * torch.randn(N, 2, generator=g), "bwd_flow": 3 * torch.randn(N, 2, generator=g),
        "fwd_mask": (torch.rand(N, generator=g) > 0.2).float(), "bwd_mask": (torch.rand(N, generator=g) > 0.2).float(),
        "invdepths": torch.rand(N, generator=g) + 0.1,
        "cam2world": torch.cat([sixD_to_mtx(r), t[..., None]], -1), "starting_id": starting_id,
    }
    if R <= 3:
        # x and g ordered alike tie d structurally: for R = 2 xn = gn = {0, 2} and d is rounding noise of 0; for
        # R = 3 xn and gn are {-a, 0, 3 - a} and the two nonzero d are equal, so which one is cut is rounding
        # noise.  g = 0.2 depth orders them oppositely (x = 1 / depth).
        kw["invdepths"] = 0.2 * kw["depth_map"]
    return kw


def run(kw, fw=FW, dw=DW):
    """supervision_losses on the device with fresh leaves -> (device inputs, losses, arrays, gradients)."""
    from localrf_b200 import supervision_losses
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}
    for k in O.GRAD_NAMES:
        d[k].requires_grad_()
    args = {k: v for k, v in d.items() if k not in ("rgb_map", "rgb_train", "loss_weights")}
    *losses, arr = supervision_losses(d["rgb_map"], d["rgb_train"], d["loss_weights"], **args, flow_weight=fw,
                                      depth_weight=dw, return_arrays=True)
    sum(l for l in losses if l is not None).backward()
    grads = {k: d[k].grad for k in O.GRAD_NAMES}
    return d, losses, arr, grads


def check_decisions(d, arr, flow, depth):
    V = d["view_ids"].shape[0]
    for on, key, q in ((flow, "flow", 0.9), (depth, "depth", 0.8)):
        if not on:
            continue
        rows, tau = arr[key], arr[f"{key}_tau"]
        want = torch.quantile(rows, q, dim=1)
        assert torch.equal(tau.view(torch.int32), want.view(torch.int32)), (key, tau, want)
        assert torch.equal(rows > tau[:, None], rows > want[:, None]), key
    if depth:
        x = 1 / d["depth_map"].detach().view(V, -1).clamp(1e-6)
        g = d["invdepths"].view(V, -1)
        idx = arr["depth_median_index"].long()
        for col, rows in ((0, x), (1, g)):
            med = torch.median(rows, dim=1).values
            got = rows.gather(1, idx[:, col:col + 1])[:, 0]
            assert torch.equal(got.isnan(), med.isnan()), col
            assert torch.equal(got[~got.isnan()], med[~med.isnan()]), col
            holds = (rows == med[:, None]) | (rows.isnan() & med.isnan()[:, None])
            assert torch.equal(idx[:, col], holds.int().argmax(dim=1)), (col, idx[:, col], holds.int().argmax(1))


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64).reshape(np.shape(a))
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def check(kw, fw=FW, dw=DW, ties=False, grad_bars=None):
    """Runs one case through every check of the module docstring; returns what run() returned.  grad_bars:
    {name: bar} for a gradient that needs a looser bar than 1e-5 (its test says why)."""
    flow, depth = fw != 0, dw != 0
    d, losses, arr, grads = run(kw, fw, dw)
    assert (losses[1] is not None) == flow and (losses[2] is not None) == depth
    check_decisions(d, arr, flow, depth)
    on = [0] + [1] * flow + [2] * depth
    got = torch.stack([losses[i] for i in on]).detach().cpu().double()

    # torch's block on the device: the same NaN / inf / finite pattern, and within 1e-5 where nothing ties
    with torch.no_grad():
        plain = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in d.items()}
        tb = torch.stack(O.torch_block(dict(plain, flow_weight=fw, depth_weight=dw))).cpu().double()[on]
    assert torch.equal(got.isnan(), tb.isnan()) and torch.equal(got.isinf(), tb.isinf()), (got, tb)
    assert torch.equal(got[got.isinf()], tb[tb.isinf()])
    fin = got.isfinite()
    if not ties:
        assert ((got - tb).abs()[fin] <= 1e-5 * tb.abs()[fin]).all(), (got, tb)

    # float64 arithmetic on the kernel's decisions
    case = {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in kw.items()}
    l64, g64 = O.losses_f64(case, flow_weight=fw, depth_weight=dw,
                            decisions=O.decisions_of(arr, flow=flow, depth=depth))
    l64 = l64[on]
    assert ((got - l64).abs()[fin] <= 1e-6 * l64.abs()[fin]).all(), (got, l64, (got - l64).abs() / l64.abs())
    if fin.all():
        for k in ("rgb_map", "depth_map") + (FLOW_NAMES if flow else ()):
            bar = (grad_bars or {}).get(k, 1e-5)
            assert rel_err(grads[k].cpu(), g64[k]) < bar, (k, rel_err(grads[k].cpu(), g64[k]))
        for k in () if flow else FLOW_NAMES:
            assert grads[k] is None, k
    return d, losses, arr, grads


SHAPES = [(1, 2), (3, 3), (2, 255), (4, 257), (3, 511), (2, 1000), (2, 2049), (2, 4095), (4, 4096), (300, 16),
          (64, 256)]


@pytest.mark.parametrize("V,R", SHAPES)
def test_shapes(V, R):
    """Both terms.  One looser bar: at R = 2 the depth term is the constant 4 (xn and gn are {0, 2} whatever the
    inputs), so its exact gradient is 0 and the kernel's is fp32 cancellation of terms of about 0.1.  That noise
    is 4e-8 absolute; against the flow term's depth gradient (max 4e-4) it measured 1.1e-4 on an H100, so the
    depth_map bar is 3e-4 there."""
    check(batch(V * 1000 + R, V, R), grad_bars={"depth_map": 3e-4} if R == 2 else None)


@pytest.mark.parametrize("V,R", [(3, 3), (4, 257), (2, 4095), (300, 16)])
@pytest.mark.parametrize("term", ["flow_only", "depth_only"])
def test_shapes_one_term(V, R, term):
    fw, dw = (FW, 0.0) if term == "flow_only" else (0.0, DW)
    check(batch(V * 1000 + R + 1, V, R), fw=fw, dw=dw)


# ---- ties ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("V,R", [(4, 256), (3, 511)])
def test_quantised_depths_tie(V, R):
    """Depths and inverse depths on 8 values each: x, g, their normalised values and d tie in long runs, so the
    medians and the depth threshold fall inside runs."""
    kw = batch(11 + R, V, R)
    g = torch.Generator().manual_seed(R)
    kw["depth_map"] = torch.tensor([0.6, 0.9, 1.3, 1.7, 2.2, 2.9, 3.5, 4.4])[torch.randint(0, 8, (V * R,), generator=g)]
    kw["invdepths"] = torch.linspace(0.15, 1.0, 8)[torch.randint(0, 8, (V * R,), generator=g)]
    _, _, arr, _ = check(kw, ties=True)
    idx = arr["depth_median_index"].long().cpu()
    x = 1 / kw["depth_map"].view(V, R)
    assert ((x == x.gather(1, idx[:, :1])).sum(1) > 1).all()          # every x median is one of a run
    # and the ray at the lower median's sorted position is not the run's lowest index: the tie-break is exercised
    assert (torch.sort(x, dim=1, stable=True).indices[:, (R - 1) // 2] != idx[:, 0]).any()


def test_masked_view_cuts_every_nonzero_residual():
    """95 % of view 0's rays are masked on both flows: the 0.9 quantile lies in the run of zeros, tau = 0 and every
    nonzero residual of the view is cut."""
    V, R = 4, 256
    kw = batch(21, V, R)
    masked = torch.randperm(R, generator=torch.Generator().manual_seed(2))[:int(0.95 * R)]
    for k in ("fwd_mask", "bwd_mask"):
        kw[k].view(V, R)[0] = 1.0
        kw[k].view(V, R)[0, masked] = 0.0
    _, _, arr, _ = check(kw, ties=True)
    e = arr["flow"][0]
    assert arr["flow_tau"][0].item() == 0.0
    assert (e > 0).sum().item() == R - len(masked) and (e[masked] == 0).all()


def tiled_view(kw, v, R, pool, seed):
    """View v's rays become its first `pool` rays, each repeated R / pool times in a random order: every per-ray
    value ties in runs of R / pool."""
    src = v * R + torch.arange(R) % pool
    src = src[torch.randperm(R, generator=torch.Generator().manual_seed(seed))]
    for k, t in kw.items():
        if torch.is_tensor(t) and k not in ("view_ids", "cam2world", "focal", "center"):
            t[v * R:(v + 1) * R] = t[src].clone()


def test_flow_threshold_equals_residual():
    """View 1 holds 16 distinct rays, 16 times each: both neighbours of the 0.9 rank (229 and 230 of 256) lie in
    the run [224, 240), so tau equals that residual exactly, its 16 rays are kept and the 16 above are cut."""
    V, R = 4, 256
    kw = batch(31, V, R)
    tiled_view(kw, 1, R, 16, 5)
    _, _, arr, _ = check(kw, ties=True)
    e, tau = arr["flow"][1], arr["flow_tau"][1]
    s = torch.sort(e).values
    lo = int(np.floor(np.float32(0.9) * np.float32(R - 1)))
    assert s[lo] == s[lo + 1] == tau
    assert (e == tau).sum().item() == 16 and (e > tau).sum().item() == 16


# ---- clamped depths --------------------------------------------------------------------------------------------

def test_clamped_depth_run_holds_the_median():
    """60 % of view 0's depths are <= 1e-6 (zeros, tiny and negative values, never 1e-6 itself): x clamps to 1e6
    for all of them, the lower median lies in that run, and those rays get no gradient from the depth term (their
    depth gradient is the flow term's alone, bit for bit)."""
    V, R = 4, 256
    kw = batch(41, V, R)
    g = torch.Generator().manual_seed(7)
    clamped = torch.randperm(R, generator=g)[:int(0.6 * R)]
    low = torch.rand(len(clamped), generator=g) * 9e-7
    low[:5], low[5:10] = 0.0, -0.5
    kw["depth_map"].view(V, R)[0, clamped] = low
    _, _, arr, grads = check(kw, ties=True)
    mx = arr["depth_median_index"][0, 0].item()
    assert mx == int(clamped.min()) and (clamped == mx).any()
    _, _, _, flow_only = run(kw, FW, 0.0)
    assert torch.equal(grads["depth_map"].view(V, R)[0, clamped], flow_only["depth_map"].view(V, R)[0, clamped])
    assert not torch.equal(grads["depth_map"].view(V, R)[1], flow_only["depth_map"].view(V, R)[1])


# ---- non-finite values -----------------------------------------------------------------------------------------

def test_inf_flow_is_cut():
    """One ray of view 0 with an infinite forward flow (and its mask on): an infinite residual, sorted last and
    cut; every loss stays finite."""
    V, R = 4, 256
    kw = batch(51, V, R)
    kw["fwd_flow"][9, 0] = float("inf")
    kw["fwd_mask"][9] = 1.0
    d, losses, arr, _ = check(kw)
    assert torch.isinf(arr["flow"][0, 9]) and arr["flow"][0, 9] > arr["flow_tau"][0]
    assert all(torch.isfinite(l).item() for l in losses)


@pytest.mark.parametrize("R", [256, 257])
def test_inf_quantile_neighbour(R):
    """The upper neighbour of view 0's 0.9 rank is infinite.  R = 256: weight 0.5, ATen's large-weight lerp, inf -
    inf = NaN; R = 257: weight 0.4, the small-weight lerp gives +inf.  Either way nothing is cut and the flow loss
    is +inf, as torch's."""
    V = 4
    kw = batch(61 + R, V, R)
    r = np.float32(np.float32(0.9) * np.float32(R - 1))
    hi = int(np.ceil(r))
    assert (float(r - np.floor(r)) < 0.5) == (R == 257)
    rays = torch.arange(R - hi)                        # the largest R - hi residuals become +inf
    kw["fwd_flow"].view(V, R, 2)[0, rays, 0] = float("inf")
    kw["fwd_mask"].view(V, R)[0, rays] = 1.0
    _, losses, arr, _ = check(kw)
    tau = arr["flow_tau"][0].item()
    assert np.isnan(tau) if R == 256 else tau == float("inf")
    assert losses[1].item() == float("inf")


@pytest.mark.parametrize("bits", [0x7fc00000, 0xffc00000 - (1 << 32)], ids=["nan", "negative_nan"])
def test_nan_invdepth(bits):
    """A NaN among view 0's inverse depths, with its sign bit clear and set: torch.median gives NaN, so the g
    median is that ray (a NaN with the sign bit set used to sort first, below -inf, and leave a finite median),
    and the depth loss is NaN; the others stay finite."""
    V, R = 4, 256
    kw = batch(71, V, R)
    kw["invdepths"].view(torch.int32)[5] = bits
    d, losses, arr, _ = check(kw)
    assert d["invdepths"].view(torch.int32)[5].item() == bits
    assert arr["depth_median_index"][0, 1].item() == 5
    assert torch.isnan(losses[2]).item() and torch.isfinite(losses[0]).item() and torch.isfinite(losses[1]).item()


def test_nan_depth():
    """A NaN depth in view 0: its flow residual and x are NaN, so both thresholds of the view and the flow and
    depth losses are NaN, as torch's."""
    V, R = 4, 256
    kw = batch(81, V, R)
    kw["depth_map"][7] = float("nan")
    _, losses, arr, _ = check(kw)
    assert torch.isnan(arr["flow_tau"][0]) and torch.isnan(arr["depth_tau"][0])
    assert arr["depth_median_index"][0, 0].item() == 7
    assert torch.isnan(losses[1]).item() and torch.isnan(losses[2]).item() and torch.isfinite(losses[0]).item()


# ---- cameras ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("where", ["one_camera", "all_at_starting_id", "all_at_n_cams_minus_1", "all_at_last"])
def test_edge_cameras(where):
    """one_camera: n_cams = 1, both cam2cams are the identity.  all_at_starting_id: every backward flow clamps to
    the view's own camera.  all_at_n_cams_minus_1: every view's absolute id is n_cams - 1, so the reference zeroes
    every forward mask.  all_at_last: every view at the last camera, whose forward flow clamps to itself."""
    V, R = 8, 256
    n_frames, sid = (13, 12) if where == "one_camera" else (40, 12)
    n_cams = n_frames - sid
    vid = {"one_camera": sid, "all_at_starting_id": sid, "all_at_n_cams_minus_1": n_cams - 1,
           "all_at_last": n_frames - 1}[where]
    kw = batch(91, V, R, n_frames=n_frames, starting_id=sid, view_ids=torch.full((V,), vid))
    _, _, _, grads = check(kw)
    touched = grads["cam2world"].abs().sum(dim=(1, 2)) != 0
    assert touched[vid - sid].item()
    if where in ("all_at_starting_id", "all_at_last"):
        assert touched.sum().item() == 2                # the view's camera and its one clamped neighbour


# ---- repeatability ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("V,R", [(4, 4096), (300, 16)])
def test_bitwise_repeatable(V, R):
    kw = batch(101, V, R)
    outs = []
    for _ in range(2):
        _, losses, arr, grads = run(kw)
        outs.append([torch.stack(losses).detach()] + [arr[k] for k in sorted(arr)] + [grads[k] for k in O.GRAD_NAMES])
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
