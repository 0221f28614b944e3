"""-m gpu: lrf_test_panels across the sizes, cameras and values its C ABI accepts.  Three references: np.quantile and
torch.median directly; panels_oracle's rows on the kernel's own predicted flows, bit for bit
(test_gpu_panels.check_against_own_arrays); panels_oracle.pred_flow in float64, within flow_bound.  Covers numpy's
three choices of the quantile's upper neighbour (hi_mode 0, 1, 2, reached only above 2^24 values), frames where the
MAD kernel hits its block cap, one camera and the clamped neighbours of the first and last, depths that are 0,
negative, infinite or NaN, odd masks and ground truth, extreme nearest-map ratios, and the ABI itself: canaries
around every output, NULL optional outputs, pinned outputs, scratch left dirty by other frames, a non-default
stream."""
import ctypes as C

import numpy as np
import pytest
import torch

import panels_oracle as PO
from test_gpu_panels import check_against_own_arrays, run_case, stat_equal, zero_flow_case
from test_panels_cpu import INF_OFFSETS, NEAREST_EXTREMES, NEIGHBOUR_SIZES, bits_equal

pytestmark = pytest.mark.gpu
F32 = np.float32
CANARY = np.array([0xDEADBEEF], np.uint32).view(np.float32)[0]


@pytest.mark.parametrize("W,H,mode", NEIGHBOUR_SIZES)
def test_quantile_upper_neighbour(W, H, mode):
    """Zero predicted flow and ground truth whose first +inf lies 1, 2 or 3 ranks above numpy's lower rank (or
    nowhere), one arrangement per statistic.  gamma is 0 at these sizes, so numpy's quantile is NaN exactly when its
    upper neighbour is an infinity: at hi_mode 0 only the lower rank counts (a kernel that took the next rank would
    give NaN for offset 1), at hi_mode 2 the neighbour is two ranks up (a kernel that took the next rank would give a
    finite value for offset 2)."""
    assert PO.hi_mode(W, H) == mode
    lo, hi, gamma = PO.quantile_ranks(2 * W * H)
    assert gamma == 0
    gts = [PO.neighbour_gt(W, H, None if off is None else lo + off, k) for k, off in enumerate(INF_OFFSETS)]
    c = zero_flow_case(W, H, H, W, gts[0], gts[1])
    c["bwd_flow"] = np.stack([gts[2], gts[3]], -1).reshape(H, W, 2)
    _, _, _, arr = run_case(c)
    assert not arr["fwd_pred"].any() and not arr["bwd_pred"].any()
    for i, (g, off) in enumerate(zip(gts, INF_OFFSETS)):
        with np.errstate(invalid="ignore"):
            want = np.quantile(np.concatenate([np.zeros(W * H, F32), g]), 0.9)
        assert np.isnan(want) == (off is not None and lo + off <= hi), (i, off, want)
        assert stat_equal(arr["stats"][i], want), (mode, i, off, arr["stats"][i], want)


def pred_bound(c, offset):
    """-> (reference pred [H, W, 2], bound): panels_oracle.pred_flow and a bound on an fp32 evaluation's distance
    from it.  flow_bound, plus for each coordinate 16 eps of the sum of |terms| of q (cam2cam and the point in fp32),
    carried through q / z * f, with z's own error where it is not clamped: what a point near or behind the camera
    (z clamped to 1e-6) amplifies."""
    W, H = c["W"], c["H"]
    ref = PO.pred_flow(c["depth"], c["directions"], c["cam2world"], c["idx"], offset, c["focal"], c["center"], W, H)
    m = PO.cam2cam(c["cam2world"], c["idx"], offset)
    with np.errstate(invalid="ignore", over="ignore"):
        p = c["directions"].astype(np.float64) * c["depth"].astype(np.float64)[:, None]
        q = p @ m[:, :3].T + m[:, 3]
        S = np.abs(p) @ np.abs(m[:, :3]).T + np.abs(m[:, 3])
        z = np.maximum(-q[:, 2], 1e-6)
        e = 16 * PO.EPS * abs(float(c["focal"])) / z
        du = e * (S[:, 0] + np.abs(q[:, 0]) * S[:, 2] / z)
        dv = e * (S[:, 1] + np.abs(q[:, 1]) * S[:, 2] / z)
        b = PO.flow_bound(ref, W, H) + np.stack([du, dv], -1).reshape(H, W, 2)
    return ref, np.nan_to_num(b, nan=np.inf)


def check_preds(c, arr):
    for off, key in ((1, "fwd_pred"), (-1, "bwd_pred")):
        ref, b = pred_bound(c, off)
        got = arr[key]
        assert np.array_equal(np.isinf(got), np.isinf(ref)) and np.array_equal(np.signbit(got[np.isinf(got)]),
                                                                                np.signbit(ref[np.isinf(ref)])), key
        assert PO.within(got, ref, b), key


def check_all(c):
    out = run_case(c)
    check_against_own_arrays(c, *out)
    check_preds(c, out[3])
    return out


def test_large_frame_depth_statistics():
    """3840 x 2160 with half-size ground truth: 8.3 M pixels, so panels_mad_kernel runs at its cap of 1024 blocks.
    The medians are torch.median's, the MAD scales within 1 ulp of float64 fsum, every row bit for bit."""
    W, H = 3840, 2160
    assert (W * H + 4095) // 4096 > 1024
    c = PO.build_case(11, W, H, H // 2, W // 2, 6, 2)
    check_all(c)


@pytest.mark.parametrize("n_cams,idx", [(1, 0), (5, 0), (5, 4), (2, 1)])
def test_cameras(n_cams, idx):
    """One camera (both neighbours are the frame itself), and the first and last frames, whose backward / forward
    neighbour clamps to the frame: that flow is the identity reprojection, a few ulps from 0."""
    c = PO.build_case(30 + n_cams + idx, 64, 48, 96, 128, n_cams, idx)
    check_all(c)
    for off, clamps in ((-1, idx == 0), (1, idx == n_cams - 1)):
        if clamps:
            ref, b = pred_bound(c, off)
            assert np.all(np.abs(ref) <= b), off


DEPTHS = {
    "zero_negative_inf": np.array([0.0, -0.0, -1.0, -1e-3, -50.0, np.inf, 1e-7, 1e-6, 3e-7], F32),
    "nan": np.array([np.nan, 0.0, -1.0, np.inf], F32),
    "behind": np.array([-0.5, -2.0, -5.0], F32),
}


@pytest.mark.parametrize("kind", list(DEPTHS))
def test_depth_values(kind):
    """Depths of 0, negative, inf or NaN among normal ones.  A negative depth puts the point behind the camera, where
    -z is clamped to 1e-6 and the flow reaches 1e8 or overflows; x = 1 / max(depth, 1e-6) is 1e6 there."""
    c = PO.build_case(40 + len(kind), 64, 48, 96, 128, 4, 2)
    g = np.random.default_rng(len(kind))
    k = g.permutation(64 * 48)[:300]
    c["depth"][k] = DEPTHS[kind][np.arange(k.size) % DEPTHS[kind].size]
    check_all(c)


def _masks_and_gt(c, g, kind):
    n = c["fwd_mask"].shape
    if kind == "fractional_masks":
        c["fwd_mask"] = g.uniform(-0.5, 1.5, n).astype(F32)
        c["bwd_mask"] = g.uniform(0, 1, n).astype(F32)
    elif kind == "nan_masks":
        c["fwd_mask"][g.random(n) < 0.01] = np.nan
        c["bwd_mask"][g.random(n) < 0.1] = -2.0
    elif kind == "nan_flow":
        c["fwd_flow"][4, 6, 0] = np.nan                       # even row and column: in the 64 x 48 nearest map
        c["bwd_flow"][8, 2, 1] = -np.nan
    elif kind == "inf_flow":
        c["fwd_flow"][g.random(n) < 0.2] = np.inf
        c["bwd_flow"][g.random(n) < 0.05] = -np.inf
    elif kind == "constant_invdepth":
        c["invdepth"][:] = F32(0.75)
    return c


@pytest.mark.parametrize("kind", ["fractional_masks", "nan_masks", "nan_flow", "inf_flow", "constant_invdepth"])
def test_masks_and_ground_truth(kind):
    """Masks that are fractional, negative or NaN; NaN or infinite ground-truth flow; a constant inverse depth, whose
    MAD is 0 and whose rows are then 0 / 0 = NaN."""
    c = _masks_and_gt(PO.build_case(50, 64, 48, 96, 128, 4, 1), np.random.default_rng(51), kind)
    _, _, dep, arr = check_all(c)
    if kind == "nan_flow":
        assert np.isnan(arr["stats"][0]) and np.isnan(arr["stats"][3]) and not np.isnan(arr["stats"][1])
    if kind == "constant_invdepth":
        assert arr["stats"][6] == F32(0.75) and arr["stats"][7] == 0
        assert np.isnan(dep[48:]).all()


@pytest.mark.parametrize("src,dst", NEAREST_EXTREMES)
def test_nearest_map_extremes(src, dst):
    """The ground truth's nearest map at extreme ratios, against panels_oracle.nearest_index (which equals cv2's,
    test_panels_cpu): a zero-flow frame whose ground truth holds every source index once, so each error row's value
    names the source pixel, and the whole panel must equal the restatement's bit for bit."""
    (h0, w0), (H, W) = src, dst
    e = int(np.ceil(np.log2(h0 * w0 + 1)))
    gt = (np.arange(h0 * w0, dtype=np.float64) * 2.0 ** -e).astype(F32)
    c = zero_flow_case(W, H, h0, w0, gt)
    fwd, bwd, _, arr = run_case(c)
    assert not arr["fwd_pred"].any()
    flow = PO.resize_nearest(c["fwd_flow"], W, H)
    want, _ = PO.flow_panel(arr["fwd_pred"], flow, PO.resize_nearest(c["fwd_mask"], W, H), W)
    assert bits_equal(fwd, want) and bits_equal(bwd, want)
    idx = PO.nearest_index(h0, H)[:, None] * w0 + PO.nearest_index(w0, W)[None, :]
    assert np.array_equal(flow[..., 0], gt[idx])
    if W == 1:                                               # err = gt / 1: the source index itself, read back
        assert np.array_equal(np.rint(fwd[2 * H:, :1].astype(np.float64) * 2.0 ** e)[:, 0], idx[:, 0])


# ---- through ctypes ---------------------------------------------------------------------------------------------
OUTS = ("fwd_panel", "bwd_panel", "depth_panel", "fwd_pred", "bwd_pred", "stats")
PAD = 67


def out_sizes(W, H):
    return dict(fwd_panel=6 * W * H, bwd_panel=6 * W * H, depth_panel=3 * W * H, fwd_pred=2 * W * H,
                bwd_pred=2 * W * H, stats=8)


def device_inputs(c):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, F32)).cuda()
    ins = {k: t(c[k]) for k in ("depth", "directions", "cam2world", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask",
                                "invdepth")}
    ins["intrinsics"] = torch.tensor([float(c["focal"]), *map(float, c["center"])], device="cuda")
    return ins


def guarded_outputs(W, H, pin=False, names=OUTS):
    """-> {name: (buffer with PAD canaries on each side, the output inside it)}."""
    out = {}
    for k in names:
        n = out_sizes(W, H)[k]
        buf = torch.full((n + 2 * PAD,), float(CANARY), device="cpu" if pin else "cuda")
        if pin:
            buf = buf.pin_memory()
        out[k] = (buf, buf[PAD:PAD + n])
    return out


def panels_abi(c, ins, outs, scratch, stream=None, branches=("flow", "depth")):
    from localrf_b200 import _lib
    f = _lib.LrfPanelFrame()
    f.W, f.H = c["W"], c["H"]
    f.h0, f.w0 = c["fwd_flow"].shape[:2]
    f.n_cams, f.idx = len(c["cam2world"]), c["idx"]
    keep = {"depth", "directions", "cam2world", "intrinsics"}
    if "flow" in branches:
        keep |= {"fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"}
    if "depth" in branches:
        keep |= {"invdepth"}
    for k, v in ins.items():
        setattr(f, k, v.data_ptr() if k in keep else None)
    for k in OUTS:
        v = outs.get(k)
        setattr(f, k, v[1].data_ptr() if v is not None else None)
    _lib.check(_lib.lib().lrf_test_panels(C.byref(f), scratch.data_ptr(), scratch.numel(), stream))


def scratch_for(W, H, fill=0):
    from localrf_b200 import _lib
    n = int(_lib.lib().lrf_test_panels_scratch_bytes(W, H))
    return torch.full((n,), fill, dtype=torch.uint8, device="cuda")


def host_outs(outs):
    torch.cuda.synchronize()
    return {k: (b.cpu().numpy(), v.cpu().numpy()) for k, (b, v) in outs.items()}


def assert_same(got, want, names=OUTS):
    for k in names:
        buf, v = got[k]
        assert bits_equal(v, want[k]), k
        assert np.all(buf[:PAD].view(np.uint32) == CANARY.view(np.uint32)) and \
            np.all(buf[PAD + v.size:].view(np.uint32) == CANARY.view(np.uint32)), ("canary", k)


@pytest.fixture(scope="module")
def small():
    """A 37 x 23 frame with 61 x 100 ground truth, its device inputs, and the outputs of a plain ABI call."""
    c = PO.build_case(60, 37, 23, 61, 100, 5, 2)
    ins = device_inputs(c)
    outs = guarded_outputs(37, 23)
    panels_abi(c, ins, outs, scratch_for(37, 23))
    want = {k: v for k, (_, v) in host_outs(outs).items()}
    return c, ins, want


def test_abi_outputs_match_the_binding_and_keep_canaries(small):
    c, ins, want = small
    fwd, bwd, dep, arr = run_case(c)
    for k, v in (("fwd_panel", fwd), ("bwd_panel", bwd), ("depth_panel", dep), ("fwd_pred", arr["fwd_pred"]),
                 ("bwd_pred", arr["bwd_pred"]), ("stats", arr["stats"])):
        assert bits_equal(want[k], v.reshape(-1)), k
    outs = guarded_outputs(37, 23)
    panels_abi(c, ins, outs, scratch_for(37, 23))
    assert_same(host_outs(outs), want)


def test_abi_null_optional_outputs(small):
    """With stats and the predicted flows NULL the panels have the same bits."""
    c, ins, want = small
    for drop in (("stats",), ("fwd_pred", "bwd_pred"), ("stats", "fwd_pred", "bwd_pred")):
        names = tuple(k for k in OUTS if k not in drop)
        outs = guarded_outputs(37, 23, names=names)
        panels_abi(c, ins, outs, scratch_for(37, 23))
        assert_same(host_outs(outs), want, names)


def test_abi_pinned_outputs(small):
    c, ins, want = small
    outs = guarded_outputs(37, 23, pin=True)
    panels_abi(c, ins, outs, scratch_for(37, 23))
    assert_same(host_outs(outs), want)


def test_abi_dirty_scratch(small):
    """Scratch filled with 0xFF, scratch last used by a larger frame, and scratch last used by one branch alone give
    the same bits as fresh zeroed scratch."""
    c, ins, want = small
    outs = guarded_outputs(37, 23)
    panels_abi(c, ins, outs, scratch_for(37, 23, 0xFF))
    assert_same(host_outs(outs), want)
    big = PO.build_case(61, 480, 270, 540, 960, 8, 5)
    shared = scratch_for(480, 270, 0xFF)
    panels_abi(big, device_inputs(big), guarded_outputs(480, 270), shared)
    outs = guarded_outputs(37, 23)
    panels_abi(c, ins, outs, shared)
    assert_same(host_outs(outs), want)
    for first in (("depth",), ("flow",)):
        shared = scratch_for(37, 23)
        names = ("depth_panel", "stats") if first == ("depth",) else ("fwd_panel", "bwd_panel", "stats")
        panels_abi(c, ins, guarded_outputs(37, 23, names=names), shared, branches=first)
        outs = guarded_outputs(37, 23)
        panels_abi(c, ins, outs, shared)
        assert_same(host_outs(outs), want)


def test_abi_dirty_scratch_at_hi_mode_2():
    """The extra selection jobs of hi_mode 2 with scratch filled with 0xFF, against zeroed scratch."""
    W, H = 4096, 2304
    lo, _, _ = PO.quantile_ranks(2 * W * H)
    c = zero_flow_case(W, H, H, W, PO.neighbour_gt(W, H, lo + 3, 0), PO.neighbour_gt(W, H, None, 1))
    c["invdepth"] = (np.random.default_rng(2).random((H, W)) + 0.1).astype(F32)
    ins = device_inputs(c)
    res = []
    for fill in (0, 0xFF):
        outs = guarded_outputs(W, H)
        panels_abi(c, ins, outs, scratch_for(W, H, fill))
        res.append(host_outs(outs))
    assert_same(res[1], {k: v for k, (_, v) in res[0].items()})
    with np.errstate(invalid="ignore"):
        want = np.quantile(np.concatenate([np.zeros(W * H, F32), c["fwd_flow"][..., 0].ravel()]), 0.9)
    assert np.isfinite(want) and stat_equal(res[0]["stats"][1][0], want)


def test_abi_non_default_stream(small):
    """On a non-blocking stream whose earlier work (a spin, then the copy that fills depth) the kernels must wait
    for."""
    c, ins, want = small
    stream = torch.cuda.Stream()
    depth = torch.full_like(ins["depth"], float("nan"))
    outs = guarded_outputs(37, 23)
    scratch = scratch_for(37, 23)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(20_000_000)
        depth.copy_(ins["depth"])
        panels_abi(c, {**ins, "depth": depth}, outs, scratch, stream=stream.cuda_stream)
    stream.synchronize()
    assert_same(host_outs(outs), want)
