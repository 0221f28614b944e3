"""-m gpu: the test-frame comparison panels on the device (lrf_test_panels, metrics.test_panels, FramePipeline with
panels=) against np.quantile / torch.median bit for bit, against the numpy expressions of renderer.py:79-124 on the
kernel's own predicted flows, against the reference's block (tests/golden/test_panels.npz) and against the
unmodified reference renderer."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import panels_oracle as PO
from test_panels_cpu import bits_equal, golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def stat_equal(a, b):
    """An order statistic against torch's / numpy's: bitwise, except that -0 and +0 are one value.  Both select by
    comparison (torch sorts with -0 == +0, np.partition compares), so which zero they return depends on where the
    zeros lie in the input; the kernel's keys order -0 before +0.  Ranks are unaffected: the two keys are adjacent."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return bits_equal(a, b) or bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def row_median(v):
    """compute_depth_loss's median: torch.median over the last dimension of a [1, n] row (the reduction without dim
    is another code path, which on CUDA does not see a NaN whose sign bit is set)."""
    return torch.median(v.reshape(1, -1), dim=-1).values[0].item()


def run_case(c, **over):
    import localrf_b200 as L
    c = {**c, **over}
    W, H = c["W"], c["H"]
    depth = torch.from_numpy(np.asarray(c["depth"], F32)).cuda()
    dirs = torch.from_numpy(np.asarray(c["directions"], F32)).cuda() if c.get("directions") is not None else None
    c2w = torch.from_numpy(np.asarray(c["cam2world"], F32)).cuda()
    focal = torch.tensor([float(c["focal"])], device="cuda")
    center = torch.from_numpy(np.asarray(c["center"], F32)).cuda()
    gts = {k: c.get(k) for k in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask", "invdepth")}
    fwd, bwd, dep, arr = L.metrics.test_panels(depth, dirs, c2w, c["idx"], focal, center, W, H, return_arrays=True,
                                               **gts)
    torch.cuda.synchronize()
    cpu = lambda t: None if t is None else t.cpu().numpy()
    return cpu(fwd), cpu(bwd), cpu(dep), {k: cpu(v) for k, v in arr.items()}


def zero_flow_case(W, H, h0, w0, gt0, gt1=None, seed=0):
    """Identity camera, unit depth, rays through the pixel centres (focal 1, centre 0): the predicted flow is exactly
    0, so the 0.9 quantile of [pred; gt] is the quantile of [zeros; gt] for an arbitrary gt."""
    p = np.arange(W * H)
    i, j = (p % W).astype(F32), (p // W).astype(F32)
    gt1 = gt0 if gt1 is None else gt1
    flow = np.stack([gt0, gt1], -1).astype(F32).reshape(h0, w0, 2)
    return dict(W=W, H=H, idx=0, cam2world=np.concatenate([np.eye(3), np.zeros((3, 1))], 1)[None].astype(F32),
                focal=F32(1.0), center=np.zeros(2, F32), depth=np.ones(W * H, F32),
                directions=np.stack([i + F32(0.5), -(j + F32(0.5)), -np.ones_like(i)], -1).astype(F32),
                fwd_flow=flow, fwd_mask=np.ones((h0, w0), F32), bwd_flow=flow.copy(),
                bwd_mask=np.ones((h0, w0), F32), invdepth=None)


def value_class(rng, n, kind):
    special = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, np.inf, -np.inf, 1.0, -1.0], np.float32)
    if kind == "normal":
        a = rng.standard_normal(n)
    elif kind == "ties":
        a = rng.integers(-3, 4, n).astype(np.float64)
    elif kind == "special":
        a = rng.standard_normal(n)
        k = rng.integers(0, n, max(1, n // 7))
        a[k] = rng.choice(special, k.size)
    elif kind == "subnormal":
        a = rng.choice(special[:6], n)
    elif kind == "nan":
        a = rng.standard_normal(n)
        a[rng.integers(0, n)] = -np.nan if n % 2 else np.nan
    else:
        a = rng.choice(np.array([np.inf, -np.inf, 0.0, 1.0]), n)
    return a.astype(F32)


KINDS = ("normal", "ties", "special", "subnormal", "nan", "infs")
SIZES = (2, 3, 255, 256, 257, 4095, 2 ** 16 - 1, 2 ** 16 + 1, 2 * 960 * 540, 2 * 1920 * 1080)


@pytest.mark.parametrize("n", SIZES)
def test_median_selection_bitwise(n):
    """torch.median over n arbitrary values: the depth branch with the ground truth at the render size (W = n,
    H = 1: the nearest map is the identity), so g is the array itself; stats[6] is its median."""
    rng = np.random.default_rng(n)
    for kind in KINDS:
        g = value_class(rng, n, kind)
        depth = (0.5 + rng.random(n)).astype(F32)
        _, _, _, arr = run_case(dict(W=n, H=1, idx=0, cam2world=np.zeros((1, 3, 4), F32), focal=1.0,
                                     center=np.zeros(2, F32), depth=depth, directions=None,
                                     invdepth=g.reshape(1, n)))
        want = row_median(torch.from_numpy(g).cuda())
        assert stat_equal(arr["stats"][6], want), (kind, arr["stats"][6], want)
        x = torch.from_numpy(depth).cuda()
        assert stat_equal(arr["stats"][4], row_median(1 / x.clamp(1e-6)))


@pytest.mark.parametrize("n", [s for s in SIZES if s % 2 == 0])
def test_quantile_selection_bitwise(n):
    """np.quantile(., 0.9) over [zeros(n/2); gt] for arbitrary gt of every value class, both channels.  n = 2 is a
    1 x 1 frame: index 0.9, neighbours 0 and 1."""
    rng = np.random.default_rng(n + 1)
    half = n // 2
    W = 960 if half % 960 == 0 else half
    H = half // W
    for kind in KINDS:
        g0, g1 = value_class(rng, half, kind), value_class(rng, half, KINDS[(KINDS.index(kind) + 1) % 6])
        c = zero_flow_case(W, H, H, W, g0, g1)
        _, _, _, arr = run_case(c)
        assert np.all(arr["fwd_pred"] == 0)
        for ch, g in ((0, g0), (1, g1)):
            with np.errstate(invalid="ignore"):
                want = np.quantile(np.concatenate([np.zeros(half, F32), g]), 0.9)
            assert stat_equal(arr["stats"][ch], want) and stat_equal(arr["stats"][2 + ch], want), (kind, ch)


def check_against_own_arrays(c, fwd, bwd, dep, arr):
    """Every statistic equals np.quantile / torch.median over the kernel's own arrays, and every row equals the
    numpy expression on those arrays, bit for bit."""
    W, H = c["W"], c["H"]
    stats = arr["stats"]
    for d, (panel, pred) in enumerate(((fwd, arr["fwd_pred"]), (bwd, arr["bwd_pred"]))):
        name = ("fwd", "bwd")[d]
        flow = PO.resize_nearest(c[f"{name}_flow"], W, H)
        mask = PO.resize_nearest(c[f"{name}_mask"], W, H)
        want, qs = PO.flow_panel(pred, flow, mask, W)
        for ch in range(2):
            with np.errstate(invalid="ignore"):
                q = np.quantile(np.vstack([pred[..., ch], flow[..., ch]]), 0.9)
            assert stat_equal(stats[2 * d + ch], q) and stat_equal(qs[ch], q)
        assert bits_equal(panel, want), name
    x = 1 / torch.from_numpy(c["depth"]).cuda().clamp(1e-6)
    g = torch.from_numpy(PO.resize_nearest(c["invdepth"], W, H).reshape(-1)).cuda()
    for i, v in ((4, x), (6, g)):
        t = torch.median(v.reshape(1, -1), dim=-1).values[0]
        assert stat_equal(stats[i], t.item())
        r = torch.abs(v - t).double().cpu().numpy()
        mean = math.fsum(r.tolist()) / r.size if np.isfinite(r).all() else float(np.mean(r))
        assert bits_equal(stats[i + 1], F32(mean)) or PO.ulps(stats[i + 1], F32(mean)) <= 1
    xs, gs = x.cpu().numpy(), g.cpu().numpy()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        xn = (xs - stats[4]) / stats[5]
        gn = (gs - stats[6]) / stats[7]
        want = np.clip(np.vstack([(F32(0.5) * xn).reshape(H, W), (F32(0.5) * gn).reshape(H, W),
                                  ((xn - gn) * (xn - gn)).reshape(H, W)]), 0, 1)
    assert bits_equal(dep, want)


@pytest.mark.parametrize("name", list(PO.CASES))
def test_thresholds_and_rows_bitwise_on_own_arrays(name):
    c = PO.make_case(name)
    check_against_own_arrays(c, *run_case(c))


def flow_panel_bound(ref_pred, ref_q, flow, mask, W):
    """Bound on |panel - reference panel| when the predicted flows differ by at most PO.flow_bound: the order
    statistics are 1-Lipschitz in the largest change, so |dq| <= dp_max; a scaled row v / q moves by at most
    (|dv| + |dq|) / |q| plus two roundings; an error row by |dv| mask / W plus one.  Rows with q = 0 must match
    exactly (inf / NaN)."""
    H = ref_pred.shape[0]
    cols = []
    for ch in range(2):
        dp = PO.flow_bound(ref_pred[..., ch], W, H)
        dq = float(dp.max())
        q = abs(float(ref_q[ch]))
        if q == 0:
            cols.append(np.zeros((3 * H, W)))
            continue
        pred_rows = (dp + dq) / q + 2 * PO.EPS
        gt_rows = dq / q + 2 * PO.EPS + 0 * dp
        err_rows = dp * np.abs(mask) / W + 2 * PO.EPS
        cols.append(np.vstack([pred_rows, gt_rows, err_rows]))
    return np.hstack(cols)


@pytest.mark.parametrize("name", list(PO.CASES))
def test_against_reference_block(name):
    g = golden()
    c = PO.make_case(name)
    W, H = c["W"], c["H"]
    fwd, bwd, dep, arr = run_case(c)
    full = W * H <= PO.FULL_OUTPUT_PIXELS
    pick = (lambda a: a) if full else (lambda a: a.reshape(-1)[PO.sample_index(name, a.size)])
    ref_stats = g[f"{name}.stats"]
    for key in ("fwd_pred", "bwd_pred"):
        ref = g[f"{name}.{key}"]
        assert np.all(np.abs(pick(arr[key]) - ref) <= PO.flow_bound(ref, W, H)), key
    assert stat_equal(arr["stats"][[4, 6]], ref_stats[[4, 6]])                         # medians: bitwise
    k = 1
    for i in (5, 7):                                            # MAD scales: torch's fp32 mean vs the fp64 one
        if not bits_equal(arr["stats"][i], ref_stats[i]):
            k = max(k, PO.ulps(arr["stats"][i], ref_stats[i]))
    assert k <= 4
    bound = PO.depth_bound(c["depth"], PO.resize_nearest(c["invdepth"], W, H), W, H, s_ulps=k)
    assert PO.within(pick(dep), g[f"{name}.depth_cmp"], pick(bound))
    if not full:
        return
    for d, (panel, name_d) in enumerate(((fwd, "fwd"), (bwd, "bwd"))):
        ref_pred = g[f"{name}.{name_d}_pred"]
        flow, mask = PO.resize_nearest(c[f"{name_d}_flow"], W, H), PO.resize_nearest(c[f"{name_d}_mask"], W, H)
        b = flow_panel_bound(ref_pred, ref_stats[2 * d: 2 * d + 2], flow, mask, W)
        for ch in range(2):
            assert abs(float(arr["stats"][2 * d + ch]) - float(ref_stats[2 * d + ch])) <= \
                float(PO.flow_bound(ref_pred[..., ch], W, H).max()) or bits_equal(arr["stats"][2 * d + ch],
                                                                                  ref_stats[2 * d + ch])
        assert PO.within(panel, g[f"{name}.{name_d}_cmp"], b), name_d


def test_nearest_map_equals_cv2():
    """The ground truth's nearest map, read back through the error rows of a zero-flow frame: gt = index * 2^-e
    with unit masks gives err = gt / W < 1, so round(err * W * 2^e) is the source index of every pixel."""
    cv2 = pytest.importorskip("cv2")
    for (h0, w0) in ((96, 128), (61, 100), (15, 20), (1, 1), (7, 3), (270, 480)):
        e = int(math.ceil(math.log2(h0 * w0 + 1)))
        src = np.arange(h0 * w0, dtype=np.float64).reshape(h0, w0)
        for (W, H) in ((64, 48), (37, 23), (1, 1), (3, 7), (2 * w0 + 1, 3 * h0), (max(1, w0 // 3), max(1, h0 // 2))):
            gt = (src * 2.0 ** -e).astype(F32)
            c = zero_flow_case(W, H, h0, w0, gt)
            fwd, _, _, _ = run_case(c)
            got = np.rint(fwd[2 * H:, :W].astype(np.float64) * W * 2.0 ** e)
            want = cv2.resize(src.astype(F32), (W, H), interpolation=cv2.INTER_NEAREST).reshape(H, W)
            assert np.array_equal(got, want), (h0, w0, W, H)


def test_repeatable():
    c = PO.make_case("big_480x270")
    a, b = run_case(c), run_case(c)
    for x, y in zip(a[:3], b[:3]):
        assert bits_equal(x, y)
    for k in a[3]:
        assert bits_equal(a[3][k], b[3][k])


def test_branches_and_errors():
    import localrf_b200 as L
    c = PO.make_case("base_64x48")
    fwd, bwd, dep, arr = run_case(c, invdepth=None)
    assert dep is None and fwd.shape == (3 * 48, 128) and np.isnan(arr["stats"][4:]).all()
    full = run_case(c)
    assert bits_equal(fwd, full[0]) and bits_equal(bwd, full[1])
    fwd, bwd, dep, arr = run_case(c, fwd_flow=None, fwd_mask=None, bwd_flow=None, bwd_mask=None)
    assert fwd is None and bwd is None and bits_equal(dep, full[2]) and np.isnan(arr["stats"][:4]).all()
    with pytest.raises(ValueError):
        run_case(c, bwd_mask=None)
    with pytest.raises(ValueError, match="idx"):
        run_case(c, idx=6)


def test_inputs_on_the_wrong_device_raise_before_launch():
    """The kernel dereferences every input pointer: a pageable host tensor or another device's tensor must be refused
    before anything is enqueued (a host pointer read on the device would be an illegal address)."""
    import localrf_b200 as L
    c = PO.make_case("base_64x48")
    W, H = c["W"], c["H"]
    depth = torch.from_numpy(c["depth"]).cuda()
    dirs = torch.from_numpy(c["directions"]).cuda()
    c2w = torch.from_numpy(c["cam2world"]).cuda()
    focal, center = torch.tensor([float(c["focal"])], device="cuda"), torch.from_numpy(c["center"]).cuda()
    gts = {k: c[k] for k in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask", "invdepth")}
    torch.cuda.synchronize()
    for bad in (dict(cam2world=c2w.cpu()), dict(directions=dirs.cpu()), dict(depth=depth.cpu())):
        args = dict(depth=depth, directions=dirs, cam2world=c2w, **gts)
        args.update(bad)
        with pytest.raises(ValueError):
            L.metrics.test_panels(args.pop("depth"), args.pop("directions"), args.pop("cam2world"), c["idx"], focal,
                                  center, W, H, **args)
    if torch.cuda.device_count() > 1:
        other = torch.from_numpy(c["fwd_flow"]).to("cuda:1")
        with pytest.raises(ValueError, match="cuda:1"):
            L.metrics.test_panels(depth, dirs, c2w, c["idx"], focal, center, W, H, **{**gts, "fwd_flow": other})
    # pinned host inputs are read in place, and give the device inputs' results
    want = run_case(c)
    got = L.metrics.test_panels(depth, dirs.cpu().pin_memory(), c2w.cpu().pin_memory(), c["idx"], focal, center, W, H,
                                **{k: torch.from_numpy(v).pin_memory() for k, v in gts.items()})
    for g_, w_ in zip(got, want[:3]):
        assert bits_equal(g_.cpu().numpy(), w_)


def test_pipeline_panels_match_direct_calls():
    import bench
    import localrf_b200 as L
    wl = bench.Workload("cfg5", 48)
    lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
    W, H = 96, 80
    rng = np.random.default_rng(3)
    gts = {}
    for f in (5, 30, 63):
        gts[f] = dict(fwd_flow=(3 * rng.standard_normal((160, 192, 2))).astype(F32),
                      fwd_mask=(rng.random((160, 192)) > 0.2).astype(F32),
                      bwd_flow=(3 * rng.standard_normal((160, 192, 2))).astype(F32),
                      bwd_mask=(rng.random((160, 192)) > 0.2).astype(F32),
                      invdepth=(rng.random((160, 192)) + 0.1).astype(F32))
    gt_rgb = rng.random((H, W, 3)).astype(F32)

    def run(with_panels):
        pipe = L.FramePipeline(lt, W, H, n_buffers=2, keep_float=True)
        out = []
        for f in gts:
            if pipe.in_flight() == 2:
                out.append({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pipe.fetch().items()})
            extra = {"panels": dict(idx=f, **gts[f])} if with_panels else {}
            pipe.submit(torch.tensor([f], device="cuda"), gt=gt_rgb, tag=f, test_id=True, **extra)
        while pipe.in_flight():
            out.append({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pipe.fetch().items()})
        return out

    plain, with_p = run(False), run(True)
    ids = torch.arange(W * H, device="cuda")
    for a, b in zip(plain, with_p):
        for k in ("rgb8", "depth8", "rgb", "depth"):
            assert np.array_equal(a[k], b[k]), k
        assert a["mse"] == b["mse"] and a["ssim"] == b["ssim"]
        assert "fwd_flow_cmp" not in a
        f = b["tag"]
        with torch.no_grad():
            _, depth, dirs, _ = lt(ids, torch.tensor([f], device="cuda"), W, H, is_train=False, test_id=True)
            want = L.metrics.test_panels(depth, dirs, lt.get_cam2world(), f, lt.focal(W), lt.center(W, H), W, H,
                                         **gts[f])
        for key, w in zip(("fwd_flow_cmp", "bwd_flow_cmp", "depth_cmp"), want):
            assert bits_equal(b[key], w.cpu().numpy()), key


SCRIPT = r'''
import sys, types
import numpy as np, torch
ROOT, REF = sys.argv[1], sys.argv[2]
sys.path[:0] = [ROOT + "/dropin", ROOT, ROOT + "/tests", REF]
from oracle import ref_loader
for name, attrs in (("kornia", dict(create_meshgrid=None)), ("matplotlib", dict(use=lambda *a, **k: None)),
                    ("matplotlib.pyplot", {}), ("matplotlib.cm", {}), ("plyfile", {}), ("skimage", {}),
                    ("skimage.measure", {}), ("imageio", {}), ("lpips", {})):
    ref_loader._stub(name, **attrs)
import renderer                                     # the reference's module, unmodified
import local_tensorfs, localrf_b200 as L
import panels_oracle as PO
assert local_tensorfs.LocalTensorfs is L.LocalTensorfs and renderer.__file__.startswith(REF)
import bench
W, H, h0, w0 = 64, 48, 96, 128
renderer.draw_poses = lambda poses, colours: np.zeros((H, W, 3), np.uint8)      # matplotlib plot: stubbed I/O
wl = bench.Workload("cfg5", 40)
lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
n = len(lt.r_c2w)
rng = np.random.default_rng(0)
test_ids = [0, 9, n - 1]
train_ds = types.SimpleNamespace(all_fbases={f"{i:04d}": i for i in range(n)}, get_frame_fbase=lambda i: f"{i:04d}")
mk = lambda *s: [rng.standard_normal(s).astype(np.float32) * 3 for _ in test_ids]
test_ds = types.SimpleNamespace(
    all_fbases={f"{i:04d}": k for k, i in enumerate(test_ids)},
    all_fwd_flow=mk(h0, w0, 2), all_bwd_flow=mk(h0, w0, 2),
    all_fwd_mask=[(rng.random((h0, w0)) > 0.2).astype(np.float32) for _ in test_ids],
    all_bwd_mask=[(rng.random((h0, w0)) > 0.2).astype(np.float32) for _ in test_ids],
    all_invdepths=[(rng.random((h0, w0)) + 0.1).astype(np.float32) for _ in test_ids],
    all_rgbs=[rng.random((h0, w0, 3)).astype(np.float32) for _ in test_ids])
args = types.SimpleNamespace(batch_size=4096, device="cuda")
poses = lt.get_cam2world().detach()
out = renderer.render(test_ds, poses, lt, args, W=W, H=H, savePath=None, save_video=False, save_frames=False,
                      test=True, train_dataset=train_ds, start=0, floater_thresh=0, add_frame_to_list=True)
fwd_tb, bwd_tb, dep_tb = out[3], out[4], out[5]
assert len(fwd_tb) == len(bwd_tb) == len(dep_tb) == len(test_ids)
ids = torch.arange(W * H, device="cuda")
for k, idx in enumerate(test_ids):
    with torch.no_grad():
        _, depth, dirs, _ = lt(ids, torch.tensor([idx], device="cuda"), W, H, is_train=False, test_id=True,
                               chunk=4096)
        gts = dict(fwd_flow=test_ds.all_fwd_flow[k], fwd_mask=test_ds.all_fwd_mask[k],
                   bwd_flow=test_ds.all_bwd_flow[k], bwd_mask=test_ds.all_bwd_mask[k],
                   invdepth=test_ds.all_invdepths[k])
        fwd, bwd, dep, arr = L.metrics.test_panels(depth, dirs, lt.get_cam2world(), idx, lt.focal(W),
                                                   lt.center(W, H), W, H, return_arrays=True, **gts)
    stats = arr["stats"].cpu().numpy()
    ref_dep = dep_tb[k].cpu().numpy()
    # the depth panel: the kernel's MAD scales are within 4 ulps of torch's fp32 mean (see test_against_reference_block)
    inv = PO.resize_nearest(gts["invdepth"], W, H)
    bound = PO.depth_bound(depth.cpu().numpy(), inv, W, H, s_ulps=4)
    assert PO.within(dep.cpu().numpy(), ref_dep, bound), ("depth", idx)
    # the flow panels: recompute the reference's rows from the kernel's predicted flows would be exact; the
    # reference's own predicted flows differ by PO.flow_bound, which bounds the rows as in the golden test
    for d, (mine, ref) in enumerate(((fwd, fwd_tb[k]), (bwd, bwd_tb[k]))):
        mine, ref = mine.cpu().numpy(), ref.numpy()
        nm = ("fwd", "bwd")[d]
        pred = arr[nm + "_pred"].cpu().numpy()
        dp = PO.flow_bound(pred, W, H).max()
        for ch in range(2):
            q = abs(float(stats[2 * d + ch]))
            assert q > 0
            b = (2 * dp) / q + 1e-6
            cols = slice(ch * W, ch * W + W)
            assert np.all(np.abs(mine[:2 * H, cols] - ref[:2 * H, cols]) <= b), (nm, ch, idx)
            assert np.all(np.abs(mine[2 * H:, cols] - ref[2 * H:, cols]) <= dp / W + 1e-6), (nm, ch, idx)
print("PANELS_RENDER_OK", len(fwd_tb))
'''


def test_reference_renderer_panels_match():
    ref = os.path.join(ROOT, "oracle", "_ref", "localTensoRF")
    if not os.path.isfile(os.path.join(ref, "renderer.py")):
        pytest.skip("no staged reference (oracle/_ref) on this box")
    out = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, ref], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "PANELS_RENDER_OK 3" in out.stdout, (out.stdout[-1500:], out.stderr[-3000:])
