"""-m gpu: test-frame MSE and SSIM on the device (localrf_b200/metrics.py, lrf_image_metrics) against the
reference's rgb_ssim (utils/utils.py:232-287) and renderer.py's MSE stored in tests/golden/ssim.npz, against the
oracle on a rendered 800x800 frame, and inside FramePipeline and the unmodified reference renderer."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_metrics_cpu import golden_cases

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fp64_mse(img, gt):
    d = np.asarray(gt, np.float32) - np.asarray(img, np.float32)
    return float(np.sum((d * d).astype(np.float64)) / d.size)


@pytest.mark.parametrize("name", [c[0] for c in golden_cases()])
def test_golden_cases_match_reference(name):
    from localrf_b200 import metrics
    case, params = next((c, p) for n, c, p in golden_cases() if n == name)
    gt, img = (torch.from_numpy(case[k]).cuda() for k in ("gt", "img"))
    out = metrics.image_metrics(img, gt, **params).cpu().numpy()
    assert abs(out[1] - float(case["ssim"])) <= 1e-12
    mse_ref = float(case["mse"])
    assert abs(out[0] - mse_ref) <= 1e-6 * mse_ref
    want = _fp64_mse(case["img"], case["gt"])
    assert abs(out[0] - want) <= 1e-12 * want
    # the reference's own signature: numpy in, float / numpy map out (renderer.py:163 passes gt first)
    s = metrics.rgb_ssim(case["gt"], case["img"], params["max_val"], params["filter_size"], params["filter_sigma"],
                         params["k1"], params["k2"])
    assert isinstance(s, float) and s == out[1]
    m = metrics.rgb_ssim(case["gt"], case["img"], params["max_val"], params["filter_size"], params["filter_sigma"],
                         params["k1"], params["k2"], return_map=True)
    assert isinstance(m, np.ndarray) and m.dtype == np.float64 and m.shape == case["ssim_map"].shape
    np.testing.assert_allclose(m, case["ssim_map"], rtol=0, atol=1e-12)
    # CUDA tensors: 0-d tensor / map tensor on the device
    t = metrics.rgb_ssim(gt, img, params["max_val"], params["filter_size"], params["filter_sigma"], params["k1"],
                         params["k2"])
    assert t.is_cuda and t.dim() == 0 and t.dtype == torch.float64 and float(t) == out[1]


def test_identical_frames_give_exactly_one_and_zero():
    from localrf_b200 import metrics
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.rand(123, 77, 3, device="cuda", generator=g)
    out = metrics.image_metrics(a, a.clone()).cpu()
    assert out[0].item() == 0.0 and out[1].item() == 1.0


@pytest.fixture(scope="module")
def frame800():
    import bench
    lt = bench.build_scene("cuda")                                   # cfg2: the bench's 300^3 field
    W = H = 800
    ids = torch.arange(W * H, device="cuda")
    with torch.no_grad():
        rgb, _, _, _ = lt(ids, torch.tensor([0], device="cuda"), W, H, is_train=False, chunk=4096)
    g = torch.Generator(device="cuda").manual_seed(11)
    gt = (rgb + 0.03 * torch.randn(rgb.shape, device="cuda", generator=g)).clamp(0, 1)
    return rgb.reshape(H, W, 3).contiguous(), gt.reshape(H, W, 3).contiguous()


def test_800x800_render_matches_oracle(frame800):
    from localrf_b200 import metrics
    import metrics_oracle as orc
    rgb, gt = frame800
    out = metrics.image_metrics(rgb, gt).cpu().numpy()
    m = metrics.rgb_ssim(gt, rgb, 1.0, return_map=True).cpu().numpy()
    a, b = gt.cpu().numpy(), rgb.cpu().numpy()
    want_map = orc.ssim(a, b, 1.0, return_map=True)
    np.testing.assert_allclose(m, want_map, rtol=0, atol=1e-12)
    assert abs(out[1] - orc.ssim(a, b, 1.0)) <= 1e-12
    want = orc.mse(b, a)
    assert abs(out[0] - want) <= 1e-12 * want
    t = float(((gt.cpu() - rgb.cpu()) ** 2).mean())                # renderer.py:162 (torch fp32)
    assert abs(out[0] - t) <= 1e-6 * t


def test_repeated_calls_are_bit_identical(frame800):
    from localrf_b200 import metrics
    rgb, gt = frame800
    outs = [metrics.image_metrics(rgb, gt).cpu() for _ in range(3)]
    maps = [metrics.rgb_ssim(gt, rgb, 1.0, return_map=True).cpu() for _ in range(3)]
    for o, m in zip(outs[1:], maps[1:]):
        assert torch.equal(o, outs[0]) and torch.equal(m, maps[0])


def test_stride4_view_and_pinned_gt_are_bit_identical(frame800):
    from localrf_b200 import metrics
    rgb, gt = frame800
    H, W = rgb.shape[:2]
    pix = torch.full((H * W, 4), -7.0, device="cuda")                 # the interleaved [N,4] pix layout
    pix[:, :3] = rgb.reshape(-1, 3)
    want = metrics.image_metrics(rgb, gt).cpu()
    assert torch.equal(metrics.image_metrics(pix[:, :3], gt, W=W).cpu(), want)
    assert torch.equal(metrics.image_metrics(rgb, gt.cpu().pin_memory()).cpu(), want)
    assert torch.equal(metrics.image_metrics(rgb.reshape(-1, 3).cpu().pin_memory(), gt.cpu().pin_memory(),
                                             W=W).cpu(), want)


def test_pipeline_metrics_match_direct_render():
    import bench
    import localrf_b200 as L
    from localrf_b200 import metrics
    wl = bench.Workload("cfg5", 48)
    lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
    W, H = 96, 80
    ids = torch.arange(W * H, dtype=torch.int64, device="cuda")
    views = [0, 5, 30, 63]
    g = torch.Generator().manual_seed(5)
    gts = [torch.rand(H, W, 3, generator=g) for _ in views]
    kinds = [lambda t: t.numpy(), lambda t: t.pin_memory(), lambda t: t.cuda(), lambda t: t.numpy().tolist()]
    frames = [torch.tensor([v], device="cuda") for v in views]

    def run(with_gt):
        pipe = L.FramePipeline(lt, W, H, n_buffers=2, keep_float=True)
        items = [(f, {"gt": k(t)} if with_gt else {}) for f, k, t in zip(frames, kinds, gts)]
        return [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in fr.items()}
                for fr in pipe.render(items, floater_thresh=0.5)]

    plain, scored = run(False), run(True)
    for view, gt, p, s in zip(frames, gts, plain, scored):
        assert "mse" not in p and "ssim" not in p
        for k in ("rgb8", "depth8", "rgb", "depth"):
            np.testing.assert_array_equal(s[k], p[k])
        with torch.no_grad():
            rgb, _, _, _ = lt(ids, view, W, H, is_train=False, floater_thresh=0.5)
        want = metrics.image_metrics(rgb, gt.cuda(), W=W).cpu().numpy()
        assert isinstance(s["mse"], float) and isinstance(s["ssim"], float)
        assert s["mse"] == want[0] and s["ssim"] == want[1]


SCRIPT = r'''
import sys, types
import numpy as np, torch
ROOT, REF = sys.argv[1], sys.argv[2]
sys.path[:0] = [ROOT + "/dropin", ROOT, REF]
from oracle import ref_loader
for name, attrs in (("kornia", dict(create_meshgrid=None)), ("matplotlib", dict(use=lambda *a, **k: None)),
                    ("matplotlib.pyplot", {}), ("matplotlib.cm", {}), ("plyfile", {}), ("skimage", {}),
                    ("skimage.measure", {}), ("imageio", {}), ("lpips", {})):
    ref_loader._stub(name, **attrs)
import renderer                                     # the reference's module, unmodified
import localrf_b200 as L
import bench
W, H = 64, 48
renderer.draw_poses = lambda poses, colours: np.zeros((H, W, 3), np.uint8)      # matplotlib plot: stubbed I/O
lt = bench.Workload("cfg5", 40).build(L.LocalTensorfs, quiet=True).to("cuda")
n = len(lt.r_c2w)
test_idx = (9, 30, 50)
train_ds = types.SimpleNamespace(all_fbases={f"{i:04d}": i for i in range(n)})
train_ds.get_frame_fbase = lambda i: f"{i:04d}"
ids = torch.arange(W * H, device="cuda")
g = torch.Generator().manual_seed(9)
rgbs = []
with torch.no_grad():
    for i in test_idx:
        rgb, _, _, _ = lt(ids, torch.tensor([i], device="cuda"), W, H, is_train=False, test_id=True, chunk=4096,
                          floater_thresh=0.5)
        rgb = rgb.reshape(H, W, 3).cpu()
        rgbs.append((rgb + 0.05 * torch.randn(rgb.shape, generator=g)).clamp(0, 1).numpy())
test_ds = types.SimpleNamespace(all_fbases={f"{i:04d}": k for k, i in enumerate(test_idx)}, all_rgbs=rgbs,
                                all_fwd_flow=None, all_invdepths=None)
args = types.SimpleNamespace(batch_size=4096, device="cuda")
poses = lt.get_cam2world().detach()
kw = dict(savePath=None, save_video=False, save_frames=False, test=True, train_dataset=train_ds, start=0,
          floater_thresh=0.5, add_frame_to_list=True)
ref = renderer.render(test_ds, poses, lt, args, W=W, H=H, **kw)[-1]
renderer.rgb_ssim = L.metrics.rgb_ssim
ours = renderer.render(test_ds, poses, lt, args, W=W, H=H, **kw)[-1]
assert sorted(ref) == sorted(ours) == sorted(test_ds.all_fbases), (sorted(ref), sorted(ours))
worst = 0.0
for fb in ref:
    assert isinstance(ours[fb]["ssim"], float)
    worst = max(worst, abs(ours[fb]["ssim"] - ref[fb]["ssim"]))
    assert torch.equal(ours[fb]["mse"], ref[fb]["mse"])
assert worst <= 1e-12, worst
print("RENDER_METRICS_OK", len(ref), worst)
'''


def test_reference_renderer_test_metrics_with_device_ssim():
    ref = os.path.join(ROOT, "oracle", "_ref", "localTensoRF")
    if not os.path.isfile(os.path.join(ref, "renderer.py")):
        pytest.skip("no staged reference (oracle/_ref) on this box")
    out = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, ref], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "RENDER_METRICS_OK 3" in out.stdout, (out.stdout[-1500:], out.stderr[-3000:])
