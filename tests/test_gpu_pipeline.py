"""-m gpu: the frame-render pipeline (localrf_b200/pipeline.py): frames rendered through the ring of pinned
buffers equal direct LocalTensorfs.forward calls; the device-side 8-bit conversions equal the host-side
conversions renderer.py applies (cv2.imwrite's saturating round of 255 * rgb[..., ::-1]; visualize_depth =
cv2.applyColorMap of the truncated, clipped, normalised depth, utils/utils.py:179-197)."""
import numpy as np
import pytest
import torch

import metrics_oracle as orc

pytestmark = pytest.mark.gpu


def test_pipeline_frames_match_direct_calls_and_host_conversions():
    import cv2
    import bench
    import localrf_b200 as L
    wl = bench.Workload("cfg5", 48)                       # 8 small fields, 64 frames, cross-fades
    lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
    W, H = 96, 80
    pipe = L.FramePipeline(lt, W, H, depth_minmax=(0.0, 5.0), n_buffers=3, keep_float=True)
    frames = [torch.tensor([f], device="cuda") for f in (0, 5, 6, 7, 8, 30, 63)]
    # the yielded arrays are views of the ring's pinned buffers (valid until n_buffers more submits): copy
    got = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in fr.items()}
           for fr in pipe.render(frames, floater_thresh=0.5)]
    assert len(got) == len(frames) and pipe.in_flight() == 0
    ids = torch.arange(W * H, dtype=torch.int64, device="cuda")
    for view, fr in zip(frames, got):
        with torch.no_grad():
            rgb, depth, _, _ = lt(ids, view, W, H, is_train=False, floater_thresh=0.5)
        rgb, depth = rgb.cpu().numpy().reshape(H, W, 3), depth.cpu().numpy().reshape(H, W)
        np.testing.assert_array_equal(fr["rgb"], rgb)                     # zero-copy float outputs, bit-exact
        np.testing.assert_array_equal(fr["depth"], depth)
        np.testing.assert_array_equal(fr["rgb8"], orc.rgb8(rgb))
        x = (np.nan_to_num(depth) - 0) / (5 - 0 + 1e-8)                  # visualize_depth(depth, [0, 5])
        idx = (255 * np.clip(x, 0, 1)).astype(np.uint8)
        np.testing.assert_array_equal(fr["depth8"], cv2.applyColorMap(idx, cv2.COLORMAP_JET))


def test_pipeline_depth_ranges_other_than_0_5():
    """Depth ranges other than renderer.py's (0, 5), with a colour map that names its index: every pixel picks
    the index visualize_depth picks.  (0.3, 2.9) lies below this scene's depths, so every pixel saturates; the
    second range is the frames' 5th to 95th depth percentile, rounded to Python numbers, and spans most indices."""
    import bench
    import localrf_b200 as L
    wl = bench.Workload("cfg5", 48)
    lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
    W, H = 96, 80
    lut = np.stack([np.arange(256), np.arange(256)[::-1], np.full(256, 7)], -1).astype(np.uint8)
    frames = [torch.tensor([f], device="cuda") for f in (0, 6, 30, 63)]

    def run(lo, hi):
        pipe = L.FramePipeline(lt, W, H, depth_minmax=(lo, hi), n_buffers=2, lut=lut, keep_float=True)
        got = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in fr.items()}
               for fr in pipe.render(frames, floater_thresh=0.5)]
        for fr in got:
            np.testing.assert_array_equal(fr["depth8"], orc.depth8(fr["depth"], lo, hi, lut))
            np.testing.assert_array_equal(fr["rgb8"], orc.rgb8(fr["rgb"]))
        return got, np.concatenate([fr["depth8"][..., 0].ravel() for fr in got])

    got, _ = run(0.3, 2.9)
    d = np.concatenate([fr["depth"].ravel() for fr in got])
    lo, hi = (round(float(v), 2) for v in np.percentile(d[np.isfinite(d)], [5, 95]))
    _, idx = run(lo, hi)
    assert lo < hi and len(np.unique(idx)) > 64, (lo, hi, len(np.unique(idx)))


def test_pipeline_refuses_overflow_and_cpu_model():
    import bench
    import localrf_b200 as L
    lt = bench.build_scene("cuda", 32)
    pipe = L.FramePipeline(lt, 32, 24, n_buffers=2)
    v = torch.tensor([0], device="cuda")
    pipe.submit(v); pipe.submit(v)
    with pytest.raises(RuntimeError, match="in flight"):
        pipe.submit(v)
    assert pipe.fetch() is not None and pipe.fetch() is not None and pipe.fetch() is None
    with pytest.raises(RuntimeError, match="CUDA"):
        L.FramePipeline(bench.build_scene("cpu", 16), 8, 8)
