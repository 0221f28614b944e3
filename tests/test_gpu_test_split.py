"""GPU: the test split on the device.  lrf_resize_linear against tests/resize_oracle.py (which equals cv2.resize without
IPP, tests/test_resize_cpu.py), DeviceFrameDataset(split="test") against the arrays the unmodified reference's
read_meta built from the golden scenes (tests/golden/ingest.npz), and the held-out loop of FramePipeline fed from the
device split against the same loop fed the reference's host arrays."""
import json
import os

import numpy as np
import pytest
import torch

import ingest_oracle as io
import resize_oracle as ro
from test_resize_cpu import GRID

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ingest.npz")
F32 = np.float32


@pytest.fixture
def ipp_off():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.ascontiguousarray(a).view(np.uint32)


def frame(w0, h0, seed):
    a = np.random.default_rng(seed).random((h0, w0, 3), dtype=np.float32)
    return a if seed % 2 == 0 else (a * 4000 - 2000).astype(F32)


@pytest.mark.parametrize("w0,h0,W,H", GRID)
def test_kernel_equals_the_restatement(w0, h0, W, H):
    from localrf_b200.metrics import resize_linear
    for seed in range(2):
        a = frame(w0, h0, seed)
        want = bits(ro.resize(a, W, H))
        src = torch.from_numpy(a).cuda()
        got = resize_linear(src, W, H)
        assert got.shape == (H, W, 3) and got.dtype == torch.float32 and got.is_cuda
        assert np.array_equal(bits(got), want), (w0, h0, W, H, seed)
        assert np.array_equal(bits(resize_linear(src, W, H)), want)              # bitwise repeatable
        # rows further apart than 3 w0 floats, in and out
        big = torch.full((h0 + 2, w0 + 5, 3), float("nan"), device="cuda")
        big[1:h0 + 1, 2:w0 + 2] = src
        out_big = torch.full((H + 1, W + 3, 3), -7.0, device="cuda")
        out = out_big[:H, 1:W + 1]
        assert resize_linear(big[1:h0 + 1, 2:w0 + 2], W, H, out=out) is out
        assert np.array_equal(bits(out), want)
        rest = out_big.clone()
        rest[:H, 1:W + 1] = -7.0
        assert bool((rest == -7.0).all())                                         # nothing outside `out` written
        # a pinned source, read in place
        pinned = torch.from_numpy(a).pin_memory()
        assert np.array_equal(bits(resize_linear(pinned, W, H)), want)


def test_binding_refuses_bad_inputs():
    from localrf_b200.metrics import resize_linear
    a = torch.rand(8, 6, 3, device="cuda")
    with pytest.raises(TypeError):
        resize_linear(a.double(), 3, 4)
    with pytest.raises(ValueError):
        resize_linear(a.cpu(), 3, 4)                                              # pageable host memory
    with pytest.raises(ValueError):
        resize_linear(a[..., :2], 3, 4)
    with pytest.raises(ValueError):
        resize_linear(a, 3, 4, out=torch.empty(4, 3, 3))                         # host out
    with pytest.raises(ValueError):
        resize_linear(a, 3, 4, out=torch.empty(3, 4, 3, device="cuda"))           # wrong shape
    with pytest.raises(ValueError):
        resize_linear(a, 0, 4)                                                    # refused by the C ABI


def golden():
    z = np.load(GOLDEN)
    return z, [(str(c), str(s)) for c, s in zip(z["cases"], z["scenes"])]


def make_test_split(z, case, scene, d):
    from localrf_b200 import DeviceFrameDataset
    cfg = json.loads(str(z[f"{case}.config"]))
    io.write_golden_scene(z, scene, d)
    ds = DeviceFrameDataset(d, split="test", downsampling=cfg["downsampling"], load_depth=cfg["load_depth"],
                            load_flow=cfg["load_flow"], frames_chunk=cfg["frames_chunk"],
                            n_init_frames=cfg["n_init_frames"], test_frame_every=cfg["test_frame_every"])
    return ds, cfg


def golden_test_frames(z, case, cfg):
    """The golden train-split arrays at the test frames, in np.stack's shapes: key -> [N, h, w(, k)]."""
    w, h = cfg["img_wh"]
    sel = np.flatnonzero(z[f"{case}.test_mask"] == 1)
    out = {}
    for key, attr in (("rgbs", "all_rgbs"), ("invdepths", "all_invdepths"), ("fwd_flow", "all_fwd_flow"),
                      ("fwd_mask", "all_fwd_mask"), ("bwd_flow", "all_bwd_flow"), ("bwd_mask", "all_bwd_mask")):
        name = f"{case}.frames.{key}"
        if name in z:
            a = z[name][sel]
            k = a.shape[-1]
            out[attr] = a.reshape(len(sel), h, w, k) if k > 1 else a.reshape(len(sel), h, w)
    return sel, out


def test_test_split_equals_the_reference(tmp_path):
    z, cases = golden()
    for case, scene in cases:
        ds, cfg = make_test_split(z, case, scene, str(tmp_path / case))
        sel, want = golden_test_frames(z, case, cfg)
        n = len(sel)
        assert n == 3 and ds.num_images == n and ds.img_wh == cfg["img_wh"]
        assert ds.n_px_per_frame == cfg["img_wh"][0] * cfg["img_wh"][1]
        assert ds.all_fbases == {f"{i:05d}": k for k, i in enumerate(sel)}
        assert [ds.get_frame_fbase(k) for k in range(n)] == [f"{i:05d}" for i in sel]
        assert np.array_equal(ds.test_mask, z[f"{case}.test_mask"])
        assert ds.active_frames_bounds == [0, min(cfg["n_init_frames"], n)] and ds.loaded_frames == n
        assert ds.has_left_frames() == (min(cfg["n_init_frames"], n) < n)
        assert ds.all_loss_weights is None
        for attr in ("all_rgbs", "all_invdepths", "all_fwd_flow", "all_fwd_mask", "all_bwd_flow", "all_bwd_mask"):
            t = getattr(ds, attr)
            if attr not in want:
                assert t is None, (case, attr)
                continue
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), (case, attr)
            assert tuple(t.shape) == want[attr].shape, (case, attr, tuple(t.shape))
            assert np.array_equal(bits(t), want[attr].view(np.uint32)), (case, attr)
        assert not ds._raw and not ds._scratch                   # every decoded plane and the scratch dropped
        floats = [k for k, v in vars(ds).items() if isinstance(v, np.ndarray) and v.dtype.kind == "f"]
        assert not floats, floats                                # the host keeps no float copy


def test_sampler_refuses_the_test_split_and_other_splits_raise(tmp_path):
    from localrf_b200 import DeviceFrameDataset, DeviceRaySampler
    z, cases = golden()
    case, scene = cases[0]
    ds, _ = make_test_split(z, case, scene, str(tmp_path / "a"))
    with pytest.raises(ValueError, match="train split"):
        DeviceRaySampler(ds, "cuda")
    with pytest.raises(ValueError, match="split='val'"):
        DeviceFrameDataset(str(tmp_path / "a"), split="val")


@pytest.mark.parametrize("W,H", [(20, 15), (27, 19)])
def test_held_out_loop_equals_the_host_path(tmp_path, ipp_off, W, H):
    """Two FramePipeline runs over every test frame: ground truth from the device split through resize_linear and the
    panels from its all_* tensors, against the reference's host arrays resized with cv2.resize (IPP off) and handed
    over as numpy.  rgb8, mse, ssim and the three panels are bitwise equal.  20 x 15 is the exact 2x of the 40 x 30
    frames (INTER_AREA), 27 x 19 the linear rule."""
    import bench
    import localrf_b200 as L
    from localrf_b200.metrics import resize_linear
    wl = bench.Workload("cfg5", 48)
    lt = wl.build(L.LocalTensorfs, quiet=True).to("cuda")
    z, cases = golden()
    for case, scene in cases:
        ds, cfg = make_test_split(z, case, scene, str(tmp_path / case))
        sel, host = golden_test_frames(z, case, cfg)

        def run(device_split):
            pipe = L.FramePipeline(lt, W, H, n_buffers=2)
            out = []
            for k, f in enumerate(sel):
                if pipe.in_flight() == 2:
                    out.append({a: (b.copy() if isinstance(b, np.ndarray) else b) for a, b in pipe.fetch().items()})
                src = ds if device_split else None
                arrays = {a: (getattr(src, a)[k] if src is not None else host[a][k]) for a in host}
                gt = resize_linear(arrays["all_rgbs"], W, H) if device_split else \
                    cv2.resize(arrays["all_rgbs"], (W, H))
                panels = {name: arrays["all_" + name] for name in ("fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask")
                          if "all_" + name in arrays}
                if "all_invdepths" in arrays:
                    panels["invdepth"] = arrays["all_invdepths"]
                pipe.submit(torch.tensor([int(f)], device="cuda"), gt=gt, tag=int(f), test_id=True,
                            panels=dict(idx=int(f), **panels))
            while pipe.in_flight():
                out.append({a: (b.copy() if isinstance(b, np.ndarray) else b) for a, b in pipe.fetch().items()})
            return out

        dev_run, host_run = run(True), run(False)
        assert len(dev_run) == len(host_run) == len(sel)
        for a, b in zip(dev_run, host_run):
            assert a["tag"] == b["tag"]
            assert np.array_equal(a["rgb8"], b["rgb8"]) and np.array_equal(a["depth8"], b["depth8"])
            assert np.array_equal(np.float64(a["mse"]).view(np.uint64), np.float64(b["mse"]).view(np.uint64))
            assert np.array_equal(np.float64(a["ssim"]).view(np.uint64), np.float64(b["ssim"]).view(np.uint64))
            for key in ("fwd_flow_cmp", "bwd_flow_cmp", "depth_cmp"):
                if b[key] is None:
                    assert a[key] is None, (case, key)
                else:
                    assert np.array_equal(bits(a[key]), bits(b[key])), (case, a["tag"], key)
