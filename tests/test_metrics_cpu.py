"""CPU-only: the numpy SSIM / MSE (tests/metrics_oracle.py) against the reference's rgb_ssim and renderer.py's
torch-fp32 MSE stored in tests/golden/ssim.npz; lrf_image_metrics' argument checks and scratch size without a
device; metrics.rgb_ssim refusing to run without one."""
import ctypes as C

import numpy as np
import pytest
import torch

from localrf_b200 import _lib
import metrics_oracle as orc

GOLDEN = "tests/golden/ssim.npz"


def golden_cases():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), GOLDEN))
    for name in g["names"]:
        name = str(name)
        p = g[f"{name}.params"]
        params = dict(max_val=float(p[0]), filter_size=int(p[1]), filter_sigma=float(p[2]), k1=float(p[3]),
                      k2=float(p[4]))
        yield name, {k.split(".", 1)[1]: g[k] for k in g.files if k.startswith(name + ".")}, params


@pytest.mark.parametrize("name", [c[0] for c in golden_cases()])
def test_oracle_matches_reference_rgb_ssim_and_mse(name):
    case, params = next((c, p) for n, c, p in golden_cases() if n == name)
    gt, img = case["gt"], case["img"]
    assert abs(orc.ssim(gt, img, **params) - float(case["ssim"])) <= 1e-13
    m = orc.ssim(gt, img, **params, return_map=True)
    assert m.shape == case["ssim_map"].shape == (gt.shape[0] - params["filter_size"] + 1,
                                                  gt.shape[1] - params["filter_size"] + 1, 3)
    # scipy's horizontal pass rounds its sums in a different order than any plain loop: one rounding of a
    # moment near 1, divided by 2 s01 + c2 ~ 1e-3 where the windows are nearly flat, moves the smooth case's
    # map by up to ~3e-13; the others stay below 1e-14
    np.testing.assert_allclose(m, case["ssim_map"], rtol=0, atol=1e-12)
    assert abs(orc.mse(img, gt) - float(case["mse"])) <= 1e-6 * float(case["mse"])


def _call(L, img=1, img_stride=3, gt=1, gt_stride=3, H=32, W=32, fs=11, out=1, scratch=8, nbytes=1 << 20):
    p = lambda v: C.c_void_p(v) if v else None
    return L.lrf_image_metrics(p(img), img_stride, p(gt), gt_stride, H, W, 1.0, fs, 1.5, 0.01, 0.03, p(out), None,
                               p(scratch), nbytes, None)


@pytest.mark.parametrize("kw, code, word", [
    (dict(img=0), -1, b"img"), (dict(gt=0), -1, b"gt"), (dict(out=0), -1, b"out"),
    (dict(img_stride=2), -1, b"img_stride"), (dict(gt_stride=1), -1, b"gt_stride"),
    (dict(H=10), -1, b"filter_size"), (dict(W=5), -1, b"filter_size"),
    (dict(nbytes=8), -1, b"scratch_bytes"), (dict(scratch=0), -1, b"scratch"),
    (dict(fs=0), -2, b"filter_size"), (dict(fs=17), -2, b"filter_size"),
])
def test_image_metrics_validation_without_gpu(kw, code, word):
    L = _lib.lib()
    assert _call(L, **kw) == code
    assert word in L.lrf_last_error()


def test_image_metrics_scratch_bytes():
    L = _lib.lib()
    f = L.lrf_image_metrics_scratch_bytes
    assert f(10, 32, 11) == 0 and f(32, 10, 11) == 0 and f(32, 32, 0) == 0 and f(64, 64, 17) == 0
    assert f(11, 11, 11) > 0 and f(1, 1, 1) > 0
    small, big = f(100, 100, 11), f(800, 800, 11)
    assert 0 < small < big and f(1600, 800, 11) > big and f(800, 800, 16) == big


def test_rgb_ssim_needs_a_cuda_device(monkeypatch):
    from localrf_b200 import metrics
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    a = np.zeros((16, 16, 3), np.float32)
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.rgb_ssim(a, a, 1)
