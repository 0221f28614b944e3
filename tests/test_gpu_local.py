"""-m gpu: LocalTensorfs.forward (ray generation + multi-field blend + exposure + clamp) against the
reference goldens, restored through the reference's checkpoint path (`load`)."""
import numpy as np
import pytest
import torch

from helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module", params=["local3", "local3_fov360"])
def scene(request):
    from gpu_helpers import local_from_golden
    g = load_golden(request.param)
    return g, local_from_golden(g)


def _call(lt, g, case, ids, view_ids, **kw):
    W, H = int(g["W"]), int(g["H"])
    with torch.no_grad():
        rgb, depth, dirs, ij = lt(torch.from_numpy(ids).cuda(), torch.as_tensor(view_ids).cuda(),
                                  W, H, **kw)
    torch.cuda.synchronize()
    assert rel_err(rgb.cpu().numpy(), g[f"{case}.rgb"]) < TOL, case
    assert rel_err(depth.cpu().numpy(), g[f"{case}.depth"]) < TOL, case
    np.testing.assert_allclose(dirs.cpu().numpy(), g[f"{case}.directions"], rtol=2e-6, atol=1e-6)
    assert np.array_equal(ij.cpu().numpy(), g[f"{case}.ij"])


def test_state_dict_keys_match_reference(scene):
    g, lt = scene
    ref_keys = sorted(k[3:] for k in g if k.startswith("sd."))
    assert sorted(lt.state_dict().keys()) == ref_keys


def test_blend3(scene):
    g, lt = scene
    bw = torch.from_numpy(g["blend3"]).cuda()
    _call(lt, g, "blend3", g["ray_ids"], [2], is_train=False, blending_weights=bw, chunk=256)
    _call(lt, g, "blend3_testid", g["ray_ids"], [2], is_train=False, blending_weights=bw,
          chunk=256, test_id=True, floater_thresh=0.5)


@pytest.mark.parametrize("fr", [0, 3, 5])
def test_natural_rows_external_pose(scene, fr):
    g, lt = scene
    if f"frame{fr}.rgb" not in g:
        pytest.skip("not in this fixture")
    c2w = torch.from_numpy(g[f"frame{fr}.cam2world"]).cuda()
    _call(lt, g, f"frame{fr}", g["ray_ids"], [fr], is_train=False, cam2world=c2w, chunk=128)


def test_train_mode_multi_view(scene):
    g, lt = scene
    z = torch.from_numpy(g["train.z0"]).cuda()
    rf = lt.tensorfs[-1]
    orig = rf.sample_table
    rf.sample_table = lambda *a, **k: z          # the reference's own jittered table
    try:
        _call(lt, g, "train", g["train.ray_ids"], g["train.view_ids"], is_train=True)
    finally:
        rf.sample_table = orig


def test_repeated_call_refuses_pageable_id_copy(scene, monkeypatch):
    """A repeated eval call reuses the first call's plan.  Pinned int32 ids convert to a pageable int64 copy, which
    the kernel cannot read: the repeated call refuses it like the first call does, before anything is launched."""
    from localrf_b200 import _lib
    g, lt = scene
    W, H = int(g["W"]), int(g["H"])
    ids = torch.from_numpy(g["ray_ids"]).to(torch.int64).pin_memory()
    with torch.no_grad():
        lt(ids, [2], W, H, is_train=False)
    torch.cuda.synchronize()
    real = _lib.lib()

    class NoRender:
        def __getattr__(self, name):
            if name == "lrf_render":
                def launched(*args):
                    raise AssertionError("launched")
                return launched
            return getattr(real, name)

    monkeypatch.setattr(_lib, "lib", NoRender)
    with torch.no_grad(), pytest.raises(RuntimeError, match="must be pinned"):
        lt(ids.to(torch.int32).pin_memory(), [2], W, H, is_train=False)
