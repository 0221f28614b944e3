"""CPU-only: host-side logic of the Python mirror against the reference goldens -- the sample table,
the progressive-schedule bookkeeping (append_frame / append_rf blending rows), checkpoint restore,
test-frame exposure rule, pose math.  No CUDA calls (the render path itself refuses CPU tensors)."""
import numpy as np
import pytest
import torch

import localrf_b200 as L
from helpers import field_scalars, load_golden
from oracle import oracle as orc


def test_render_path_refuses_cpu_tensors():
    from gpu_helpers import module_from_golden
    m = module_from_golden(load_golden("opaque_32"), device="cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(4, 6))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.compute_densityfeature(torch.zeros(4, 3))


def test_constructor_matches_reference_init_and_table():
    """Same seed -> same parameters as the reference constructor (the goldens hold its init), same
    nSamples, same eval distance table, same state_dict keys."""
    from gpu_helpers import AABB, field_kwargs
    g = load_golden("cfg1_64")
    sc = field_scalars(g)
    torch.manual_seed(0)
    m = L.TensorVMSplit("cpu", AABB.clone(), sc["gridSize"], **field_kwargs(sc))
    assert m.nSamples == int(g["nSamples"])
    for k, v in m.state_dict().items():
        assert k in g, k
        np.testing.assert_array_equal(v.numpy(), g[k])
    np.testing.assert_array_equal(m.sample_table(False).numpy(), g["eval.z"])
    assert m.density_plane[0].is_contiguous(memory_format=torch.channels_last)
    assert m.density_plane[0].shape == (1, 8, 64, 64)


def test_train_table_consumes_rng_like_reference():
    from gpu_helpers import AABB, field_kwargs
    g = load_golden("cfg1_64")
    sc = field_scalars(g)
    torch.manual_seed(0)
    m = L.TensorVMSplit("cpu", AABB.clone(), sc["gridSize"], **field_kwargs(sc))
    torch.manual_seed(2)
    np.testing.assert_allclose(m.sample_table(True).numpy(), g["train.z"], rtol=2e-7, atol=0)


def test_upsample_keeps_layout_and_updates_sampling():
    from gpu_helpers import module_from_golden
    m = module_from_golden(load_golden("opaque_32"), device="cpu")
    m.upsample_volume_grid([40, 44, 48])
    assert m.gridSize.tolist() == [40, 44, 48] and m._grid_host == [40, 44, 48]
    assert m.app_plane[1].shape == (1, 24, 48, 40)          # [1, C, G_z, G_x]
    assert m.app_plane[1].is_contiguous(memory_format=torch.channels_last)
    assert m.density_line[0].shape == (1, 8, 48, 1)
    f = orc.Field({**{k: v.detach().numpy() for k, v in m.state_dict().items()},
                   "gridSize": [40, 44, 48], "step_ratio": 0.5})
    assert m.nSamples == f.n_samples()


def test_checkpoint_restore_and_bookkeeping_vs_reference():
    from gpu_helpers import local_from_golden
    g = load_golden("local3")
    lt = local_from_golden(g, device="cpu")
    assert len(lt.tensorfs) == 3 and len(lt.r_c2w) == 6
    np.testing.assert_array_equal(lt.blending_weights.numpy(), g["sd.blending_weights"])
    assert sorted(lt.state_dict().keys()) == sorted(k[3:] for k in g if k.startswith("sd."))
    # cam2world of the mirror == the oracle's restatement of sixD_to_mtx
    c2w = lt.get_cam2world(torch.tensor([1, 4, 5, 2])).detach().numpy()
    r6 = np.stack([g[f"sd.r_c2w.{i}"] for i in (1, 4, 5, 2)])
    np.testing.assert_allclose(c2w[:, :, :3], orc.sixD_to_mtx(r6), rtol=2e-6, atol=2e-7)


def test_progressive_schedule_blending_rows():
    """append_frame / append_rf reproduce the reference's blending matrix (the golden's was built by
    the reference's own calls: 4 frames, append_rf(2), frame, append_rf(1), frame)."""
    import bench
    g = load_golden("local3")
    aabb = 2 * torch.tensor([[-1.0, -1, -1], [1, 1, 1]])
    lt = L.LocalTensorfs(camera_prior=None, fov=85.6, n_init_frames=4, n_overlap=30, WH=(48, 40),
                         n_iters_per_frame=600, n_iters_reg=100, lr_R_init=5e-3, lr_t_init=5e-4,
                         lr_i_init=0, lr_exposure_init=1e-3, rf_lr_init=2e-2, rf_lr_basis=1e-3,
                         lr_decay_target_ratio=0.1, N_voxel_list={}, update_AlphaMask_list=[],
                         lr_upsample_reset=True, device="cpu", aabb=aabb, gridSize=[8, 8, 8],
                         **bench.field_kwargs())
    lt.append_rf(2); lt.append_frame(); lt.append_rf(1); lt.append_frame()
    np.testing.assert_allclose(lt.blending_weights.numpy(), g["sd.blending_weights"], atol=1e-7)
    assert lt.pose_linked_rf == [0, 0, 0, 0, 1, 2]


def test_test_frame_exposure_rule():
    from gpu_helpers import local_from_golden
    g = load_golden("local3")
    lt = local_from_golden(g, device="cpu")
    E = torch.stack(list(lt.exposure)).detach()
    n = len(lt.exposure)
    for v in range(n):
        out = lt._exposure_for([v], True, torch.device("cpu"))[0]
        vm = max(v - 1, 0); vm = 1 if vm == v else vm
        vp = min(v + 1, n - 1); vp = n - 2 if vm == v else vp
        torch.testing.assert_close(out, (E[vm] + E[vp]) / 2)


def test_field_tensor_table_matches_modules():
    """TensorBase._tensors reads the module attributes _FIELD_TENSORS names, in its order, which is _grad_params'
    and the order the gradients of the fused backward come back in; after an upsample too (new grid tensors)."""
    from gpu_helpers import module_from_golden
    from localrf_b200.tensorf import _FIELD_TENSORS
    m = module_from_golden(load_golden("cfg1_64"), device="cpu")
    for _ in range(2):
        grids, mlp = m._tensors()
        assert len(grids) == 12 and len(mlp) == 7
        assert all(t is m.get_parameter(attr) for (_, _, attr), t in zip(_FIELD_TENSORS, grids + mlp))
        assert m._grad_params() == grids + mlp
        m.upsample_volume_grid([20, 24, 28])


def test_grid_storage_setting_host_side():
    """set_grid_storage: validation, propagation through LocalTensorfs, inheritance by appended fields; the
    parameters and the state_dict are untouched (the 16-bit copies are an inference cache)."""
    from gpu_helpers import module_from_golden, local_from_golden
    m = module_from_golden(load_golden("opaque_32"), device="cpu")
    keys = set(m.state_dict().keys())
    assert m.grid_storage == "fp32"
    with pytest.raises(ValueError):
        m.set_grid_storage("fp16")
    assert m.set_grid_storage("bf16") is m and m.grid_storage == "bf16"
    assert set(m.state_dict().keys()) == keys and all(p.dtype == torch.float32 for p in m.parameters())
    m.set_grid_storage("fp32")
    pe = module_from_golden(load_golden("aniso_pe"), device="cpu")
    with pytest.raises(NotImplementedError):
        pe.set_grid_storage("bf16")
    lt = local_from_golden(load_golden("local3"), device="cpu")
    lt.set_grid_storage("bf16")
    assert all(rf.grid_storage == "bf16" for rf in lt.tensorfs)
    n = len(lt.tensorfs)
    lt.append_frame(); lt.append_rf(1)
    assert len(lt.tensorfs) == n + 1 and lt.tensorfs[-1].grid_storage == "bf16"
