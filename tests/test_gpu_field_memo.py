"""What a TensorVMSplit derives from its tensors and keeps between calls -- its LrfFields (with and without a distance
table, over fp32 or bf16 grids), the bf16 grid copies, the host copies of the aabbs and the prepared MLP blocks --
follows every change to the field.  After each event that changes one (an Adam step, an upsample, an alpha-mask
rebuild, load_state_dict, a grid-storage switch) the field computes bit for bit what a field rebuilt from its
state_dict computes."""
import pytest
import torch

import localrf_b200 as L
from gpu_helpers import AABB, field_kwargs, module_from_golden
from helpers import field_scalars, load_golden
from localrf_b200.optim import adam_step

pytestmark = pytest.mark.gpu


def _rebuilt(m, kw):
    """A new field from m.state_dict(), built as LocalTensorfs.load builds one (gridSize from the planes, an
    AlphaGridMask from the mask entries), with m's grid storage."""
    sd = m.state_dict()
    plane0, line0 = sd["density_plane.0"], sd["density_line.0"]
    f = L.TensorVMSplit("cuda", AABB.clone().cuda(), [plane0.shape[3], plane0.shape[2], line0.shape[2]], **kw)
    if "alphaMask.aabb" in sd:
        f.alphaMask = L.AlphaGridMask("cuda", sd["alphaMask.aabb"], sd["alphaMask.alpha_volume"])
    f.load_state_dict(sd)
    return f.set_grid_storage(m.grid_storage)


def _outputs(f, rays, xyz):
    rgb32, depth32 = f(rays)            # autograd records: the fused node, which reads the fp32 grids
    with torch.no_grad():
        rgb, depth = f(rays)            # eval: the grids of the field's grid storage
        out = dict(rgb32=rgb32.detach(), depth32=depth32.detach(), rgb=rgb, depth=depth,
                   density=f.compute_densityfeature(xyz), app=f.compute_appfeature(xyz), alpha=f.getDenseAlpha())
    out["l1"] = f.density_L1().detach()
    torch.cuda.synchronize()
    return out


def test_memoised_field_state_follows_every_change():
    g = load_golden("cfg1_64")
    kw = field_kwargs(field_scalars(g))
    m = module_from_golden(g).set_grid_storage("bf16")
    gen = torch.Generator().manual_seed(0)
    rays = torch.cat([0.1 * torch.randn(512, 3, generator=gen), torch.randn(512, 3, generator=gen)], -1).cuda()
    xyz = (torch.rand(4096, 3, generator=gen) * 2.2 - 1.1).cuda()
    seen = [_outputs(m, rays, xyz)]

    def check(event):
        ours, ref = _outputs(m, rays, xyz), _outputs(_rebuilt(m, kw), rays, xyz)
        for k in ours:
            if k != "l1":
                assert torch.equal(ours[k], ref[k]), (event, k, float((ours[k] - ref[k]).abs().max()))
        # density_L1 adds fp64 block partials atomically: two calls may differ in the last bit of the fp32 result
        ulp = torch.nextafter(ref["l1"], torch.tensor(float("inf"), device="cuda")) - ref["l1"]
        assert float((ours["l1"] - ref["l1"]).abs()) <= float(ulp), (event, float(ours["l1"]), float(ref["l1"]))
        assert not torch.equal(ours["rgb"], seen[-1]["rgb"]), f"{event} left the render unchanged"
        seen.append(ours)

    opt = torch.optim.Adam(m.get_optparam_groups(0.02, 1e-3), betas=(0.9, 0.99))
    rgb, depth = m(rays)
    ((rgb - 0.5).square().sum() + depth.sum() + m.density_L1()).backward()
    adam_step([opt])
    check("adam_step")

    m.upsample_volume_grid([80, 72, 96])
    check("upsample_volume_grid")

    # a threshold that keeps about half the lattice, so the new mask changes the render: the mask keeps the voxels
    # whose 3x3x3 max-pooled alpha reaches it (tensorBase.py:517-536)
    dims = (40, 36, 48)
    pooled = torch.nn.functional.max_pool3d(m.getDenseAlpha(dims)[None, None], 3, stride=1, padding=1)
    kw["alphaMask_thres"] = m.alphaMask_thres = float(pooled.median())
    m.updateAlphaMask(dims)
    kept = float(m.alphaMask.alpha_volume.mean())
    assert 0 < kept < 1, kept
    check("updateAlphaMask")

    sd = {k: v.clone() for k, v in m.state_dict().items()}
    gen = torch.Generator(device="cuda").manual_seed(1)
    for k, v in sd.items():
        if not k.startswith(("aabb", "invaabbSize", "alphaMask")):
            v.add_(0.01 * torch.randn(v.shape, generator=gen, device="cuda"))
    sd["aabb"] *= 1.25
    sd["invaabbSize"] = 2.0 / (sd["aabb"][1] - sd["aabb"][0])
    sd["alphaMask.aabb"] *= 0.9
    sd["alphaMask.invgridSize"] = 2.0 / (sd["alphaMask.aabb"][1] - sd["alphaMask.aabb"][0])
    sd["alphaMask.alpha_volume"] = sd["alphaMask.alpha_volume"].flip(-1).contiguous()
    m.load_state_dict(sd)
    check("load_state_dict")

    m.set_grid_storage("bf16")
    m.set_grid_storage("fp32")
    check("set_grid_storage bf16 -> fp32")
