"""Helpers for the -m gpu parity tests (build product modules from golden fixtures)."""
import math

import numpy as np
import torch

import localrf_b200 as L
from helpers import FIELD_KEYS, field_scalars

AABB = 2 * torch.tensor([[-1.0, -1, -1], [1, 1, 1]])


def field_kwargs(sc):
    return dict(density_n_comp=[8, 8, 8], appearance_n_comp=[24, 24, 24], app_dim=int(sc["app_dim"]),
                shadingMode="MLP_Fea_late_view", near_far=[0.1, 1e3],
                density_shift=float(sc["density_shift"]), alphaMask_thres=1e-4,
                distance_scale=float(sc["distance_scale"]),
                rayMarch_weight_thres=float(sc["rayMarch_weight_thres"]), pos_pe=0,
                view_pe=int(sc["view_pe"]), fea_pe=int(sc["fea_pe"]), featureC=int(sc["featureC"]),
                step_ratio=float(sc["step_ratio"]), fea2denseAct=sc["fea2denseAct"])


def module_from_golden(g, device="cuda"):
    """TensorVMSplit (product) populated through load_state_dict with the golden's parameters."""
    sc = field_scalars(g)
    m = L.TensorVMSplit(device, AABB.clone().to(device), sc["gridSize"], **field_kwargs(sc))
    sd = {k: torch.from_numpy(np.asarray(g[k])) for k in FIELD_KEYS}
    sd["invaabbSize"] = m.invaabbSize.detach().cpu()
    if "alphaMask.alpha_volume" in g:
        m.alphaMask = L.AlphaGridMask(device, torch.from_numpy(g["alphaMask.aabb"]),
                                      torch.from_numpy(g["alphaMask.alpha_volume"]))
        for k in ("alphaMask.aabb", "alphaMask.invgridSize", "alphaMask.alpha_volume"):
            sd[k] = torch.from_numpy(g[k])
    m.load_state_dict(sd)
    return m.to(device)


def local_from_golden(g, device="cuda"):
    sc = field_scalars(g)
    kw = field_kwargs(sc)
    lt = L.LocalTensorfs(camera_prior=None, fov=float(g["fov"]), n_init_frames=4, n_overlap=30,
                         WH=tuple(int(v) for v in g["WH"]), n_iters_per_frame=600, n_iters_reg=100,
                         lr_R_init=5e-3, lr_t_init=5e-4, lr_i_init=0, lr_exposure_init=1e-3,
                         rf_lr_init=2e-2, rf_lr_basis=1e-3, lr_decay_target_ratio=0.1,
                         N_voxel_list={}, update_AlphaMask_list=[], lr_upsample_reset=True,
                         device=device, aabb=AABB.clone().to(device), gridSize=sc["gridSize"], **kw)
    sd = {k[3:]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("sd.")}
    lt.load(sd)           # the reference's own checkpoint-restore path (local_tensorfs.py:331-356)
    return lt.to(device)


def oracle_field(rf):
    """One (product) TensorVMSplit as an oracle Field (reference layout, numpy; its alpha mask included)."""
    from oracle import oracle as orc
    fd = {k: v.detach().cpu().numpy() for k, v in rf.state_dict().items()}
    kw = rf.get_kwargs()
    for k in ("density_shift", "distance_scale", "rayMarch_weight_thres", "fea_pe", "view_pe",
              "featureC", "app_dim", "step_ratio", "fea2denseAct", "gridSize"):
        fd[k] = kw[k]
    return orc.Field(fd)


def oracle_fields(lt):
    """Every field of a (product) LocalTensorfs as an oracle Field (reference layout, numpy)."""
    return [oracle_field(rf) for rf in lt.tensorfs]


def oracle_local(lt, fields, ids, view, W, H, world2rf=None, blend=None, floater_thresh=0.0):
    """LocalTensorfs.forward (eval) through the CPU oracle, with each ray's threshold margin."""
    from oracle import oracle as orc
    n = len(fields)
    zs = [orc.sample_table(f.n_samples()) for f in fields]
    focal = float(lt.focal(W).detach().cpu())
    cx, cy = [float(v) for v in lt.center(W, H).detach().cpu()]
    c2w = lt.get_cam2world(torch.tensor([view])).detach().cpu().numpy()
    expo = torch.stack(list(lt.exposure))[[view]].detach().cpu().numpy()
    if world2rf is None:
        world2rf = torch.stack([w.detach().cpu() for w in lt.world2rf]).numpy()
    if blend is None:
        blend = lt.blending_weights.detach().cpu().numpy()[[view]]
    return orc.local_forward(fields, zs, np.asarray(ids, np.int64), W, H, lt.fov == 360, focal, cx, cy,
                             c2w, np.asarray(world2rf, np.float32).reshape(n, 3),
                             np.asarray(blend, np.float32).reshape(1, n), exposure=expo,
                             floater_thresh=floater_thresh, with_margin=True)


def components_scene(n_init_frames=2, grid=64):
    """The bench's LocalTensorfs scene on the device, its init frames moved apart (the connected-components tests)."""
    import bench
    torch.manual_seed(0)
    lt = bench._scene(L.LocalTensorfs, "cpu", grid, n_init_frames=n_init_frames, density_shift=2.0)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for i in range(n_init_frames):
            lt.t_c2w[i].add_(0.3 * torch.randn(3, generator=g))
    return lt.to("cuda")


def components_boxes(rf, boxes, z_half):
    """relu density S P(x, y) L(z) in the field's frame: P 1 inside the (x0, x1, y0, y1) rectangles, L 1 for |z| <=
    z_half, ramps one grid cell wide; S puts alpha = 0.005 at P L = 1/2 (test_gpu_mesh's cylinder, as boxes)."""
    G = rf.gridSize.tolist()[0]
    cell = 4.0 / (G - 1)
    c = torch.linspace(-2, 2, G, dtype=torch.float64)
    yy, xx = torch.meshgrid(c, c, indexing="ij")
    ramp = lambda d: (0.5 + d / cell).clamp(0, 1)
    P = torch.zeros(G, G, dtype=torch.float64)
    for x0, x1, y0, y1 in boxes:
        P = torch.maximum(P, torch.minimum(ramp(torch.minimum(xx - x0, x1 - xx)), ramp(torch.minimum(yy - y0, y1 - yy))))
    Lz = ramp(z_half - c.abs())
    S = -math.log(1 - 0.005) / (float(rf.stepSize) * 0.5)
    with torch.no_grad():
        for i in range(3):
            rf.density_plane[i].zero_()
            rf.density_line[i].zero_()
        rf.density_plane[0][0, 0] = P.float().cuda()
        rf.density_line[0][0, 0, :, 0] = (S * Lz).float().cuda()
    rf.fea2denseAct = "relu"
