"""Generate tests/golden/train_losses.npz: the supervision losses of train.py:369-423 and their autograd gradients,
computed on the CPU in float32 by the UNMODIFIED reference's get_fwd_bwd_cam2cams, get_pred_flow and
compute_depth_loss (utils/utils.py:15-59).  The block's inline rgb term, cuts and means are restated from their
formulas around those calls.

Run in the build container only (needs the reference, see oracle/ref_loader.py):

    python tests/golden/make_golden_losses.py

Each case stores its inputs, the three losses and the gradients of their sum with respect to rgb_map, depth_map,
directions, cam2world, focal and center.  Recorded environment: the `meta` entry.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
import utils.utils as ref_utils  # noqa: E402  (the reference's module, top-level name after load_reference)

META = f"torch {torch.__version__} cpu; reference facebookresearch/localrf @ 3905e39"
GRAD_NAMES = ("rgb_map", "depth_map", "directions", "cam2world", "focal", "center")


def make_case(seed, V, R, n_cams, starting_id, view_ids, W=960, H=540, tiny_depths=0, behind=0):
    """Near-identity cameras stepping along -z; camera-space directions (x, y, -1); random flows around zero."""
    g = torch.Generator().manual_seed(seed)
    N = V * R
    rot = []
    for _ in range(n_cams):
        q, r = torch.linalg.qr(torch.eye(3, dtype=torch.float64) + 0.05 * torch.randn(3, 3, generator=g, dtype=torch.float64))
        rot.append(q * torch.sign(torch.diagonal(r))[None, :])
    t = torch.stack([0.02 * torch.randn(3, generator=g, dtype=torch.float64) + torch.tensor([0.0, 0.0, -0.1 * i],
                                                                                            dtype=torch.float64)
                     for i in range(n_cams)])
    cam2world = torch.cat([torch.stack(rot), t[..., None]], -1).float()
    directions = torch.cat([torch.rand(N, 2, generator=g) - 0.5, -torch.ones(N, 1)], 1)
    depth = 0.5 + 4.5 * torch.rand(N, generator=g)
    if tiny_depths:
        idx = torch.randperm(N, generator=g)[:tiny_depths]
        depth[idx] = torch.tensor([1e-6, 0.0, 5e-7, 1e-7])[torch.arange(tiny_depths) % 4]
    if behind:                                    # points behind the target camera: the z clip of pts2px
        idx = torch.randperm(N, generator=g)[:behind]
        directions[idx, 2] = 0.5
        depth[idx] = 0.3
    return {
        "rgb_map": torch.rand(N, 3, generator=g), "rgb_train": torch.rand(N, 3, generator=g),
        "loss_weights": 0.2 + torch.rand(N, 1, generator=g),
        "view_ids": torch.tensor(view_ids, dtype=torch.int64), "starting_id": np.int64(starting_id),
        "depth_map": depth, "directions": directions,
        "ij": torch.stack([torch.randint(0, W, (N,), generator=g), torch.randint(0, H, (N,), generator=g)], 1),
        "cam2world": cam2world, "focal": torch.tensor([500.0]), "center": torch.tensor([W / 2.0, H / 2.0]),
        "fwd_flow": 3 * torch.randn(N, 2, generator=g), "bwd_flow": 3 * torch.randn(N, 2, generator=g),
        "fwd_mask": (torch.rand(N, generator=g) > 0.2).float(), "bwd_mask": (torch.rand(N, generator=g) > 0.2).float(),
        "invdepths": torch.rand(N, generator=g) + 0.1,
        "flow_weight": np.float32(1.0 / ((W + H) / 2)), "depth_weight": np.float32(0.1),
    }


def reference_block(c):
    """train.py:369-423 around the reference's functions -> (losses [3], {name: gradient})."""
    p = {k: c[k].clone().requires_grad_() for k in GRAD_NAMES}
    V = c["view_ids"].shape[0]
    view_ids, w = c["view_ids"], c["loss_weights"]
    rgb = (0.25 * (torch.abs(p["rgb_map"] - c["rgb_train"]) * w) / w.mean()).mean()
    depth_map = p["depth_map"].view(V, -1)
    directions = p["directions"].view(V, -1, 3)
    ij = c["ij"].view(V, -1, 2)
    fwd_mask = c["fwd_mask"].view(V, -1).clone()
    fwd_mask[view_ids == len(p["cam2world"]) - 1] = 0
    fwd_c2c, bwd_c2c = ref_utils.get_fwd_bwd_cam2cams(p["cam2world"], view_ids - int(c["starting_id"]))
    pts = directions * depth_map[..., None]
    pred_fwd = ref_utils.get_pred_flow(pts, ij, fwd_c2c, p["focal"], p["center"])
    pred_bwd = ref_utils.get_pred_flow(pts, ij, bwd_c2c, p["focal"], p["center"])
    e = torch.sum(torch.abs(pred_bwd - c["bwd_flow"].view(V, -1, 2)), dim=-1) * c["bwd_mask"].view(V, -1)
    e = e + torch.sum(torch.abs(pred_fwd - c["fwd_flow"].view(V, -1, 2)), dim=-1) * fwd_mask
    e = torch.where(e > torch.quantile(e, 0.9, dim=1)[..., None], 0, e)
    flow = e.mean() * float(c["flow_weight"])
    _, _, d = ref_utils.compute_depth_loss(1 / depth_map.clamp(1e-6), c["invdepths"].view(V, -1))
    d = torch.where(d > torch.quantile(d, 0.8, dim=1)[..., None], 0, d)
    depth = d.mean() * float(c["depth_weight"])
    (rgb + flow + depth).backward()
    return torch.stack([rgb, flow, depth]).detach(), {k: p[k].grad for k in GRAD_NAMES}


def main():
    cases = {
        # 20 cameras from frame 5: view 19 is the last ABSOLUTE id (fwd-mask quirk), view 5 the first camera
        # (bwd clamp), view 24 the last camera (fwd clamp); views 7 and 11 appear twice
        "train_16x256": make_case(1, 16, 256, 20, 5, [5, 19, 24, 7, 7, 8, 11, 11, 12, 14, 15, 16, 17, 20, 22, 23]),
        "odd_4x37": make_case(2, 4, 37, 6, 0, [0, 2, 5, 3]),
        "single_1x4096": make_case(3, 1, 4096, 3, 0, [1]),
        "clip_8x64": make_case(4, 8, 64, 10, 2, [2, 3, 4, 6, 8, 9, 10, 11], tiny_depths=12, behind=3),
    }
    out = {}
    for name, c in cases.items():
        losses, grads = reference_block(c)
        for k, v in c.items():
            out[f"{name}.{k}"] = v.numpy() if isinstance(v, torch.Tensor) else v
        out[f"{name}.losses"] = losses.numpy()
        for k, v in grads.items():
            out[f"{name}.grad_{k}"] = v.numpy()
        print(name, losses.tolist())
    path = os.path.join(HERE, "train_losses.npz")
    np.savez_compressed(path, meta=np.array(META), names=np.array(list(cases)), **out)
    print(f"train_losses: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
