"""Generate tests/golden/test_panels.npz: the flow and depth comparison panels renderer.render(test=True) builds for a
held-out frame (renderer.py:79-124), computed on the CPU by the UNMODIFIED reference's get_fwd_bwd_cam2cams,
get_pred_flow and compute_depth_loss (utils/utils.py:15-59).  The block's inline lines (cv2.resize with
INTER_NEAREST, np.vstack / np.quantile / np.hstack, the clamp) are restated around those calls.

Run in the build container only (needs the reference, see oracle/ref_loader.py):

    python tests/golden/make_golden_panels.py

The inputs are regenerated from seeds by tests/panels_oracle.make_case; the fixture stores their sha256, the
predicted flows, the statistics (four 0.9 quantiles, then median and mean absolute deviation of x and of g) and the
panels -- whole for the small cases, at panels_oracle.sample_index positions for the 480x270 one.
"""
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]
from oracle.ref_loader import load_reference  # noqa: E402
import panels_oracle as PO  # noqa: E402

load_reference()
import utils.utils as ref_utils  # noqa: E402  (the reference's module, top-level name after load_reference)

META = f"torch {torch.__version__} cpu, numpy {np.__version__}, opencv {cv2.__version__}; " \
       "reference facebookresearch/localrf @ 3905e39"


def reference_block(c):
    """renderer.py:79-124 for one frame around the reference's functions -> dict of outputs."""
    W, H, idx = c["W"], c["H"], c["idx"]
    depth_map = torch.from_numpy(c["depth"])
    directions = torch.from_numpy(c["directions"])
    p = torch.arange(W * H)
    ij = torch.stack([p % W, p // W], -1)
    cam2world = torch.from_numpy(c["cam2world"])
    focal, center = torch.tensor([float(c["focal"])]), torch.from_numpy(c["center"])
    view_ids = torch.tensor([idx], dtype=torch.long)
    fwd_c2c, bwd_c2c = ref_utils.get_fwd_bwd_cam2cams(cam2world, view_ids)
    pts = directions[None] * depth_map[None, ..., None]
    pred = {}
    pred["fwd"] = ref_utils.get_pred_flow(pts, ij, fwd_c2c, focal, center).numpy().reshape(H, W, 2)
    pred["bwd"] = ref_utils.get_pred_flow(pts, ij, bwd_c2c, focal, center).numpy().reshape(H, W, 2)
    out, qs = {}, []
    for d in ("fwd", "bwd"):
        flow = cv2.resize(c[f"{d}_flow"], (W, H), interpolation=cv2.INTER_NEAREST)
        mask = cv2.resize(c[f"{d}_mask"], (W, H), interpolation=cv2.INTER_NEAREST)
        cols = []
        with np.errstate(divide="ignore", invalid="ignore"):
            for ch in range(2):
                cmp = np.vstack([pred[d][..., ch], flow[..., ch]])
                q = np.quantile(cmp, 0.9)
                qs.append(q)
                cmp /= q
                cols.append(np.vstack([cmp, np.abs(pred[d][..., ch] - flow[..., ch]) * mask / W]))
        out[f"{d}_cmp"] = torch.from_numpy(np.hstack(cols)).clamp(0, 1).numpy()
        out[f"{d}_pred"] = pred[d]
    inv = torch.from_numpy(cv2.resize(c["invdepth"], (W, H), interpolation=cv2.INTER_NEAREST)).view(1, -1)
    x = 1 / depth_map[None].clamp(1e-6)
    xn, gn, err = ref_utils.compute_depth_loss(x, inv)
    out["depth_cmp"] = torch.vstack([0.5 * xn[0].reshape(H, W), 0.5 * gn[0].reshape(H, W),
                                     err[0].reshape(H, W)]).clamp(0, 1).numpy()
    tx = torch.median(x, dim=-1).values[0]
    tg = torch.median(inv, dim=-1).values[0]
    sx = torch.mean(torch.abs(x - tx))
    sg = torch.mean(torch.abs(inv - tg))
    out["stats"] = np.array([*qs, tx, sx, tg, sg], np.float32)
    return out


def main():
    out = {}
    for name in PO.CASES:
        c = PO.make_case(name)
        r = reference_block(c)
        out[f"{name}.digest"] = np.array(PO.input_digest(c))
        out[f"{name}.stats"] = r["stats"]
        W, H = c["W"], c["H"]
        for k in ("fwd_pred", "bwd_pred", "fwd_cmp", "bwd_cmp", "depth_cmp"):
            v = r[k]
            if W * H > PO.FULL_OUTPUT_PIXELS:
                v = v.reshape(-1)[PO.sample_index(name, v.size)]
            out[f"{name}.{k}"] = v
        print(name, r["stats"].tolist())
    path = os.path.join(HERE, "test_panels.npz")
    np.savez_compressed(path, meta=np.array(META), names=np.array(list(PO.CASES)), **out)
    print(f"test_panels: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
