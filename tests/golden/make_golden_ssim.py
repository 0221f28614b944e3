"""Generate tests/golden/ssim.npz by running the UNMODIFIED reference's rgb_ssim (utils/utils.py:232-287) and
renderer.py:162's torch-fp32 MSE on the CPU.

Run in the build container only (needs the reference, see oracle/ref_loader.py):

    python tests/golden/make_golden_ssim.py

Each case stores the two frames, the parameters (max_val, filter_size, filter_sigma, k1, k2), the reference's
ssim and map, and the MSE.  Recorded environment: the `meta` entry.
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


def main():
    rng = np.random.default_rng(7)
    u = lambda *s: rng.random(s, dtype=np.float32)
    yy, xx = np.meshgrid(np.linspace(0, 1, 96), np.linspace(0, 1, 80), indexing="ij")
    smooth = np.stack([0.5 + 0.4 * np.sin(3 * xx + c) * np.cos(2 * yy - c) for c in range(3)], -1).astype(np.float32)
    noisy = np.clip(smooth + 0.05 * rng.standard_normal(smooth.shape), 0, 1).astype(np.float32)
    same = u(40, 33, 3)
    cases = {                                    # name: (gt, img, max_val, filter_size, filter_sigma, k1, k2)
        "rand_37x53": (u(37, 53, 3), u(37, 53, 3), 1.0, 11, 1.5, 0.01, 0.03),
        "one_11x11": (u(11, 11, 3), u(11, 11, 3), 1.0, 11, 1.5, 0.01, 0.03),
        "smooth_96x80": (smooth, noisy, 1.0, 11, 1.5, 0.01, 0.03),
        "identical": (same, same.copy(), 1.0, 11, 1.5, 0.01, 0.03),
        "constant": (np.full((24, 30, 3), 0.3, np.float32), np.full((24, 30, 3), 0.7, np.float32), 1.0, 11, 1.5,
                     0.01, 0.03),
        "even_255": ((255 * u(29, 41, 3)).round(), (255 * u(29, 41, 3)).round(), 255.0, 8, 1.0, 0.02, 0.05),
    }
    out = {}
    for name, (gt, img, max_val, fs, sigma, k1, k2) in cases.items():
        gt, img = gt.astype(np.float32), img.astype(np.float32)
        out[f"{name}.gt"], out[f"{name}.img"] = gt, img
        out[f"{name}.params"] = np.array([max_val, fs, sigma, k1, k2])
        # renderer.py:163 calls rgb_ssim(gt_rgb, rgb_map, 1)
        out[f"{name}.ssim"] = np.float64(ref_utils.rgb_ssim(gt, img, max_val, fs, sigma, k1, k2))
        out[f"{name}.ssim_map"] = ref_utils.rgb_ssim(gt, img, max_val, fs, sigma, k1, k2, return_map=True)
        out[f"{name}.mse"] = np.float32(((torch.from_numpy(gt) - torch.from_numpy(img)) ** 2).mean().item())
    path = os.path.join(HERE, "ssim.npz")
    np.savez_compressed(path, meta=np.array(META), names=np.array(list(cases)), **out)
    print(f"ssim: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
