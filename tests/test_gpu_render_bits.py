"""-m gpu: the fused render kernel's cfg2 output, bit for bit.  Changes to how the kernel distributes
work (warp roles, producer / consumer counts, ray scheduling, shared-memory layout) must not change a
single bit of what a ray computes: the composite is fixed point, so the result of every ray is
independent of which warp marched it and in which order its rows were shaded.

tests/golden/cfg2_300_render_bits.npz holds rgb / depth of batches 80 and 155 (4096 rays each) of the
bench.py cfg2 scene (300^3, seed 0, 800x800 frame) as rendered on an H100 by the kernel of commit ce960d2
(12 producer warps, one consumer warpgroup).  To regenerate it, save what this test renders, from a build
that is known to be right."""
import numpy as np
import pytest
import torch

from helpers import load_golden

pytestmark = pytest.mark.gpu


def test_cfg2_batches_bit_identical_to_stored_render():
    import bench
    g = load_golden("cfg2_300_render_bits")
    lt = bench.build_scene(torch.device("cuda", 0), 300)
    for b in g["batches"]:
        ids = torch.arange(int(b) * 4096, (int(b) + 1) * 4096, dtype=torch.int64, device="cuda")
        with torch.no_grad():
            rgb, depth, _, _ = lt(ids, torch.tensor([0], device="cuda"), 800, 800, is_train=False)
        rgb, depth = rgb.cpu().numpy(), depth.cpu().numpy()
        n_rgb = int((rgb != g[f"b{b}.rgb"]).any(-1).sum())
        n_depth = int((depth != g[f"b{b}.depth"]).sum())
        assert n_rgb == 0 and n_depth == 0, f"batch {b}: {n_rgb} rgb / {n_depth} depth values differ"
        assert np.array_equal(rgb, g[f"b{b}.rgb"]) and np.array_equal(depth, g[f"b{b}.depth"])
