"""CPU-only: the float64 restatement of the supervision losses (tests/losses_oracle.py) agrees with the golden
values and gradients of the reference (tests/golden/train_losses.npz), and the fp32 selection formulas the kernels
use are bit-exact against torch.quantile / torch.median."""
import os

import numpy as np
import pytest
import torch

import losses_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_losses.npz")


def golden_cases():
    z = np.load(GOLDEN)
    for name in z["names"]:
        yield str(name), {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(f"{name}.")}


CASES = dict(golden_cases())
# In the clip case the reference's fp32 gradients of depth_map and cam2world cancel catastrophically: rays at depth
# <= 1e-6 (x = 1/depth up to 1e6, |d depth| up to 1e3) and near the clipped camera plane.  Measured: 7.3e-5 and
# 2.0e-3 of the max; the float64 restatement is the better value there.
LOOSE = {("clip_8x64", "depth_map"): 1e-4, ("clip_8x64", "cam2world"): 3e-3}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden(name):
    c = CASES[name]
    losses, grads = O.losses_f64(c)
    # fp32 reference vs float64: the residuals and the sums round differently in the last bits
    np.testing.assert_allclose(losses.numpy(), c["losses"].astype(np.float64), rtol=2e-6, atol=0)
    for k in O.GRAD_NAMES:
        ref = c[f"grad_{k}"].astype(np.float64)
        err = np.abs(grads[k].numpy().reshape(ref.shape) - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err < LOOSE.get((name, k), 1e-5), (k, err)


def _rows(R, ties, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(40, R, generator=g) * torch.rand(40, 1, generator=g) * 10
    if ties:                                    # a few values only: long runs of equal entries
        x = torch.round(x * 2) / 2
    return x


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("R", [1, 2, 255, 256, 4096])
def test_quantile_formula_bit_exact(R, ties):
    x = _rows(R, ties, R)
    for q in (0.8, 0.9):
        want = torch.quantile(x, q, dim=1).numpy()
        got = O.quantile_fp32(x.numpy(), q)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (q, np.nonzero(got != want))


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("R", [1, 2, 255, 256, 4096])
def test_lower_median_bit_exact(R, ties):
    x = _rows(R, ties, 100 + R)
    vals, idx = O.lower_median(x.numpy())
    want = torch.median(x, dim=1).values.numpy()
    assert np.array_equal(vals.view(np.int32), want.view(np.int32))
    assert np.array_equal(x.numpy()[np.arange(x.shape[0]), idx], vals)


def test_quantile_nan_row():
    x = torch.rand(3, 17)
    x[1, 4] = float("nan")
    got = O.quantile_fp32(x.numpy(), 0.9)
    assert np.isnan(got[1]) and not np.isnan(got[[0, 2]]).any()
    assert np.array_equal(np.isnan(torch.quantile(x, 0.9, dim=1).numpy()), np.isnan(got))
