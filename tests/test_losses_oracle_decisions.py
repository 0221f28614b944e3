"""CPU-only: losses_f64's decisions= argument (tests/losses_oracle.py).  Fed its own float64 cuts and medians it
reproduces its default output bit for bit, and fed other decisions it uses them."""
import numpy as np
import pytest
import torch

import losses_oracle as O
from test_losses_cpu import CASES


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


@pytest.mark.parametrize("name", sorted(CASES))
def test_own_decisions_reproduce_default_bit_for_bit(name):
    c = CASES[name]
    l0, g0, a0 = O.losses_f64(c, return_arrays=True)
    own = a0["decisions"]
    V, R = a0["flow"].shape
    assert own["flow_cut"].shape == own["depth_cut"].shape == (V, R)
    assert own["median_x"].shape == own["median_g"].shape == (V,)
    l1, g1 = O.losses_f64(c, decisions={k: v.clone() for k, v in own.items()})
    assert _same(l1, l0)
    for k in O.GRAD_NAMES:
        assert _same(g1[k], g0[k]), k


def test_given_decisions_are_used():
    """No ray cut: the flow loss is the plain mean; a median index moved to another ray moves the depth term.
    A part left out is selected in float64 as by default."""
    c = CASES["odd_4x37"]
    l0, _, a0 = O.losses_f64(c, return_arrays=True)
    V, R = a0["flow"].shape
    none_cut = {"flow_cut": torch.zeros(V, R, dtype=torch.bool)}
    l1, _ = O.losses_f64(c, decisions=none_cut)
    assert abs(l1[1].item() - a0["flow"].mean().item() * float(c["flow_weight"])) <= 1e-15 * abs(l1[1].item())
    assert l1[1] > l0[1] and _same(l1[[0, 2]], l0[[0, 2]])
    moved = dict(a0["decisions"], median_x=(a0["decisions"]["median_x"] + 1) % R)
    l2, _ = O.losses_f64(c, decisions=moved)
    assert l2[2] != l0[2] and _same(l2[:2], l0[:2])
