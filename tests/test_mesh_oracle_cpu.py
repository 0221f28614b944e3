"""CPU-only: the vectorised restatements of tests/mesh_oracle.py (cells_np / extract_np, owner32, probe_slots) against
the scalar restatement they stand in for in the GPU tests at sizes the scalar one cannot reach."""
import numpy as np
import pytest
import torch

import mesh_oracle as mo

H = mo.HALF


def _lattice(seed, dims=(12, 12, 12), special=True):
    rng = np.random.default_rng(seed)
    v = rng.random(dims).astype(np.float32)
    level = np.float32(rng.uniform(0.3, 0.7))
    if special:
        v[rng.random(dims) < 0.05] = level
        v[rng.random(dims) < 0.02] = np.nan
        v[rng.random(dims) < 0.02] = np.inf
        v[rng.random(dims) < 0.02] = -np.inf
    return v, level


def _same(a, b):
    return np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]) and \
        a[0].dtype == b[0].dtype == np.float32 and a[1].dtype == b[1].dtype == np.int32


@pytest.mark.parametrize("seed", range(12))
def test_cells_np_equals_mesh_lattice(seed):
    """The 12 random lattices of test_random_lattices_mesh_closed_and_oriented, then the same with values on the level,
    NaN and +-inf, at negative lo and at both key limits."""
    rng = np.random.default_rng(seed)
    n = 12
    v = rng.random((n, n, n)).astype(np.float32)
    v[[0, -1]] = v[:, [0, -1]] = v[:, :, [0, -1]] = 0.0
    level = np.float32(rng.uniform(0.3, 0.7))
    args = ((-5, 0, 7), level, (0.5, -0.25, 0.0), 0.125)
    assert _same(mo.cells_np(v, *args), mo.mesh_lattice(v, *args))
    v, level = _lattice(seed, (13, 11, 12))
    lo = [(-H, -H, -H), (H - 13, H - 11, H - 12), (-7, -6, -5), (-H, 3, H - 12)][seed % 4]
    args = (lo, level, (0.1, -0.2, 0.3), 0.03125 * (seed + 1))
    want = mo.mesh_lattice(v, *args)
    assert len(want[1]) > 500 and _same(mo.cells_np(v, *args), want)


def test_cells_np_small_slabs_and_empty():
    """Slabs of one x-layer of cells give the same mesh; a lattice with no cut edge gives empty arrays."""
    v, level = _lattice(3, (9, 10, 11))
    args = ((-4, 2, -1), level, (0.0, 0.5, -0.5), 0.25)
    old = mo.SLAB_CELLS
    try:
        mo.SLAB_CELLS = 1
        assert _same(mo.cells_np(v, *args), mo.mesh_lattice(v, *args))
    finally:
        mo.SLAB_CELLS = old
    xyz, faces = mo.cells_np(np.zeros((4, 5, 6), np.float32), *args)
    assert xyz.shape == (0, 3) and faces.shape == (0, 3) and xyz.dtype == np.float32 and faces.dtype == np.int32


@pytest.mark.parametrize("seed", range(3))
def test_cells_np_in_bricks_equals_one_brick(seed):
    """2 x 3 x 2 bricks sharing their boundary points (each edge computed once per brick that holds it), merged by
    extract_np, give the one-brick mesh; so does the scalar merge()."""
    v, level = _lattice(seed, (21, 22, 23))
    lo, origin, vs = (-7 + seed, 3, -H), (0.1, -0.2, 0.3), 0.03125 * (seed + 1)
    want = mo.cells_np(v, lo, level, origin, vs)
    parts, scalar = [], []
    for x0, x1 in ((0, 11), (10, 21)):
        for y0, y1 in ((0, 8), (7, 15), (14, 22)):
            for z0, z1 in ((0, 12), (11, 23)):
                sub, sl = v[x0:x1, y0:y1, z0:z1], (lo[0] + x0, lo[1] + y0, lo[2] + z0)
                parts.append(mo.cells_parts(sub, sl, level, origin, vs))
                scalar.append(mo.cells(sub, sl, level, origin, vs))
    assert _same(mo.extract_np(parts), want)
    assert _same(mo.extract(*mo.merge(scalar)), want)


def test_owner32_agrees_with_mesh_value64():
    """owner32 picks mesh_value64's owner wherever that point is not flagged (mesh_value64's owner is -1 beyond
    max_norm; owner32 has no cut, so it is compared through the norms there), with exact ties to the lowest field,
    NaN and infinite rows."""
    rng = np.random.default_rng(0)
    w = rng.uniform(-1, 1, (9, 3)).astype(np.float32)
    w[3] = w[1]                                                           # an exact tie: never owns
    w[5] = [np.nan, 0.0, 0.0]
    w[7] = [np.inf, 0.0, 0.0]
    p = rng.uniform(-2, 2, (20000, 3)).astype(np.float32)
    p[:100] = np.round(p[:100] * 8) / 8                                  # lattice-like points: exact norm ties
    own, norm = mo.owner32(p, w)
    assert not np.isin(own, [3, 5, 7]).any() and (own >= 0).all()
    finite = [k for k in range(9) if np.isfinite(w[k]).all() and k != 3]
    _, o64, flagged = mo.mesh_value64([], [], w[finite], torch.from_numpy(p.astype(np.float64)), 10.0)
    ok = ~flagged.numpy()
    assert ok.mean() > 0.99
    assert np.array_equal(own[ok], np.asarray(finite)[o64.numpy()[ok]])
    want = np.abs(p.astype(np.float64)[:, None] + w[finite].astype(np.float64)).max(-1).min(-1)
    assert np.all(np.abs(norm - want) <= 2.0 ** -22 * (1 + want))
    o, n = mo.owner32(p[:5], np.full((4, 3), np.nan, np.float32))
    assert (o == -1).all() and (n == np.inf).all()


def test_probe_slots_wraps_from_the_last_slot():
    import export_oracle as eo
    cap = 64
    keys = np.nonzero((eo.mix64(np.arange(1 << 20, dtype=np.uint64)) & np.uint64(cap - 1)) == cap - 1)[0][:3].tolist()
    assert mo.probe_slots(keys, cap) == {cap - 1, 0, 1}
    assert mo.probe_slots(keys + [keys[0]], cap) == {cap - 1, 0, 1}
