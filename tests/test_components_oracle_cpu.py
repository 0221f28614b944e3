"""CPU-only: the pieces of tests/components_oracle.py that the device tests lean on hardest -- probe_start (splitmix64's
finaliser), table_ok (the cell table a point-cloud run leaves), colliding_cells (cells that share a probe start) and
the ranking / selection rule of lrf_components_select on hand-built label / size arrays."""
import numpy as np
import pytest

import components_oracle as co

M64 = (1 << 64) - 1
GOLDEN = 0x9e3779b97f4a7c15
NO_INDEX = 0x7fffffff


def test_probe_start_on_hand_worked_constants():
    # splitmix64 seeded with 0 returns the finaliser of GOLDEN, 2 GOLDEN, 3 GOLDEN (mod 2^64): its published first outputs
    want = {0: 0, GOLDEN: 0xe220a8397b1dcdaf, 2 * GOLDEN & M64: 0x6e789e6aa1b965f4, 3 * GOLDEN & M64: 0x06c45d188009454f,
            1: 0x5692161d100b05e5}
    keys = np.array(list(want), np.uint64)
    assert co.probe_start(keys).tolist() == list(want.values())
    assert int(co.probe_start(np.uint64(GOLDEN))) == 0xe220a8397b1dcdaf                  # a scalar, no warning
    # the key of cell (0, 0, 0) is 2^20 on each axis: 0x4000020000100000
    assert int(co.cell_keys([[0, 0, 0]])[0]) == 0x4000020000100000
    assert co.cell_keys([[-(1 << 20)] * 3, [(1 << 20) - 1] * 3]).tolist() == [0, (1 << 63) - 1]


def _insert(cells_k, capacity):
    """A table built the way find_or_claim fills it one key at a time: (tags, first, xyz) for one point per cell at
    its centre (cell_size 1, origin 0), points in the order of `cells_k`."""
    keys = co.cell_keys(cells_k)
    tags = np.zeros(capacity, np.uint64)
    first = np.full(capacity, NO_INDEX, np.int64)
    for p, k in enumerate(keys):
        s = int(co.probe_start(k)) & (capacity - 1)
        while tags[s] not in (0, k + np.uint64(1)):
            s = (s + 1) % capacity
        tags[s] = k + np.uint64(1)
        first[s] = min(first[s], p)
    return tags, first, np.asarray(cells_k, np.float32) + np.float32(0.5)


def test_table_ok_accepts_a_table_built_by_linear_probing():
    rng = np.random.default_rng(0)
    cells_k = rng.integers(-50, 50, (40, 3))
    cells_k = np.concatenate([cells_k, cells_k[:7]])                   # repeated cells: the lowest point is kept
    tags, first, xyz = _insert(cells_k, 128)
    assert co.table_ok(tags.view(np.int64), first, xyz, (0, 0, 0), 1.0, 128)
    assert co.table_ok(np.zeros(16, np.int64), np.full(16, NO_INDEX), np.zeros((0, 3), np.float32), (0, 0, 0), 1.0, 16)


def test_table_ok_on_a_chain_that_wraps_past_the_last_slot():
    cap = 32
    chain = co.colliding_cells(cap, cap - 2, (-8, -8, -8), (8, 8, 8))[:5]
    assert len(chain) == 5 and (co.probe_start(co.cell_keys(chain)) & np.uint64(cap - 1) == cap - 2).all()
    tags, first, xyz = _insert(chain, cap)
    assert np.nonzero(tags)[0].tolist() == [0, 1, 2, cap - 2, cap - 1]
    assert co.table_ok(tags, first, xyz, (0, 0, 0), 1.0, cap)
    t, f = tags.copy(), first.copy()
    t[4], f[4], t[2], f[2] = t[2], f[2], 0, NO_INDEX                   # slot 2's key past the now empty slot 2
    with pytest.raises(AssertionError, match="off its probe path"):
        co.table_ok(t, f, xyz, (0, 0, 0), 1.0, cap)


@pytest.mark.parametrize("damage, text", [
    ("drop", "keys are not"), ("duplicate", "keys are not"), ("first", "lowest point"), ("empty_first", "empty slot"),
    ("stranger", "keys are not"),
])
def test_table_ok_names_a_damaged_table(damage, text):
    rng = np.random.default_rng(1)
    cells_k = rng.integers(-20, 20, (30, 3))
    tags, first, xyz = _insert(np.concatenate([cells_k, cells_k[:3]]), 64)
    occ, empty = np.nonzero(tags)[0], np.nonzero(tags == 0)[0]
    if damage == "drop":
        tags[occ[0]], first[occ[0]] = 0, NO_INDEX
    elif damage == "duplicate":
        tags[empty[0]], first[empty[0]] = tags[occ[0]], first[occ[0]]
    elif damage == "first":
        first[occ[0]] += 1
    elif damage == "empty_first":
        first[empty[0]] = 0
    else:
        tags[empty[0]], first[empty[0]] = co.cell_keys([[100, 0, 0]])[0] + np.uint64(1), 0
    with pytest.raises(AssertionError, match=text):
        co.table_ok(tags, first, xyz, (0, 0, 0), 1.0, 64)


def test_colliding_cells_share_their_probe_start():
    for cap, slot in ((2, 1), (64, 0), (64, 63), (1024, 517)):
        k = co.colliding_cells(cap, slot, (-4, 10, -20), (4, 40, 0))
        keys = co.cell_keys(k)
        assert len(k) > 0 and (keys[1:] > keys[:-1]).all()                  # lexicographic, each once
        assert ((co.probe_start(co.cell_keys(k)) & np.uint64(cap - 1)) == slot).all()
        assert (k >= (-4, 10, -20)).all() and (k < (4, 40, 0)).all()
    every = sum(len(co.colliding_cells(16, s, (0, 0, 0), (4, 4, 4))) for s in range(16))
    assert every == 64


def test_select_ties_rank_by_label():
    label = np.arange(6)
    s = co.select(label, [3, 5, 3, 5, 0, 3])
    assert s["sizes"].tolist() == [5, 5, 3, 3, 3, 0] and s["rank"].tolist() == [2, 0, 3, 1, 5, 4]
    s = co.select(label, [3, 5, 3, 5, 0, 3], keep=3)
    assert s["new_index"].tolist() == [0, 1, -1, 2, -1, -1] and s["counts"] == [3, 3, 6, 13]
    s = co.select(label, [3, 5, 3, 5, 0, 3], min_size=4)
    assert s["counts"] == [2, 2, 6, 10] and s["rank"].tolist() == [0, 1]


def test_select_clamps_large_and_negative_sizes():
    big = [2 ** 31 - 2, 2 ** 31 - 1, 2 ** 31, 2 ** 63 - 1, 0, -1, -(2 ** 63), 7]
    s = co.select(np.arange(8), big)
    top = 2 ** 31 - 1
    # 2^31 - 1, 2^31 and 2^63 - 1 tie at 2^31 - 1 (by label), then 2^31 - 2, 7, and 0, -1, -2^63 tie at 0
    assert s["sizes"].tolist() == [top, top, top, top - 1, 7, 0, 0, 0]
    assert s["rank"].tolist() == [3, 0, 1, 2, 5, 6, 7, 4]
    assert s["counts"] == [8, 8, 8, 3 * top + top - 1 + 7]
    s = co.select(np.arange(8), big, min_size=1)                       # a negative size is 0: dropped by min_size 1
    assert s["new_index"].tolist() == [0, 1, 2, 3, -1, -1, -1, 4] and s["counts"][3] == 4 * top - 1 + 7
    s = co.select(np.arange(3), [-5, 1, 0], keep=1)                    # a negative size never ranks first
    assert s["new_index"].tolist() == [-1, 0, -1] and s["counts"] == [1, 1, 3, 1]
    s = co.select(np.arange(3), [-5, 0, 0], min_size=0)
    assert s["rank"].tolist() == [0, 1, 2] and s["counts"] == [3, 3, 3, 0]


def test_select_drops_vertices_whose_label_is_not_a_root_in_range():
    n = 9
    label = np.array([0, 0, -1, n, 4, 4, 4, 5, -(2 ** 31)])             # 5 is not a root (label[5] = 4)
    size = np.array([2, 9, 9, 9, 1, 9, 9, 9, 9])                       # sizes at non-roots are not read
    s = co.select(label, size)
    assert s["sizes"].tolist() == [2, 1] and s["counts"] == [5, 2, 2, 3]
    assert s["new_index"].tolist() == [0, 1, -1, -1, 2, 3, 4, -1, -1] and s["rank"].tolist() == [0, 0, 1, 1, 1]
    s = co.select(np.full(4, -1), np.ones(4, np.int64))                # no roots at all
    assert s["counts"] == [0, 0, 0, 0] and (s["new_index"] == -1).all() and len(s["sizes"]) == 0


@pytest.mark.parametrize("keep, min_size, want", [
    (0, 0, [5, 3, 3, 12]), (1, 0, [1, 1, 3, 5]), (2, 0, [4, 2, 3, 9]), (3, 0, [5, 3, 3, 12]), (4, 0, [5, 3, 3, 12]),
    (2 ** 62, 0, [5, 3, 3, 12]), (0, 4, [4, 2, 3, 9]), (0, 2 ** 31 - 1, [0, 0, 3, 0]), (0, 2 ** 31, [0, 0, 3, 0]),
    (0, 2 ** 62, [0, 0, 3, 0]), (1, 5, [1, 1, 3, 5]), (1, 6, [0, 0, 3, 0]),
])
def test_select_keep_and_min_size_edges(keep, min_size, want):
    label = np.array([0, 0, 0, 3, 4])
    assert co.select(label, [4, 0, 0, 3, 5], keep, min_size)["counts"] == want
