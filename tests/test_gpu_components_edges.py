"""GPU: the connected-components entries (lrf_mesh_components / lrf_point_components / lrf_components_select and
export.keep_components) at the sizes and edges where a lock-free union-find, an open-addressing table and a radix-sort
ranking go wrong, bit for bit against tests/components_oracle.py.

Every output buffer starts as random bytes with canary words after it, and the select scratch sits at an offset inside
a larger block of random bytes at exactly the size lrf_components_select_scratch_bytes reports, with guard bytes on
both sides.  Each case runs twice on the same buffers, the second time on the first run's leftovers, so nothing has
to be zeroed first.  Large graphs whose components are known in closed form (a few triangles among 2^27 vertices, a
dense block of cells) are checked against that form instead of scipy."""
import ctypes as C

import numpy as np
import pytest
import torch

import components_oracle as co
from gpu_helpers import components_boxes, components_scene
from localrf_b200 import _lib
from localrf_b200.export import keep_components, mesh

pytestmark = pytest.mark.gpu
PAD = 16
CANARY = -123456789
GUARD = 4096
TOP = 2 ** 31 - 1


def _out(n, dtype):
    """n elements of random bytes, then PAD canary words."""
    t = torch.empty(n + PAD, dtype=dtype, device="cuda")
    t.view(torch.uint8).random_(0, 256)
    t[n:] = CANARY
    return t


def _intact(t, n, what):
    assert (t[n:] == CANARY).all(), f"a canary word past {what} changed"


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _stream(s):
    return None if s is None else C.c_void_p(s.cuda_stream)


# ---- ctypes wrappers -------------------------------------------------------------------------------------------------
class Mesh:
    """lrf_mesh_components into buffers that persist between runs."""

    def __init__(self, faces, V):
        self.f = faces if torch.is_tensor(faces) else _dev(np.asarray(faces, np.int64).reshape(-1, 3), torch.int32)
        self.V, self.T = V, self.f.shape[0]
        self.label, self.size, self.stats = _out(V, torch.int32), _out(V, torch.int64), _out(1, torch.int64)

    def launch(self, stream=None):
        _lib.check(_lib.lib().lrf_mesh_components(self.f.data_ptr() if self.T else None, self.T, self.V,
                                                  self.label.data_ptr(), self.size.data_ptr(), self.stats.data_ptr(),
                                                  _stream(stream)))

    def result(self):
        torch.cuda.synchronize()
        for t, n, w in ((self.label, self.V, "label"), (self.size, self.V, "size"), (self.stats, 1, "stats")):
            _intact(t, n, w)
        return self.label[:self.V].cpu().numpy(), self.size[:self.V].cpu().numpy(), int(self.stats[0])


class Points:
    """lrf_point_components into buffers (the table included) that persist between runs."""

    def __init__(self, xyz, origin, cell, capacity):
        self.x = _dev(np.asarray(xyz, np.float32).reshape(-1, 3), torch.float32)
        self.n, self.origin, self.cell, self.cap = self.x.shape[0], origin, cell, capacity
        self.keys, self.first = _out(capacity, torch.int64), _out(capacity, torch.int32)
        self.label, self.size, self.stats = _out(self.n, torch.int32), _out(self.n, torch.int64), _out(2, torch.int64)

    def launch(self):
        _lib.check(_lib.lib().lrf_point_components(
            self.x.data_ptr() if self.n else None, self.n, (C.c_float * 3)(*self.origin), self.cell,
            self.keys.data_ptr(), self.first.data_ptr(), self.cap, self.label.data_ptr(), self.size.data_ptr(),
            self.stats.data_ptr(), None))

    def result(self):
        torch.cuda.synchronize()
        for t, m, w in ((self.keys, self.cap, "keys"), (self.first, self.cap, "first"), (self.label, self.n, "label"),
                        (self.size, self.n, "size"), (self.stats, 2, "stats")):
            _intact(t, m, w)
        return (self.label[:self.n].cpu().numpy(), self.size[:self.n].cpu().numpy(), int(self.stats[0]),
                int(self.stats[1]))

    def table(self):
        return self.keys[:self.cap].cpu().numpy(), self.first[:self.cap].cpu().numpy()


class Select:
    """lrf_components_select into outputs and a guarded scratch block that persist between runs."""

    def __init__(self, n):
        self.n = n
        self.nb = _lib.lib().lrf_components_select_scratch_bytes(n) if n else 0
        assert (self.nb > 0 and self.nb % 256 == 0) or n == 0
        self.block = torch.empty(self.nb + 2 * GUARD, dtype=torch.uint8, device="cuda").random_(0, 256)
        self.guards = (self.block[:GUARD].clone(), self.block[GUARD + self.nb:].clone())
        self.new_index, self.rank = _out(n, torch.int32), _out(n, torch.int32)
        self.sizes, self.counts = _out(n, torch.int64), _out(4, torch.int64)

    def launch(self, label, size, keep=0, min_size=0, stream=None):
        n = self.n
        _lib.check(_lib.lib().lrf_components_select(
            label.data_ptr() if n else None, size.data_ptr() if n else None, n, keep, min_size,
            self.new_index.data_ptr(), self.rank.data_ptr(), self.sizes.data_ptr(), self.counts.data_ptr(),
            self.block[GUARD:].data_ptr() if n else None, self.nb, _stream(stream)))

    def result(self):
        torch.cuda.synchronize()
        n = self.n
        c = self.counts[:4].cpu().tolist()
        for t, m, w in ((self.new_index, n, "new_index"), (self.rank, n, "rank"), (self.sizes, n, "sizes"),
                        (self.counts, 4, "counts")):
            _intact(t, m, w)
        assert torch.equal(self.block[:GUARD], self.guards[0]), "the guard before the scratch changed"
        assert torch.equal(self.block[GUARD + self.nb:], self.guards[1]), "the guard after the scratch changed"
        return dict(new_index=self.new_index[:n].cpu().numpy(), rank=self.rank[:c[0]].cpu().numpy(),
                    sizes=self.sizes[:c[2]].cpu().numpy(), counts=c)


def same_selection(got, want):
    assert got["counts"] == list(want["counts"]), (got["counts"], want["counts"])
    for k in ("new_index", "rank", "sizes"):
        assert np.array_equal(got[k], want[k]), k


def run_select(label, size, cases, want_fn):
    """Each (keep, min_size) of `cases` twice on one Select (the second on the first's leftovers) against want_fn."""
    n = len(label)
    lb, sz = _dev(label, torch.int32), _dev(size, torch.int64)
    s = Select(n)
    for keep, min_size in cases:
        want = want_fn(keep, min_size)
        for _ in range(2):
            s.launch(lb, sz, keep, min_size)
            same_selection(s.result(), want)


def check_mesh(faces, V, cases=((0, 0), (1, 0), (0, 2))):
    """lrf_mesh_components twice on one set of buffers and the selections, against the oracle."""
    m = Mesh(faces, V)
    f = faces.cpu().numpy() if torch.is_tensor(faces) else faces
    wl, ws, wb = co.mesh_components(f, V)
    for _ in range(2):
        m.launch()
        label, size, bad = m.result()
        assert bad == wb and np.array_equal(label, wl) and np.array_equal(size, ws)
    run_select(wl, ws, cases, lambda k, s: co.select(wl, ws, k, s))
    return wl, ws


# ---- the mesh union-find under contention ---------------------------------------------------------------------------
@pytest.mark.parametrize("divisor", [8, 6, 4])
def test_random_hypergraphs_around_the_giant_component_threshold(divisor):
    """3-uniform random hypergraphs on 2^24 vertices with V/8, V/6, V/4 triangles: below, at and above the point
    (V/6) where a giant component appears, so component sizes spread from 0 to millions."""
    V, T = 1 << 24, (1 << 24) // divisor
    f = np.random.default_rng(divisor).integers(0, V, (T, 3)).astype(np.int32)
    label, size = check_mesh(f, V, cases=((0, 0), (0, 2)))
    if divisor == 4:
        assert size.max() > T // 4                                        # a giant component
    if divisor == 8:
        assert size.max() < T // 1000                                     # none


def test_one_triangle_repeated_4m_times():
    V = 1000
    f = np.tile(np.array([[V - 1, V // 2, 7]], np.int32), (1 << 22, 1))
    label, size = check_mesh(f, V)
    assert size[7] == 1 << 22 and label[V - 1] == 7


def test_star_at_the_highest_vertex():
    """Every triangle joins a leaf to hub V - 1: each union re-hooks the root the hub already has."""
    V = 1 << 22
    leaves = np.random.default_rng(1).permutation(V - 1)
    label, size = check_mesh(np.stack([leaves, np.full(V - 1, V - 1), leaves], 1).astype(np.int32), V)
    assert (label == 0).all() and size[0] == V - 1


def test_comb_of_paths_hooked_in_descending_order():
    """1024 paths of 4096 vertices each, their first vertices joined by a spine, every triangle in descending order."""
    P, Lp = 1024, 4096
    V = P * Lp
    v = np.arange(V).reshape(P, Lp)
    teeth = np.stack([v[:, 1:].ravel(), v[:, :-1].ravel(), v[:, :-1].ravel()], 1)
    spine = np.stack([v[1:, 0], v[:-1, 0], v[:-1, 0]], 1)
    f = np.concatenate([teeth, spine])
    f = f[np.argsort(-f.max(1), kind="stable")].astype(np.int32)
    label, size = check_mesh(f, V)
    assert (label == 0).all() and size[0] == V - 1


def test_binary_tree_merges():
    """Level l joins i and i + 2^l for i a multiple of 2^(l+1): the roots of the two halves the level before made."""
    V = 1 << 22
    f = []
    for lev in range(22):
        i = np.arange(0, V, 2 << lev)
        f.append(np.stack([i + (1 << lev), i, i], 1))
    label, size = check_mesh(np.concatenate(f).astype(np.int32), V)
    assert (label == 0).all() and size[0] == V - 1


def test_2e24_vertices_without_triangles_all_tie():
    """2^24 components of size 0: every one ties, so the ranking is the label order."""
    V = 1 << 24
    m = Mesh(np.zeros((0, 3), np.int32), V)
    for _ in range(2):
        m.launch()
        label, size, bad = m.result()
        assert bad == 0 and np.array_equal(label, np.arange(V)) and not size.any()
    ident = np.arange(V, dtype=np.int32)

    def want(keep, min_size):
        k = V if keep == 0 else min(keep, V)
        if min_size > 0:
            k = 0
        ni = np.where(ident < k, ident, -1)
        return dict(new_index=ni, rank=ident[:k], sizes=np.zeros(V, np.int64), counts=[k, k, V, 0])
    run_select(label, size, ((0, 0), (1, 0), (1000, 0), (0, 1)), want)


def _sparse_want(faces, V):
    """The oracle on the vertices the triangles touch, the other vertices of 2^27 left alone: (label, size, the
    selection for keep / min_size in closed form)."""
    f = np.asarray(faces, np.int64)
    used = np.unique(f)
    sub = np.searchsorted(used, f)                                 # an order-preserving renumbering
    sl, ss, _ = co.mesh_components(sub, len(used))
    label = np.arange(V, dtype=np.int32)
    label[used] = used[sl]
    size = np.zeros(V, np.int64)
    size[used] = ss

    def want(keep, min_size):
        roots = used[sl == np.arange(len(used))]
        big = roots[np.lexsort((roots, -size[roots]))]             # the touched components, ranked first
        t, K = len(big), V - len(used) + len(roots)
        comp = np.empty(V, np.int64)
        free = np.ones(V, bool)
        free[used] = False
        comp[free] = t + np.arange(free.sum())                     # untouched vertices: size-0 roots by label
        by_label = np.argsort(big)
        comp[used] = by_label[np.searchsorted(big, label[used], sorter=by_label)]
        sizes = np.concatenate([size[big], np.zeros(K - t, np.int64)])
        kept_comp = (sizes >= min_size) & ((keep == 0) | (np.arange(K) < keep))
        keep_v = kept_comp[comp]
        ni = np.where(keep_v, np.cumsum(keep_v) - 1, -1).astype(np.int32)
        return dict(new_index=ni, rank=comp[keep_v].astype(np.int32), sizes=sizes,
                    counts=[int(keep_v.sum()), int(kept_comp.sum()), K, int(sizes[kept_comp].sum())])
    return label, size, want


@pytest.mark.parametrize("where", ["one_triangle", "near_the_top"])
def test_2e27_vertices_with_a_few_triangles(where):
    """2^27 vertices, nearly all isolated: the grid of every launch at its largest, peak device memory under 8 GB."""
    V = 1 << 27
    top = V - 1
    if where == "one_triangle":
        f = np.array([[5, 1 << 26, top]])
    else:
        f = np.array([[top, top - 1, top - 2], [top - 5, top - 3, top - 5], [top - 2, top - 7, top - 7],
                      [top - 9, top - 9, top - 9], [0, top - 11, top - 12]])
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    wl, ws, want = _sparse_want(f, V)
    m = Mesh(f, V)
    for _ in range(2):
        m.launch()
        torch.cuda.synchronize()
        _intact(m.label, V, "label")
        _intact(m.size, V, "size")
        assert int(m.stats[0]) == 0
        assert torch.equal(m.label[:V], _dev(wl, torch.int32)) and torch.equal(m.size[:V], _dev(ws, torch.int64))
    s = Select(V)
    for keep, min_size in ((0, 0), (1, 0), (0, 1)):
        w = want(keep, min_size)
        for _ in range(2):
            s.launch(m.label, m.size, keep, min_size)
            same_selection(s.result(), w)
    peak = torch.cuda.max_memory_allocated()
    print(f"2^27 vertices ({where}): peak device memory {peak / 2 ** 30:.2f} GiB")
    assert peak < 8 * 2 ** 30


# ---- determinism -----------------------------------------------------------------------------------------------------
def _hypergraph(seed, V, T):
    return np.random.default_rng(seed).integers(0, V, (T, 3)).astype(np.int32)


def test_same_input_three_times_is_bitwise_equal():
    V = 1 << 22
    f = _hypergraph(30, V, V // 6)
    runs = []
    for _ in range(3):
        m = Mesh(f, V)
        m.launch()
        label, size, _ = m.result()
        s = Select(V)
        s.launch(m.label, m.size, 0, 2)
        runs.append((label, size, s.result()))
    for label, size, sel in runs[1:]:
        assert np.array_equal(label, runs[0][0]) and np.array_equal(size, runs[0][1])
        same_selection(sel, runs[0][2])
    wl, ws, _ = co.mesh_components(f, V)
    assert np.array_equal(runs[0][0], wl) and np.array_equal(runs[0][1], ws)


def test_two_inputs_on_two_streams_at_once():
    V = 1 << 22
    inputs = [_hypergraph(31, V, V // 6), _hypergraph(32, V, V // 5)]
    single = []
    for f in inputs:
        m = Mesh(f, V)
        m.launch()
        s = Select(V)
        s.launch(m.label, m.size, 3, 1)
        single.append((m.result(), s.result()))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ms, ss = [Mesh(f, V) for f in inputs], [Select(V) for _ in inputs]
    torch.cuda.synchronize()                                       # the random fills are on the default stream
    for m, st in zip(ms, streams):
        m.launch(st)
    for m, s, st in zip(ms, ss, streams):
        s.launch(m.label, m.size, 3, 1, st)
    for m, s, (mr, sr) in zip(ms, ss, single):
        got = m.result()
        assert np.array_equal(got[0], mr[0]) and np.array_equal(got[1], mr[1]) and got[2] == mr[2]
        same_selection(s.result(), sr)


# ---- point clouds ----------------------------------------------------------------------------------------------------
def check_points(xyz, origin, cell, capacity, cases=((0, 0), (1, 0), (0, 3)), want=None):
    """lrf_point_components twice on one set of buffers against the oracle (or `want`), the table it leaves checked
    by table_ok, and the selections."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    wl, ws, wc, wo = want if want is not None else co.point_components(xyz, origin, cell)
    p = Points(xyz, origin, cell, capacity)
    for _ in range(2):
        p.launch()
        label, size, cells, out = p.result()
        assert (cells, out) == (wc, wo)
        assert np.array_equal(label, wl) and np.array_equal(size, ws)
        assert co.table_ok(*p.table(), xyz, origin, cell, capacity)
    run_select(wl, ws, cases, lambda k, s: co.select(wl, ws, k, s))
    return wl, ws


def _centres(k, per_cell, rng):
    """per_cell points in each cell k (cell_size 1, origin 0) at random offsets in [1/8, 7/8), in random order."""
    k = np.repeat(np.asarray(k, np.float32), per_cell, 0)
    p = k + rng.uniform(0.125, 0.875, k.shape).astype(np.float32)
    return p[rng.permutation(len(p))]


def test_probe_chain_of_half_the_capacity_wrapping_past_the_last_slot():
    """capacity / 2 cells whose probes all start two slots before the end: one chain as long as the table allows,
    wrapping from the last slot to 0; one cell more overflows, and keep_components names `capacity`."""
    cap = 256
    k = co.colliding_cells(cap, cap - 2, (0, 0, 0), (64, 64, 64))
    assert len(k) > cap // 2
    rng = np.random.default_rng(40)
    full = _centres(k[:cap // 2], 3, rng)
    check_points(full, (0.0, 0.0, 0.0), 1.0, cap)
    over = np.concatenate([full, _centres(k[cap // 2:cap // 2 + 1], 1, rng)])
    p = Points(over, (0.0, 0.0, 0.0), 1.0, cap)
    p.launch()
    assert p.result()[2] > cap // 2
    cloud = dict(xyz=_dev(over, torch.float32))
    with pytest.raises(RuntimeError, match="capacity"):
        keep_components(cloud, cell_size=1.0, capacity=cap)
    assert len(keep_components(cloud, cell_size=1.0, capacity=2 * cap)["xyz"]) == len(over)


def test_capacity_two_with_one_cell_and_4m_points_in_one_cell():
    rng = np.random.default_rng(41)
    check_points(_centres([[-3, 5, 0]], 7, rng), (0.0, 0.0, 0.0), 1.0, 2)
    n = 1 << 22
    p = _centres([[0, 0, 0]], n, rng)
    label, size = check_points(p, (0.0, 0.0, 0.0), 1.0, 16, cases=((0, 0), (1, n + 1)),
                               want=(np.zeros(n, np.int32), np.r_[n, np.zeros(n - 1, np.int64)], 1, 0))
    assert size[0] == n


def test_dense_block_of_2e24_points():
    """256^3 cells with one point each, in random order, in a table of 2^25 slots: one component."""
    g = np.arange(256, dtype=np.float32) + np.float32(0.5)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    p = p[np.random.default_rng(42).permutation(len(p))]
    n = len(p)
    check_points(p, (0.0, 0.0, 0.0), 1.0, 1 << 25, cases=((1, 0),),
                 want=(np.zeros(n, np.int32), np.r_[n, np.zeros(n - 1, np.int64)], n, 0))


def test_cells_on_the_key_field_limits():
    """Cells at key fields 0 and 2^21 - 1 on each axis.  (x, y, 2^20 - 1) and (x, y + 1, -2^20) have adjacent packed
    keys but are not neighbours; nor are (x, 2^20 - 1, z) and (x + 1, -2^20, z)."""
    lo, hi = -(1 << 20), (1 << 20) - 1
    corners = [[a, b, c] for a in (lo, hi) for b in (lo, hi) for c in (lo, hi)]
    pairs = [[7, 9, hi], [7, 10, lo], [3, hi, -4], [4, lo, -4], [hi, 0, 0], [hi - 1, 1, 1], [lo, 2, 2], [lo + 1, 3, 3]]
    cells_k = np.array(corners + pairs, np.float64)
    p = (cells_k + 0.5).astype(np.float32)
    assert np.array_equal(np.floor(p), cells_k)
    label, _ = check_points(p, (0.0, 0.0, 0.0), 1.0, 64)
    i = len(corners)
    assert label[i] != label[i + 1] and label[i + 2] != label[i + 3]          # adjacent keys, not neighbours
    assert label[i + 4] == label[i + 5] and label[i + 6] == label[i + 7]      # true neighbours at the limits
    assert len(np.unique(label[:i])) == 8


def test_subnormal_huge_and_signed_zero_coordinates():
    fmax = np.finfo(np.float32).max
    tiny = np.float32(1e-40)                                              # subnormal
    k = np.arange(-6, 7, dtype=np.float32)
    sub = np.stack([k * tiny, -k * tiny, np.zeros_like(k)], 1)             # multiples of a subnormal cell size
    check_points(sub, (0.0, 0.0, 0.0), float(tiny), 64)
    check_points(np.concatenate([sub, [[1e-30, 0, 0], [fmax, 0, 0]]]).astype(np.float32), (0.0, 0.0, 0.0),
                 float(tiny), 64)                                         # quotients past the key range and inf
    small = np.array([[1e-39, 2e-39, -1e-39], [0.0, -0.0, 0.0], [-0.0, -0.0, -0.0], [3e-38, 0, 0], [-1e-45, 0, 0]],
                     np.float32)                                          # subnormal p - origin
    check_points(small, (0.0, 0.0, 0.0), 1e-38, 64)
    odd = np.array([[fmax, 0, 0], [-fmax, 0, 0], [0, fmax, -fmax], [1e38, 1e38, 1e38], [-0.0, 0, 0], [0, 0, 0]],
                   np.float32)
    label, size = check_points(odd, (-1e38, 0.0, 0.0), 1e32, 64)          # fmax - (-1e38) overflows to inf
    origin = (0.1, -0.3, 0.7)
    h = np.float32(0.25)
    kk = np.arange(-5, 6, dtype=np.float32)
    on = np.stack(np.meshgrid(kk, kk, kk, indexing="ij"), -1).reshape(-1, 3) * h + np.asarray(origin, np.float32)
    check_points(on, origin, float(h), 1 << 12)                             # on cell boundaries, non-zero origin


# ---- selection on hand-written arrays --------------------------------------------------------------------------------
def _hand_written(n, rng):
    """Labels mostly roots, some pointing at roots, at non-roots, at -1, n and INT32_MIN; sizes spread over the clamp
    limits, negatives included."""
    label = np.arange(n, dtype=np.int64)
    r = rng.random(n)
    label[r < 0.3] = rng.integers(0, n, (r < 0.3).sum())
    odd = rng.choice([-1, n, -(2 ** 31)], n)
    label[r > 0.95] = odd[r > 0.95]
    size = rng.choice(np.array([0, 1, 2, 3, 5, TOP - 1, TOP, TOP + 1, 2 ** 63 - 1, -1, -(2 ** 40)], np.int64), n)
    return label, size


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 31, 32, 33, 255, 256, 257, (1 << 20) + 1])
def test_select_hand_written(n):
    rng = np.random.default_rng(n)
    label, size = _hand_written(n, rng)
    K = int((label == np.arange(n)).sum())
    cases = [(0, 0), (1, 0), (K, 0), (K + 1, 0), (2 ** 62, 0), (0, 1), (0, TOP), (0, 2 ** 31), (0, 2 ** 62), (2, 3)]
    run_select(label, size, cases, lambda k, s: co.select(label, size, k, s))


@pytest.mark.parametrize("n_kept", [32, 256, 512, 33])
def test_select_kept_prefix_ending_on_a_warp_or_block_boundary(n_kept):
    """1000 roots of distinct sizes: min_size and keep cut the ranking after exactly n_kept components."""
    n = 1000
    rng = np.random.default_rng(50)
    size = rng.permutation(n).astype(np.int64) + 10
    label = np.arange(n)
    cut = np.sort(size)[::-1][n_kept - 1]
    cases = [(0, int(cut)), (n_kept, 0), (n_kept, int(cut))]
    run_select(label, size, cases, lambda k, s: co.select(label, size, k, s))
    assert co.select(label, size, 0, int(cut))["counts"][1] == n_kept


@pytest.mark.parametrize("value", [7, 2 ** 63 - 1, -3])
def test_select_2e24_tied_components_and_their_summed_sizes(value):
    """2^24 roots of one size: ranked by label; counts[3] sums 2^24 clamped sizes (2^24 (2^31 - 1) for 2^63 - 1)."""
    n = 1 << 24
    label = np.arange(n, dtype=np.int32)
    size = np.full(n, value, np.int64)
    c = min(max(value, 0), TOP)

    def want(keep, min_size):
        k = n if keep == 0 else min(keep, n)
        k = k if c >= min_size else 0
        return dict(new_index=np.where(label < k, label, -1), rank=label[:k], sizes=np.full(n, c, np.int64),
                    counts=[k, k, n, k * c])
    run_select(label, size, ((0, 0), (1000, 0), (0, 1)), want)


# ---- through keep_components -----------------------------------------------------------------------------------------
def test_mesh_three_floaters_min_size_drops_the_smaller_two():
    lt = components_scene(grid=128)
    components_boxes(lt.tensorfs[0], [(-0.6, 0.2, -0.5, 0.5), (0.5, 0.7, 0.3, 0.5), (0.5, 0.62, -0.2, -0.08),
                                      (0.45, 0.85, -0.75, -0.45)], 0.4)
    w = lt.world2rf[0].detach().cpu().double().numpy()
    m = mesh(lt, voxel_size=1 / 64, origin=tuple(float(-x) for x in w))
    xyz, f = m["xyz"].cpu().numpy(), m["faces"].cpu().numpy()
    c = xyz[f[:, 0]].astype(np.float64) + w
    part = np.where(c[:, 0] < 0.35, 0, np.where(c[:, 1] > 0.2, 1, np.where(c[:, 1] > -0.35, 2, 3)))
    n_part = np.bincount(part, minlength=4)
    label, size, _ = co.mesh_components(f, len(xyz))
    assert co.select(label, size)["counts"][2] == 4
    assert sorted(co.select(label, size)["sizes"].tolist()) == sorted(n_part.tolist())
    floaters = sorted(range(1, 4), key=lambda i: n_part[i])
    assert n_part[floaters[0]] < n_part[floaters[1]] < n_part[floaters[2]] < n_part[0]
    clean = keep_components(m, min_size=int(n_part[floaters[1]]) + 1)
    gone = np.isin(part, floaters[:2])
    want = co.select(label, size, 0, int(n_part[floaters[1]]) + 1)
    kx, kf, (kn, kc) = co.keep_mesh(xyz, f, want["new_index"], (m["normals"].cpu().numpy(), m["rgb"].cpu().numpy()))
    assert len(kf) == int((~gone).sum())
    assert np.array_equal(kx[kf].view(np.uint32), xyz[f[~gone]].view(np.uint32))
    assert np.array_equal(clean["xyz"].cpu().numpy(), kx) and np.array_equal(clean["faces"].cpu().numpy(), kf)
    assert np.array_equal(clean["normals"].cpu().numpy(), kn) and np.array_equal(clean["rgb"].cpu().numpy(), kc)
    assert np.array_equal(clean["sizes"].cpu().numpy(), want["sizes"])
    # idempotent: applied to its own output it keeps every row and face, and the sizes are the kept prefix
    again = keep_components(clean, min_size=int(n_part[floaters[1]]) + 1)
    for k in ("xyz", "faces", "normals", "rgb", "component"):
        assert torch.equal(again[k], clean[k]), k
    assert again["sizes"].tolist() == want["sizes"][:want["counts"][1]].tolist()


def test_keep_components_empty_all_dropped_and_keep_past_k():
    dev = "cuda"
    empty = dict(xyz=torch.zeros(0, 3, device=dev), faces=torch.zeros(0, 3, dtype=torch.int32, device=dev))
    out = keep_components(empty, keep=1)
    assert out["xyz"].shape == (0, 3) and out["faces"].shape == (0, 3) and len(out["sizes"]) == 0
    out = keep_components(dict(xyz=torch.zeros(0, 3, device=dev)), cell_size=1.0)
    assert out["xyz"].shape == (0, 3) and len(out["component"]) == 0
    with pytest.raises(ValueError, match="outside"):
        keep_components(dict(empty, faces=torch.zeros(1, 3, dtype=torch.int32, device=dev)))
    rng = np.random.default_rng(60)
    V = 3000
    f = rng.integers(0, V, (800, 3)).astype(np.int32)
    xyz = torch.from_numpy(rng.standard_normal((V, 3)).astype(np.float32)).to(dev)
    g = dict(xyz=xyz, faces=_dev(f, torch.int32))
    label, size, _ = co.mesh_components(f, V)
    K = co.select(label, size)["counts"][2]
    out = keep_components(g, min_size=10 ** 9)                            # every component dropped
    assert out["xyz"].shape == (0, 3) and out["faces"].shape == (0, 3)
    assert out["sizes"].tolist() == co.select(label, size)["sizes"].tolist()
    out = keep_components(g, keep=K + 5)                                  # keep past the component count
    assert torch.equal(out["xyz"], xyz) and torch.equal(out["faces"], g["faces"])


def test_keep_components_non_contiguous_inputs_and_extra_keys():
    rng = np.random.default_rng(61)
    V = 4000
    f = rng.integers(0, V, (1200, 3)).astype(np.int32)
    big = torch.from_numpy(rng.standard_normal((V, 6)).astype(np.float32)).cuda()
    xyz = big[:, ::2]                                                     # stride 2 along a row
    wide = torch.zeros(len(f), 6, dtype=torch.int32, device="cuda")
    wide[:, ::2] = _dev(f, torch.int32)
    faces = wide[:, ::2]                                                  # stride 2 along a row
    assert not xyz.is_contiguous() and not faces.is_contiguous()
    extra = torch.arange(V, device="cuda").reshape(V, 1).expand(V, 5)      # a per-vertex key, stride 0
    g = dict(xyz=xyz, faces=faces, ids=extra, note="kept as is", scale=2.5)
    label, size, _ = co.mesh_components(f, V)
    want = co.select(label, size, 0, 3)
    out = keep_components(g, min_size=3)
    rows = want["new_index"] >= 0
    kx, kf, (ki,) = co.keep_mesh(xyz.cpu().numpy(), f, want["new_index"], (extra.cpu().numpy(),))
    assert np.array_equal(out["xyz"].cpu().numpy(), kx) and np.array_equal(out["faces"].cpu().numpy(), kf)
    assert np.array_equal(out["ids"].cpu().numpy(), ki) and out["note"] == "kept as is" and out["scale"] == 2.5
    assert np.array_equal(out["component"].cpu().numpy(), want["rank"]) and rows.sum() == len(kx)
    cloud = dict(xyz=xyz, ids=extra, tag=None)
    wl, ws, _, _ = co.point_components(xyz.cpu().numpy(), (0, 0, 0), 0.5)
    want = co.select(wl, ws, 2, 0)
    out = keep_components(cloud, keep=2, cell_size=0.5)
    rows = want["new_index"] >= 0
    assert np.array_equal(out["xyz"].cpu().numpy(), xyz.cpu().numpy()[rows]) and out["tag"] is None
    assert np.array_equal(out["ids"].cpu().numpy(), extra.cpu().numpy()[rows])
