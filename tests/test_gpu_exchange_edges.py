"""-m gpu, one device: the fused pixel exchange of the ray-sharded render (lrf_render's peer stores and step flags,
lrf_peer_barrier / lrf_peer_signal_wait, dist.PixelExchange, dist.render_sharded and the exchange branch of
LocalTensorfs.forward) with W simulated ranks on one GPU.

The kernels see a peer only as addresses (peer_pix[p], peer_flags[p]), so W ordinary buffers stand in for the
peers' gathered buffers, and every rank's launches are enqueued in rank order on ONE stream.  The gathered pixel
buffers are device memory filled with a NaN-payload canary (rows a launch must not touch keep it); every flag array
any launch may wait on is zeroed pinned host memory.  Before a launch with a nonzero wait is enqueued the harness
synchronises and asserts on the host that the flags it reads already hold the step it waits for, so a correct build
never spins; after it, the launch's event is polled against a deadline, and on a timeout every flag is set to
2^64-1 from the host (which releases any spin) before the test fails with the flags it saw.

  1. C ABI, lag 0: per step every rank renders its shard (shard_bounds) with n_peers = W and signal_seq = s, then
     every rank closes the step with lrf_peer_signal_wait(s, s) (one step with lrf_peer_barrier).  Every peer's
     buffer holds each shard bitwise as its rank's local pix and as the unsharded render; guard rows and the other
     rotating buffer keep the canary; slot r of every flag array is s and the other 16 - W slots stay 0; the stats
     summed over the ranks are the unsharded call's.  Small n leaves ranks with empty shards, which publish their
     step through lrf_render's n_rays = 0 path.  Non-final launches of a multi-field scene must not store to peers.
  2. C ABI, lag L in {1, 3}: the render kernel waits for step s - 1 - L itself; 2L + 4 buffers rotate over more than
     two rounds, and every buffer holds the last step that used it.
  3. The Python layer on hand-made PixelExchange instances (buffers and flags in pinned host memory): gathered()
     after step s is bitwise the unsharded render of step s - 1 - L; empty shards, a repeated batch (the cached
     plan), the bench's weak layout (row = rank * n), multi-view batches through render_sharded on both paths, and
     a batch no field renders (NotImplementedError with an exchange before anything is enqueued; out= filled).
  4. One gathered three-field image against the float64 restatement (tests/render64.py) at the bars of
     test_gpu_render_edges.py, so bitwise agreement with the unsharded render is not agreement with a shared wrong
     answer."""
import ctypes as C
import time

import pytest
import torch

import render64 as R
from localrf_b200 import _lib
from localrf_b200 import dist as xdist
from localrf_b200.dist import ExchangeSchedule, PixelExchange, render_sharded, shard_bounds

pytestmark = pytest.mark.gpu

CANARY = 0x7FC0DEAD              # a quiet NaN whose payload no rendered pixel carries
GUARD = 8                        # canary rows before and after the n rows of every gathered buffer
GRID = 64
IMG_W, IMG_H = 200, 150
DEADLINE_S = 30.0
WORLDS = [1, 2, 3, 5, 8, 16]


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def batch_sizes(W):
    return sorted({1, 7, 8, 9, 8 * W - 1, 8 * n_sms() + 1, 4096, 20000})


def ray_ids(n, seed, pinned=False):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, IMG_W * IMG_H, (n,), generator=g, dtype=torch.int64)
    return ids.pin_memory() if pinned else ids.cuda()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- scenes ------------------------------------------------------------------------------------------------------
def _exposure():
    """An exposure that pushes the first channel above 1 and the second below 0 (both clamp bounds)."""
    return torch.tensor([[4.0, 0.0, 0.0], [0.0, -0.5, 0.0], [0.2, 0.2, 0.6]])


SCENES = ["fp32", "three_fields", "floater", "bf16", "pe22", "exposure", "black_bg", "pinned_ids"]
_built = {}


def scene(name):
    """-> (LocalTensorfs on cuda, forward kwargs, pinned ids?)"""
    if name in _built:
        return _built[name]
    import bench
    over = dict(density_shift=-2)
    if name == "pe22":
        over.update(fea_pe=2, view_pe=2)
    with torch.random.fork_rng():
        lt = bench.build_scene("cpu", GRID, **over)
        if name == "three_fields":                  # as bench.py's cfg3
            for k in (1, 2):
                lt.append_frame()
                torch.manual_seed(k)
                lt.append_rf(1)
            # render64.random_field's safe MLP (hidden units biased +-1, small weights): no pre-activation near 0, so
            # the float64 anchor below compares nearly every ray
            sign = torch.where(torch.arange(128) % 2 == 0, 1.0, -1.0)
            with torch.no_grad():
                for rf in lt.tensorfs:
                    for layer in (rf.renderModule.mlp[0], rf.renderModule.mlp[2]):
                        layer.weight.mul_(0.05)
                        layer.bias.copy_(sign)
    lt = lt.to("cuda")
    kw = dict(is_train=False)
    if name == "three_fields":
        kw["world2rf"] = [torch.zeros(3, device="cuda"), torch.tensor([-0.3, 0.0, 0.0], device="cuda"),
                          torch.tensor([-0.6, 0.0, 0.0], device="cuda")]
        kw["blending_weights"] = torch.tensor([[0.2, 0.5, 0.3]], device="cuda")
    if name == "floater":
        kw["floater_thresh"] = 0.5
    if name == "bf16":
        lt.set_grid_storage("bf16")
    if name == "exposure":
        with torch.no_grad():
            lt.exposure[0].copy_(_exposure())
    if name == "black_bg":
        kw["white_bg"] = False
    _built[name] = (lt, kw, name == "pinned_ids")
    return _built[name]


VIEW = {}


def view0():
    if "v" not in VIEW:
        VIEW["v"] = torch.tensor([0], device="cuda")
    return VIEW["v"]


def unsharded(lt, kw, ids):
    """The unsharded eval render of `ids` -> (pix [n, 4] fp32, stats [2], the launch plan's launches, the plan)."""
    lt.__dict__.pop("_plans", None)
    stats = torch.zeros(2, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        rgb, depth, _, _ = lt(ids, view0(), IMG_W, IMG_H, stats=stats, **kw)
    (plan,) = lt.__dict__["_plans"].values()
    torch.cuda.synchronize()
    return torch.cat([rgb, depth[:, None]], 1).cuda(), stats, plan.launches, plan


def unsharded_pix(lt, kw, ids, views=None):
    """The unsharded eval render of `ids` as pix [n, 4] (leaves the plan cache alone)."""
    with torch.no_grad():
        rgb, depth, _, _ = lt(ids, view0() if views is None else views, IMG_W, IMG_H, **kw)
    return torch.cat([rgb, depth[:, None]], 1)


def bits(t):
    return t.contiguous().view(torch.int32)


# ---- the harness ---------------------------------------------------------------------------------------------------
class Peers:
    """W simulated ranks: gathered buffers [n_buf][GUARD + rows + GUARD][4] in device memory, one 16-slot flag array
    per rank in pinned host memory."""

    def __init__(self, W, n_buf, rows):
        self.W, self.n_buf, self.rows = W, n_buf, rows
        self.span = GUARD + rows + GUARD
        self.pix = [torch.full((n_buf, self.span, 4), CANARY, dtype=torch.int32, device="cuda") for _ in range(W)]
        self.flags = torch.zeros(W, 16, dtype=torch.int64).pin_memory()
        self.flag_ptrs = (C.c_void_p * 16)(*[self.flags.data_ptr() + 128 * p for p in range(W)])

    def refill(self):
        for p in self.pix:
            p.fill_(CANARY)

    def peer_pix(self, p, buf, row):
        return self.pix[p].data_ptr() + ((buf * self.span) + GUARD + row) * 16

    def fill(self, o, rank, buf, row, signal=0, wait=0):
        o.n_peers = self.W
        for p in range(self.W):
            o.peer_pix[p] = self.peer_pix(p, buf, row)
            o.peer_flags[p] = self.flag_ptrs[p]
        o.rank, o.signal_seq, o.wait_seq = rank, signal, wait

    def before_wait(self, rank, wait):
        """A launch of `rank` that waits for step `wait` is only enqueued once its flags already hold it."""
        if wait:
            torch.cuda.synchronize()
            seen = self.flags[rank, :self.W].tolist()
            assert all(v >= wait for v in seen), f"rank {rank} would wait for step {wait}; its flags hold {seen}"

    def watch(self, what):
        ev = torch.cuda.Event()
        ev.record()
        t0 = time.monotonic()
        while not ev.query():
            if time.monotonic() - t0 > DEADLINE_S:
                seen = self.flags.tolist()
                self.flags.fill_(-1)                            # 2^64 - 1 in every slot: releases any spinning wait
                torch.cuda.synchronize()
                pytest.fail(f"{what} did not finish within {DEADLINE_S} s; flags seen {seen}")
            time.sleep(0.001)

    def check_flags(self, s):
        f = self.flags.tolist()
        for p in range(self.W):
            assert f[p][:self.W] == [s] * self.W, (p, f[p])
            assert f[p][self.W:] == [0] * (16 - self.W), (p, f[p])

    def check_buffer(self, buf, want, bounds, local=None):
        """Buffer `buf` of every peer holds `want` [n, 4] in rows [0, n) (bitwise, and each shard as its rank's local
        pix when given) and the canary in its guard rows and rows past n."""
        n = want.shape[0]
        for p in range(self.W):
            b = self.pix[p][buf]
            assert torch.equal(b[GUARD:GUARD + n], bits(want)), f"peer {p}, buffer {buf}: rows differ from the render"
            assert bool((b[:GUARD] == CANARY).all()) and bool((b[GUARD + n:] == CANARY).all()), \
                f"peer {p}, buffer {buf}: a row outside [0, {n}) was written"
            if local is not None:
                for r, (lo, hi) in enumerate(bounds):
                    assert torch.equal(b[GUARD + lo:GUARD + hi], local[r][:hi - lo]), (p, r)

    def check_canary(self, buf):
        for p in range(self.W):
            assert bool((self.pix[p][buf] == CANARY).all()), f"peer {p}: buffer {buf} was written"


def render_rank(peers, launches, ids, lo, hi, rank, buf, signal, wait, stats):
    """Enqueues rank `rank`'s launches of one step (its shard [lo, hi) of `ids`): every launch gets the peers, only
    the finalize launch stores to them (checked after each earlier launch) and only it signals.  -> local pix (int32
    view, GUARD canary rows after the shard)."""
    lib = _lib.lib()
    n = hi - lo
    pix = torch.full((max(n, 1) + GUARD, 4), CANARY, dtype=torch.int32, device="cuda")
    ids_ptr = ids.data_ptr() + 8 * lo
    for rf, z, b, _, last in launches:
        bb = _lib.LrfBatch.from_buffer_copy(b)
        bb.n_rays, bb.ray_ids = n, ids_ptr
        o = _lib.LrfOutputs(pix=pix.data_ptr(), stats=stats.data_ptr())
        peers.fill(o, rank, buf, lo, signal if last else 0, wait if last else 0)
        if last:
            peers.before_wait(rank, o.wait_seq)
        fs, prep = rf.field_and_prepared(z)
        before = None if last else [q[buf].clone() for q in peers.pix]     # (the canary, or an older step's pixels)
        _lib.check(lib.lrf_render(C.byref(fs), C.c_void_p(prep.data_ptr()), C.byref(bb), C.byref(o), _stream()))
        if last and o.wait_seq:
            peers.watch(f"rank {rank}'s render of step {signal} (wait {wait})")
        if not last:
            torch.cuda.synchronize()
            for p in range(peers.W):
                assert torch.equal(peers.pix[p][buf], before[p]), "a non-final launch stored to a peer"
    return pix


# ---- 1. C ABI, lag 0 -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", WORLDS)
@pytest.mark.parametrize("name", SCENES)
def test_cabi_lag0(name, W):
    lt, kw, pinned = scene(name)
    sizes = batch_sizes(W)
    peers = Peers(W, 2, max(sizes))
    lib = _lib.lib()
    for s, n in enumerate(sizes, start=1):
        ids = ray_ids(n, 100 * W + s, pinned)
        want, want_stats, launches, _ = unsharded(lt, kw, ids)
        bounds = [shard_bounds(n, r, W) for r in range(W)]
        buf = s % 2
        peers.refill()
        stats = torch.zeros(W, 2, dtype=torch.int64, device="cuda")
        local = [render_rank(peers, launches, ids, lo, hi, r, buf, s, 0, stats[r]) for r, (lo, hi) in enumerate(bounds)]
        torch.cuda.synchronize()
        peers.check_flags(s)
        for r in range(W):
            peers.before_wait(r, s)
            if s == 3:
                _lib.check(lib.lrf_peer_barrier(peers.flag_ptrs, r, W, s, _stream()))
            else:
                _lib.check(lib.lrf_peer_signal_wait(peers.flag_ptrs, r, W, s, s, _stream()))
            peers.watch(f"rank {r}'s close of step {s}")
        torch.cuda.synchronize()
        peers.check_flags(s)
        peers.check_buffer(buf, want, bounds, local)
        peers.check_canary(1 - buf)
        for r, (lo, hi) in enumerate(bounds):
            assert torch.equal(local[r][:hi - lo], bits(want[lo:hi])), (n, r)
            assert bool((local[r][hi - lo:] == CANARY).all()), (n, r)
        assert stats.sum(0).tolist() == want_stats.tolist(), (n, stats.tolist(), want_stats.tolist())


# ---- 2. C ABI, the render kernel's own wait (lag >= 1) ---------------------------------------------------------------
@pytest.mark.parametrize("W,n", [(1, 4096), (2, 9), (3, 1057), (5, 4096), (8, 63), (16, 20000), (16, 100)])
@pytest.mark.parametrize("lag", [1, 3])
def test_cabi_lag(lag, W, n):
    lt, kw, _ = scene("three_fields" if W in (3, 16) and n > 1000 else "fp32")
    sch = ExchangeSchedule(lag)
    peers = Peers(W, sch.n_buf, n)
    bounds = [shard_bounds(n, r, W) for r in range(W)]
    history, last_used = {}, {}
    for s in range(1, 2 * sch.n_buf + 2):
        ids = ray_ids(n, 1000 * W + s)
        want, want_stats, launches, _ = unsharded(lt, kw, ids)
        buf, sig, wait = sch.next_step()
        assert sig == s and wait == max(s - 1 - lag, 0)
        stats = torch.zeros(W, 2, dtype=torch.int64, device="cuda")
        local = [render_rank(peers, launches, ids, lo, hi, r, buf, s, wait, stats[r]) for r, (lo, hi) in enumerate(bounds)]
        sch.advance()
        torch.cuda.synchronize()
        history[s], last_used[buf] = want, s
        peers.check_flags(s)
        for b in range(sch.n_buf):
            if b in last_used:        # every buffer holds the last step that used it
                peers.check_buffer(b, history[last_used[b]], bounds, local if b == buf else None)
            else:
                peers.check_canary(b)
        g = sch.gathered_step()
        if g >= 1:
            peers.check_buffer(sch.gathered_buffer(), history[g], bounds)
        assert stats.sum(0).tolist() == want_stats.tolist()


# ---- 3. the Python layer ----------------------------------------------------------------------------------------------
def exchanges(W, lag, max_rays):
    """W hand-made PixelExchange instances (as tests/test_exchange_protocol.py builds them), each `mem` in pinned host
    memory: the gathered buffers filled with the canary, the flags zeroed; `ptrs` are the W mems."""
    sch = ExchangeSchedule(lag)
    buf_bytes = (max_rays * 16 + 255) // 256 * 256
    total = sch.n_buf * buf_bytes + PixelExchange.FLAG_BYTES
    mems = []
    for _ in range(W):
        m = torch.zeros(total, dtype=torch.uint8).pin_memory()
        m[:sch.n_buf * buf_bytes].view(torch.int32).fill_(CANARY)
        mems.append(m)
    xs = []
    for r in range(W):
        x = PixelExchange.__new__(PixelExchange)
        x.world, x.rank, x.max_rays, x.device = W, r, max_rays, torch.device("cuda", 0)
        x.buf_bytes, x.sched = buf_bytes, ExchangeSchedule(lag)
        x.lag, x.n_buf = x.sched.lag, x.sched.n_buf
        x.mem, x.ptrs, x.mc_ptr = mems[r], [m.data_ptr() for m in mems], 0
        x._flag_ptrs = (C.c_void_p * W)(*[p + x.n_buf * buf_bytes for p in x.ptrs])
        x._lib = _lib
        xs.append(x)
    return xs


def x_flags(x):
    return x.mem[x.n_buf * x.buf_bytes:].view(torch.int64)


class Ranks:
    """Simulated ranks for dist.render_sharded: torch.distributed's rank and world size as the test sets them."""

    def __init__(self, monkeypatch, W):
        self.W, self.rank = W, 0
        monkeypatch.setattr(xdist.dist, "get_world_size", lambda group=None: self.W)
        monkeypatch.setattr(xdist.dist, "get_rank", lambda group=None: self.rank)


def step_rank(x, what, fn):
    """Runs one rank's call `fn` of the next step: the host check of its wait before, the deadline after."""
    wait = x.sched.next_step()[2]
    if wait:
        torch.cuda.synchronize()
        seen = x_flags(x)[:x.world].tolist()
        assert all(v >= wait for v in seen), f"{what} would wait for step {wait}; its flags hold {seen}"
    out = fn()
    ev = torch.cuda.Event()
    ev.record()
    t0 = time.monotonic()
    while not ev.query():
        if time.monotonic() - t0 > DEADLINE_S:
            seen = x_flags(x).tolist()
            x_flags(x).fill_(-1)                                # its render waits on its own flags only
            torch.cuda.synchronize()
            pytest.fail(f"{what} did not finish within {DEADLINE_S} s; flags seen {seen}")
        time.sleep(0.001)
    return out


def release_all(xs):
    for x in xs:
        x_flags(x).fill_(-1)


def gathered_bits(x, n):
    return x.gathered(n).contiguous().view(torch.int32)


@pytest.mark.parametrize("W", [1, 2, 5, 16])
@pytest.mark.parametrize("lag", [1, 3])
def test_render_sharded_lag(monkeypatch, lag, W):
    """render_sharded through W hand-made exchanges: small batches give empty shards (skip_step), a batch repeated
    with the same tensors reuses the cached plan; after step s every rank's gathered() is bitwise the unsharded
    render of step s - 1 - lag."""
    lt, kw, _ = scene("fp32")
    ranks = Ranks(monkeypatch, W)
    xs = exchanges(W, lag, 20000)
    view = view0()
    repeat = ray_ids(4096, 7)
    batches = [repeat, ray_ids(9, 1), repeat, ray_ids(1, 2), ray_ids(20000, 3), repeat, ray_ids(8 * W - 1, 4)]
    batches += [ray_ids(777 + s, 10 + s) for s in range(2 * xs[0].n_buf + 1 - len(batches))]
    history = {}
    lt.__dict__.pop("_plans", None)
    try:
        for s, ids in enumerate(batches, start=1):
            history[s] = unsharded_pix(lt, kw, ids)
            plans = len(lt.__dict__["_plans"])
            for r in range(W):
                ranks.rank = r
                with torch.no_grad():
                    step_rank(xs[r], f"rank {r} step {s}",
                              lambda: render_sharded(lt, ids, view, IMG_W, IMG_H, exchange=xs[r], **kw))
            if s == 3:                                          # the batch of step 1 again: every shard's plan is cached
                assert len(lt.__dict__["_plans"]) == plans
            torch.cuda.synchronize()
            g = s - 1 - lag
            for x in xs:
                assert x.seq == s and x.gathered_step() == max(g, 0)
                assert x_flags(x)[:W].tolist() == [s] * W and x_flags(x)[W:].tolist() == [0] * (16 - W)
                if g >= 1:
                    n = history[g].shape[0]
                    assert torch.equal(gathered_bits(x, n), bits(history[g]).cpu()), (x.rank, s, g)
    except BaseException:
        release_all(xs)
        raise


@pytest.mark.parametrize("W", [2, 5, 16])
@pytest.mark.parametrize("lag", [1, 3])
def test_weak_layout(lag, W):
    """The bench's weak scaling: every rank renders its own batch of n rays into rows rank * n of the gathered
    buffer, through LocalTensorfs.forward(exchange=(x, rank * n))."""
    lt, kw, _ = scene("fp32")
    n = 1000
    xs = exchanges(W, lag, W * n)
    history = {}
    try:
        for s in range(1, 2 * xs[0].n_buf + 2):
            batches = [ray_ids(n, 50 * s + r) for r in range(W)]
            history[s] = torch.cat([unsharded_pix(lt, kw, b) for b in batches])
            for r in range(W):
                with torch.no_grad():
                    step_rank(xs[r], f"rank {r} step {s}",
                              lambda: lt(batches[r], view0(), IMG_W, IMG_H, exchange=(xs[r], r * n), **kw))
            torch.cuda.synchronize()
            g = s - 1 - lag
            if g >= 1:
                for x in xs:
                    assert torch.equal(gathered_bits(x, W * n), bits(history[g]).cpu()), (x.rank, s)
    except BaseException:
        release_all(xs)
        raise


def test_render_sharded_lag0_one_rank(monkeypatch):
    """Lag 0 through Python (one rank: close_step's wait kernel follows the render of the same stream)."""
    lt, kw, _ = scene("three_fields")
    Ranks(monkeypatch, 1)
    (x,) = exchanges(1, 0, 20000)
    try:
        for s, n in enumerate([4096, 1, 20000, 9, 4096], start=1):
            ids = ray_ids(n, 300 + s)
            want = unsharded_pix(lt, kw, ids)
            with torch.no_grad():
                rgb, depth = step_rank(x, f"step {s}", lambda: render_sharded(lt, ids, view0(), IMG_W, IMG_H,
                                                                              exchange=x, **kw))
            torch.cuda.synchronize()
            assert x.gathered_step() == s and x_flags(x)[0] == s
            assert torch.equal(gathered_bits(x, n), bits(want).cpu())
            assert torch.equal(rgb, want[:, :3].cpu()) and torch.equal(depth, want[:, 3].cpu())
    except BaseException:
        release_all([x])
        raise


def _views_scene():
    if "views16" not in _built:
        import bench
        import localrf_b200 as L
        with torch.random.fork_rng():
            lt = bench.Workload("incoherent", grid=GRID).build(L.LocalTensorfs, quiet=True)
        _built["views16"] = lt.to("cuda")
    return _built["views16"]


def _views_batch(seed, V=16, per=256):
    g = torch.Generator().manual_seed(seed)
    px = torch.randint(0, IMG_W * IMG_H, (V, per), generator=g)
    return (px + torch.arange(V)[:, None] * IMG_W * IMG_H).reshape(-1).cuda()


@pytest.mark.parametrize("W", [2, 3, 5, 16])
def test_render_sharded_multiview_exchange(monkeypatch, W):
    """16 views x 256 rays: each rank renders whole views (shard_views) at the rows of its first ray, and the
    gathered image equals the unsharded call bitwise."""
    lt = _views_scene()
    ranks = Ranks(monkeypatch, W)
    lag = 1
    xs = exchanges(W, lag, 4096)
    views = torch.arange(16, device="cuda")
    history = {}
    try:
        for s in range(1, lag + 5):
            ids = _views_batch(s)
            history[s] = unsharded_pix(lt, dict(is_train=False), ids, views)
            for r in range(W):
                ranks.rank = r
                with torch.no_grad():
                    step_rank(xs[r], f"rank {r} step {s}",
                              lambda: render_sharded(lt, ids, views, IMG_W, IMG_H, exchange=xs[r], is_train=False))
            torch.cuda.synchronize()
            g = s - 1 - lag
            if g >= 1:
                for x in xs:
                    assert torch.equal(gathered_bits(x, 4096), bits(history[g]).cpu()), (x.rank, s)
    except BaseException:
        release_all(xs)
        raise


@pytest.mark.parametrize("W", [2, 3, 5, 16])
def test_render_sharded_multiview_gather(monkeypatch, W):
    """The all-gather path of the same batches: each rank's forward renders its whole views, and the bounds it hands
    to gather_pixels place them (the gather itself is the host logic test_dist_gloo.py covers)."""
    lt = _views_scene()
    ranks = Ranks(monkeypatch, W)
    parts = {}

    def gather(rgb, depth, n_total, group=None, bounds=None):
        parts[ranks.rank] = (rgb.clone(), depth.clone(), n_total, bounds)
        return rgb, depth

    monkeypatch.setattr(xdist, "gather_pixels", gather)
    views = torch.arange(16, device="cuda")
    ids = _views_batch(99)
    with torch.no_grad():
        rgb, depth, _, _ = lt(ids, views, IMG_W, IMG_H, is_train=False)
        for r in range(W):
            ranks.rank = r
            render_sharded(lt, ids, views, IMG_W, IMG_H, is_train=False)
    bounds = parts[0][3]
    assert bounds is not None and all(parts[r][3] == bounds for r in range(W))
    assert bounds[0][0] == 0 and bounds[-1][1] == 4096 and all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
    assert all((hi - lo) % 256 == 0 for lo, hi in bounds)
    got_rgb = torch.cat([parts[r][0] for r in range(W)])
    got_depth = torch.cat([parts[r][1] for r in range(W)])
    assert torch.equal(got_rgb, rgb) and torch.equal(got_depth, depth)


def test_no_field_renders_the_batch():
    """A batch whose blending row is zero: with an exchange, NotImplementedError before anything is enqueued (no
    step is counted or published); with out=, the ones the reference returns land in the caller's buffers (device
    and pinned host)."""
    lt, kw, _ = scene("fp32")
    (x,) = exchanges(1, 1, 4096)
    zero = torch.zeros(1, 1, device="cuda")
    ids = ray_ids(100, 5)
    with torch.no_grad(), pytest.raises(NotImplementedError):
        lt(ids, view0(), IMG_W, IMG_H, is_train=False, blending_weights=zero, exchange=(x, 0))
    torch.cuda.synchronize()
    assert x.seq == 0 and x_flags(x).tolist() == [0] * 16
    assert bool((x.mem[:x.n_buf * x.buf_bytes].view(torch.int32) == CANARY).all())
    for dev_out in (True, False):
        rgb, depth = torch.full((100, 3), 7.0), torch.full((100,), 7.0)
        rgb, depth = (rgb.cuda(), depth.cuda()) if dev_out else (rgb.pin_memory(), depth.pin_memory())
        with torch.no_grad():
            r, d, _, _ = lt(ids, view0(), IMG_W, IMG_H, is_train=False, blending_weights=zero, out=(rgb, depth))
        torch.cuda.synchronize()
        assert r.data_ptr() == rgb.data_ptr() and d.data_ptr() == depth.data_ptr()
        assert bool((rgb == 1).all()) and bool((depth == 1).all()), dev_out


# ---- 4. the float64 anchor ---------------------------------------------------------------------------------------------
TOL = 1e-4
MARGIN, BOUND = 2.0 ** 6, 2.0           # test_gpu_render_edges.py's margins (EPS units / propagated-bound units)
MARGIN_MLP = BOUND * 96                  # (the tensor-core path's three bf16 products)
MAX_EXCLUDED = 0.08


def scale_err(a, b, floor=1e-30):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(floor))


def test_gathered_three_fields_vs_float64():
    lt, kw, _ = scene("three_fields")
    W, n = 5, 4096
    ids = ray_ids(n, 77)
    want, _, launches, plan = unsharded(lt, kw, ids)
    peers = Peers(W, 2, n)
    bounds = [shard_bounds(n, r, W) for r in range(W)]
    stats = torch.zeros(W, 2, dtype=torch.int64, device="cuda")
    for r, (lo, hi) in enumerate(bounds):
        render_rank(peers, launches, ids, lo, hi, r, 1, 1, 0, stats[r])
    torch.cuda.synchronize()
    peers.check_buffer(1, want, bounds)
    got = peers.pix[W - 1][1, GUARD:GUARD + n].view(torch.float32)
    c2w, intr, E, blend = plan.keep[:4]
    w2rf = plan.keep[4:]
    z = launches[0][1]
    assert all(torch.equal(l[1], z) for l in launches)
    fields = [R.Field64.from_module(rf, "cuda") for rf in lt.tensorfs]
    ref = R.render_views(fields, z.double(), ids, IMG_W, IMG_H, lt.fov == 360, intr, c2w, w2rf, blend, E, True)
    keep = torch.ones_like(ref["thres"], dtype=torch.bool)
    for k in R.MARGIN_KEYS:                 # (not the contraction: both of its branches give 1 at max|p| = 1)
        if k != "contract":
            keep &= ref[k] >= (MARGIN_MLP if k == "mlp" else BOUND if k in R.BOUND_KEYS else MARGIN)
    frac = 1 - float(keep.double().mean())
    tol = max(TOL, 2 * z.numel() * R.EPS)
    e_rgb = scale_err(got[:, :3][keep], ref["rgb"][keep], 0.1)
    e_dep = scale_err(got[:, 3][keep], ref["depth"][keep])
    print(f"three fields, gathered over {W} ranks: excluded {100 * frac:.2f} %, rgb {e_rgb:.1e} depth {e_dep:.1e} "
          f"(bar {tol:.1e})")
    assert frac <= MAX_EXCLUDED and e_rgb < tol and e_dep < tol
