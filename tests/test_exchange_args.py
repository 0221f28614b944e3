"""CPU-only: the fused pixel exchange arguments of the C ABI -- the exchange fields of LrfOutputs that lrf_render
checks, for a batch of rays and for an empty one (a rank whose shard is empty still publishes its step, so its
fields are checked the same way), and the arguments of lrf_peer_barrier / lrf_peer_signal_wait.  Every refusal is
LRF_ERR_INVALID with its message before any device work (the fake pointers below are never dereferenced, and no
call here is given a valid set of arguments, so none reaches a device)."""
import ctypes as C

import pytest

from localrf_b200 import _lib

OK, INVALID = 0, -1
FAKE = 0x10000                       # 16-byte aligned, never read
WORLD = 4


def _field():
    s = _lib.LrfField()
    s.grid[:] = [8, 8, 8]
    s.aabb[:] = [-1, -1, -1, 1, 1, 1]
    s.n_dcomp, s.n_acomp, s.app_dim, s.featureC = 8, 24, 27, 128
    for name in ("dplane", "dline", "aplane", "aline"):
        for i in range(3):
            getattr(s, name)[i] = FAKE
    for name in ("basis", "w1", "b1", "w2", "b2", "w3", "b3", "z_vals"):
        setattr(s, name, FAKE)
    s.n_samples = 64
    return s


def _batch(n):
    b = _lib.LrfBatch()
    b.n_rays, b.rays, b.n_views, b.finalize = n, FAKE, 1, 1
    return b


def _outputs(signal=True):
    """A valid exchange: WORLD peers, this rank 1, peer stores at rows of 16 bytes, flags 8-byte aligned."""
    o = _lib.LrfOutputs()
    o.pix = FAKE
    o.n_peers = WORLD
    for p in range(WORLD):
        o.peer_pix[p] = FAKE + 0x100000 * (p + 1) + 16 * 7
        o.peer_flags[p] = FAKE + 0x1000 * (p + 1) + 8
    o.rank = 1
    if signal:
        o.signal_seq, o.wait_seq = 9, 5
    return o


def _render(o, n):
    return _lib.lib().lrf_render(C.byref(_field()), FAKE, C.byref(_batch(n)), C.byref(o), None)


def _err():
    return _lib.lib().lrf_last_error().decode()


# case -> (how to spoil a valid exchange, a piece of the message)
CASES = {
    "n_peers_-1": (lambda o: setattr(o, "n_peers", -1), "n_peers out of range"),
    "n_peers_17": (lambda o: setattr(o, "n_peers", 17), "n_peers out of range"),
    "no_pix": (lambda o: setattr(o, "pix", None), "needs the interleaved `pix` output"),
    "peer_pix_null": (lambda o: o.peer_pix.__setitem__(3, None), "peer_pix pointers must be non-NULL"),
    "peer_pix_misaligned": (lambda o: o.peer_pix.__setitem__(2, FAKE + 8), "16-byte aligned"),
    "mc_pix_misaligned": (lambda o: setattr(o, "mc_pix", FAKE + 4), "mc_pix must be 16-byte aligned"),
    "signal_without_peers": (lambda o: setattr(o, "n_peers", 0), "in-kernel signalling needs n_peers >= 1"),
    "rank_-1": (lambda o: setattr(o, "rank", -1), "0 <= rank < n_peers"),
    "rank_n_peers": (lambda o: setattr(o, "rank", WORLD), "0 <= rank < n_peers"),
    "wait_above_signal": (lambda o: setattr(o, "wait_seq", 10), "wait_seq <= signal_seq"),
    "peer_flags_null": (lambda o: o.peer_flags.__setitem__(0, None), "peer_flags pointers must be non-NULL"),
    "peer_flags_misaligned": (lambda o: o.peer_flags.__setitem__(3, FAKE + 4), "8-byte aligned"),
}


@pytest.mark.parametrize("n", [64, 0])
@pytest.mark.parametrize("case", list(CASES))
def test_render_refuses_bad_exchange_fields(case, n):
    spoil, msg = CASES[case]
    o = _outputs()
    spoil(o)
    assert _render(o, n) == INVALID, case
    assert msg in _err(), (case, _err())


def test_empty_batch_without_signal_enqueues_nothing():
    """Without signal_seq the flag array, rank and wait step are not read: on an empty batch a NULL flag pointer, a
    rank out of range and a wait step above the (zero) signal step give LRF_OK, and nothing is enqueued."""
    o = _outputs(signal=False)
    o.peer_flags[0], o.rank, o.wait_seq = None, WORLD + 3, 7
    assert _render(o, 0) == OK, _err()
    o.n_peers = 0
    assert _render(o, 0) == OK, _err()


def _flags(world, bad=None, value=None):
    arr = (C.c_void_p * 16)(*[FAKE + 0x100 * p for p in range(16)])
    if bad is not None:
        arr[bad] = value
    return arr


BARRIER_CASES = {
    "world_0": dict(world=0),
    "world_17": dict(world=17),
    "rank_-1": dict(rank=-1),
    "rank_world": dict(rank=WORLD),
    "flags_array_null": dict(flags=None),
    "flag_null": dict(flags=_flags(WORLD, 2, None)),
    "flag_misaligned": dict(flags=_flags(WORLD, 3, FAKE + 4)),
}


def _barrier(entry, world=WORLD, rank=1, flags="valid", seq=3, wait=3):
    L = _lib.lib()
    flags = _flags(WORLD) if flags == "valid" else flags
    if entry == "barrier":
        return L.lrf_peer_barrier(flags, rank, world, seq, None)
    return L.lrf_peer_signal_wait(flags, rank, world, seq, wait, None)


@pytest.mark.parametrize("entry", ["barrier", "signal_wait"])
@pytest.mark.parametrize("case", list(BARRIER_CASES))
def test_peer_barrier_refuses_bad_arguments(case, entry):
    assert _barrier(entry, **BARRIER_CASES[case]) == INVALID, case
    assert "bad peer_flags / rank / world" in _err() or "8-byte aligned" in _err(), _err()


def test_signal_wait_refuses_a_wait_above_its_signal():
    assert _barrier("signal_wait", seq=3, wait=4) == INVALID
    assert "wait_seq must not exceed seq" in _err()
