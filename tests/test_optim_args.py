"""CPU-only: lrf_adam_step refuses bad arguments with LRF_ERR_INVALID and a message before it touches a device (the
non-NULL pointers below are never dereferenced), and localrf_b200.adam_step hands optimisers it cannot run on the
device to their own step()."""
import copy
import ctypes as C
import struct

import torch

from localrf_b200 import _lib, optim

INVALID = -1
FAKE = 0x10000                       # 16-byte aligned, never read


def _table(n, numel=64):
    t = (_lib.LrfAdamTensor * max(n, 1))()
    for e in t:
        e.param = e.grad = e.exp_avg = e.exp_avg_sq = FAKE
        e.numel = numel
    return t


def test_struct_mirror():
    L = _lib.lib()
    assert L.lrf_sizeof(6) == C.sizeof(_lib.LrfAdamTensor) == 4 * 8 + 8 + 6 * 4
    assert struct.calcsize("<" + optim._ENTRY) == C.sizeof(_lib.LrfAdamTensor)


def test_invalid():
    L = _lib.lib()
    assert L.lrf_adam_step(_table(1), -1, None) == INVALID
    assert b"bad tensor table" in L.lrf_last_error()
    assert L.lrf_adam_step(None, 2, None) == INVALID
    t = _table(3)
    t[2].numel = -1
    assert L.lrf_adam_step(t, 3, None) == INVALID
    assert b"numel < 0" in L.lrf_last_error()
    for name in ("param", "grad", "exp_avg", "exp_avg_sq"):
        t = _table(3)
        setattr(t[1], name, None)
        assert L.lrf_adam_step(t, 3, None) == INVALID, name
        assert b"is NULL" in L.lrf_last_error()


def test_nothing_to_do():
    L = _lib.lib()
    assert L.lrf_adam_step(None, 0, None) == 0
    t = _table(2, numel=0)                        # empty tensors are skipped: their pointers may be NULL
    t[0].param = t[1].grad = None
    assert L.lrf_adam_step(t, 2, None) == 0


def test_cpu_optimizers_take_their_own_step():
    """CPU parameters are not the kernel's: adam_step is the per-optimiser loop, zero_grad is zero_grad()."""
    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(3, 2)), torch.nn.Parameter(torch.randn(3))]
    opts = [torch.optim.Adam([ps[0]], lr=1e-2), torch.optim.Adam([ps[1]], lr=1e-3, betas=(0.9, 0.99))]
    refs = copy.deepcopy(opts)
    for _ in range(3):
        for o, r in zip(opts, refs):
            for p, q in zip(o.param_groups[0]["params"], r.param_groups[0]["params"]):
                p.grad = torch.randn(p.shape)
                q.grad = p.grad.clone()
        optim.adam_step(opts)
        for r in refs:
            r.step()
    for o, r in zip(opts, refs):
        p, q = o.param_groups[0]["params"][0], r.param_groups[0]["params"][0]
        assert torch.equal(p, q)
        assert torch.equal(o.state[p]["exp_avg_sq"], r.state[q]["exp_avg_sq"])
        assert o.state[p]["step"].item() == 3.0
    optim.zero_grad(opts)
    assert all(p.grad is None for p in ps)
