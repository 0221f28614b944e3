"""Adam steps of a training iteration in one launch.

    adam_step(optimizers)      # == for o in optimizers: o.step(), bit for bit
    zero_grad(optimizers)      # == for o in optimizers: o.zero_grad()

A LocalTensorfs iteration steps the field's optimiser and, for every live frame, one Adam each for its rotation,
translation and exposure, plus the intrinsics' (local_tensorfs.py:245,272-284): up to about 300 `Adam.step()`
calls, each of them seven foreach kernels.  `adam_step` keeps the optimisers as they are -- real
`torch.optim.Adam` objects whose `param_groups`, `state` and `state_dict()` callers keep reading and writing --
and performs their update with one lrf_adam_step launch per device: the state is created as `Adam._init_group`
creates it, every `step` counter is incremented in one `torch._foreach_add_` on the CPU, each group's `lr` is read
at the call, and the per-tensor scalars are folded in double precision as torch 2.11's `_multi_tensor_adam` folds
them.  The kernel rounds as torch's foreach sequence does, so parameters and state are bit-identical to `step()`'s.
Nothing synchronises the host.

An optimiser goes through its own `step()` instead when the one-launch update would not be what that call does:
an option other than the default (amsgrad, maximize, weight_decay, foreach=False, fused, capturable,
differentiable, a tensor lr or betas), a parameter with a gradient that is not a dense fp32 CUDA tensor laid out
like its gradient and state, a parameter that appears twice among the optimisers, a subclass or an overridden
`step`, or step hooks (the optimiser's own or global ones).
"""
import struct

import torch
from torch.optim import optimizer as _optimizer

from . import _lib
from .tensorf import _stream

_ENTRY = "4Qq6f"                         # LrfAdamTensor: 4 pointers, numel, 6 floats (64 bytes)
_ONE = torch.tensor(1.0)                 # the increment torch adds to CPU step counters


def _plain(opt):
    """opt.step() / opt.zero_grad() are torch.optim.Adam's own, with no hook around them."""
    return (type(opt) is torch.optim.Adam and "step" not in vars(opt) and "zero_grad" not in vars(opt)
            and not opt._optimizer_step_pre_hooks and not opt._optimizer_step_post_hooks)


def _default_options(group):
    return not (group["amsgrad"] or group["maximize"] or group["weight_decay"] != 0 or group["foreach"] is False
                or group["fused"] or group["capturable"] or group["differentiable"] or torch.is_tensor(group["lr"])
                or any(torch.is_tensor(b) for b in group["betas"]))


def _dense(t):
    """t's elements fill [data_ptr, data_ptr + numel) exactly once (any order of the dimensions)."""
    if t.is_contiguous() or t.is_contiguous(memory_format=torch.channels_last):
        return True
    expected = 1
    for size, stride in sorted((d for d in zip(t.shape, t.stride()) if d[0] != 1), key=lambda d: d[1]):
        if stride != expected:
            return False
        expected *= size
    return True


def _same_layout(t, p):
    return (t.dtype == torch.float32 and t.device == p.device and not t.is_sparse and t.shape == p.shape
            and t.stride() == p.stride())


def _fusable(opt, seen_twice):
    """The parameters with a gradient of `opt`, or None when opt must go through its own step()."""
    if not _plain(opt):
        return None
    out = []
    for group in opt.param_groups:
        if not _default_options(group):
            return None
        for p in group["params"]:
            if id(p) in seen_twice:
                return None
            g = p.grad
            if g is None:
                continue
            if not (p.is_cuda and p.dtype == torch.float32 and _same_layout(g, p) and _dense(p)):
                return None
            st = opt.state.get(p)
            if st:
                step = st.get("step")
                if (step is None or not torch.is_tensor(step) or step.is_cuda or "exp_avg" not in st
                        or "exp_avg_sq" not in st or not _same_layout(st["exp_avg"], p)
                        or not _same_layout(st["exp_avg_sq"], p)):
                    return None
            out.append((group, p, g))
    return out


def _twice(optimizers):
    seen, twice = set(), set()
    for opt in optimizers:
        for group in opt.param_groups:
            for p in group["params"]:
                (twice if id(p) in seen else seen).add(id(p))
    return twice


def adam_step(optimizers):
    """Does what `for o in optimizers: o.step()` does, with one kernel launch per device for every optimiser that
    allows it (see the module docstring); the others run their own step() after the launch.  Enqueued on the
    current stream of each parameter's device."""
    optimizers = list(optimizers)
    hooked = bool(_optimizer._global_optimizer_pre_hooks or _optimizer._global_optimizer_post_hooks)
    twice = _twice(optimizers) if len(optimizers) > 1 else set()
    fused, rest = [], []
    for opt in optimizers:
        items = None if hooked else _fusable(opt, twice)
        if items is None:
            rest.append(opt)
        else:
            fused.append((opt, items))

    entries = []                           # (device, group, p, g, state)
    for opt, items in fused:
        for group, p, g in items:
            st = opt.state[p]
            if len(st) == 0:               # as Adam._init_group creates it
                st["step"] = torch.tensor(0.0, dtype=_optimizer._get_scalar_dtype())
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            entries.append((p.device, group, p, g, st))
    if entries:
        with torch.no_grad():
            torch._foreach_add_([e[4]["step"] for e in entries], _ONE, alpha=1.0)
        scalars = {}
        by_device = {}
        for dev, group, p, g, st in entries:
            lr, (beta1, beta2), eps = group["lr"], group["betas"], group["eps"]
            step = st["step"].item()
            key = (lr, beta1, beta2, eps, step)
            s = scalars.get(key)
            if s is None:                  # _multi_tensor_adam's non-capturable branch, in double
                bias_correction1 = 1 - beta1 ** step
                bias_correction2 = 1 - beta2 ** step
                s = scalars[key] = (1 - beta1, beta2, 1 - beta2, eps, (lr / bias_correction1) * -1,
                                    bias_correction2 ** 0.5)
            m, v = st["exp_avg"], st["exp_avg_sq"]
            by_device.setdefault(dev, []).append((p, g, m, v, s))
        L = _lib.lib()
        for dev, rows in by_device.items():
            flat, touched = [], []
            for p, g, m, v, s in rows:
                flat += (p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel())
                flat += s
                touched += (p, m, v)
            table = struct.pack("<" + _ENTRY * len(rows), *flat)
            with torch.cuda.device(dev):
                _lib.check(L.lrf_adam_step(table, len(rows), _stream(dev)))
            torch._C._increment_version(touched)     # as the in-place foreach ops do
    for opt in rest:
        opt.step()


def zero_grad(optimizers):
    """Does what `for o in optimizers: o.zero_grad()` does (set_to_none=True) in one pass over the parameters;
    an optimiser that adam_step would hand to its own step() calls its own zero_grad()."""
    for opt in optimizers:
        if _plain(opt):
            for group in opt.param_groups:
                for p in group["params"]:
                    if p.grad is not None:
                        p.grad = None
        else:
            opt.zero_grad()
