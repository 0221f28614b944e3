"""-m gpu: localrf_b200.adam_step (lrf_optim.cu) where a multi-tensor kernel goes wrong: tables of more tensors
than one launch takes, empty tensors among them, chunk boundaries, operands that are not 16-byte aligned, scalar
tails past the first chunk, and hyperparameters off the scene model's (lerp weights on both sides of ATen's 0.5
branch and exactly at it, eps 0, lr 0, a restored step of 1e6).

The oracle is test_gpu_optim's: deep copies of the same optimisers stepped one by one with `o.step()`, compared as
bit patterns, with no tolerance anywhere."""
import copy

import pytest
import torch

from localrf_b200 import optim
from test_gpu_optim import CountingLib, assert_same, params_of, set_grads, special_grad

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHUNK = 16384                       # ADAM_CHUNK: elements per work item
MAX_T = 448                         # ADAM_MAX_T: tensors per launch


@pytest.fixture
def counting(monkeypatch):
    from localrf_b200 import _lib
    c = CountingLib(_lib.lib())
    monkeypatch.setattr(_lib, "lib", lambda: c)
    return c


def step_both(opts, refs, grads):
    set_grads(opts, refs, grads)
    optim.adam_step(opts)
    for r in refs:
        r.step()


def test_launch_split(counting):
    """1000 parameters over six optimisers, numel from {0, 1, 2, 3, 5, 16383, 16384, 16385, 32771} and random
    sizes: each adam_step call is one lrf_adam_step call, which launches adam_kernel once per 448 non-empty
    tensors (the empty ones are skipped), and every bit matches torch's for 5 steps."""
    from torch.profiler import ProfilerActivity, profile
    gen = torch.Generator().manual_seed(0)
    fixed = [0, 1, 2, 3, 5, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 3]
    sizes = [fixed[i % len(fixed)] if i % 4 else int(torch.randint(1, 3000, (1,), generator=gen)) for i in range(1000)]
    ps = [torch.nn.Parameter(0.1 * torch.randn(n, generator=gen).to(DEV)) for n in sizes]
    cuts = [0, 100, 450, 451, 700, 990, 1000]
    opts = []
    for k, (a, b) in enumerate(zip(cuts, cuts[1:])):
        lr, betas = 10.0 ** -(1 + k % 3), ((0.9, 0.99), (0.8, 0.999))[k % 2]
        half = (a + b) // 2
        opts.append(torch.optim.Adam([{"params": ps[a:half]}, {"params": ps[half:b], "lr": 2 * lr}], lr=lr,
                                     betas=betas))
    refs = copy.deepcopy(opts)
    non_empty = sum(n > 0 for n in sizes)
    launches_per_step = -(-non_empty // MAX_T)
    assert launches_per_step == 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for step in range(5):
            step_both(opts, refs, [special_grad(p, gen, step) for p in ps])
            assert_same(opts, refs)
        torch.cuda.synchronize()
    assert counting.calls == 5
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert sum("adam_kernel" in n for n in names) == 5 * launches_per_step


def _views(n, offsets):
    """Views of n floats at the given float offsets into one shared buffer (each in its own 16-byte aligned
    stretch of it, so that the offset alone sets the view's alignment)."""
    stride = (n + 8 + 3) // 4 * 4
    buf = torch.empty(stride * len(offsets), device=DEV)
    return [buf[i * stride + off:i * stride + off + n] for i, off in enumerate(offsets)]


@pytest.mark.parametrize("layout", ["param_misaligned", "grad_misaligned", "aligned_tails"])
def test_alignment(layout, counting):
    """param_misaligned: nn.Parameter views at float offsets 1, 2 and 3 into one buffer (their gradients and state
    are aligned); grad_misaligned: aligned parameters whose gradients are same-stride views at offsets 1, 2, 3.
    Either sends every chunk of the tensor down the scalar loop.  aligned_tails: all four operands aligned, numel
    % 4 = 1, 2, 3 and numel > 16384, so the scalar tail after the 16-byte loop lies in the second chunk."""
    gen = torch.Generator().manual_seed(1)
    n = 2 * CHUNK + 1234
    if layout == "param_misaligned":
        ps = [torch.nn.Parameter(v.copy_(0.1 * torch.randn(n, generator=gen))) for v in _views(n, (1, 2, 3))]
        assert all(p.data_ptr() % 16 for p in ps) and all(optim._dense(p) for p in ps)
    elif layout == "grad_misaligned":
        ps = [torch.nn.Parameter(0.1 * torch.randn(n, generator=gen).to(DEV)) for _ in range(3)]
    else:
        ps = [torch.nn.Parameter(0.1 * torch.randn(CHUNK + 4 * k + r, generator=gen).to(DEV))
              for k, r in ((100, 1), (200, 2), (900, 3), (CHUNK // 4 + 7, 3))]
        assert all(p.data_ptr() % 16 == 0 for p in ps) and [p.numel() % 4 for p in ps] == [1, 2, 3, 3]
    opts = [torch.optim.Adam(ps[:2], lr=1e-2, betas=(0.9, 0.99)), torch.optim.Adam(ps[2:], lr=1e-3)]
    refs = copy.deepcopy(opts)
    for step in range(4):
        grads = [special_grad(p, gen, step) for p in ps]
        if layout == "grad_misaligned":
            grads = [v.copy_(g) for v, g in zip(_views(n, (1, 2, 3)), grads)]
            assert all(g.data_ptr() % 16 and g.stride() == p.stride() for g, p in zip(grads, ps))
        step_both(opts, refs, grads)
        assert_same(opts, refs)
    assert counting.calls == 4


HYPER = {
    "betas_0.3_0.999": dict(betas=(0.3, 0.999)),       # lerp weight 0.7: ATen's large-weight branch
    "betas_0.5_0.5": dict(betas=(0.5, 0.5)),           # weight exactly 0.5: the large-weight branch too
    "betas_0_0": dict(betas=(0.0, 0.0)),               # weight 1: exp_avg = grad, exp_avg_sq = grad^2
    "betas_0.99_0.9999": dict(betas=(0.99, 0.9999)),   # weight 0.01
    "eps_0": dict(eps=0.0),                            # 0 / 0 where a gradient is 0 from the start
    "eps_1e-30": dict(eps=1e-30),
    "lr_0": dict(lr=0.0),                              # step size -0.0
    "lr_10": dict(lr=10.0),
}


def hyper_params(gen):
    sizes = (1, 3, 5, 64, CHUNK + 1, 4 * 1000 + 2)
    return [torch.nn.Parameter(0.1 * torch.randn(n, generator=gen).to(DEV)) for n in sizes]


@pytest.mark.parametrize("name", list(HYPER))
def test_hyperparameters_20_steps(name, counting):
    """20 steps from step 0 with special_grad's zeros, denormals, +-1e-30 and +-1e20; the options under test on
    one optimiser, the scene model's on another in the same call."""
    gen = torch.Generator().manual_seed(2)
    ps = hyper_params(gen)
    opts = [torch.optim.Adam(ps[:4], **HYPER[name]), torch.optim.Adam(ps[4:], lr=1e-3, betas=(0.9, 0.99))]
    refs = copy.deepcopy(opts)
    for step in range(20):
        step_both(opts, refs, [special_grad(p, gen, step) for p in ps])
        assert_same(opts, refs)
    assert counting.calls == 20


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.5, 0.5)])
def test_restored_large_step(betas, counting):
    """A state restored through load_state_dict with step = 1e6: both bias corrections round to 1 in double."""
    gen = torch.Generator().manual_seed(3)
    ps = hyper_params(gen)
    seed = torch.optim.Adam(ps, lr=1e-3, betas=betas)
    for p in ps:
        p.grad = special_grad(p, gen, 0)
    seed.step()
    sd = copy.deepcopy(seed.state_dict())
    for st in sd["state"].values():
        st["step"] = torch.tensor(1e6)
    assert 1 - betas[0] ** 1e6 == 1.0 and 1 - betas[1] ** 1e6 == 1.0
    opts = [torch.optim.Adam(ps, lr=1e-3, betas=betas)]
    opts[0].load_state_dict(sd)
    refs = copy.deepcopy(opts)
    for step in range(3):
        step_both(opts, refs, [special_grad(p, gen, step) for p in ps])
        assert_same(opts, refs)
    assert opts[0].state[ps[0]]["step"].item() == 1e6 + 3
    assert counting.calls == 3
