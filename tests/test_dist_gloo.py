"""CPU, world_size 2, gloo: the host-side sharding / all-gather logic of the multi-GPU path."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from localrf_b200.dist import gather_pixels, shard_bounds, shard_views


@pytest.mark.parametrize("n,world", [(4096, 1), (4096, 2), (4096, 8), (640000, 8), (1000, 3), (7, 4), (0, 2)])
def test_shard_bounds_partition(n, world):
    bounds = [shard_bounds(n, r, world) for r in range(world)]
    assert bounds[0][0] == 0 and bounds[-1][1] == n
    for (lo, hi), (lo2, _) in zip(bounds, bounds[1:]):
        assert hi == lo2 and lo <= hi
    sizes = [hi - lo for lo, hi in bounds]
    assert max(sizes) - min(sizes) <= 8
    assert all(lo % 8 == 0 or lo == n for lo, _ in bounds)


def test_shard_views_whole_views():
    v = torch.arange(16)
    covered = []
    for r in range(4):
        v_lo, v_hi, lo, hi = shard_views(v, 4096, r, 4)
        assert (hi - lo) == (v_hi - v_lo) * 256
        covered += list(range(lo, hi))
    assert covered == list(range(4096))


def _fake_render(ids):
    """Stand-in for the kernel on CPU: a deterministic per-ray function of the ray id."""
    x = ids.to(torch.float32)
    return torch.stack([torch.sin(x), torch.cos(x), x / 1000.0], -1), torch.sqrt(x + 1.0)


def _worker(rank, world, port, n, q, n_views=1):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ids = torch.arange(n)
        bounds = None
        if n_views > 1:                              # whole views per rank: shards of any length, empty ones included
            bounds = [shard_views(torch.arange(n_views), n, r, world)[2:] for r in range(world)]
            lo, hi = bounds[rank]
        else:
            lo, hi = shard_bounds(n, rank, world)
        rgb, depth = _fake_render(ids[lo:hi])
        full_rgb, full_depth = gather_pixels(rgb, depth, n, bounds=bounds)
        ref_rgb, ref_depth = _fake_render(ids)
        ok = torch.equal(full_rgb, ref_rgb) and torch.equal(full_depth, ref_depth)
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def _run_gather(n, world, n_views):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, q, n_views)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    return sorted(results)


@pytest.mark.parametrize("n", [4096, 1001])
def test_gather_pixels_equals_single_process(n):
    assert _run_gather(n, 2, 1) == [(0, True), (1, True)]


@pytest.mark.parametrize("n,world,n_views", [(300, 2, 3), (4096, 3, 16), (74, 3, 2)])
def test_gather_pixels_whole_view_shards(n, world, n_views):
    """Whole-view shards of a multi-view batch (shard_views, the bounds handed to gather_pixels): 200 + 100 rays,
    6 + 5 + 5 views of 256, and 37 + 37 + 0 rays (a rank without a view)."""
    assert _run_gather(n, world, n_views) == [(r, True) for r in range(world)]


def test_shard_views_uneven_and_empty():
    """Views that do not divide evenly give the first ranks one view more; more ranks than views leave the last
    ones empty, at the end of the batch; a list of view ids shards like a tensor."""
    assert [shard_views(torch.arange(3), 300, r, 2) for r in range(2)] == [(0, 2, 0, 200), (2, 3, 200, 300)]
    assert [shard_views([4, 9], 74, r, 3) for r in range(3)] == [(0, 1, 0, 37), (1, 2, 37, 74), (2, 2, 74, 74)]


def _grad_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import bench
        from localrf_b200.dist import allreduce_gradients, trainable_parameters
        lt = bench.build_scene("cpu", 12)
        params = trainable_parameters(lt)
        names = {id(p): n for n, p in lt.named_parameters()}
        assert any("density_plane" in names[id(p)] for p in params) and any("r_c2w" in names[id(p)] for p in params)
        gen = torch.Generator().manual_seed(100 + rank)
        mine = []
        for i, p in enumerate(params):
            if i % 5 == 4 and rank == 1:
                p.grad = None                        # a parameter this rank got no gradient for
                mine.append(torch.zeros_like(p))
            else:
                g = torch.randn(p.shape, generator=gen)
                p.grad = g.clone().contiguous(memory_format=torch.channels_last) if p.dim() == 4 else g.clone()
                mine.append(g)
        n_calls = allreduce_gradients(lt, bucket_bytes=4096)
        # expected: mean over ranks of what each rank held
        ok = n_calls > 1
        for i, p in enumerate(params):
            parts = []
            for r in range(world):
                gr = torch.Generator().manual_seed(100 + r)
                for j, pj in enumerate(params):
                    g = torch.randn(pj.shape, generator=gr) if not (j % 5 == 4 and r == 1) else None
                    if j == i:
                        parts.append(torch.zeros_like(pj) if g is None else g)
                        break
            ok &= bool(torch.allclose(p.grad, sum(parts) / world, atol=1e-6))
            if p.dim() == 4:
                ok &= p.grad.is_contiguous(memory_format=torch.channels_last)
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_dp_gradient_allreduce_averages_in_place():
    world = 2
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_grad_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(0, True), (1, True)]
