"""Ray-batch data parallelism over the GPUs of one node (SURVEY.md §8e).

The render path has no cross-ray term, so the field is replicated on every rank, each rank renders
a contiguous shard of the batch's rays and ONE all-gather of the rendered [rays, 4] pixels
(rgb + depth) closes the step.  No collective touches the data path itself.  The reference has no
distributed code at all (its only multi-GPU mode is one scene per process, scripts/train_all.sh).

Two ways to close a step:

  * `PixelExchange` (the fused path): the gathered [rays, 4] buffer lives in symmetric memory
    (peer-mapped over NVLink / NVSwitch); the thread of the render kernel that finishes a ray stores
    its (r,g,b,depth) straight into every peer's copy -- one 16-byte store per peer, or one NVLS
    multimem store for all of them -- and `lrf_peer_barrier` (a one-CTA kernel over peer-mapped
    flags) closes the step.  The all-gather IS the kernel's epilogue; no collective is launched.
  * `gather_pixels`: one NCCL all-gather (fallback when peer access is unavailable; gloo in the CPU
    tests of this host logic).
"""
import ctypes as C

import torch
import torch.distributed as dist


def shard_bounds(n_rays, rank, world, align=8):
    """Contiguous shard [lo, hi) of rank `rank`; boundaries aligned to `align` rays (the kernel's
    ray-tile size) so that every rank's launch covers whole tiles; the union is exactly
    [0, n_rays) and shards differ by at most one aligned block."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    blocks = (n_rays + align - 1) // align
    base, extra = divmod(blocks, world)
    lo_b = rank * base + min(rank, extra)
    hi_b = lo_b + base + (1 if rank < extra else 0)
    return min(lo_b * align, n_rays), min(hi_b * align, n_rays)


def shard_views(view_ids, n_rays, rank, world):
    """Shard of a training-style batch (rays grouped by view): whole views per rank, so the
    kernel's view indexing (ray // rays_per_view) stays valid inside the shard.  -> (v_lo, v_hi, lo, hi)"""
    n_views = len(view_ids)
    per_view = n_rays // n_views
    v_lo, v_hi = shard_bounds(n_views, rank, world, align=1)
    return v_lo, v_hi, v_lo * per_view, v_hi * per_view


def gather_pixels(rgb, depth, n_total, group=None, bounds=None):
    """One all-gather of the rendered pixels: local [n_local,3] + [n_local] -> [n_total,3], [n_total].

    `bounds` = every rank's shard [lo, hi), in rank order, contiguous over [0, n_total) (default: shard_bounds).
    Shards may differ in length, so every rank pads to the largest shard."""
    world = dist.get_world_size(group)
    if world == 1:
        return rgb, depth
    rank = dist.get_rank(group)
    if bounds is None:
        bounds = [shard_bounds(n_total, r, world) for r in range(world)]
    width = max(hi - lo for lo, hi in bounds)
    pix = torch.zeros(width, 4, dtype=rgb.dtype, device=rgb.device)
    n_local = bounds[rank][1] - bounds[rank][0]
    pix[:n_local, :3] = rgb
    pix[:n_local, 3] = depth
    out = torch.empty(world * width, 4, dtype=rgb.dtype, device=rgb.device)
    dist.all_gather_into_tensor(out, pix, group=group)
    out = out.view(world, width, 4)
    parts = [out[r, : hi - lo] for r, (lo, hi) in enumerate(bounds)]
    full = torch.cat(parts, dim=0)
    return full[:, :3].contiguous(), full[:, 3].contiguous()


class ExchangeSchedule:
    """The step bookkeeping of the fused pixel exchange, free of any device state (PixelExchange owns one;
    tests/test_dist_gloo.py drives N of them through randomly interleaved simulated ranks to check the
    protocol's two claims: a gathered image is complete when it is read, and no buffer is overwritten before
    every rank has read it -- for any N, any lag, any relative speed of the ranks).

    Steps are numbered from 1.  `seq` = steps this rank has launched."""

    def __init__(self, lag=0):
        self.lag = int(lag)
        if self.lag < 0:
            raise ValueError("lag must be >= 0")
        self.n_buf = 2 if self.lag == 0 else 2 * self.lag + 4
        self.seq = 0

    def next_step(self):
        """-> (buffer index the NEXT step's pixels go to, the step number its last CTA publishes, the step of
        the peers its prologue waits for (0 = no wait: lag 0 closes the step with a separate wait kernel))"""
        step = self.seq + 1
        wait = max(self.seq - self.lag, 0) if self.lag >= 1 else 0
        return step % self.n_buf, step, wait

    def advance(self):
        self.seq += 1

    def gathered_step(self):
        """The step whose complete image is readable now (after the launch of step `seq`, in stream order)."""
        return self.seq if self.lag == 0 else max(self.seq - 1 - self.lag, 0)

    def gathered_buffer(self):
        return self.gathered_step() % self.n_buf


class PixelExchange:
    """Gathered pixel buffer in symmetric memory + the step barrier (fused pixel exchange).

    `lag` = steps of slack between a rank and its slowest peer.
    lag 0 (render_sharded): the kernel publishes step i, a small wait kernel closes it when every peer has
    published step i -- every rank returns the complete image of the same step; 2 buffers alternate.
    lag L >= 1 (a renderer's steady state, no extra launch at all): the render kernel of step s first waits
    until every peer has published step s-1-L (so a rank never stalls on a peer that is less than L steps
    behind: with different batches per rank the step time is the MEAN over the ranks' batches, not the
    per-step maximum), then stores its pixels, and its last CTA publishes step s.  After the launch of
    step s, `gathered()` is the complete image of step s-1-L.  2L+4 buffers rotate.  Safety: step s is
    stored into the buffer step u = s-2L-4 used; a peer reads step u between its launches u+1+L and u+2+L
    and publishes flag u+2+L after that read (stream order); before launching step s this rank has seen
    every peer's flag s-1-L >= u+2+L  (needs 2L+3 buffers; one more keeps the count even).
    """
    FLAG_BYTES = 16 * 8

    def __init__(self, max_rays, group=None, device=None, use_multicast=True, lag=0):
        import torch.distributed._symmetric_memory as symm_mem
        from . import _lib
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if self.world > 16:
            raise ValueError("PixelExchange covers the GPUs of one node (<= 16 peers)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.max_rays = int(max_rays)
        self.buf_bytes = (self.max_rays * 16 + 255) // 256 * 256
        self.sched = ExchangeSchedule(lag)
        self.lag, self.n_buf = self.sched.lag, self.sched.n_buf
        total = self.n_buf * self.buf_bytes + self.FLAG_BYTES
        self.mem = symm_mem.empty(total, dtype=torch.uint8, device=self.device)
        self.mem.zero_()
        torch.cuda.synchronize(self.device)
        self.handle = symm_mem.rendezvous(self.mem, self.group)
        self.ptrs = [int(p) for p in self.handle.buffer_ptrs]
        mc = 0
        if use_multicast:
            try:
                mc = int(self.handle.multicast_ptr) if self.handle.has_multicast_support(
                    self.device.type, self.device.index) else 0
            except Exception:
                mc = 0
        self.mc_ptr = mc
        self._flag_ptrs = (C.c_void_p * self.world)(*[p + self.n_buf * self.buf_bytes for p in self.ptrs])
        self._lib = _lib
        dist.barrier(self.group)          # every rank has zeroed + mapped before anybody stores

    def fill_outputs(self, o, ray_lo):
        """Points an LrfOutputs at the NEXT step's buffer: peer p receives this rank's rays at row
        `ray_lo` of its gathered buffer."""
        buf, signal_seq, wait_seq = self.sched.next_step()
        off = buf * self.buf_bytes + ray_lo * 16
        o.n_peers = self.world
        for p in range(self.world):
            o.peer_pix[p] = self.ptrs[p] + off
            o.peer_flags[p] = self.ptrs[p] + self.n_buf * self.buf_bytes
        o.mc_pix = (self.mc_ptr + off) if self.mc_ptr else None
        # the kernel itself publishes the step (its last CTA release-stores the flags after all pixel
        # stores) and, when the consumer lags, first waits for the peers to be done with this buffer
        o.rank = self.rank
        o.signal_seq = signal_seq
        o.wait_seq = wait_seq

    def close_step(self, stream):
        """Closes the step the render kernel has just published.  lag 0: enqueues the wait for every peer's
        flag of THIS step (one small kernel); lag >= 1: nothing to enqueue.  `gathered(n)` then refers to
        step (this - 0) resp. (this - 1 - lag), which is complete at that point of the stream."""
        self.sched.advance()
        if self.lag == 0:
            self._lib.check(self._lib.lib().lrf_peer_signal_wait(self._flag_ptrs, self.rank, self.world, self.seq,
                                                                 self.seq, stream))

    def skip_step(self, stream):
        """A rank whose shard of this step is empty renders nothing but still publishes the step."""
        self.sched.advance()
        self._lib.check(self._lib.lib().lrf_peer_signal_wait(self._flag_ptrs, self.rank, self.world, self.seq,
                                                             self.seq if self.lag == 0 else 0, stream))

    @property
    def seq(self):
        return self.sched.seq

    def gathered_step(self):
        """The step whose complete image `gathered()` returns now."""
        return self.sched.gathered_step()

    def gathered(self, n_rays):
        off = self.sched.gathered_buffer() * self.buf_bytes
        return self.mem[off:off + n_rays * 16].view(torch.float32).view(n_rays, 4)


def render_sharded(local_tensorfs, ray_ids, view_ids, W, H, group=None, exchange=None, **kw):
    """LocalTensorfs.forward with the rays of an eval batch sharded over the ranks; every rank returns the
    full (rgb, depth).  A single-view batch is sharded by `shard_bounds`, a multi-view one (rays grouped by
    view) by whole views (`shard_views`), since the kernel takes a ray's view from its position in the
    launch.  With a `PixelExchange` the pixels are exchanged by the render kernel itself (returned tensors
    are views of the exchange buffer, valid until the step after next); without one, by one NCCL all-gather."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n = ray_ids.shape[0]
    if len(view_ids) > 1:
        parts = [shard_views(view_ids, n, r, world) for r in range(world)]
        bounds = [(lo, hi) for _, _, lo, hi in parts]
        v_lo, v_hi = parts[rank][:2]
        views = view_ids[v_lo:v_hi]
    else:
        bounds = [shard_bounds(n, r, world) for r in range(world)]
        views = view_ids
    lo, hi = bounds[rank]
    if exchange is None:
        rgb, depth, _, _ = local_tensorfs(ray_ids[lo:hi], views, W, H, **kw)
        return gather_pixels(rgb, depth, n, group, bounds)
    if n > exchange.max_rays:
        raise ValueError(f"batch of {n} rays exceeds the exchange buffer ({exchange.max_rays})")
    local_tensorfs(ray_ids[lo:hi], views, W, H, exchange=(exchange, lo), **kw)   # (an empty shard only signals)
    full = exchange.gathered(n)
    return full[:, :3], full[:, 3]


# ---- data-parallel training (SURVEY.md 8f rank 1: "+ DP gradient all-reduce") ---------------------------
def trainable_parameters(local_tensorfs):
    """The tensors one optimisation step updates (local_tensorfs.py:193-290): the newest field's
    parameters (rf_optimizer), the poses / exposures still linked to it, the intrinsics."""
    lt = local_tensorfs
    params = [p for g in lt.rf_optimizer.param_groups for p in g["params"]]
    for i in lt._live_pose_ids():
        params += [lt.r_c2w[i], lt.t_c2w[i], lt.exposure[i]]
    params += [lt.focal_offset, lt.center_rel]
    return [p for p in params if p.requires_grad]


def allreduce_gradients(local_tensorfs, group=None, bucket_bytes=64 << 20):
    """Averages the gradients of one training step over the ranks (each rank rendered its own shard of
    the ray batch): flat buckets of <= bucket_bytes, one all-reduce each (NCCL over NVLink / NVSwitch;
    NVLS reduces inside the switch when available).  A parameter without a gradient on this rank
    contributes zeros (every rank must issue the same collectives).  Call between loss.backward() and
    the optimiser steps; LocalTensorfs.optimizer_step does so when `dp_group` is set."""
    world = dist.get_world_size(group)
    if world == 1:
        return 0
    views = []
    for p in trainable_parameters(local_tensorfs):
        if p.grad is None:
            p.grad = torch.zeros_like(p)              # preserves the parameter's memory format
        g = p.grad
        # a dense view of the gradient in its OWN memory order (no NCHW round trip for channel-last grids)
        v = g.permute(0, 2, 3, 1) if (g.dim() == 4 and not g.is_contiguous()
                                      and g.is_contiguous(memory_format=torch.channels_last)) else g
        if not v.is_contiguous():
            p.grad = g = g.contiguous()
            v = g
        views.append(v)
    n_calls, lo = 0, 0
    while lo < len(views):
        hi, size = lo, 0
        while hi < len(views) and (hi == lo or size + views[hi].numel() * 4 <= bucket_bytes):
            size += views[hi].numel() * views[hi].element_size()
            hi += 1
        flat = torch.cat([v.reshape(-1) for v in views[lo:hi]])
        dist.all_reduce(flat, group=group)
        flat.div_(world)
        off = 0
        for v in views[lo:hi]:
            v.copy_(flat[off:off + v.numel()].view(v.shape))      # writes through the view into p.grad
            off += v.numel()
        n_calls += 1
        lo = hi
    return n_calls
