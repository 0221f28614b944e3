"""GPU: localrf_b200.DeviceRaySampler and lrf_gather_rays against the unmodified reference's LocalRFDataset.sample
(golden blobs) and against its host restatement (tests/sample_oracle.py) at training size."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import sample_oracle as so

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ray_sample.npz")


class Frames:
    """Distinct, cheaply made frames: frame f of quantity `key` is pool[f % 7] + f, built when sliced."""

    def __init__(self, n_frames, n_px, w, seed):
        self.shape = (n_frames, n_px, w)
        self.pool = np.random.default_rng(seed).random((7, n_px, w), dtype=np.float32)

    def __getitem__(self, sl):
        return np.stack([self.pool[f % 7] + np.float32(f) for f in range(*sl.indices(self.shape[0]))])


def frame_dataset(n_frames, W, H, n_init, chunk, flow=True, depth=True, test_every=10):
    frames = {key: Frames(n_frames, W * H, w, i) for i, (_, key, w) in enumerate(so.QUANTITIES)}
    test_mask = np.array([1 if f % test_every == 0 else 0 for f in range(n_frames)])
    return so.FrameDataset(frames, test_mask, depth, flow, chunk, n_init)


def host(blob):
    return {k: (blob[k].cpu().numpy() if blob[k] is not None else None) for k in so.BLOB_ARRAYS}


def assert_blob_equal(got, want, what=""):
    """got: a DeviceRaySampler blob; want: a host blob (golden or oracle)."""
    assert bool(got["train_test_poses"]) == bool(want["train_test_poses"]), what
    assert np.array_equal(got["view_ids_host"], want["view_ids"]), what
    g = host(got)
    for k in so.BLOB_ARRAYS:
        if want[k] is None:
            assert g[k] is None, (what, k)
            continue
        assert g[k].dtype == want[k].dtype and g[k].shape == want[k].shape, (what, k, g[k].shape, want[k].shape)
        assert np.array_equal(g[k], want[k]), (what, k)


def paired(sampler, ds, *args):
    """The sampler's blob and the oracle's from the same RNG state; both must consume the RNG identically."""
    state = random.getstate(), np.random.get_state()
    got = sampler.sample(*args)
    after = random.getstate(), np.random.get_state()
    random.setstate(state[0])
    np.random.set_state(state[1])
    want = so.sample(ds, *args)
    assert random.getstate() == after[0]
    np_after = np.random.get_state()
    assert np.array_equal(np_after[1], after[1][1]) and np_after[2] == after[1][2]
    return got, want


@pytest.mark.parametrize("case", ["flow_depth", "rgb_only"])
def test_golden_replay(case):
    from localrf_b200 import DeviceRaySampler
    ds, ops, want = so.golden_case(np.load(GOLDEN), case)
    sampler = DeviceRaySampler(ds, "cuda")
    got = list(so.replay(ds, ops, sampler.sample))
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert_blob_equal(a, b, f"{case}[{i}]")
        assert a["view_ids"].dtype == torch.int64 and a["idx"].dtype == torch.int64 and a["idx"].is_cuda
        floats = [a[k] for k in ("rgbs", "loss_weights", "invdepths", "fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask")
                  if a[k] is not None]
        assert all(t.is_contiguous() and t.dtype == torch.float32 for t in floats)
        assert len({t.untyped_storage().data_ptr() for t in floats}) == 1     # one allocation


def test_training_size_with_growth():
    """800x800 frames, flow and depth on, 4096 rays x 16 views, 200 calls while the active span grows to 100
    frames, is cut back and grows again; the ring starts at the initial span and must grow."""
    from localrf_b200 import DeviceRaySampler
    ds = frame_dataset(112, 800, 800, n_init=10, chunk=20)
    sampler = DeviceRaySampler(ds, "cuda")
    cap0 = sampler.capacity
    random.seed(3)
    np.random.seed(3)
    max_span = 0
    for i in range(200):
        if i % 2 == 0 and ds.active_frames_bounds[1] < ds.num_images:
            ds.activate_frames(1)
        b0, b1 = ds.active_frames_bounds
        if b1 - b0 > 100:
            ds.deactivate_frames(b0 + 40)
        max_span = max(max_span, ds.active_frames_bounds[1] - ds.active_frames_bounds[0])
        got, want = paired(sampler, ds, 4096, i % 3 == 0, i % 4 != 1, 16)
        assert_blob_equal(got, want, str(i))
    assert max_span == 100
    assert sampler.capacity > cap0                                   # grew at least once
    assert max_span <= sampler.capacity < 2 * max_span               # growth policy: max(span, 2 * capacity)


def test_no_host_synchronisation():
    from localrf_b200 import DeviceRaySampler
    ds = frame_dataset(40, 64, 48, n_init=8, chunk=8)
    sampler = DeviceRaySampler(ds, "cuda")
    random.seed(0)
    np.random.seed(0)
    for _ in range(3):
        sampler.sample(4096, False, True)
    torch.cuda.synchronize()
    blobs = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        blobs.append(paired(sampler, ds, 4096, False, True))
        ds.activate_frames(1)                                        # one new frame to upload
        blobs.append(paired(sampler, ds, 4096, True, True))
        ds.activate_frames(8)                                        # past the capacity: the ring grows
        blobs.append(paired(sampler, ds, 4096, False, False))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for i, (got, want) in enumerate(blobs):
        assert_blob_equal(got, want, str(i))


def test_host_running_ahead():
    """32 calls enqueued behind ~50 ms of device sleep: a pinned ids or frame buffer reused while its copy is still
    in flight would corrupt an earlier blob."""
    from localrf_b200 import DeviceRaySampler
    ds = frame_dataset(60, 64, 48, n_init=12, chunk=4)
    sampler = DeviceRaySampler(ds, "cuda", capacity=64)
    random.seed(5)
    np.random.seed(5)
    sampler.sample(256, True, False)
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)
    blobs = []
    for i in range(32):
        if i % 4 == 3:
            ds.activate_frames(2)                                    # frame uploads in flight too
        if i == 20:
            ds.deactivate_frames(ds.active_frames_bounds[0] + 5)
        blobs.append(paired(sampler, ds, 1024, i % 2 == 0, True, 16))
    torch.cuda.synchronize()
    for i, (got, want) in enumerate(blobs):
        assert_blob_equal(got, want, str(i))


def test_bad_ids_give_nan_rows():
    """Through the C entry: a view whose slot holds another frame, and pixels outside the frame, give NaN for
    those rays only; every other ray is exact."""
    from localrf_b200 import _lib
    from localrf_b200.tensorf import _ptr, _stream
    dev = "cuda"
    n_px, cap, V, R = 100, 4, 4, 8
    g = torch.Generator().manual_seed(0)
    q = {k: torch.rand((cap, n_px, w) if w > 1 else (cap, n_px), generator=g).to(dev)
         for _, k, w in so.QUANTITIES}
    slot_frame = torch.tensor([8, 5, 6, 7], dtype=torch.int64, device=dev)   # frame 4's slot holds frame 8
    views = torch.tensor([5, 4, 7, 8], dtype=torch.int64)
    px = torch.randint(0, n_px, (V * R,), generator=g)
    px[3], px[17], px[30] = n_px, -1, n_px + 7                           # outside the frame
    ids = torch.cat([views, px]).to(dev)
    out = {k: torch.full((V * R, w) if w > 1 else (V * R,), 7.0, device=dev) for _, k, w in so.QUANTITIES}
    idx = torch.empty(V * R, dtype=torch.int64, device=dev)
    s = _lib.LrfFrameStore()
    s.n_px, s.capacity, s.slot_frame = n_px, cap, _ptr(slot_frame).value
    b = _lib.LrfRayGather()
    b.n_rays, b.n_views, b.ids, b.idx = V * R, V, _ptr(ids).value, _ptr(idx).value
    names = {"rgbs": "rgb", "loss_weights": "loss_weight", "invdepths": "invdepth"}
    for k in q:
        setattr(s, names.get(k, k), _ptr(q[k]).value)
        setattr(b, names.get(k, k), _ptr(out[k]).value)
    _lib.check(_lib.lib().lrf_gather_rays(C.byref(s), C.byref(b), _stream(torch.device(dev))))
    torch.cuda.synchronize()
    view_of_ray = views.repeat_interleave(R)
    assert torch.equal(idx.cpu(), view_of_ray * n_px + px)
    bad = (view_of_ray == 4) | (px < 0) | (px >= n_px)
    assert int(bad.sum()) == R + 3                                     # view 4's rays and the three pixels
    for k, t in out.items():
        t = t.cpu()
        assert torch.isnan(t[bad]).all(), k
        good = (~bad).nonzero()[:, 0]
        want = q[k].cpu()[view_of_ray[good] % cap, px[good]]
        assert torch.equal(t[good], want), k


def test_one_training_iteration():
    """The forward and the supervision losses of one iteration, fed once from the sampler and once from the
    oracle's blob uploaded by hand, with the same torch seed, are equal."""
    import bench
    import localrf_b200 as L
    W, H = bench.IMG_W, bench.IMG_H
    lt = bench._scene(L.LocalTensorfs, "cpu", 64, n_init_frames=8).to("cuda")
    ds = frame_dataset(8, W, H, n_init=8, chunk=8, test_every=4)
    sampler = L.DeviceRaySampler(ds, "cuda")
    random.seed(1)
    np.random.seed(1)
    got, want = paired(sampler, ds, 4096, False, True, 16)
    dev = torch.device("cuda")
    up = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in want.items()}

    def iteration(blob, view_ids_host):
        torch.manual_seed(0)
        rgb, depth, dirs, ij = lt(blob["idx"], view_ids_host, W, H, is_train=True)
        cr = lt.center_rel
        losses = L.supervision_losses(
            rgb, blob["rgbs"], blob["loss_weights"], view_ids=blob["view_ids"], depth_map=depth, directions=dirs,
            ij=ij, cam2world=lt.get_cam2world(starting_id=0), starting_id=0, focal=lt.focal(W),
            center=torch.stack([cr[0] * W, cr[1] * H]), fwd_flow=blob["fwd_flow"], fwd_mask=blob["fwd_mask"],
            bwd_flow=blob["bwd_flow"], bwd_mask=blob["bwd_mask"], flow_weight=1.0 / ((W + H) / 2),
            invdepths=blob["invdepths"], depth_weight=0.1)
        return [t.detach() for t in (rgb, depth, dirs, ij) + tuple(losses)]

    a = iteration(got, got["view_ids_host"])
    b = iteration(up, want["view_ids"])
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i
    assert all(torch.isfinite(t).all() for t in a[4:])
