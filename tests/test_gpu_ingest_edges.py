"""GPU: lrf_ingest_frame called directly through the C ABI, bit for bit against tests/ingest_oracle.py (which
tests/test_ingest_cpu.py holds to cv2 and numpy), at what files decoded by cv2.imread never look like: rows further
apart than their width in buffers that do not start at their allocation, every shape of the variance's summation tree
from one pixel to 3840 x 2160, constant and checkerboard frames, sparse masks, inverse depth and flows at the ratios
and values where a weight, a rounding tie or the mask threshold decides the result -- with canaries around everything
the call must not write.  Then the branches of DeviceFrameDataset's file reading that no other test reaches."""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import ingest_oracle as io
from test_ingest_cpu import ENLARGEMENTS, extreme_planes, flow_planes

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

CANARY = 0x7FC5A5A5                  # a NaN no kernel here produces
WIDTHS = {"rgbs": 3, "loss_weights": 1, "invdepths": 1, "fwd_flow": 2, "fwd_mask": 1, "bwd_flow": 2, "bwd_mask": 1}
FIELDS = {"rgbs": "rgb", "loss_weights": "loss_weight", "invdepths": "invdepth", "fwd_flow": "fwd_flow",
          "fwd_mask": "fwd_mask", "bwd_flow": "bwd_flow", "bwd_mask": "bwd_mask"}
PYTHON_VAR_MAX = 110_000             # above this many pixels the expected variance is numpy's own .var()


def place(a, sentinel):
    """numpy plane [h][w](c) -> (its device copy inside a larger buffer filled with `sentinel`, that buffer, the row
    stride in elements): 2 rows above, 1 below, 3 elements left and 4 right of the plane."""
    h, row = a.shape[0], int(np.prod(a.shape[1:]))
    dtype = torch.uint8 if a.dtype == np.uint8 else torch.int16
    big = torch.full((h + 3, row + 7), sentinel, dtype=dtype, device="cuda")
    view = big[2:h + 2, 3:row + 3]
    view.copy_(torch.from_numpy(np.ascontiguousarray(a).reshape(h, row).view(np.uint8 if a.dtype == np.uint8
                                                                             else np.int16)))
    return view, big, row + 7


class Ring:
    """A frame store of `capacity` slots filled with CANARY, and lrf_ingest_frame into one of them."""

    def __init__(self, w, h, capacity=1, depth=False, flow=False):
        self.w, self.h, self.n_px, self.capacity = w, h, w * h, capacity
        self.keys = ["rgbs", "loss_weights"] + (["invdepths"] if depth else []) + \
            (["fwd_flow", "fwd_mask", "bwd_flow", "bwd_mask"] if flow else [])
        self.store = {k: torch.full((capacity, self.n_px, WIDTHS[k]), CANARY, dtype=torch.int32, device="cuda")
                      for k in self.keys}
        self.slot_frame = torch.full((capacity,), -1, dtype=torch.int64, device="cuda")
        self.filled = set()                              # slots a call has written
        self.cstore = _lib().LrfFrameStore()
        self.cstore.n_px, self.cstore.capacity, self.cstore.slot_frame = self.n_px, capacity, self.slot_frame.data_ptr()
        for k in self.keys:
            setattr(self.cstore, FIELDS[k], self.store[k].data_ptr())

    def scratch(self):
        """Scratch of exactly the size the library asks for, with 64 canary bytes after it."""
        need = _lib().lib().lrf_ingest_scratch_bytes(self.n_px)
        assert need >= 16 + 5 * self.n_px and need % 8 == 0
        return torch.full((need + 64,), 0xC3, dtype=torch.uint8, device="cuda"), need

    def ingest(self, slot, bgr, depth=None, fwd=None, bwd=None, mask=None, scratch=None, stream=None):
        """-> {key: uint32 bits [n_px, width]} of `slot` after the call; asserts that the other slots, the source
        buffers (padding included) and the bytes after the scratch are bit-unchanged."""
        L = _lib()
        fr = L.LrfIngestFrame()
        fr.slot, fr.w, fr.h = slot, self.w, self.h
        sources = {}
        v, big, stride = place(bgr, 0x5A)
        sources["image"] = (big, big.clone())
        fr.image, fr.h0, fr.w0, fr.image_stride = v.data_ptr(), bgr.shape[0], bgr.shape[1], stride
        if depth is not None:
            v, big, stride = place(depth, 0x7A7A)
            sources["invdepth"] = (big, big.clone())
            fr.invdepth, fr.hd, fr.wd, fr.invdepth_stride = v.data_ptr(), depth.shape[0], depth.shape[1], stride
        if fwd is not None:
            assert fwd.shape == bwd.shape
            # one stride serves both flows: the backward plane sits in a buffer of the same geometry
            v, big, stride = place(fwd, 0x7A7A)
            sources["fwd_flow"] = (big, big.clone())
            vb, bigb, _ = place(bwd, 0x1B1B)
            sources["bwd_flow"] = (bigb, bigb.clone())
            fr.fwd_flow, fr.bwd_flow = v.data_ptr(), vb.data_ptr()
            fr.hf, fr.wf, fr.flow_stride = fwd.shape[0], fwd.shape[1], stride
            fr.flow_scale = float(np.float32(self.h / fwd.shape[0]))
        if mask is not None:
            v, big, stride = place(mask, 0xFF)           # a kernel that ignored the stride would read "on"
            sources["mask"] = (big, big.clone())
            fr.mask, fr.hm, fr.wm, fr.mask_stride = v.data_ptr(), mask.shape[0], mask.shape[1], stride
        s, need = scratch if scratch is not None else self.scratch()
        handle = None
        if stream is not None:
            stream.wait_stream(torch.cuda.current_stream())          # the uploads above
            handle = C.c_void_p(stream.cuda_stream)
        L.check(L.lib().lrf_ingest_frame(C.byref(self.cstore), C.byref(fr), C.c_void_p(s.data_ptr()), need, handle))
        torch.cuda.synchronize()
        for name, (big, before) in sources.items():
            assert torch.equal(big, before), f"the {name} buffer was written"
        assert bool((s[need:] == 0xC3).all()), "bytes after the scratch were written"
        out = {}
        for k in self.keys:
            t = self.store[k]
            for other in range(self.capacity):
                if other != slot and other not in self.filled:
                    assert bool((t[other] == CANARY).all()), f"slot {other} of {k} was written"
            out[k] = t[slot].cpu().numpy().view(np.uint32)
        self.filled.add(slot)
        return out


def _lib():
    from localrf_b200 import _lib
    return _lib


def assert_frame(got, want, what=""):
    assert sorted(got) == sorted(want), (sorted(got), sorted(want))
    for key, a in want.items():
        a = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
        g = got[key]
        assert g.shape == a.shape, (what, key, g.shape, a.shape)
        bad = np.flatnonzero((g != a).reshape(-1))
        assert bad.size == 0, (f"{what} {key}: {bad.size} of {a.size} values differ, first at {bad[0]}: got "
                               f"{g.reshape(-1)[bad[0]:bad[0] + 1].view(np.float32)[0]!r}, want "
                               f"{a.reshape(-1)[bad[0]:bad[0] + 1].view(np.float32)[0]!r}")


def expected(bgr, k=1, depth=None, fwd=None, bwd=None, mask=None):
    n = (bgr.shape[0] // k) * (bgr.shape[1] // k)
    return io.frame(bgr, k, depth, fwd, bwd, mask, numpy_var=n > PYTHON_VAR_MAX)


def random_image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


# ---- 1. the summation tree: every shape of numpy's recursion ----------------------------------------------------

def tree_shapes():
    """n x 1, 1 x n and a 2-D factorisation of the sizes around the recursion's edges: below 8 values (no
    accumulators), one leaf, a leaf with a tail, two leaves, trees whose leaves end at different depths (257, 8193),
    and a prime well above a leaf."""
    two_d = {8: (4, 2), 9: (3, 3), 128: (16, 8), 129: (43, 3), 136: (17, 8), 143: (13, 11), 144: (12, 12),
             1000: (40, 25), 8192: (128, 64), 8193: (2731, 3)}
    out = []
    for n in (1, 2, 7, 8, 9, 127, 128, 129, 136, 143, 144, 257, 1000, 8191, 8192, 8193, 100003):
        out += [(n, 1), (1, n)] if n > 1 else [(1, 1)]
        if n in two_d:
            out.append(two_d[n])
    return out


@pytest.mark.parametrize("w,h", tree_shapes())
def test_tree_shapes(w, h):
    bgr = random_image(h, w, w * 7 + h)
    got = Ring(w, h).ingest(0, bgr)
    assert_frame(got, expected(bgr), f"{w}x{h}")


@pytest.mark.parametrize("w,h,depth", [(1920, 1080, 14), (3840, 2160, 16)])
def test_large_frames(w, h, depth):
    """Trees of 14 and 16 levels, the deepest the library builds (64 slots per thread in the tree's serial part), with
    a strided mask."""
    assert io.tree_depth(w * h) == depth
    rng = np.random.default_rng(depth)
    bgr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask = (rng.integers(0, 4, (h, w)) == 0).astype(np.uint8) * 254
    got = Ring(w, h).ingest(0, bgr, mask=mask)
    assert_frame(got, expected(bgr, mask=mask), f"{w}x{h}")


# ---- 2. values of the loss weight --------------------------------------------------------------------------------

def pattern(name, h, w):
    """uint8 BGR [h][w][3]."""
    y, x = np.mgrid[:h, :w]
    if name.startswith("const"):
        g = np.full((h, w), int(name[5:]))
    elif name == "checker1":
        g = ((x + y) % 2) * 255
    elif name == "checker2":
        g = ((x // 2 + y // 2) % 2) * 255
    elif name == "corner":
        g = np.zeros((h, w), np.int64)
        g[-1, -1] = 255
    elif name == "ramp":
        g = (x * 255) // max(w - 1, 1)
    a = np.repeat(g[..., None], 3, -1).astype(np.uint8)
    if name == "ramp":
        a[..., 1] = 255 - a[..., 1]                      # the channels differ, so the grey weights matter
    return a


# (w, h, k): one leaf, a tree whose leaves end at different depths (43 * 6 = 258 -> 128 | 130 -> 128 | 64 | 66), and
# the training size; every reduction appears
WEIGHT_SIZES = [(16, 7, 1), (16, 7, 4), (43, 6, 1), (43, 6, 2), (960, 540, 1), (480, 270, 2), (240, 135, 4)]


@pytest.mark.parametrize("name", ["const0", "const255", "const77", "checker1", "checker2", "corner", "ramp"])
@pytest.mark.parametrize("w,h,k", WEIGHT_SIZES)
def test_loss_weight_values(w, h, k, name):
    bgr = pattern(name, k * h, k * w)
    want = expected(bgr, k)
    if name.startswith("const"):
        assert want["loss_weights"].view(np.uint32).max() == 0          # +0.0, not -0.0
    got = Ring(w, h).ingest(0, bgr)
    assert_frame(got, want, f"{name} {w}x{h} k={k}")


@pytest.mark.parametrize("kind", ["off", "on", "sparse"])
@pytest.mark.parametrize("w,h,k", WEIGHT_SIZES)
def test_masks(w, h, k, kind):
    """weight = variance * (mask > 0), for the checkerboard's large variance and a random frame's: all off (+0.0
    everywhere), all on, and the values 0, 1 and 254 mixed."""
    rng = np.random.default_rng(w + h + k)
    mask = {"off": np.zeros((h, w), np.uint8), "on": np.full((h, w), 255, np.uint8),
            "sparse": rng.choice(np.array([0, 1, 254], np.uint8), (h, w))}[kind]
    for bgr in (pattern("checker1", k * h, k * w), random_image(k * h, k * w, w)):
        want = expected(bgr, k, mask=mask)
        if kind == "off":
            assert want["loss_weights"].view(np.uint32).max() == 0
        assert_frame(Ring(w, h).ingest(0, bgr, mask=mask), want, f"{kind} {w}x{h} k={k}")


# ---- 3. inverse depth ratios -------------------------------------------------------------------------------------

@pytest.mark.parametrize("hs,ws,h,w", ENLARGEMENTS + [(30, 40, 30, 40), (60, 80, 30, 40), (120, 160, 30, 40),
                                                      (24, 32, 6, 8)])
def test_invdepth_ratios(hs, ws, h, w):
    """Same size, reduced by 2 and by 4, and every enlargement of the CPU test, on random planes and on zeros next to
    65535 (where a weight of 1e-16 in place of 0 is a wrong pixel)."""
    ring = Ring(w, h, depth=True)
    bgr = random_image(h, w, hs)
    d = np.random.default_rng(hs + ws).integers(0, 65536, (hs, ws), dtype=np.uint16)
    d[0, 0] = 65535
    for name, d in dict(extreme_planes(hs, ws, hs + ws), random=d).items():
        assert_frame(ring.ingest(0, bgr, depth=d), expected(bgr, depth=d), f"{name} {ws}x{hs} -> {w}x{h}")


def test_exact_zero_weight_at_6_to_8():
    """Column 3 of 6 -> 8 takes source column 2 with the next column's weight exactly 0."""
    d = np.zeros((6, 6), np.uint16)
    d[:, 3] = 65535
    got = Ring(8, 8, depth=True).ingest(0, random_image(8, 8, 0), depth=d)["invdepths"].reshape(8, 8)
    assert got[:, 3].tolist() == [0] * 8, got[:, 3].view(np.float32)


# ---- 4. flows ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hs,ws,h,w", ENLARGEMENTS + [(135, 240, 270, 480), (20, 20, 20, 20)])
def test_flow_codes(hs, ws, h, w):
    """The planes of the CPU test (saturating codes, zeros next to 65535, codes whose blends are exact .5 ties and
    cross the mask's threshold), forward and backward different, flow_scale = float32(h / hs)."""
    ring = Ring(w, h, flow=True)
    bgr = random_image(h, w, ws)
    planes = flow_planes(hs, ws, hs * 100 + ws)
    other = flow_planes(hs, ws, hs * 100 + ws + 1)
    for name in planes:
        fwd, bwd = planes[name], other[name][::-1, ::-1].copy()
        assert_frame(ring.ingest(0, bgr, fwd=fwd, bwd=bwd), expected(bgr, fwd=fwd, bwd=bwd),
                     f"{name} {ws}x{hs} -> {w}x{h}")


# ---- 5. layout and isolation -------------------------------------------------------------------------------------

def full_frame(w, h, seed, k=1):
    rng = np.random.default_rng(seed)
    return dict(bgr=rng.integers(0, 256, (k * h, k * w, 3), dtype=np.uint8),
                depth=rng.integers(0, 65536, (2 * h, 2 * w), dtype=np.uint16),
                fwd=rng.integers(0, 65536, (h // 2, w // 2, 3), dtype=np.uint16),
                bwd=rng.integers(0, 65536, (h // 2, w // 2, 3), dtype=np.uint16),
                mask=rng.integers(0, 2, (h, w), dtype=np.uint8) * 255)


def test_middle_slot_and_neighbours():
    """Slot 1 of 3, then slot 2, then slot 0: each call writes its own slot only (ingest() checks the slots not yet
    filled, the sources and the scratch's end); afterwards all three hold their frames."""
    w, h = 46, 30
    ring = Ring(w, h, capacity=3, depth=True, flow=True)
    frames = {slot: full_frame(w, h, slot) for slot in (1, 2, 0)}
    for slot, f in frames.items():
        got = ring.ingest(slot, f["bgr"], f["depth"], f["fwd"], f["bwd"], f["mask"])
        assert_frame(got, expected(f["bgr"], 1, f["depth"], f["fwd"], f["bwd"], f["mask"]), f"slot {slot}")
    for slot, f in frames.items():
        want = expected(f["bgr"], 1, f["depth"], f["fwd"], f["bwd"], f["mask"])
        assert_frame({k: ring.store[k][slot].cpu().numpy().view(np.uint32) for k in ring.keys}, want,
                     f"slot {slot} afterwards")
    assert ring.slot_frame.tolist() == [-1, -1, -1]                 # the caller tags the slots


@pytest.mark.parametrize("depth,flow", [(False, False), (True, False), (False, True)])
def test_stores_without_groups(depth, flow):
    w, h = 46, 30
    f = full_frame(w, h, 5, k=2)
    args = dict(depth=f["depth"] if depth else None, fwd=f["fwd"] if flow else None, bwd=f["bwd"] if flow else None)
    got = Ring(w, h, capacity=2, depth=depth, flow=flow).ingest(1, f["bgr"], mask=f["mask"], **args)
    assert_frame(got, expected(f["bgr"], 2, mask=f["mask"], **args))


def test_scratch_reuse_repeat_and_stream():
    """One scratch for frame A, a different frame B of the same size, and a smaller frame C (whose tree is shallower:
    the flags of the earlier frames are stale): each equals what a fresh scratch gives.  The same call twice gives
    the same bits; a non-default stream gives them too."""
    w, h = 43, 6                                                     # leaves at different depths
    big = Ring(w, h, depth=True, flow=True)
    shared = big.scratch()
    small = Ring(16, 7, depth=True, flow=True)
    assert io.tree_depth(16 * 7) < io.tree_depth(w * h)
    a, b, c = full_frame(w, h, 1), full_frame(w, h, 2), full_frame(16, 7, 3)
    a["bgr"] = pattern("checker1", h, w)                             # A's sums dwarf B's
    for ring, f in ((big, a), (big, b), (small, c), (big, b)):
        want = expected(f["bgr"], 1, f["depth"], f["fwd"], f["bwd"], f["mask"])
        reused = ring.ingest(0, f["bgr"], f["depth"], f["fwd"], f["bwd"], f["mask"], scratch=shared)
        assert_frame(reused, want, "reused scratch")
        fresh = ring.ingest(0, f["bgr"], f["depth"], f["fwd"], f["bwd"], f["mask"])
        assert all(np.array_equal(reused[k], fresh[k]) for k in ring.keys)
    stream = torch.cuda.Stream()
    on_stream = big.ingest(0, b["bgr"], b["depth"], b["fwd"], b["bwd"], b["mask"], stream=stream)
    assert all(np.array_equal(on_stream[k], fresh[k]) for k in big.keys)


# ---- 6. through the classes: what files can also be --------------------------------------------------------------

def write_scene(d, names, w=12, h=10, depth_dtype=np.uint8, step=1, mask_of=None, flow_sizes=None, seed=0):
    """Writes images/, depth/, flow_ds/ and masks/ under d and returns, per kept frame (every `step`-th of names),
    the planes as cv2.imread will decode them: dict(bgr, depth, fwd, bwd, mask).  mask_of(i, name) -> (file name,
    array) or None; flow_sizes(i) -> ((hf, wf) forward, (hf, wf) backward)."""
    rng = np.random.default_rng(seed)
    for sub in ("images", "depth", "flow_ds", "masks"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    kept = names[::step]
    prefix = f"step{step}_" if step != 1 else ""
    fwd_of, planes = {}, []
    for i, name in enumerate(kept):
        base = os.path.splitext(name)[0]
        (fh, fw), (bh, bw) = flow_sizes(i) if flow_sizes else ((h // 2, w // 2), (h // 2, w // 2))
        p = dict(bgr=rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
                 depth=rng.integers(0, np.iinfo(depth_dtype).max + 1, (h, w)).astype(depth_dtype),
                 bwd=rng.integers(0, 65536, (bh, bw, 3), dtype=np.uint16), mask=None)
        fwd_of[base] = rng.integers(0, 65536, (fh, fw, 3), dtype=np.uint16)   # the flow INTO this frame: fwd_<base>
        assert cv2.imwrite(os.path.join(d, "images", name), p["bgr"])
        assert cv2.imwrite(os.path.join(d, "depth", base + ".png"), p["depth"])
        assert cv2.imwrite(os.path.join(d, "flow_ds", f"fwd_{prefix}{base}.png"), fwd_of[base])
        assert cv2.imwrite(os.path.join(d, "flow_ds", f"bwd_{prefix}{base}.png"), p["bwd"])
        m = mask_of(i, name) if mask_of else None
        if m is not None:
            assert cv2.imwrite(os.path.join(d, "masks", m[0]), m[1])
            p["mask"] = m[1] if m[1].ndim == 2 else m[1][..., 0]
        planes.append(p)
    for i, name in enumerate(names):                                 # the frames frame_step skips: decoys
        if name not in kept:
            assert cv2.imwrite(os.path.join(d, "images", name), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    for i, p in enumerate(planes):                                   # fwd_<next kept frame>, wrapping to the first
        p["fwd"] = fwd_of[os.path.splitext(kept[(i + 1) % len(kept)])[0]]
    return planes


def want_frame(p, load_depth=True, load_flow=True):
    depth = p["depth"].astype(np.uint16) if load_depth else None
    m = None if p["mask"] is None else (p["mask"] > 0).astype(np.uint8)
    return io.frame(p["bgr"], 1, depth, p["fwd"] if load_flow else None, p["bwd"] if load_flow else None, m)


def check_both_splits(d, planes, test_frames, **kw):
    """The train split through DeviceRaySampler's ring and the test split's stacked tensors against the oracle fed
    the planes written to the files."""
    from localrf_b200 import DeviceFrameDataset, DeviceRaySampler
    from test_gpu_ingest import slots
    n = len(planes)
    ds = DeviceFrameDataset(d, split="train", load_depth=True, load_flow=True, n_init_frames=n, **kw)
    assert ds.num_images == n and ds.test_mask.tolist() == [int(i in test_frames) for i in range(n)]
    sampler = DeviceRaySampler(ds, "cuda")
    random.seed(0), np.random.seed(0)
    sampler.sample(32, True, False)
    got = slots(sampler)
    assert sorted(got) == list(range(n))
    for f in range(n):
        assert_frame({k: a.view(np.uint32) for k, a in got[f].items()}, want_frame(planes[f]), f"train frame {f}")
    ts = DeviceFrameDataset(d, split="test", load_depth=True, load_flow=True, n_init_frames=n, **kw)
    assert ts.num_images == len(test_frames)
    for row, f in enumerate(test_frames):
        want = want_frame(planes[f])
        want.pop("loss_weights")
        got = {"rgbs": ts.all_rgbs[row], "invdepths": ts.all_invdepths[row], "fwd_flow": ts.all_fwd_flow[row],
               "fwd_mask": ts.all_fwd_mask[row], "bwd_flow": ts.all_bwd_flow[row], "bwd_mask": ts.all_bwd_mask[row]}
        got = {k: t.reshape(-1, WIDTHS[k]).cpu().numpy().view(np.uint32) for k, t in got.items()}
        assert_frame(got, want, f"test frame {f}")


def test_files_8bit_depth_colour_mask_names_and_subsequence(tmp_path):
    """8-bit depth PNGs, a 3-channel masks/all.png (its first channel counts), file names that are not numbers (the
    test split goes by position) and a subsequence of the directory."""
    names = [f"shot_{c}.png" for c in "abcdefgh"]
    rng = np.random.default_rng(1)
    colour = rng.choice(np.array([0, 3, 255], np.uint8), (10, 12, 3))
    colour[..., 1:] = 255 - colour[..., :1]                          # only channel 0 may decide
    planes = write_scene(str(tmp_path), names, depth_dtype=np.uint8,
                         mask_of=lambda i, name: ("all.png", colour) if i == 0 else None)
    for p in planes:
        p["mask"] = colour[..., 0]
    sub = planes[1:7]
    sub[-1] = dict(sub[-1], fwd=planes[0]["fwd"])                    # wraps to the subsequence's first: fwd_shot_b
    check_both_splits(str(tmp_path), sub, [0, 3], subsequence=[1, 7], test_frame_every=3)


def test_files_16bit_mask_and_frame_step(tmp_path):
    """frame_step = 2 keeps every second image and reads the fwd_step2_ / bwd_step2_ flows; a 16-bit per-frame mask
    whose low byte is 0 where it is on; flows smaller than the image by 41 / 13 on one axis."""
    names = [f"{i:05d}.png" for i in range(9)]
    m16 = (np.random.default_rng(2).integers(0, 3, (41, 12)) * 256).astype(np.uint16)
    planes = write_scene(str(tmp_path), names, w=12, h=41, depth_dtype=np.uint16, step=2,
                         flow_sizes=lambda i: ((13, 5), (13, 5)),
                         mask_of=lambda i, name: (name, m16) if i in (1, 3) else None)   # 00002.png and 00006.png
    assert len(planes) == 5 and planes[1]["mask"] is m16 and planes[0]["mask"] is None
    check_both_splits(str(tmp_path), planes, [0, 2, 4], frame_step=2, test_frame_every=4)


def test_files_refused_layouts(tmp_path):
    """A mask of another size and forward / backward flows of different sizes raise NotImplementedError naming the
    layout, before anything is launched, in both splits."""
    from localrf_b200 import DeviceFrameDataset, DeviceRaySampler
    names = [f"{i:05d}.png" for i in range(3)]
    a, b = str(tmp_path / "mask"), str(tmp_path / "flows")
    write_scene(a, names, mask_of=lambda i, name: ("all.png", np.full((5, 6), 255, np.uint8)))
    write_scene(b, names, flow_sizes=lambda i: ((5, 6), (10, 12)))
    for d, text in ((a, "the mask must be w x h"), (b, "forward and backward flows differ in size")):
        ds = DeviceFrameDataset(d, split="train", load_depth=True, load_flow=True, n_init_frames=3,
                                test_frame_every=0)
        with pytest.raises(NotImplementedError, match=text):
            DeviceRaySampler(ds, "cuda").sample(32, True, False)
        with pytest.raises(NotImplementedError, match=text):
            DeviceFrameDataset(d, split="test", load_depth=True, load_flow=True, n_init_frames=3, test_frame_every=2)
