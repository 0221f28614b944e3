"""GPU: localrf_b200.DeviceFrameDataset and lrf_ingest_frame against the arrays the unmodified reference's
LocalRFDataset.read_meta built from the same files (tests/golden/ingest.npz), against the numpy restatement
(tests/ingest_oracle.py) at training size, and the sampler's blobs against the reference's sampling over those
arrays."""
import json
import os
import random

import numpy as np
import pytest
import torch

import ingest_oracle as io
import sample_oracle as so

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ingest.npz")


def golden():
    z = np.load(GOLDEN)
    return z, [(str(c), str(s)) for c, s in zip(z["cases"], z["scenes"])]


def dataset(z, case, scene, d):
    from localrf_b200 import DeviceFrameDataset
    cfg = json.loads(str(z[f"{case}.config"]))
    io.write_golden_scene(z, scene, d)
    ds = DeviceFrameDataset(d, split="train", downsampling=cfg["downsampling"], load_depth=cfg["load_depth"],
                            load_flow=cfg["load_flow"], frames_chunk=cfg["frames_chunk"],
                            n_init_frames=cfg["n_init_frames"], test_frame_every=cfg["test_frame_every"])
    return ds, cfg


def slots(sampler):
    """frame -> {key: host array [n_px, w]} of every resident frame."""
    torch.cuda.synchronize()
    out = {}
    for f in range(*sampler.resident):
        out[f] = {key: sampler.store[key][f % sampler.capacity].cpu().numpy().reshape(sampler.n_px, w)
                  for _, key, w in sampler.quantities}
    return out


def ingest_all(z, case, scene, d):
    from localrf_b200 import DeviceRaySampler
    ds, _ = dataset(z, case, scene, d)
    sampler = DeviceRaySampler(ds, "cuda", capacity=ds.num_images)
    random.seed(0)
    np.random.seed(0)
    while True:
        sampler.sample(64, True, False)
        if not ds.has_left_frames():
            break
        ds.activate_frames(2)
    return ds, sampler


def test_slots_equal_the_reference(tmp_path):
    z, cases = golden()
    for case, scene in cases:
        ds, sampler = ingest_all(z, case, scene, str(tmp_path / case))
        cfg = json.loads(str(z[f"{case}.config"]))
        assert ds.img_wh == cfg["img_wh"] and not ds._raw            # every frame handed over, none kept
        got = slots(sampler)
        assert sorted(got) == list(range(ds.num_images))
        for f, arrays in got.items():
            for key, a in arrays.items():
                want = z[f"{case}.frames.{key}"][f]
                assert a.dtype == want.dtype and np.array_equal(a.view(np.uint32), want.view(np.uint32)), \
                    (case, f, key)


def test_blobs_and_rng_equal_the_reference(tmp_path):
    """One activate / deactivate / sample script against the reference's arrays (sample_oracle's stand-in dataset
    holding the golden frames, sampled by DeviceRaySampler and by the numpy restatement) and against
    DeviceFrameDataset + DeviceRaySampler: same blobs, same RNG consumption."""
    from localrf_b200 import DeviceRaySampler
    from test_gpu_sample import assert_blob_equal
    z, cases = golden()
    ops = ([["seed", 3], ["sample", 64, False, True, 16], ["sample", 48, True, True, 8], ["activate", 2],
            ["sample", 64, True, False, 16], ["deactivate", 2], ["sample", 64, False, True, 16], ["activate", 3],
            ["sample", 32, True, True, 16], ["sample", 64, False, False, 16]])
    for case, scene in cases:
        cfg = json.loads(str(z[f"{case}.config"]))
        frames = {key: z[f"{case}.frames.{key}"] for _, key, _ in so.QUANTITIES if f"{case}.frames.{key}" in z}
        def stand_in():
            return so.FrameDataset(frames, z[f"{case}.test_mask"], cfg["load_depth"], cfg["load_flow"],
                                   cfg["frames_chunk"], cfg["n_init_frames"])
        runs = {}
        for name, ds in (("oracle", stand_in()), ("reference", stand_in()),
                         ("device", dataset(z, case, scene, str(tmp_path / case))[0])):
            sample = (lambda *a, _ds=ds: so.sample(_ds, *a)) if name == "oracle" else \
                DeviceRaySampler(ds, "cuda").sample
            blobs, states = [], []
            for b in so.replay(ds, ops, sample):
                blobs.append(b)
                states.append((random.getstate(), np.random.get_state()[1].copy(), np.random.get_state()[2]))
            runs[name] = (blobs, states)
        want_blobs, want_states = runs["oracle"]
        for name in ("reference", "device"):
            blobs, states = runs[name]
            assert len(blobs) == len(want_blobs) == 6
            for i, (b, w) in enumerate(zip(blobs, want_blobs)):
                w = dict(w, view_ids_host=w["view_ids"])
                assert_blob_equal(b, w, f"{case} {name} [{i}]")
            for s, w in zip(states, want_states):
                assert s[0] == w[0] and np.array_equal(s[1], w[1]) and s[2] == w[2]


@pytest.mark.parametrize("k,flow_div", [(1, 2), (2, 1), (4, 2)])
def test_training_size_against_the_restatement(tmp_path, k, flow_div):
    """960 x 540 frames (k = 1; 480 x 270 for k = 2 and 4): image (reduced by k), depth at the image size, flows at
    1 / flow_div of it, a motion mask on frame 1 only; every slot against tests/ingest_oracle.py, and twice."""
    import cv2
    from localrf_b200 import DeviceFrameDataset, DeviceRaySampler
    W, H = (960, 540) if k == 1 else (480, 270)
    rng = np.random.default_rng(k)
    d = str(tmp_path)
    for sub in ("images", "depth", "masks", "flow_ds"):
        os.makedirs(os.path.join(d, sub))
    raw = []
    for i in range(3):
        f = f"{i:05d}"
        img = rng.integers(0, 256, (k * H, k * W, 3), dtype=np.uint8)
        dep = rng.integers(0, 65536, (H, W), dtype=np.uint16)
        flows = [rng.integers(0, 65536, (H // flow_div, W // flow_div, 3), dtype=np.uint16) for _ in range(2)]
        cv2.imwrite(os.path.join(d, "images", f + ".png"), img)
        cv2.imwrite(os.path.join(d, "depth", f + ".png"), dep)
        cv2.imwrite(os.path.join(d, "flow_ds", f"fwd_{f}.png"), flows[0])
        cv2.imwrite(os.path.join(d, "flow_ds", f"bwd_{f}.png"), flows[1])
        m = None
        if i == 1:
            m = rng.integers(0, 2, (H, W), dtype=np.uint8) * 255
            cv2.imwrite(os.path.join(d, "masks", f + ".png"), m)
        raw.append((img, dep, flows, m))
    results = []
    for _ in range(2):
        ds = DeviceFrameDataset(d, downsampling=k if k > 1 else -1, load_depth=True, load_flow=True,
                                n_init_frames=3, test_frame_every=0)
        sampler = DeviceRaySampler(ds, "cuda")
        sampler.sample(64, True, False)
        results.append(slots(sampler))
    for f in range(3):
        img, dep, flows, m = raw[f]
        want = io.frame(img, k, dep, raw[(f + 1) % 3][2][0], flows[1], m)   # fwd_<next frame>, bwd_<frame>
        for key, a in results[0][f].items():
            assert np.array_equal(a.view(np.uint32), want[key].view(np.uint32)), (f, key)
            assert np.array_equal(a.view(np.uint32), results[1][f][key].view(np.uint32)), (f, key)
