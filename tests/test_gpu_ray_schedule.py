"""-m gpu: the render kernel's ray distribution.  Producer warps draw rays from a per-launch counter and
the grid is min(ceil(n / 8), SMs) CTAs; these batch sizes exercise its edges (a single ray, fewer rays
than one CTA's producers, one ray more or less than a whole 4096-ray batch, a whole frame in one
launch).  Every ray must be written exactly once and come out bit-identical to the same ray rendered
inside an ordinary 4096-ray batch: the outputs are prefilled with NaN, so a ray that is never written
shows, and a ray composited twice changes its colour."""
import pytest
import torch

pytestmark = pytest.mark.gpu

W = H = 800
BATCH = 4096
FIRST = 40 * BATCH + 1234          # the sized batches start mid-batch, so they straddle two ordinary batches


@pytest.fixture(scope="module")
def scene300():
    import bench
    return bench.build_scene(torch.device("cuda", 0), 300)


def _render(lt, ids):
    """rgb, depth of `ids` in one call, written into NaN-filled `out=` buffers"""
    n = ids.numel()
    rgb = torch.full((n, 3), float("nan"), device="cuda")
    depth = torch.full((n,), float("nan"), device="cuda")
    with torch.no_grad():
        lt(ids, torch.tensor([0], device="cuda"), W, H, is_train=False, out=(rgb, depth))
    torch.cuda.synchronize()
    return rgb, depth


def _in_batches(lt, lo, hi):
    """rgb, depth of rays lo .. hi-1 of the frame, rendered in the ordinary 4096-ray batches that hold them"""
    b0 = lo // BATCH * BATCH
    rgbs, depths = [], []
    for b in range(b0, hi, BATCH):
        r, d = _render(lt, torch.arange(b, min(b + BATCH, W * H), dtype=torch.int64, device="cuda"))
        rgbs.append(r); depths.append(d)
    return torch.cat(rgbs)[lo - b0:hi - b0], torch.cat(depths)[lo - b0:hi - b0]


def _check(got, want, what):
    for g, w, name in zip(got, want, ("rgb", "depth")):
        unwritten = int(torch.isnan(g).any(-1).sum() if g.dim() > 1 else torch.isnan(g).sum())
        assert unwritten == 0, f"{what}: {unwritten} rays never written ({name})"
        diff = int((g != w).reshape(g.shape[0], -1).any(-1).sum())
        assert diff == 0, f"{what}: {diff} rays differ from the same rays in 4096-ray batches ({name})"


@pytest.mark.parametrize("n", [1, 11, 12, 13, 1000, 4095, 4097])
def test_batch_sizes_bit_identical_to_full_batches(scene300, n):
    want = _in_batches(scene300, FIRST, FIRST + n)
    got = _render(scene300, torch.arange(FIRST, FIRST + n, dtype=torch.int64, device="cuda"))
    _check(got, want, f"{n}-ray batch")


def test_whole_frame_in_one_launch(scene300):
    want = _in_batches(scene300, 0, W * H)
    got = _render(scene300, torch.arange(W * H, dtype=torch.int64, device="cuda"))
    _check(got, want, "640000-ray frame")
