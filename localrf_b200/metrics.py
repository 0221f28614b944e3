"""Test-frame metrics on the device: the MSE and SSIM that renderer.py:162-163 computes for every held-out frame.

The reference computes them on the host, with `rgb_ssim` (utils/utils.py:232-287: numpy and
scipy.signal.convolve2d).  Here one kernel (lrf_image_metrics) computes both, following the reference's
arithmetic: fp32 squares and cross products, an fp64 separable Gaussian filter and an fp64 SSIM map.

    image_metrics(img, gt)          -> float64 device tensor [mse, ssim], no host synchronisation
    rgb_ssim(img0, img1, max_val)   -> the reference's function (numpy in, float / numpy map out), on the GPU
    test_panels(depth, directions, ...) -> the flow and depth comparison panels of renderer.py:79-124
                                       (lrf_test_panels), device tensors, no host synchronisation
    resize_linear(src, W, H)        -> cv2.resize(src, (W, H)) of a held-out frame's ground truth (renderer.py:157)
                                       as OpenCV computes it without IPP (lrf_resize_linear), no synchronisation

`renderer.rgb_ssim = localrf_b200.metrics.rgb_ssim` puts it into the reference's renderer.  There is no CPU
fallback: without a CUDA device these raise RuntimeError.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .tensorf import _ptr, _stream


def _frame(t, W):
    """-> (t, H, W, stride) for an fp32 [H,W,3] or [H*W,3] frame on a CUDA device or in pinned host memory.
    The pixels may be `stride` >= 3 floats apart, e.g. the rgb columns of the interleaved [N,4] pix buffer."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"expected a torch tensor, got {type(t).__name__}")
    if t.dtype != torch.float32:
        raise TypeError(f"frames must be float32, got {t.dtype}")
    if not (t.is_cuda or t.is_pinned()):
        raise ValueError("frames must be CUDA tensors or pinned host tensors")
    if t.dim() == 3 and t.shape[2] == 3:
        H, W = int(t.shape[0]), int(t.shape[1])
        ok = t.stride(2) == 1 and t.stride(1) >= 3 and (H == 1 or t.stride(0) == W * t.stride(1))
        stride = t.stride(1)
    elif t.dim() == 2 and t.shape[1] == 3:
        if W is None or W < 1 or t.shape[0] % W:
            raise ValueError("a flat [H*W,3] frame needs W= dividing its pixel count")
        H, W = int(t.shape[0]) // W, int(W)
        ok = t.stride(1) == 1 and t.stride(0) >= 3
        stride = t.stride(0)
    else:
        raise ValueError(f"frames must be [H,W,3] or [H*W,3], got {tuple(t.shape)}")
    if not ok:
        t = t.contiguous() if t.is_cuda else t.contiguous().pin_memory()
        stride = 3
    return t, H, W, stride


def _enqueue(img, gt, out, ssim_map=None, W=None, max_val=1.0, filter_size=11, filter_sigma=1.5, k1=0.01,
             k2=0.03):
    """Enqueues lrf_image_metrics on the current stream: out[0] = mse, out[1] = ssim (out: 2 doubles, device
    or pinned); ssim_map, when given, receives the fp64 [H-fs+1, W-fs+1, 3] map."""
    img, H, W_, s_img = _frame(img, W)
    gt, Hg, Wg, s_gt = _frame(gt, W)
    if (H, W_) != (Hg, Wg):
        raise ValueError(f"img is {H}x{W_} but gt is {Hg}x{Wg}")
    devs = {t.device for t in (img, gt, out) + ((ssim_map,) if ssim_map is not None else ()) if t.is_cuda}
    if len(devs) > 1:
        raise ValueError(f"tensors on different devices: {sorted(map(str, devs))}")
    dev = devs.pop() if devs else torch.device("cuda", torch.cuda.current_device())
    L = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = L.lrf_image_metrics_scratch_bytes(H, W_, int(filter_size))
        scratch = torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device=dev)
        _lib.check(L.lrf_image_metrics(_ptr(img), s_img, _ptr(gt), s_gt, H, W_, float(max_val), int(filter_size),
                                       float(filter_sigma), float(k1), float(k2), _ptr(out), _ptr(ssim_map),
                                       _ptr(scratch), int(nbytes), _stream(dev)))


def resize_linear(src, W, H, out=None):
    """cv2.resize(src, (W, H)) as OpenCV computes it without IPP (INTER_LINEAR, exact 2x as INTER_AREA; rules and the
    documented difference from an IPP build in include/localrf_b200.h, lrf_resize_linear), bit for bit: the ground
    truth renderer.py:157 resizes for every held-out frame.  src: float32 [h0,w0,3] on a CUDA device or pinned
    (rows may be further apart than 3 w0 floats).  -> [H,W,3] float32 on src's device (the current CUDA device for a
    pinned src), or `out` (a CUDA float32 [H,W,3] tensor with 3-float pixels), enqueued without synchronising."""
    W, H = int(W), int(H)
    if not isinstance(src, torch.Tensor):
        raise TypeError(f"src must be a torch tensor, got {type(src).__name__}")
    if src.dtype != torch.float32:
        raise TypeError(f"src must be float32, got {src.dtype}")
    if not (src.is_cuda or src.is_pinned()):
        raise ValueError("src must be a CUDA tensor or a pinned host tensor")
    if src.dim() != 3 or src.shape[2] != 3:
        raise ValueError(f"src must be [h0,w0,3], got {tuple(src.shape)}")
    h0, w0 = int(src.shape[0]), int(src.shape[1])
    if not (src.stride(2) == 1 and src.stride(1) == 3 and (h0 == 1 or src.stride(0) >= 3 * w0)):
        src = src.contiguous() if src.is_cuda else src.contiguous().pin_memory()
    s_src = src.stride(0) if h0 > 1 else 3 * w0
    dev = _device_of(src, *(() if out is None else (out,)))
    if out is None:
        out = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.dtype == torch.float32 and
              tuple(out.shape) == (H, W, 3) and out.stride(2) == 1 and out.stride(1) == 3 and
              (H == 1 or out.stride(0) >= 3 * W)):
        raise ValueError(f"out must be a CUDA float32 [{H},{W},3] tensor with 3-float pixels")
    elif out.device != dev:
        raise ValueError(f"out is on {out.device} but src is on {dev}")
    s_out = out.stride(0) if H > 1 else 3 * W
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().lrf_resize_linear(_ptr(src), w0, h0, s_src, _ptr(out), W, H, s_out, _stream(dev)))
    return out


def _device_of(*ts):
    for t in ts:
        if t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        raise RuntimeError("localrf_b200.metrics needs a CUDA device (there is no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def image_metrics(img, gt, max_val=1.0, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, W=None):
    """MSE and SSIM of one rendered frame `img` against `gt` -> float64 tensor [2] = (mse, ssim) on the frames'
    CUDA device, without synchronising.  Frames: float32 [H,W,3], or [H*W,3] with W=, on a CUDA device or in
    pinned host memory.  mse = mean((gt - img)^2) over every value (renderer.py:162); ssim = rgb_ssim(gt, img,
    max_val, filter_size, filter_sigma, k1, k2) (utils/utils.py:232-287)."""
    out = torch.empty(2, dtype=torch.float64, device=_device_of(img, gt))
    _enqueue(img, gt, out, None, W, max_val, filter_size, filter_sigma, k1, k2)
    return out


def rgb_ssim(img0, img1, max_val, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False):
    """The reference's rgb_ssim (utils/utils.py:232-287) on the GPU, with its signature.

    numpy [H,W,3] float32 inputs (what renderer.py passes) are copied to the current CUDA device, and the
    result is what the reference returns: a float, or the float64 map [H-fs+1, W-fs+1, 3] as numpy.  CUDA
    tensors give a 0-d float64 tensor or the map tensor, without synchronising."""
    on_device = all(isinstance(t, torch.Tensor) and t.is_cuda for t in (img0, img1))
    if not on_device:
        if not torch.cuda.is_available():
            raise RuntimeError("localrf_b200.metrics.rgb_ssim needs a CUDA device (there is no CPU fallback)")
        a, b = np.asarray(img0), np.asarray(img1)
        if a.dtype != np.float32 or b.dtype != np.float32:
            raise TypeError(f"rgb_ssim takes float32 frames, got {a.dtype} and {b.dtype}")
        dev = torch.device("cuda", torch.cuda.current_device())
        img0, img1 = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (a, b))
    if img0.dim() != 3 or img0.shape[-1] != 3 or img0.shape != img1.shape:
        raise ValueError(f"rgb_ssim takes two [H,W,3] frames of one shape, got {tuple(img0.shape)} and "
                         f"{tuple(img1.shape)}")
    H, W = int(img0.shape[0]), int(img0.shape[1])
    out = torch.empty(2, dtype=torch.float64, device=img0.device)
    ssim_map = None
    if return_map:
        ssim_map = torch.empty(max(H - filter_size + 1, 0), max(W - filter_size + 1, 0), 3, dtype=torch.float64,
                               device=img0.device)
    _enqueue(img0, img1, out, ssim_map, None, max_val, filter_size, filter_sigma, k1, k2)
    if on_device:
        return ssim_map if return_map else out[1]
    return ssim_map.cpu().numpy() if return_map else float(out[1])


def _readable(t, dev, name):
    """t as a contiguous float32 tensor the kernel can read on `dev`: a CUDA tensor on `dev`, or a pinned host tensor.
    Anything else raises ValueError: the kernel would dereference a pageable host or another device's pointer."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(t).__name__}")
    if t.is_cuda:
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device} but the frame is on {dev}")
        return t.detach().to(torch.float32).contiguous()
    if not t.is_pinned():
        raise ValueError(f"{name} must be a CUDA tensor on {dev} or a pinned host tensor")
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.detach().to(torch.float32).contiguous().pin_memory()
    return t


def _gt_map(a, dev, name, shape, stage=None):
    """A ground-truth array of the test dataset as a contiguous float32 tensor the kernel can read: CUDA tensors on
    `dev` and pinned tensors as they are (CUDA tensors on another device raise ValueError); numpy arrays and pageable
    tensors copied to `dev` (as rgb_ssim stages its inputs), or handed to `stage(name, array)`, which returns a pinned
    copy (FramePipeline: a host copy into the frame slot's buffer, which does not wait for the device)."""
    if a is None:
        return None
    if isinstance(a, torch.Tensor) and (a.is_cuda or a.is_pinned()):
        if a.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {a.dtype}")
        a = _readable(a, dev, name)
    else:
        x = a.detach().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        if x.dtype != np.float32:
            raise TypeError(f"{name} must be float32, got {x.dtype}")
        if shape is not None and tuple(x.shape) != shape:
            raise ValueError(f"{name} is {tuple(x.shape)}, expected {shape}")
        a = stage(name, x) if stage is not None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    if shape is not None and tuple(a.shape) != shape:
        raise ValueError(f"{name} is {tuple(a.shape)}, expected {shape}")
    return a


def _intrinsics(focal, center, dev):
    """[focal, cx, cy] as a float32 device tensor, built on the device from tensors (no synchronisation)."""
    parts = [torch.as_tensor(v, dtype=torch.float32).reshape(-1).to(dev) for v in (focal, center)]
    intr = torch.cat(parts)
    if intr.numel() != 3:
        raise ValueError("focal must hold 1 value and center 2")
    return intr


def _enqueue_panels(depth, directions, cam2world, idx, intrinsics, W, H, gts, outs, dev):
    """Enqueues lrf_test_panels on the current stream of `dev`.  gts: (fwd_flow, fwd_mask, bwd_flow, bwd_mask,
    invdepth) staged by _gt_map; outs: dict of fwd_panel / bwd_panel / depth_panel / fwd_pred / bwd_pred / stats
    (device or pinned).  Returns the scratch tensor, which must stay alive until the work has run."""
    fwd_flow, fwd_mask, bwd_flow, bwd_mask, invdepth = gts
    first = next(g for g in gts if g is not None)
    h0, w0 = int(first.shape[0]), int(first.shape[1])
    f = _lib.LrfPanelFrame()
    f.W, f.H, f.h0, f.w0 = int(W), int(H), h0, w0
    f.n_cams = int(cam2world.shape[0]) if cam2world is not None else int(idx) + 1   # depth only: no camera read
    f.idx = int(idx)
    for name, t in (("depth", depth), ("directions", directions), ("cam2world", cam2world),
                    ("intrinsics", intrinsics), ("fwd_flow", fwd_flow), ("fwd_mask", fwd_mask),
                    ("bwd_flow", bwd_flow), ("bwd_mask", bwd_mask), ("invdepth", invdepth)):
        setattr(f, name, _ptr(t).value if t is not None else None)
    for name in ("fwd_panel", "bwd_panel", "depth_panel", "fwd_pred", "bwd_pred", "stats"):
        t = outs.get(name)
        setattr(f, name, _ptr(t).value if t is not None else None)
    L = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(L.lrf_test_panels_scratch_bytes(f.W, f.H))
        if nbytes == 0:
            raise ValueError(f"W x H = {W} x {H} is out of range for lrf_test_panels")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(L.lrf_test_panels(C.byref(f), _ptr(scratch), nbytes, _stream(dev)))
    return scratch


def _panel_inputs(depth, directions, cam2world, W, H, fwd_flow, fwd_mask, bwd_flow, bwd_mask, invdepth, stage=None,
                  dev=None):
    """Checks and stages the inputs of test_panels -> (dev, depth, directions, cam2world, gts).  The frame's device is
    depth's; depth may be pinned only when `dev` names the device.  directions and cam2world must be on that device
    or pinned."""
    if not isinstance(depth, torch.Tensor) or depth.dtype != torch.float32 or depth.numel() != W * H:
        raise ValueError(f"depth must be a float32 tensor of W x H = {W * H} values")
    if depth.is_cuda:
        dev = depth.device
    elif dev is None or not depth.is_pinned():
        raise ValueError("depth must be a CUDA tensor (the frame's device)")
    depth = _readable(depth, dev, "depth")
    flows = (fwd_flow, fwd_mask, bwd_flow, bwd_mask)
    n_flow = sum(x is not None for x in flows)
    if n_flow not in (0, 4):
        raise ValueError("the flow panels need all of fwd_flow, fwd_mask, bwd_flow and bwd_mask (or none)")
    if n_flow:
        if directions is None or cam2world is None:
            raise ValueError("the flow panels need directions and cam2world")
        if not isinstance(directions, torch.Tensor) or directions.dtype != torch.float32 or \
                directions.numel() != 3 * W * H:
            raise ValueError("directions must be a float32 [W*H, 3] tensor")
        directions = _readable(directions, dev, "directions").reshape(-1, 3)
        cam2world = _readable(cam2world, dev, "cam2world")
        if cam2world.numel() == 0 or cam2world.numel() % 12:
            raise ValueError(f"cam2world must be [n_cams, 3, 4], got {tuple(cam2world.shape)}")
        cam2world = cam2world.reshape(-1, 3, 4)
    else:
        directions = cam2world = None
    first = next((np.shape(x) for x in flows + (invdepth,) if x is not None), None)
    h0, w0 = (int(first[0]), int(first[1])) if first is not None and len(first) >= 2 else (0, 0)
    gts = tuple(_gt_map(x, dev, name, shape, stage) for x, name, shape in (
        (fwd_flow, "fwd_flow", (h0, w0, 2)), (fwd_mask, "fwd_mask", (h0, w0)), (bwd_flow, "bwd_flow", (h0, w0, 2)),
        (bwd_mask, "bwd_mask", (h0, w0)), (invdepth, "invdepth", (h0, w0))))
    return dev, depth.reshape(-1), directions, cam2world, gts


@torch.no_grad()
def test_panels(depth, directions, cam2world, idx, focal, center, W, H, fwd_flow=None, fwd_mask=None, bwd_flow=None,
                bwd_mask=None, invdepth=None, return_arrays=False):
    """The comparison panels renderer.render(test=True) builds for a held-out frame (renderer.py:79-124) ->
    (fwd_flow_cmp [3H,2W] | None, bwd_flow_cmp [3H,2W] | None, depth_cmp [3H,W] | None): float32 tensors on
    depth's CUDA device, clamped to [0, 1], enqueued without synchronising.  They are what render appends to
    fwd_flow_cmp_tb, bwd_flow_cmp_tb and depth_cmp_tb.

    depth [W*H] and directions [W*H,3] come from the forward of the frame (rays_ids = arange(W*H)); cam2world =
    LocalTensorfs.get_cam2world() (every frame); idx is the frame's camera; focal = focal(W), center = center(W, H)
    (tensors or numbers).  The ground truth is the test dataset's arrays of the frame at its own resolution h0 x w0:
    fwd_flow / bwd_flow [h0,w0,2] and fwd_mask / bwd_mask [h0,w0] (all four, or none: no flow panels), invdepth
    [h0,w0] (or None: no depth panel); float32 numpy arrays (copied to the device) or CUDA / pinned tensors.
    return_arrays=True adds a dict with the unscaled predicted flows fwd_pred / bwd_pred [H,W,2] and `stats`
    [8]: the four 0.9 quantiles (fwd c0, c1, bwd c0, c1), then median and mean absolute deviation of x and of g."""
    W, H = int(W), int(H)
    dev, depth, directions, cam2world, gts = _panel_inputs(depth, directions, cam2world, W, H, fwd_flow, fwd_mask,
                                                          bwd_flow, bwd_mask, invdepth)
    flow, dep = gts[0] is not None, gts[4] is not None
    new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    outs = {}
    if flow:
        outs.update(fwd_panel=new(3 * H, 2 * W), bwd_panel=new(3 * H, 2 * W))
    if dep:
        outs["depth_panel"] = new(3 * H, W)
    if return_arrays:
        outs["stats"] = new(8)
        if flow:
            outs.update(fwd_pred=new(H, W, 2), bwd_pred=new(H, W, 2))
    if flow or dep:
        intr = _intrinsics(focal, center, dev) if flow else None
        _enqueue_panels(depth, directions, cam2world, idx, intr, W, H, gts, outs, dev)
    panels = (outs.get("fwd_panel"), outs.get("bwd_panel"), outs.get("depth_panel"))
    if return_arrays:
        return panels + ({k: outs.get(k) for k in ("fwd_pred", "bwd_pred", "stats")},)
    return panels
