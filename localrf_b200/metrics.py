"""Test-frame metrics on the device: the MSE and SSIM that renderer.py:162-163 computes for every held-out frame.

The reference computes them on the host, with `rgb_ssim` (utils/utils.py:232-287: numpy and
scipy.signal.convolve2d).  Here one kernel (lrf_image_metrics) computes both, following the reference's
arithmetic: fp32 squares and cross products, an fp64 separable Gaussian filter and an fp64 SSIM map.

    image_metrics(img, gt)          -> float64 device tensor [mse, ssim], no host synchronisation
    rgb_ssim(img0, img1, max_val)   -> the reference's function (numpy in, float / numpy map out), on the GPU

`renderer.rgb_ssim = localrf_b200.metrics.rgb_ssim` puts it into the reference's renderer.  There is no CPU
fallback: without a CUDA device these raise RuntimeError.
"""
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
