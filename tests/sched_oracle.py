"""float64 / fp32 torch restatements of the schedule-time operators (localrf_b200/csrc/lrf_sched.cu), written from
the reference formulas its header cites.  TEST INFRASTRUCTURE: tests/test_gpu_sched_sizes.py compares the kernels
against these on the device; nothing under localrf_b200/ imports it.

Every function takes the field's tensors in their logical reference shapes (planes [1,C,H,W], lines [1,C,L,1]),
whatever their memory format."""
import numpy as np
import torch
import torch.nn.functional as F

MAT_MODE = ((0, 1), (0, 2), (1, 2))     # models/tensorBase.py:274
VEC_MODE = (2, 1, 0)                    # models/tensorBase.py:275
U32 = 2.0 ** -24                        # unit roundoff of fp32


# ---- density_L1 (tensoRF.py:83-92) ---------------------------------------------------------------------
def l1_features(planes, lines):
    """f[n] = sum_i (plane_i.view(C, P_i)^T @ line_i.view(C, L_i)).view(-1)[n]: the reference's per-plane bmm
    summed over components, at the flat index n = p * L_i + l.  One [P_i, L_i] product per plane."""
    f = 0
    for p, l in zip(planes, lines):
        c = p.shape[1]
        f = f + (p.reshape(c, -1).t() @ l.reshape(c, -1)).reshape(-1)
    return f


def l1_abs_terms(planes, lines):
    """sum over i and c of |plane_i[c, p] * line_i[c, l]| at every n: the scale of the rounding in fp32 f[n]."""
    return l1_features([p.abs() for p in planes], [l.abs() for l in lines])


def density_l1(planes, lines, act, shift):
    """-> (loss, f): mean(sqrt(clamp(feature2density(f), 1e-5))) (tensorBase.py:495-499 for the activation)."""
    f = l1_features(planes, lines)
    s = F.softplus(f + shift) if act == "softplus" else F.relu(f)
    return torch.sqrt(torch.clamp(s, min=1e-5)).mean(), f


# ---- getDenseAlpha / compute_alpha (tensorBase.py:501-515, 538-558) and updateAlphaMask (:517-536) -------
def lattice_points(aabb, dims):
    """fp32 lattice of getDenseAlpha: aabb[0] * (1 - t) + aabb[1] * t, t = torch.linspace(0, 1, n) per axis.
    -> [gx, gy, gz, 3] fp32 on aabb's device."""
    ts = torch.meshgrid(*[torch.linspace(0, 1, int(n)) for n in dims], indexing="ij")
    t = torch.stack(ts, -1).to(aabb.device)
    return aabb[0] * (1 - t) + aabb[1] * t


def density_feature64(planes, lines, xyzn):
    """compute_densityfeature (tensoRF.py:112-151) in float64 at fp32 normalised coordinates [M, 3]:
    grid_sample(align_corners=True, padding_mode="border") of the fp32 parameters cast to double."""
    x = xyzn.double()
    out = torch.zeros(x.shape[0], dtype=torch.float64, device=x.device)
    for i, (m0, m1) in enumerate(MAT_MODE):
        cp = torch.stack((x[:, m0], x[:, m1]), -1).view(1, -1, 1, 2)
        cl = torch.stack((torch.zeros_like(x[:, 0]), x[:, VEC_MODE[i]]), -1).view(1, -1, 1, 2)
        pv = F.grid_sample(planes[i].detach().double(), cp, align_corners=True, padding_mode="border")
        lv = F.grid_sample(lines[i].detach().double(), cl, align_corners=True, padding_mode="border")
        out += (pv * lv).sum(1).view(-1)
    return out


def dense_alpha64(m, dims):
    """alpha = 1 - exp(-sigma * stepSize) of getDenseAlpha without a mask, float64 from the fp32 lattice and the fp32
    normalize_coord.  -> [gx, gy, gz] float64."""
    pts = lattice_points(m.aabb.detach(), dims).reshape(-1, 3)
    xyzn = (pts - m.aabb[0].detach()) * m.invaabbSize.detach() - 1
    f = density_feature64(list(m.density_plane), list(m.density_line), xyzn)
    sigma = F.softplus(f + m.density_shift) if m.fea2denseAct == "softplus" else F.relu(f)
    return (1 - torch.exp(-sigma * float(m.stepSize))).view(*[int(n) for n in dims])


def pooled_alpha64(alpha):
    """updateAlphaMask's clamp(0, 1) -> transpose(0, 2) -> max_pool3d(3, stride 1, pad 1): [gz, gy, gx]."""
    a = alpha.clamp(0, 1).permute(2, 1, 0).contiguous()[None, None]
    return F.max_pool3d(a, kernel_size=3, padding=1, stride=1)[0, 0]


# ---- up_sampling_VM: F.interpolate(bilinear, align_corners=True) (tensoRF.py:198-221) ----------------------
def _axis_taps(n, n2, device):
    """ATen's source index and weights along one axis, in fp32 as ATen forms them:
    scale = (n-1)/(n2-1) (0 for n2 == 1), src = scale * dst, i0 = (int)src, lambda1 = src - i0, lambda0 = 1 - lambda1."""
    scale = np.float32(n - 1) / np.float32(n2 - 1) if n2 > 1 else np.float32(0)
    src = np.float32(scale) * np.arange(n2, dtype=np.float32)
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n - 1)
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return t(i0), t(i1), t(l0).double(), t(l1).double()


def upsample64(src, H2, W2):
    """src [H, W, C] fp32 -> (out [H2, W2, C] float64, tap [H2, W2, C]: the largest |tap| of each output element).
    Indices and weights are ATen's fp32 values; only the blend h0 * (w0 a + w1 b) + h1 * (w0 c + w1 d) is float64."""
    H, W = src.shape[0], src.shape[1]
    y0, y1, hy, ly = _axis_taps(H, H2, src.device)
    x0, x1, hx, lx = _axis_taps(W, W2, src.device)
    s = src.double()
    a, b = s[y0][:, x0], s[y0][:, x1]
    c, d = s[y1][:, x0], s[y1][:, x1]
    hx, lx = hx[None, :, None], lx[None, :, None]
    out = hy[:, None, None] * (hx * a + lx * b) + ly[:, None, None] * (hx * c + lx * d)
    tap = torch.stack([a.abs(), b.abs(), c.abs(), d.abs()]).amax(0)
    return out, tap


# ---- TVLoss (utils/utils.py:293-312) as TV_loss_density / TV_loss_app apply it (tensoRF.py:94-110) ----------
def tv_sums64(x):
    """x [H, W, C] -> (sum (x[y+1] - x[y])^2, sum (x[:, w+1] - x[:, w])^2) in float64."""
    x = x.double()
    return float(((x[1:] - x[:-1]) ** 2).sum()), float(((x[:, 1:] - x[:, :-1]) ** 2).sum())


def tv_total(planes, lines, reg):
    """sum_i reg(plane_i^T) * 1e-2 + reg(line_i^T) * 1e-3 (the transposes of tensoRF.py:94-110); reg is the
    regulariser (a TVLoss), evaluated in the dtype of the tensors it is given."""
    total = 0
    for p, l in zip(planes, lines):
        total = total + reg(p.transpose(0, 1)) * 1e-2 + reg(l.transpose(0, 1)) * 1e-3
    return total


# ---- sample_ray (tensorBase.py:396-417) as fp32 torch ops ------------------------------------------------
def sample_ray32(rays_o, rays_d, aabb, near, far, step, S, jitter=None):
    """-> (pts [N, S, 3], z [N, S], inside [N, S]); every op rounds once, as the reference's torch ops do."""
    vec = torch.where(rays_d == 0, torch.full_like(rays_d, 1e-6), rays_d)
    rate_a = (aabb[1] - rays_o) / vec
    rate_b = (aabb[0] - rays_o) / vec
    t_min = torch.minimum(rate_a, rate_b).amax(-1).clamp(min=near, max=far)
    rng = torch.arange(S, device=rays_o.device, dtype=torch.float32)[None].repeat(rays_o.shape[0], 1)
    if jitter is not None:
        rng = rng + jitter[:, None]
    interpx = t_min[..., None] + torch.tensor(step, dtype=torch.float32, device=rays_o.device) * rng
    pts = rays_o[..., None, :] + rays_d[..., None, :] * interpx[..., None]
    out = ((aabb[0] > pts) | (pts > aabb[1])).any(dim=-1)
    return pts, interpx, ~out
