"""CPU-only: the kernels' per-sample building blocks, compiled for the HOST, against the oracle.

There is no GPU in the build container, so the CUDA kernels themselves only run in the `-m gpu` tests.  But the
arithmetic they are made of lives in two headers (localrf_b200/csrc/lrf_common.cuh, lrf_device.cuh) as small
device functions -- grid coordinates, contraction, the VM density / appearance gathers for fp32 AND bf16 texels,
the alpha-mask lookup, feature2density, ray generation, the bf16 hi/lo operand split.  tests/host_emul/ compiles
exactly those sources with g++ behind a shim of the CUDA built-ins they use (test infrastructure; nothing of it is
product code, and the product never loads it) and this file holds them to the oracle, which is pinned to the
reference.  It catches indexing / layout / formula regressions in the shared device code before a GPU is involved.
(Host g++ does not contract a*b+c into FMAs the way nvcc does, so values agree to fp32 rounding, not bitwise.)"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import full_field_dict, load_golden, rel_err
from oracle import oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_emul", "emul.cpp")
LIB = os.path.join(HERE, "host_emul", "libemul.so")
CSRC = os.path.join(os.path.dirname(HERE), "localrf_b200", "csrc")
_vp = C.c_void_p


@pytest.fixture(scope="module")
def emul():
    deps = [SRC, os.path.join(CSRC, "lrf_common.cuh"), os.path.join(CSRC, "lrf_device.cuh"),
            os.path.join(HERE, "host_emul", "shim", "cuda_runtime.h"), os.path.join(HERE, "host_emul", "shim", "cuda_bf16.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        env = dict(os.environ); env.pop("CC", None); env.pop("CXX", None)
        r = subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off",
                            "-I", os.path.join(HERE, "host_emul", "shim"), "-o", LIB, SRC],
                           capture_output=True, text=True, env=env)
        assert r.returncode == 0, r.stderr
    return C.CDLL(LIB)


def channel_last(a):
    """[1,C,H,W] (reference layout) -> contiguous [H][W][C] float32"""
    return np.ascontiguousarray(np.transpose(np.asarray(a, np.float32)[0], (1, 2, 0)))


def to_bf16_bits(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.bfloat16).view(torch.int16).numpy()


class Grids:
    """Channel-last copies of a golden field's twelve grids, fp32 or bf16, + the pointer arrays the wrappers take."""

    def __init__(self, fd, bf16=False, rounded=False):
        self.keep, self.ptrs = [], {}
        for name, key in (("dplane", "density_plane"), ("dline", "density_line"), ("aplane", "app_plane"), ("aline", "app_line")):
            arr = (_vp * 3)()
            for i in range(3):
                a = channel_last(fd[f"{key}.{i}"])
                if rounded or bf16:
                    a = torch.from_numpy(a).to(torch.bfloat16).to(torch.float32).numpy()
                buf = to_bf16_bits(a) if bf16 else a
                self.keep.append(buf)
                arr[i] = buf.ctypes.data
            self.ptrs[name] = arr
        self.grid = (C.c_int * 3)(*[int(v) for v in fd["gridSize"]])
        self.aabb = np.asarray(fd["aabb"], np.float32).reshape(6).copy()
        self.bf16 = int(bf16)

    def args(self):
        return (self.grid, _vp(self.aabb.ctypes.data), self.ptrs["dplane"], self.ptrs["dline"], self.ptrs["aplane"],
                self.ptrs["aline"], self.bf16)


def points(n, seed, span=1.1):
    g = np.random.default_rng(seed)
    return (g.random((n, 3), dtype=np.float32) * 2 * span - span).astype(np.float32)


@pytest.mark.parametrize("golden", ["cfg1_64", "aniso_pe", "opaque_32"])
def test_vm_gathers_fp32_vs_oracle(emul, golden):
    """density_feature / app_plane_features of lrf_device.cuh (incl. an anisotropic [40,52,64] grid: axis mix-ups
    show) against the oracle's compute_densityfeature / compute_appfeature."""
    fd = full_field_dict(load_golden(golden))
    f = orc.Field(fd)
    G = Grids(fd)
    xyz = points(4000, 1)                                   # incl. points beyond the border clamp
    out = np.empty(len(xyz), np.float32)
    emul.emul_density_feature(*G.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(out.ctypes.data))
    ref = orc.density_feature(f, xyz)
    assert np.abs(out - ref).max() <= 2e-6 * max(np.abs(ref).max(), 1e-3)
    prod = np.empty((len(xyz), 72), np.float32)
    emul.emul_app_products(*G.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(prod.ctypes.data))
    feat = prod.astype(np.float64) @ np.asarray(fd["basis_mat.weight"], np.float64).T
    ref_a = orc.app_feature(f, xyz)
    assert np.abs(feat - ref_a).max() <= 5e-6 * max(np.abs(ref_a).max(), 1e-3)


def test_vm_gathers_bf16_storage_equal_fp32_storage(emul):
    """The bf16-texel gathers return EXACTLY what the fp32 gathers return on the bf16-rounded field (same
    expression order; bf16 -> fp32 is exact) -- the equality tests/test_gpu_bf16.py shows for the kernels."""
    fd = full_field_dict(load_golden("aniso_pe"))
    G32, G16 = Grids(fd, rounded=True), Grids(fd, bf16=True)
    xyz = points(3000, 2)
    a, b = np.empty(len(xyz), np.float32), np.empty(len(xyz), np.float32)
    emul.emul_density_feature(*G32.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(a.ctypes.data))
    emul.emul_density_feature(*G16.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(b.ctypes.data))
    assert np.array_equal(a, b)
    pa, pb = np.empty((len(xyz), 72), np.float32), np.empty((len(xyz), 72), np.float32)
    emul.emul_app_products(*G32.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(pa.ctypes.data))
    emul.emul_app_products(*G16.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(pb.ctypes.data))
    assert np.array_equal(pa, pb)
    # ... and differs from the unrounded field (the storage really is 16-bit)
    G = Grids(fd)
    c = np.empty(len(xyz), np.float32)
    emul.emul_density_feature(*G.args(), _vp(xyz.ctypes.data), C.c_longlong(len(xyz)), _vp(c.ctypes.data))
    assert not np.array_equal(a, c) and np.abs(a - c).max() < 2e-2 * np.abs(c).max()


def test_sample_positions_and_contraction_vs_oracle(emul):
    aabb = np.array([-2, -2, -2, 2, 2, 2], np.float32)
    g = np.random.default_rng(3)
    o = (0.1 * g.standard_normal(3)).astype(np.float32)
    d = g.standard_normal(3).astype(np.float32); vd = (d / np.linalg.norm(d)).astype(np.float32)
    z = orc.sample_table(1036)                                              # the 300^3 table: 0.1 ... 147
    p, q = np.empty((len(z), 3), np.float32), np.empty((len(z), 3), np.float32)
    emul.emul_sample_pos(_vp(aabb.ctypes.data), _vp(o.ctypes.data), _vp(vd.ctypes.data), _vp(z.ctypes.data),
                         C.c_longlong(len(z)), _vp(p.ctypes.data), _vp(q.ctypes.data))
    ref = orc.contract((o[None] + vd[None] * z[:, None]).astype(np.float32))
    np.testing.assert_allclose(p, ref, rtol=2e-6, atol=1e-6)
    np.testing.assert_allclose(q, (ref - aabb[:3]) * (2.0 / (aabb[3:] - aabb[:3])) - 1.0, rtol=0, atol=2e-6)
    assert np.abs(p).max() <= 2.0 + 1e-6 and (np.abs(o[None] + vd[None] * z[:, None]).max(-1) > 1).mean() > 0.3


def test_alpha_mask_lookup_vs_oracle(emul):
    g = load_golden("alphamask_32")
    fd = full_field_dict(g)
    f = orc.Field(fd)
    vol = np.ascontiguousarray(np.asarray(fd["alphaMask.alpha_volume"], np.float32).reshape(fd["alphaMask.alpha_volume"].shape[-3:]))
    dims = (C.c_int * 3)(*vol.shape)
    ab = np.asarray(fd["alphaMask.aabb"], np.float32).reshape(6).copy()
    p = points(5000, 4, span=2.2)                                           # incl. points outside the volume (zero padding)
    out = np.empty(len(p), np.float32)
    emul.emul_alpha_mask(_vp(vol.ctypes.data), dims, _vp(ab.ctypes.data), _vp(p.ctypes.data), C.c_longlong(len(p)),
                         _vp(out.ctypes.data))
    ref = orc.alpha_mask_sample(f, p)
    assert np.abs(out - ref).max() < 2e-6
    assert ((out > 0) == (ref > 0)).all()                                   # the decision the kernel takes from it


def test_feature2density(emul):
    x = np.concatenate([np.linspace(-30, 30, 2001), [19.999, 20.0, 20.001, 25.0 + 5]]).astype(np.float32)
    out = np.empty_like(x)
    emul.emul_feature2density(_vp(x.ctypes.data), C.c_longlong(len(x)), C.c_float(-5.0), 0, _vp(out.ctypes.data))
    ref = torch.nn.functional.softplus(torch.from_numpy(x) + (-5.0)).numpy()       # tensorBase.py:495-499
    assert rel_err(out, ref, floor=1e-30) < 2e-6
    emul.emul_feature2density(_vp(x.ctypes.data), C.c_longlong(len(x)), C.c_float(-5.0), 1, _vp(out.ctypes.data))
    assert np.array_equal(out, np.maximum(x, 0))


def test_contract_backward_vs_autograd(emul):
    """contract_bwd against torch autograd through ray_utils.contract, inside and outside the unit cube."""
    from localrf_b200.ray_utils import contract
    p = np.concatenate([points(3000, 7, span=3.0), points(1000, 8, span=1.0)])
    gout = np.random.default_rng(9).standard_normal(p.shape).astype(np.float32)
    out = np.empty_like(p)
    emul.emul_contract_bwd(_vp(p.ctypes.data), _vp(gout.ctypes.data), C.c_longlong(len(p)), _vp(out.ctypes.data))
    x = torch.from_numpy(p).double().requires_grad_(True)
    contract(x).backward(torch.from_numpy(gout).double())
    ref = x.grad.numpy()
    inside = np.abs(p).max(-1) <= 1
    assert 0.2 < inside.mean() < 0.5
    np.testing.assert_array_equal(out[inside], gout[inside])
    np.testing.assert_allclose(out, ref, rtol=1e-5, atol=1e-5 * np.abs(ref).max())


def test_sample_alpha_vs_oracle(emul):
    """sample_alpha (sample position, alpha-mask validity, density feature, feature2density and alpha with the
    alpha[:, -1] = 1 rule) for every sample of the golden rays of a field with an alpha mask, against values built
    from the oracle's contract, alpha_mask_sample and density_feature."""
    gd = load_golden("alphamask_32")
    fd = full_field_dict(gd)
    f = orc.Field(fd)
    G = Grids(fd)
    vol = np.ascontiguousarray(np.asarray(fd["alphaMask.alpha_volume"], np.float32).reshape(fd["alphaMask.alpha_volume"].shape[-3:]))
    dims = (C.c_int * 3)(*vol.shape)
    ab = np.asarray(fd["alphaMask.aabb"], np.float32).reshape(6).copy()
    z = np.ascontiguousarray(gd["eval.z"], np.float32)
    S = len(z)
    rays = np.asarray(gd["rays"], np.float32)
    o, d = np.ascontiguousarray(rays[:, :3]), np.ascontiguousarray(rays[:, 3:])
    n = len(rays)
    shift, scale = float(fd["density_shift"]), float(fd["distance_scale"])
    act = {"softplus": 0, "relu": 1}[fd["fea2denseAct"]]
    alpha, fe, valid = np.empty((n, S), np.float32), np.empty((n, S), np.float32), np.empty((n, S), np.uint8)
    emul.emul_sample_alpha(G.grid, _vp(G.aabb.ctypes.data), G.ptrs["dplane"], G.ptrs["dline"], G.ptrs["aplane"],
                           G.ptrs["aline"], _vp(vol.ctypes.data), dims, _vp(ab.ctypes.data), C.c_float(shift),
                           C.c_float(scale), act, _vp(z.ctypes.data), S, _vp(o.ctypes.data), _vp(d.ctypes.data),
                           C.c_longlong(n), _vp(alpha.ctypes.data), _vp(fe.ctypes.data), _vp(valid.ctypes.data))

    vd = d / np.sqrt((d * d).sum(-1, dtype=np.float32))[:, None]
    p = orc.contract((o[:, None] + vd[:, None] * z[None, :, None]).reshape(-1, 3))
    q = (p - G.aabb[:3]) * (np.float32(2) / (G.aabb[3:] - G.aabb[:3])) - np.float32(1)
    ok = (orc.alpha_mask_sample(f, p) > 0).reshape(n, S)
    ok[:, -1] = False                                                       # ray_valid[:, -1] = 0
    fe_ref = np.where(ok, orc.density_feature(f, q).reshape(n, S), np.float32(0))
    fe_t = torch.from_numpy(fe_ref)
    sigma = torch.nn.functional.softplus(fe_t + shift) if act == 0 else fe_t.clamp(min=0)
    sigma = np.where(ok, sigma.numpy(), np.float32(0))
    dist = np.append(np.diff(z), np.float32(0))
    alpha_ref = 1 - np.exp(-sigma * dist * scale)
    alpha_ref[:, -1] = 1                                                    # alpha[:, -1] = 1

    assert ok.any() and (~ok[:, :-1]).any()                                 # the mask excludes some samples
    np.testing.assert_array_equal(valid.astype(bool), ok)
    assert np.abs(fe - fe_ref).max() <= 2e-6 * max(np.abs(fe_ref).max(), 1e-3)
    assert np.abs(alpha - alpha_ref).max() <= 5e-6
    assert alpha[:, :-1].max() > 0.1


@pytest.mark.parametrize("fov360", [0, 1])
def test_ray_generation_vs_oracle(emul, fov360):
    """setup_ray (ids2pixel, get_ray_directions_lean / _360, per-view cam2rf, get_rays_lean, normalisation)."""
    W, H, V = 96, 64, 3
    g = np.random.default_rng(5)
    per = 500
    ids = np.concatenate([g.integers(0, W * H, per) + v * W * H for v in range(V)]).astype(np.int64)   # ids carry view offsets
    focal, cx, cy = 77.7, 47.3, 31.9
    c2w = np.zeros((V, 3, 4), np.float32)
    for v in range(V):
        qm, _ = np.linalg.qr(g.standard_normal((3, 3)))
        c2w[v, :, :3] = qm; c2w[v, :, 3] = 0.2 * g.standard_normal(3)
    w2rf = np.array([0.3, -0.1, 0.2], np.float32)
    n = len(ids)
    o, vd, nrm = np.empty((n, 3), np.float32), np.empty((n, 3), np.float32), np.empty(n, np.float32)
    dirs, ij = np.empty((n, 3), np.float32), np.empty((n, 2), np.int64)
    emul.emul_setup_rays(_vp(ids.ctypes.data), C.c_longlong(n), C.c_longlong(V), W, H, fov360, C.c_float(focal),
                         C.c_float(cx), C.c_float(cy), _vp(c2w.ctypes.data), _vp(w2rf.ctypes.data), _vp(o.ctypes.data),
                         _vp(vd.ctypes.data), _vp(nrm.ctypes.data), _vp(dirs.ctypes.data), _vp(ij.ctypes.data))
    rd, rij = orc.ray_directions(ids, W, H, bool(fov360), focal, cx, cy)
    assert np.array_equal(ij, rij)
    np.testing.assert_allclose(dirs, rd, rtol=3e-6, atol=1e-6)
    view = np.repeat(np.arange(V), per)
    d_world = np.einsum("nij,nj->ni", c2w[view, :, :3].astype(np.float64), rd.astype(np.float64))
    np.testing.assert_allclose(nrm, np.linalg.norm(d_world, axis=-1), rtol=3e-6)
    np.testing.assert_allclose(vd, d_world / np.linalg.norm(d_world, axis=-1, keepdims=True), rtol=0, atol=3e-6)
    np.testing.assert_allclose(o, c2w[view, :, 3] + w2rf, rtol=0, atol=1e-6)


def test_hi_lo_split_keeps_16_mantissa_bits(emul):
    """split2: x = hi + lo with both bf16 -- what makes three bf16 tensor-core products an fp32-grade GEMM."""
    g = np.random.default_rng(6)
    v = (g.standard_normal(8) * np.array([1e-3, 1, 1e3, 0.3, 7, 1e-6, 50, 2])).astype(np.float32)
    hi, lo = np.empty(8, np.float32), np.empty(8, np.float32)
    emul.emul_split8(_vp(v.ctypes.data), _vp(hi.ctypes.data), _vp(lo.ctypes.data))
    assert np.abs((hi.astype(np.float64) + lo) - v).max() <= 2.0 ** -16 * np.abs(v).max()
    assert (np.abs(hi.astype(np.float64) + lo - v) <= 2.0 ** -16 * np.abs(v)).all()
    assert np.array_equal(hi, torch.from_numpy(v).to(torch.bfloat16).to(torch.float32).numpy())


def test_operand_image_layout_and_prepared_sizes(emul):
    """oper_offset is the canonical K-major / no-swizzle wgmma operand image: 8 x 8 core matrices of 128 contiguous
    bytes, LBO = 128 B between K-adjacent core matrices, SBO = chunks * 128 B between 8-row groups (the strides
    mlp_gemm_n128 puts into the shared-memory descriptors) -- a bijection onto the image; and the prepared-block sizes
    the C ABI reports are the ones the headers lay out."""
    from localrf_b200 import _lib
    for rows, K in ((128, 80), (128, 128), (32, 80), (128, 64)):
        chunks = K // 8
        seen = set()
        for r in range(rows):
            for k in range(K):
                off = emul.emul_oper_offset(r, k, chunks)
                assert off == (r >> 3) * chunks * 128 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2
                seen.add(off)
        assert seen == set(range(0, rows * K * 2, 2))
    L = _lib.lib()
    assert emul.emul_prep_bytes() == L.lrf_prepared_bytes()
    f = _lib.LrfField()
    for pe in (1, 3, 6, 8):
        f.fea_pe, f.view_pe = pe, 0
        assert emul.emul_pe_prepared_bytes(pe) == L.lrf_prepared_bytes_for(C.byref(f))
