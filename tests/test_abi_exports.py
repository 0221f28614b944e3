"""CPU-only: the C-ABI library builds, loads and exports every symbol include/localrf_b200.h declares
(no compute calls without a GPU), and argument validation works without touching a device."""
import ctypes as C
import os
import re

from localrf_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "localrf_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(lrf_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported():
    L = _lib.lib()
    syms = declared_symbols()
    assert "lrf_render" in syms and "lrf_field_prepare" in syms
    for s in syms:
        assert hasattr(L, s), f"{s} declared in the header but not exported"
    assert sorted(_lib.EXPORTS) == syms


def test_version_and_prepared_size():
    L = _lib.lib()
    assert L.lrf_version() == _lib.ABI_VERSION
    # bf16 hi+lo images of W1B [128][80] and W2 [128][128], then fp32 b1, b2, W3[3][132], b3[4]
    assert L.lrf_prepared_bytes() == 2 * 2 * (128 * 80 + 128 * 128) + 4 * (128 + 128 + 3 * 132 + 4)


def test_struct_sizes_match_c_layout():
    # natural-alignment layouts of the header structs (x86-64)
    # + n_peers (padded), peer_pix[16], mc_pix, peer_flags[16], rank (padded), signal_seq, wait_seq
    assert C.sizeof(_lib.LrfOutputs) == 7 * 8 + 8 + 16 * 8 + 8 + 16 * 8 + 8 + 16
    assert C.sizeof(_lib.LrfBatch) == 128                            # 116 + refine (int32), padded
    assert C.sizeof(_lib.LrfField) % 8 == 0
    # ... and the compiled library agrees with every ctypes mirror (checked again at load time)
    L = _lib.lib()
    for which, mirror in enumerate((_lib.LrfField, _lib.LrfBatch, _lib.LrfOutputs, _lib.LrfGradients)):
        assert L.lrf_sizeof(which) == C.sizeof(mirror), mirror.__name__
    assert L.lrf_sizeof(99) == 0


def test_validation_errors_without_gpu():
    L = _lib.lib()
    f = _lib.LrfField()
    f.n_dcomp, f.n_acomp = 16, 24        # unsupported component count
    rc = L.lrf_density_feature(C.byref(f), None, 0, None, None)
    assert rc == -2 and b"density_n_comp" in L.lrf_last_error()
    f.n_dcomp = 8
    rc = L.lrf_density_feature(C.byref(f), None, 0, None, None)
    assert rc == -1                       # gridSize 0
    rc = L.lrf_render(C.byref(f), None, None, None, None)
    assert rc == -1


def test_backward_sizes_with_embedded_forward_block_and_validation_without_gpu():
    L = _lib.lib()
    # the forward's prepared block (bf16 operand images of W1B and W2, fp32 b1, b2, W3, b3), then
    # (W1 @ basis)^T [72][128] and W2^T [128][128] in fp32
    assert L.lrf_prepared_backward_bytes() == L.lrf_prepared_bytes() + 4 * (72 * 128 + 128 * 128)
    n, S = 4096, 344
    need = L.lrf_backward_scratch_bytes(n, S)
    # 5 fp32 tables + 2 int32 lists + 1 byte per sample, the per-ray accumulators and the counter
    assert need % 16 == 0 and n * S * 29 + n * 24 + 16 <= need <= n * S * 29 + n * 24 + 16 + 16 * 10
    assert L.lrf_backward_scratch_bytes(2 * n, S) > need
    assert L.lrf_backward_scratch_bytes(-1, S) == 0 and L.lrf_backward_scratch_bytes(n, 1) == 0
    assert C.sizeof(_lib.LrfGradients) == 19 * 8
    f = _lib.LrfField()
    rc = L.lrf_render_backward(C.byref(f), None, None, 0, 0, None, None, None, None, 0, None)
    assert rc == -1 and b"prepared_bwd" in L.lrf_last_error()
    rc = L.lrf_field_prepare_backward(C.byref(f), None, None)
    assert rc == -1


def test_grid_dtype_validation_without_gpu():
    """bf16 grid storage (LrfField.grid_dtype) is accepted by the inference entries only; anything else
    refuses it before touching a device instead of reading 16-bit texels as fp32."""
    L = _lib.lib()
    # grid_dtype sits in what used to be tail padding: the offset is part of the ABI
    assert _lib.LrfField.grid_dtype.offset == _lib.LrfField.n_samples.offset + 4
    f = _lib.LrfField()
    f.n_dcomp, f.n_acomp = 8, 24
    f.grid_dtype = 7
    assert L.lrf_density_feature(C.byref(f), None, 0, None, None) == -1 and b"grid_dtype" in L.lrf_last_error()
    f.grid_dtype = _lib.GRID_BF16
    for call in (lambda: L.lrf_app_products(C.byref(f), None, 0, None, None),
                 lambda: L.lrf_density_l1(C.byref(f), None, None),
                 lambda: L.lrf_density_feature_backward(C.byref(f), None, None, 0, (C.c_void_p * 3)(), (C.c_void_p * 3)(), None, None)):
        assert call() == -2 and b"bf16 grid storage" in L.lrf_last_error()
    assert L.lrf_density_feature(C.byref(f), None, 0, None, None) == -1      # accepted: fails later, on gridSize 0
    assert b"gridSize" in L.lrf_last_error()
    assert L.lrf_pack_bf16(None, None, -1, None) == -1


def test_header_is_plain_c_and_struct_layout_matches(tmp_path):
    """include/localrf_b200.h compiles as C99 (gcc -pedantic -Werror: no C++-isms, no torch / CUDA types in the
    boundary) and a C program that dlopens the library sees the same struct sizes and field offsets as the
    ctypes mirrors -- i.e. a cgo / JNI / plain-C host can bind it as INTEGRATION.md describes."""
    import subprocess
    src = tmp_path / "abi_check.c"
    src.write_text(r'''
#include <dlfcn.h>
#include <stddef.h>
#include <stdio.h>
#include "localrf_b200.h"
int main(int argc, char **argv) {
  void *h = argc > 1 ? dlopen(argv[1], RTLD_NOW | RTLD_LOCAL) : NULL;
  if (!h) { fprintf(stderr, "%s\n", dlerror()); return 2; }
  size_t (*sz)(int32_t) = NULL;
  int (*ver)(void) = NULL;
  *(void **)(&sz) = dlsym(h, "lrf_sizeof");        /* the POSIX idiom for dlsym -> function pointer */
  *(void **)(&ver) = dlsym(h, "lrf_version");
  if (!sz || !ver) return 3;
  if (sz(0) != sizeof(LrfField) || sz(1) != sizeof(LrfBatch) || sz(2) != sizeof(LrfOutputs) ||
      sz(3) != sizeof(LrfGradients)) return 4;
  printf("%d %zu %zu %zu %zu %zu %zu %zu\n", ver(), sizeof(LrfField), offsetof(LrfField, grid_dtype),
         offsetof(LrfField, z_vals), offsetof(LrfBatch, refine), offsetof(LrfOutputs, peer_flags),
         offsetof(LrfOutputs, wait_seq), offsetof(LrfGradients, d_b3));
  return 0;
}
''')
    exe = tmp_path / "abi_check"
    env = dict(os.environ); env.pop("CC", None)
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                        "-o", str(exe), str(src), "-ldl"], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    _lib.lib()                                                     # (builds the library if needed)
    r = subprocess.run([str(exe), _lib.LIB_PATH], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stderr)
    got = [int(v) for v in r.stdout.split()]
    want = [_lib.ABI_VERSION, C.sizeof(_lib.LrfField), _lib.LrfField.grid_dtype.offset, _lib.LrfField.z_vals.offset,
            _lib.LrfBatch.refine.offset, _lib.LrfOutputs.peer_flags.offset, _lib.LrfOutputs.wait_seq.offset,
            _lib.LrfGradients.d_b3.offset]
    assert got == want
