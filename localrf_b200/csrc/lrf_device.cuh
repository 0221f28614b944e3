// lrf_device.cuh -- device-side building blocks shared by the kernels: PTX wrappers (mbarrier, TMA
// bulk copy, wgmma), the warpgroup MLP, ray setup, the VM density / appearance gathers, warp scans.
#pragma once
#include <cuda_bf16.h>

#include <type_traits>

#include "lrf_common.cuh"

namespace lrf {

constexpr int TM = 128;      // appearance samples per MLP tile (two wgmma M = 64 halves)
constexpr float T_EPS = 1e-10f;  // early-termination transmittance

struct RaySm {                     // one ray, as set up by setup_ray
  float o[3];                      // origin in the field's frame
  float vd[3];                     // normalised direction (tensorBase.py:578-580)
  float nrm;                       // |d| before normalisation (depth is divided by it, :615)
  float blend;                     // this field's blending weight for the ray's view
};

// ---- PTX helpers: mbarrier + TMA 1-D bulk copy ---------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes,
                                             uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}

// ---- PTX helpers: wgmma (warpgroup MMA, fp32 accumulators in registers) --------------------------
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// shared-memory matrix descriptor: K-major, no swizzle (8x8 core matrices of 128 contiguous bytes)
// lbo = byte stride between the two K-adjacent core matrices, sbo = between 8-row groups
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, A and B from shared memory (one warpgroup)
__device__ __forceinline__ void wgmma_n128_ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc));
}
// D[64 x 32] (+)= A[64 x 16] * B[32 x 16]^T, A and B from shared memory (one warpgroup)
__device__ __forceinline__ void wgmma_n32_ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc));
}
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, A from registers (the accumulator fragment layout), B from shared memory
__device__ __forceinline__ void wgmma_n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, A from registers (the accumulator fragment layout), B from shared memory
__device__ __forceinline__ void wgmma_n128_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}

// x = hi + lo with hi, lo bf16 (round-to-nearest): ~16 mantissa bits.  Packs two values per word.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  float2 hf = __bfloat1622float2(h);
  __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
// stores 8 consecutive K elements (one 16-byte chunk) of row `row` into the hi and lo operands
__device__ __forceinline__ void store_chunk(unsigned char* hi_base, unsigned char* lo_base, int row,
                                            int kc, int chunks, const float* v) {
  uint4 h, l;
  split2(v[0], v[1], h.x, l.x);
  split2(v[2], v[3], h.y, l.y);
  split2(v[4], v[5], h.z, l.z);
  split2(v[6], v[7], h.w, l.w);
  const int off = (((row >> 3) * chunks + kc) * 8 + (row & 7)) * 16;
  *reinterpret_cast<uint4*>(hi_base + off) = h;
  *reinterpret_cast<uint4*>(lo_base + off) = l;
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, A and B from shared memory; TB = 1 reads B MN-major
template <int TB>
__device__ __forceinline__ void wgmma_n64_ss_t(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc), "n"(TB));
}
// D[64 x 40] (+)= A[64 x 16] * B[40 x 16]^T, A and B from shared memory; TB = 1 reads B MN-major
template <int TB>
__device__ __forceinline__ void wgmma_n40_ss_t(float (&d)[20], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n40k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1, 0, %23;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
      : "l"(a), "l"(b), "r"(acc), "n"(TB));
}

// ---- the MLP of one 64-row half of a 128-row tile, on one warpgroup -----------------------------
// Every product is three bf16 MMAs of hi/lo-split operands (hi*hi + hi*lo + lo*hi per K-step of 16, ~16
// mantissa bits), fp32 accumulation.  Accumulator fragment of thread t of the warpgroup: row
// 16 (t / 32) + (t % 32) / 4 (+ 8 for j = 1), columns 8 i + 2 (t % 4) + {0, 1} (i < N / 8).
__device__ __forceinline__ int wg_row(int j) {
  const int t = threadIdx.x & 127;
  return (t >> 5) * 16 + ((t & 31) >> 2) + 8 * j;
}

// acc[64 x 128] = A[64 x K] * B[128 x K]^T, A and B images in shared memory with `chunks` 16-byte K-chunks
__device__ __forceinline__ void mlp_gemm_n128(float (&acc)[64], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                              uint32_t b_lo, int ksteps, int chunks) {
  const uint32_t sbo = (uint32_t)chunks * 128u;
  wgmma_fence();
  for (int ks = 0; ks < ksteps; ++ks) {
    const uint32_t ko = (uint32_t)ks * 256u;   // two 128-byte core matrices per K-step
    const uint64_t ah = gmma_desc(a_hi + ko, 128u, sbo), al = gmma_desc(a_lo + ko, 128u, sbo);
    const uint64_t bh = gmma_desc(b_hi + ko, 128u, sbo), bl = gmma_desc(b_lo + ko, 128u, sbo);
    wgmma_n128_ss(acc, ah, bh, ks > 0 ? 1u : 0u);
    wgmma_n128_ss(acc, ah, bl, 1u);
    wgmma_n128_ss(acc, al, bh, 1u);
  }
  wgmma_commit();
  wgmma_wait_all();
  fence_regs(acc);
}

// From layer 1's accumulator: h1 = relu(acc + b1) -> layer 2 (A = h1 hi/lo in registers, B = W2 image at
// b2_hi / b2_lo, two N halves of 64) -> h2 = relu(. + b2) -> s[j][c] = W3[c][:128] . h2 of fragment row j,
// reduced over the quad (all four lanes hold the same sums).  The view term and b3 are the caller's.
__device__ __forceinline__ void mlp_layers23(float (&acc)[64], const float* tail, uint32_t b2_hi,
                                             uint32_t b2_lo, float (&s)[2][3]) {
  const int q = threadIdx.x & 3;
  const float* b1 = tail + TAIL_B1;
  const float* b2 = tail + TAIL_B2;
  const float* W3 = tail + TAIL_W3;
  uint32_t ah[FC / 16][4], al[FC / 16][4];
#pragma unroll
  for (int ks = 0; ks < FC / 16; ++ks) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {        // column block 2 ks + h = the A fragment's K 16 ks + 8 h + 2q, +1
      const int i = 2 * ks + h, col = 8 * i + 2 * q;
      const float2 bb = *reinterpret_cast<const float2*>(b1 + col);
      split2(fmaxf(acc[4 * i] + bb.x, 0.0f), fmaxf(acc[4 * i + 1] + bb.y, 0.0f), ah[ks][2 * h], al[ks][2 * h]);
      split2(fmaxf(acc[4 * i + 2] + bb.x, 0.0f), fmaxf(acc[4 * i + 3] + bb.y, 0.0f), ah[ks][2 * h + 1],
             al[ks][2 * h + 1]);
    }
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) s[j][0] = s[j][1] = s[j][2] = 0.0f;
  const uint32_t sbo = (uint32_t)K2_CHUNKS * 128u;
#pragma unroll
  for (int nh = 0; nh < 2; ++nh) {
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.0f;
    const uint32_t bo = (uint32_t)nh * 8u * sbo;   // output rows 64 nh .. of W2
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < FC / 16; ++ks) {
      const uint64_t bh = gmma_desc(b2_hi + bo + ks * 256u, 128u, sbo), bl = gmma_desc(b2_lo + bo + ks * 256u, 128u, sbo);
      wgmma_n64_rs(d, ah[ks], bh, ks > 0 ? 1u : 0u);
      wgmma_n64_rs(d, ah[ks], bl, 1u);
      wgmma_n64_rs(d, al[ks], bh, 1u);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(d);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int col = 64 * nh + 8 * i + 2 * q;
      const float2 bb = *reinterpret_cast<const float2*>(b2 + col);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float h0 = fmaxf(d[4 * i + 2 * j] + bb.x, 0.0f), h1 = fmaxf(d[4 * i + 2 * j + 1] + bb.y, 0.0f);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float2 ww = *reinterpret_cast<const float2*>(W3 + c * W3_LD + col);
          s[j][c] = fmaf(ww.y, h1, fmaf(ww.x, h0, s[j][c]));
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      s[j][c] += __shfl_xor_sync(0xffffffffu, s[j][c], 1);
      s[j][c] += __shfl_xor_sync(0xffffffffu, s[j][c], 2);
    }
}

// ---- ray setup (local_tensorfs.py:397-456 / tensorBase.py:578-580) ------------------------------
// origin o, |d| and the normalised direction d / |d| (R.blend is the caller's)
__device__ __forceinline__ void normalize_ray(const float* o, const float* d, RaySm& R) {
  float n = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  R.nrm = n;
#pragma unroll
  for (int a = 0; a < 3; ++a) { R.o[a] = o[a]; R.vd[a] = __fdiv_rn(d[a], n); }
}

__device__ __forceinline__ void setup_ray(const BatchDev& B, long long r, RaySm& R) {
  float o[3], d[3];
  long long view = 0;
  if (B.rays) {
    const float* p = B.rays + 6 * r;
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
    d[0] = p[3]; d[1] = p[4]; d[2] = p[5];
    if (B.rays_per_view > 0) view = r / B.rays_per_view;
  } else {
    view = r / B.rays_per_view;
    long long id = B.ray_ids[r];
    long long col = id % B.W, row = (id / B.W) % B.H;            // ids2pixel
    float i = (float)col + 0.5f, j = (float)row + 0.5f;
    float dc[3];
    if (B.fov360) {                                               // get_ray_directions_360
      const float pi = 3.14159265358979323846f;
      float phi = j * pi / (float)B.H - pi / 2.0f;
      float theta = i * 2.0f * pi / (float)B.W + pi;
      float sp, cp, st, ct;
      sincosf(phi, &sp, &cp);
      sincosf(theta, &st, &ct);
      dc[0] = cp * st; dc[1] = sp; dc[2] = cp * ct;
    } else {                                                      // get_ray_directions_lean
      float focal = B.focal, cx = B.cx, cy = B.cy;
      if (B.intrinsics) { focal = B.intrinsics[0]; cx = B.intrinsics[1]; cy = B.intrinsics[2]; }
      dc[0] = __fdiv_rn(i - cx, focal);
      dc[1] = -__fdiv_rn(j - cy, focal);
      dc[2] = -1.0f;
    }
    if (B.dirs) { B.dirs[3 * r] = dc[0]; B.dirs[3 * r + 1] = dc[1]; B.dirs[3 * r + 2] = dc[2]; }
    if (B.ij) { B.ij[2 * r] = col; B.ij[2 * r + 1] = row; }
    const float* c = B.c2w + 12 * view;
#pragma unroll
    for (int a = 0; a < 3; ++a) {                                 // get_rays_lean
      o[a] = c[a * 4 + 3] + (B.w2rf ? B.w2rf[a] : 0.0f);
      d[a] = c[a * 4 + 0] * dc[0] + c[a * 4 + 1] * dc[1] + c[a * 4 + 2] * dc[2];
    }
  }
  normalize_ray(o, d, R);
  R.blend = B.blend ? B.blend[view * B.blend_stride] : 1.0f;
}

// sample position in the field's normalised [-1,1]^3 grid coordinates (tensorBase.py:438-440,602)
__device__ __forceinline__ void sample_pos(const FieldDev& F, const RaySm& R, float z, float* p,
                                           float* q) {
  p[0] = R.o[0] + R.vd[0] * z; p[1] = R.o[1] + R.vd[1] * z; p[2] = R.o[2] + R.vd[2] * z;
  contract(p[0], p[1], p[2]);
#pragma unroll
  for (int a = 0; a < 3; ++a) q[a] = (p[a] - F.amin[a]) * F.ainv[a] - 1.0f;
}

// AlphaGridMask.sample_alpha (tensorBase.py:51-58): trilinear, zero padding, align_corners=True
__device__ __forceinline__ float alpha_mask(const FieldDev& F, const float* p) {
  int D = F.ad[0], H = F.ad[1], W = F.ad[2];
  float ix = (((p[0] - F.aamin[0]) * F.aainv[0] - 1.0f + 1.0f) * 0.5f) * (float)(W - 1);
  float iy = (((p[1] - F.aamin[1]) * F.aainv[1] - 1.0f + 1.0f) * 0.5f) * (float)(H - 1);
  float iz = (((p[2] - F.aamin[2]) * F.aainv[2] - 1.0f + 1.0f) * 0.5f) * (float)(D - 1);
  float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
  int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
  float tx = ix - fx, ty = iy - fy, tz = iz - fz;
  float v = 0.0f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int xx = x0 + (c & 1), yy = y0 + ((c >> 1) & 1), zz = z0 + (c >> 2);
    if (xx < 0 || xx >= W || yy < 0 || yy >= H || zz < 0 || zz >= D) continue;
    float w = ((c & 1) ? tx : 1.0f - tx) * ((c & 2) ? ty : 1.0f - ty) * ((c & 4) ? tz : 1.0f - tz);
    v += __ldg(F.alpha_vol + ((size_t)zz * H + yy) * W + xx) * w;
  }
  return v;
}

// ---- the VM (plane x line) lookup (tensoRF.py:112-194) -------------------------------------------
// Grids are channel-last: plane i is [H][W][C] texels, line i is [L][C].  Component c of pair i at a point is
// (a w00 + b w01 + c w10 + d w11) * (u (1 - tl) + v tl), a..d the plane's four taps, u, v the line's two.
// Texels are fp32, or bf16 with 16-bit grid storage (LrfField.grid_dtype = LRF_GRID_BF16): half the sectors
// and half the load instructions.  bf16 -> fp32 is exact (a 16-bit shift) and the arithmetic is the same
// expressions, so a field whose parameters are bf16-representable gives the same values from either storage.
template <bool H16>
using Texel = std::conditional_t<H16, __nv_bfloat16, float>;
template <bool H16>
__device__ __forceinline__ const Texel<H16>* texels(const float* grid) {
  return reinterpret_cast<const Texel<H16>*>(grid);
}

struct VmTap {                     // one plane / line pair at one point
  size_t p00, p01, p10, p11;       // element offsets of the plane's four taps ([y][x])
  size_t l0, l1;                   // and of the line's two
  float w00, w01, w10, w11;        // bilinear weights
  float u0, tl;                    // linear weights of l0 and l1 (u0 = 1 - tl)
};

template <int C>
__device__ __forceinline__ VmTap vm_tap(const int* g3, int i, const float* q) {
  const int W = g3[mat0(i)], H = g3[mat1(i)], L = g3[vecm(i)];
  int x0, x1, y0, y1, l0, l1;
  float tx, ty, tl;
  grid_coord(q[mat0(i)], W, x0, x1, tx);
  grid_coord(q[mat1(i)], H, y0, y1, ty);
  grid_coord(q[vecm(i)], L, l0, l1, tl);
  VmTap t;
  t.p00 = ((size_t)y0 * W + x0) * C; t.p01 = ((size_t)y0 * W + x1) * C;
  t.p10 = ((size_t)y1 * W + x0) * C; t.p11 = ((size_t)y1 * W + x1) * C;
  t.l0 = (size_t)l0 * C; t.l1 = (size_t)l1 * C;
  t.w00 = (1.0f - tx) * (1.0f - ty); t.w01 = tx * (1.0f - ty);
  t.w10 = (1.0f - tx) * ty; t.w11 = tx * ty;
  t.u0 = 1.0f - tl; t.tl = tl;
  return t;
}

// one 16-byte piece of a texel as floats: 4 fp32 components, or 8 bf16 ones
__device__ __forceinline__ void ldg_texel(const float* p, float (&v)[4]) {
  const float4 r = ldg4(p);
  v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w;
}
__device__ __forceinline__ void ldg_texel(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
  v[0] = __uint_as_float(r.x << 16); v[1] = __uint_as_float(r.x & 0xffff0000u);
  v[2] = __uint_as_float(r.y << 16); v[3] = __uint_as_float(r.y & 0xffff0000u);
  v[4] = __uint_as_float(r.z << 16); v[5] = __uint_as_float(r.z & 0xffff0000u);
  v[6] = __uint_as_float(r.w << 16); v[7] = __uint_as_float(r.w & 0xffff0000u);
}

// components c .. c + N - 1 of one pair at tap t: out[e] = bilinear(plane) * linear(line), one 16-byte piece
// of each of the six texels at a time
template <int N, class T>
__device__ __forceinline__ void vm_products(const VmTap& t, const T* plane, const T* line, int c, float* out) {
  constexpr int U = 16 / sizeof(T);
  static_assert(N % U == 0, "whole 16-byte pieces");
#pragma unroll
  for (int h = c; h < c + N; h += U) {
    float a[U], b[U], cc[U], d[U], u[U], v[U];
    ldg_texel(plane + t.p00 + h, a); ldg_texel(plane + t.p01 + h, b);
    ldg_texel(plane + t.p10 + h, cc); ldg_texel(plane + t.p11 + h, d);
    ldg_texel(line + t.l0 + h, u); ldg_texel(line + t.l1 + h, v);
#pragma unroll
    for (int e = 0; e < U; ++e)
      out[h - c + e] = (a[e] * t.w00 + b[e] * t.w01 + cc[e] * t.w10 + d[e] * t.w11) * (u[e] * t.u0 + v[e] * t.tl);
  }
}

// compute_densityfeature for one point (tensoRF.py:112-151): components 0..7 of each plane, then planes 0, 1, 2
template <bool H16>
__device__ __forceinline__ float density_feature_t(const FieldDev& F, const float* q) {
  float sigma = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float v[CD];
    vm_products<CD>(vm_tap<CD>(F.g, i, q), texels<H16>(F.dplane[i]), texels<H16>(F.dline[i]), 0, v);
    float s = 0.0f;
#pragma unroll
    for (int e = 0; e < CD; ++e) s += v[e];
    sigma += s;
  }
  return sigma;
}

// one plane's 24 appearance features of one point (tensoRF.py:153-194): out[c] = plane_c * line_c
template <bool H16>
__device__ __forceinline__ void app_plane_features_t(const FieldDev& F, int i, const float* q, float* out /*[CA]*/) {
  const VmTap t = vm_tap<CA>(F.g, i, q);
#pragma unroll
  for (int c = 0; c < CA; c += 8) vm_products<8>(t, texels<H16>(F.aplane[i]), texels<H16>(F.aline[i]), c, out + c);
}

// ---- one sample of the march (tensorBase.py:581-610) ---------------------------------------------
// alpha of sample k < S of ray R; fe = its density feature and valid = whether it was looked up (not the
// last sample, inside the alpha mask), fe = 0 where not
template <bool H16>
__device__ __forceinline__ float sample_alpha(const FieldDev& F, const RaySm& R, int k, int S, float& fe,
                                              bool& valid) {
  const float z = __ldg(F.z + k);
  float p[3], q[3];
  sample_pos(F, R, z, p, q);
  valid = (k != S - 1);                                       // ray_valid[:, -1] = 0
  if (valid && F.alpha_vol) valid = alpha_mask(F, p) > 0.0f;  // tensorBase.py:593-598
  float sigma = 0.0f;
  fe = 0.0f;
  if (valid) {
    fe = density_feature_t<H16>(F, q);
    sigma = feature2density(fe, F.density_shift, F.act);
  }
  const float dist = (k + 1 < S ? __ldg(F.z + k + 1) : z) - z;    // the last sample's dist is 0 (tensorBase.py:584-587)
  float alpha = 1.0f - expf(-sigma * dist * F.distance_scale);   // tensorBase.py:610, same form
  if (k == S - 1) alpha = 1.0f;                                  // alpha[:, -1] = 1
  return alpha;
}

// ---- backward of the VM lookup (F.grid_sample align_corners=True, padding_mode="border") ----------------
// pixel coordinate, its two taps and d(pixel)/d(normalised coordinate) (0 when clipped: ATen clip_coordinates_set_grad)
__device__ __forceinline__ void grid_coord_grad(float c, int size, int& i0, int& i1, float& t,
                                                float& dcoord) {
  float x = ((c + 1.0f) * 0.5f) * (float)(size - 1);
  dcoord = (x <= 0.0f || x >= (float)(size - 1)) ? 0.0f : 0.5f * (float)(size - 1);
  x = fminf((float)(size - 1), fmaxf(x, 0.0f));
  const float f = floorf(x);
  i0 = (int)f;
  i1 = min(i0 + 1, size - 1);
  t = x - f;
}

// Device only: the gradient scatter needs global atomics, which the host build of this header
// (tests/host_emul, for the forward building blocks) does not provide.
#ifdef __CUDACC__
// 16-byte vector reduction (red.global.add.v4.f32, sm_90+): one atomic per 4 components
__device__ __forceinline__ void red4(float* p, float x, float y, float z, float w) {
  atomicAdd(reinterpret_cast<float4*>(p), make_float4(x, y, z, w));
}

// backward of one plane/line pair with C components, over the 4-component groups c_first, c_first + c_step, ...
// (UNROLL of them per loop step).  g(c) = dL/d(plane_c * line_c).  Parameter gradients are accumulated by atomic
// adds, four components at a time; the gradient of the normalised point is added to dq.
template <int C, int UNROLL = 2, class G>
__device__ __forceinline__ void vm_pair_backward(const int* g3, int i, const float* plane,
                                                 const float* line, float* d_plane, float* d_line,
                                                 const float* q, G g, float* dq, int c_first = 0, int c_step = 4) {
  const int W = g3[mat0(i)], H = g3[mat1(i)], L = g3[vecm(i)];
  int x0, x1, y0, y1, l0, l1;
  float tx, ty, tl, dx, dy, dl;
  grid_coord_grad(q[mat0(i)], W, x0, x1, tx, dx);
  grid_coord_grad(q[mat1(i)], H, y0, y1, ty, dy);
  grid_coord_grad(q[vecm(i)], L, l0, l1, tl, dl);
  const size_t o00 = ((size_t)y0 * W + x0) * C, o01 = ((size_t)y0 * W + x1) * C;
  const size_t o10 = ((size_t)y1 * W + x0) * C, o11 = ((size_t)y1 * W + x1) * C;
  const size_t ol0 = (size_t)l0 * C, ol1 = (size_t)l1 * C;
  const float w00 = (1.0f - tx) * (1.0f - ty), w01 = tx * (1.0f - ty);
  const float w10 = (1.0f - tx) * ty, w11 = tx * ty, u0 = 1.0f - tl;
  float gx = 0.0f, gy = 0.0f, gl = 0.0f;
#pragma unroll UNROLL
  for (int c = c_first; c < C; c += c_step) {
    const float4 a = ldg4(plane + o00 + c), b = ldg4(plane + o01 + c);
    const float4 cc = ldg4(plane + o10 + c), d = ldg4(plane + o11 + c);
    const float4 u = ldg4(line + ol0 + c), v = ldg4(line + ol1 + c);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
    const float cv[4] = {cc.x, cc.y, cc.z, cc.w}, dv[4] = {d.x, d.y, d.z, d.w};
    const float uv[4] = {u.x, u.y, u.z, u.w}, vv[4] = {v.x, v.y, v.z, v.w};
    float dP[4], dLc[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float P = av[e] * w00 + bv[e] * w01 + cv[e] * w10 + dv[e] * w11;
      const float Lc = uv[e] * u0 + vv[e] * tl;
      const float gc = g(c + e);
      dP[e] = gc * Lc;
      dLc[e] = gc * P;
      gx += dP[e] * ((bv[e] - av[e]) * (1.0f - ty) + (dv[e] - cv[e]) * ty);
      gy += dP[e] * ((cv[e] - av[e]) * (1.0f - tx) + (dv[e] - bv[e]) * tx);
      gl += dLc[e] * (vv[e] - uv[e]);
    }
    red4(d_plane + o00 + c, dP[0] * w00, dP[1] * w00, dP[2] * w00, dP[3] * w00);
    red4(d_plane + o01 + c, dP[0] * w01, dP[1] * w01, dP[2] * w01, dP[3] * w01);
    red4(d_plane + o10 + c, dP[0] * w10, dP[1] * w10, dP[2] * w10, dP[3] * w10);
    red4(d_plane + o11 + c, dP[0] * w11, dP[1] * w11, dP[2] * w11, dP[3] * w11);
    red4(d_line + ol0 + c, dLc[0] * u0, dLc[1] * u0, dLc[2] * u0, dLc[3] * u0);
    red4(d_line + ol1 + c, dLc[0] * tl, dLc[1] * tl, dLc[2] * tl, dLc[3] * tl);
  }
  dq[mat0(i)] += gx * dx;
  dq[mat1(i)] += gy * dy;
  dq[vecm(i)] += gl * dl;
}
#endif  // __CUDACC__

// ---- warp primitives ----------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// inclusive product scan across the warp
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= u;
  }
  return v;
}

// transmittance of one 32-sample chunk of a ray, lane = sample (tensorBase.py:23-31): T = carry times the
// product of (1 - alpha) + 1e-10 over the chunk's earlier samples, w = alpha T; then carry moves past the chunk.
// Lanes past the ray's end (in = false) take part with a factor of 1.  use() runs once T and w are set, before
// the carry's shuffle: the render producer accumulates and stores there (placed after the shuffle, that code
// made ptxas spill 60-100 B more per thread in the render kernels).
struct NoUse {
  __device__ __forceinline__ void operator()() const {}
};
template <class Use = NoUse>
__device__ __forceinline__ void transmittance_step(float alpha, bool in, int lane, float& carry, float& T,
                                                   float& w, Use use = {}) {
  const float inc = warp_scan_mul(in ? (1.0f - alpha) + 1e-10f : 1.0f, lane);
  float exc = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) exc = 1.0f;
  T = carry * exc;
  w = alpha * T;
  use();
  carry *= __shfl_sync(0xffffffffu, inc, 31);
}

}  // namespace lrf
