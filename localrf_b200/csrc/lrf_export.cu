// lrf_export.cu -- the scene's geometry as a coloured point cloud: each rendered ray's expected-depth point in the
// world frame, merged into a voxel grid on the device.
//
// lrf_ray_opacity folds a field's per-sample weights (LrfOutputs.weights of its lrf_render launch) into the ray's
// blended opacity.  lrf_frame_points back-projects each kept ray of one view and adds it to an open-addressing table
// of 64-bit integer sums keyed by voxel; integer sums commute, so the table's content does not depend on thread
// scheduling, on how the rays are chunked or on the order of the frames, and atomics are used freely.
// lrf_voxel_extract sorts the occupied slots by key (KeySlotSort, a radix sort) and writes one point per voxel:
// whatever the slot layout, the output is bitwise repeatable.  The table's conventions are lrf_table.cuh's.
//
// The back-projection and the key are written with explicit round-to-nearest fp32 operations in a fixed order (no
// FMA contraction), so a numpy float32 restatement reproduces them bit for bit; the per-voxel means are fp64, rounded
// once.
//
// lrf_frame_colours / lrf_colour_extract colour given points (a mesh's vertices, a cloud's points) from the video's
// frames: each point is projected into one rendered view, tested against the view's expected depth, and the frame's
// pixel is added to the point's integer sums; the blend is fp64, rounded once.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/localrf_b200.h"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"
#include "lrf_table.cuh"

namespace lrf {

namespace {

constexpr int OP_RAYS = 128;           // rays per CTA of ray_opacity_kernel (one per thread)
constexpr int OP_TILE = 32;            // samples per tile staged through shared memory
constexpr int PT_THREADS = 256;
constexpr int EX_THREADS = 256;
constexpr int CO_THREADS = 256;
constexpr int KEY_BITS = 21;           // per axis: keys in [-2^20, 2^20), 63 bits in all
constexpr float KEY_LIM = 1048576.0f;  // 2^20

// One thread per ray sums its weights in sample order in fp64, from -0 (the identity of IEEE addition, so a row of -0
// sums to -0 as np.cumsum does).  The [rays][S] rows are read a tile at a time, coalesced, into padded shared rows, so
// every thread's sequential sum reads its own row without bank conflicts.
__global__ void __launch_bounds__(OP_RAYS) ray_opacity_kernel(const float* __restrict__ w, long long n, int S,
                                                              long long rays_per_view, const float* __restrict__ blend,
                                                              long long blend_stride, int accumulate, float* acc) {
  __shared__ float tile[OP_RAYS][OP_TILE + 1];
  const long long r0 = (long long)blockIdx.x * OP_RAYS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double s = -0.0;
  for (int k0 = 0; k0 < S; k0 += OP_TILE) {
    __syncthreads();
    for (int row = warp; row < OP_RAYS; row += OP_RAYS / 32) {
      const long long r = r0 + row;
      const int k = k0 + lane;
      tile[row][lane] = (r < n && k < S) ? __ldg(w + r * S + k) : 0.0f;
    }
    __syncthreads();
    const int m = min(OP_TILE, S - k0);
    for (int j = 0; j < m; ++j) s += (double)tile[threadIdx.x][j];
  }
  const long long r = r0 + threadIdx.x;
  if (r >= n) return;
  const float b = blend ? blend[(r / rays_per_view) * blend_stride] : 1.0f;
  const float a = __fmul_rn(b, (float)s);
  acc[r] = accumulate ? __fadd_rn(acc[r], a) : a;
}

// The table's claim counter is stats[2], the occupied slots.
__global__ void __launch_bounds__(PT_THREADS) frame_points_kernel(const LrfPointFrame f, const LrfVoxelTable t) {
  const long long r = (long long)blockIdx.x * PT_THREADS + threadIdx.x;
  const unsigned long long half = (unsigned long long)t.capacity >> 1;
  bool keep = false, out = false;
  unsigned long long key = 0, fs[3];
  unsigned int cs[3];
  if (r < f.n_rays && claim_count(t.stats + 2) <= half) {
    const float a = f.acc[r], d = f.depth[r];
    if (a >= f.min_acc && a > 0.0f && isfinite(d)) {
      const float s = __fdiv_rn(d, a);
      float c[3], p[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) c[i] = __fmul_rn(f.directions[3 * r + i], s);
      const float* M = f.cam2world;
#pragma unroll
      for (int i = 0; i < 3; ++i)
        p[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[4 * i], c[0]), __fmul_rn(M[4 * i + 1], c[1])),
                                   __fmul_rn(M[4 * i + 2], c[2])), M[4 * i + 3]);
      bool inside = false;
      for (int k = 0; k < f.n_fields && !inside; ++k) {
        if (f.blend && !(f.blend[k] > 0.0f)) continue;
        const float* o = f.world2rf + 3 * k;         // (each comparison is false for NaN)
        inside = fabsf(__fadd_rn(p[0], o[0])) <= f.max_norm && fabsf(__fadd_rn(p[1], o[1])) <= f.max_norm &&
                 fabsf(__fadd_rn(p[2], o[2])) <= f.max_norm;
      }
      if (inside) {
        bool in_range = true;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float q = __fdiv_rn(__fsub_rn(p[i], t.origin[i]), t.voxel_size);
          const float k = floorf(q);
          in_range = in_range && k >= -KEY_LIM && k < KEY_LIM;
          if (in_range) {
            const float fr = __fsub_rn(q, k);
            const unsigned long long u = __float2ull_rz(__fmul_rn(fr, 4294967296.0f));
            fs[i] = u < 0xffffffffull ? u : 0xffffffffull;
            key = (key << KEY_BITS) | (unsigned long long)((int)k + (1 << 20));
          }
        }
        keep = in_range;
        out = !in_range;
        if (keep)
#pragma unroll
          for (int i = 0; i < 3; ++i)
            cs[i] = __float2uint_rz(__fmul_rn(fminf(fmaxf(f.rgb[3 * r + i], 0.0f), 1.0f), 16777216.0f));
      }
    }
  }
  const unsigned mk = __ballot_sync(0xffffffffu, keep), mo = __ballot_sync(0xffffffffu, out);
  if ((threadIdx.x & 31) == 0) {
    if (mk) atomicAdd(t.stats + 0, (unsigned long long)__popc(mk));
    if (mo) atomicAdd(t.stats + 1, (unsigned long long)__popc(mo));
  }
  if (!keep) return;
  find_or_claim(t.keys, t.capacity, t.stats + 2, key, [&](unsigned long long slot, bool) {
    unsigned long long* v = t.sums + 7 * slot;
    atomicAdd(v, 1ull);
#pragma unroll
    for (int i = 0; i < 3; ++i) atomicAdd(v + 1 + i, fs[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i) atomicAdd(v + 4 + i, (unsigned long long)cs[i]);
  });
}

// One thread per point: the pixel of the view that sees it, the depth test against the view's rendered depth, then
// the integer sums of lrf_frame_colours (include/localrf_b200.h, which states every operation).  Each point is one
// thread's, so the atomics never contend; they keep the sums exact when frames of one table run on several streams.
__global__ void __launch_bounds__(CO_THREADS) frame_colours_kernel(const LrfColourFrame f, const float* __restrict__ xyz,
                                                                   const float* __restrict__ normals, long long n,
                                                                   unsigned long long* sums) {
  const long long p = (long long)blockIdx.x * CO_THREADS + threadIdx.x;
  if (p >= n) return;
  const float* M = f.cam2world;
  float x[3], e[3], c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    x[a] = xyz[3 * p + a];
    e[a] = __fsub_rn(x[a], M[4 * a + 3]);
  }
#pragma unroll
  for (int b = 0; b < 3; ++b)
    c[b] = __fadd_rn(__fadd_rn(__fmul_rn(M[b], e[0]), __fmul_rn(M[4 + b], e[1])), __fmul_rn(M[8 + b], e[2]));
  long long i, j;
  float dv;
  if (f.fov360) {
    dv = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2])));
    if (!(dv > 0.0f) || !isfinite(dv)) return;
    const float pi = 3.14159265358979323846f;
    const float phi = asinf(fminf(fmaxf(__fdiv_rn(c[1], dv), -1.0f), 1.0f));
    const float theta = atan2f(c[0], c[2]);               // both finite, so are the quotients below
    j = (long long)floorf(__fdiv_rn(__fmul_rn(__fadd_rn(phi, pi / 2.0f), (float)f.H), pi));
    j = j < 0 ? 0 : (j > f.H - 1 ? f.H - 1 : j);
    i = (long long)floorf(__fdiv_rn(__fmul_rn(__fsub_rn(theta, pi), (float)f.W), __fmul_rn(2.0f, pi))) % f.W;
    if (i < 0) i += f.W;
  } else {
    if (!(c[2] < 0.0f)) return;
    dv = -c[2];
    const float* K = f.intrinsics;
    const float u = floorf(__fadd_rn(__fmul_rn(__fdiv_rn(c[0], dv), K[0]), K[1]));
    const float v = floorf(__fadd_rn(__fmul_rn(__fdiv_rn(-c[1], dv), K[0]), K[2]));
    if (!(u >= 0.0f && (double)u < (double)f.W && v >= 0.0f && (double)v < (double)f.H)) return;
    i = (long long)u;
    j = (long long)v;
  }
  const long long k = j * f.W + i;
  const float acc = f.acc[k];
  const float s = __fdiv_rn(f.depth[k], acc);
  if (!(acc >= f.min_acc && acc > 0.0f && isfinite(s) && s > 0.0f &&
        fabsf(__fsub_rn(dv, s)) <= __fmul_rn(f.depth_tol, s)))
    return;
  float w = 1.0f;
  if (normals) {
    float t[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) t[a] = __fsub_rn(M[4 * a + 3], x[a]);
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(t[0], t[0]), __fmul_rn(t[1], t[1])), __fmul_rn(t[2], t[2])));
    const float* nv = normals + 3 * p;
    w = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(nv[0], t[0]), __fmul_rn(nv[1], t[1])), __fmul_rn(nv[2], t[2])), len);
    if (!(w >= f.min_cos)) return;
  }
  const float* px = f.image + 3 * k;
  const float r = px[0], g = px[1], b = px[2];
  if (!isfinite(r) || !isfinite(g) || !isfinite(b)) return;
  const unsigned long long q = __float2uint_rz(__fmul_rn(fminf(w, 1.0f), 65536.0f));
  unsigned long long* v = sums + 5 * p;
  atomicAdd(v, 1ull);
  atomicAdd(v + 1, q);
  atomicAdd(v + 2, q * __float2uint_rz(__fmul_rn(fminf(fmaxf(r, 0.0f), 1.0f), 16777216.0f)));
  atomicAdd(v + 3, q * __float2uint_rz(__fmul_rn(fminf(fmaxf(g, 0.0f), 1.0f), 16777216.0f)));
  atomicAdd(v + 4, q * __float2uint_rz(__fmul_rn(fminf(fmaxf(b, 0.0f), 1.0f), 16777216.0f)));
}

__global__ void __launch_bounds__(CO_THREADS) colour_extract_kernel(const unsigned long long* __restrict__ sums,
                                                                    long long n, unsigned char* rgb, int* count) {
  const long long p = (long long)blockIdx.x * CO_THREADS + threadIdx.x;
  if (p >= n) return;
  const unsigned long long* v = sums + 5 * p;
  const unsigned long long views = v[0], q = v[1];
  count[p] = views < 2147483647ull ? (int)views : 2147483647;
  const double den = __dmul_rn(__ull2double_rn(q), 16777216.0);
#pragma unroll
  for (int a = 0; a < 3; ++a)
    rgb[3 * p + a] = q == 0 ? 0 : (unsigned char)floor(__dadd_rn(__dmul_rn(__ddiv_rn(__ull2double_rn(v[2 + a]), den),
                                                                            255.0), 0.5));
}

// sort input: the key of every slot holding at least min_count points, NO_KEY (sorted last) for the others
__global__ void __launch_bounds__(EX_THREADS) voxel_keys_kernel(const LrfVoxelTable t, unsigned long long min_count,
                                                                unsigned long long* keys, unsigned int* slots) {
  const long long i = (long long)blockIdx.x * EX_THREADS + threadIdx.x;
  if (i >= t.capacity) return;
  const unsigned long long tag = t.keys[i];
  keys[i] = (tag != 0 && t.sums[7 * i] >= min_count) ? tag - 1 : NO_KEY;
  slots[i] = (unsigned int)i;
}

__global__ void __launch_bounds__(EX_THREADS) voxel_write_kernel(const LrfVoxelTable t, const unsigned long long* keys,
                                                                 const unsigned int* slots, float* xyz,
                                                                 unsigned char* rgb, int* count, long long* n_out) {
  const long long i = (long long)blockIdx.x * EX_THREADS + threadIdx.x;
  if (i >= t.capacity) return;
  const unsigned long long key = keys[i];
  if (key == NO_KEY) {
    if (i == 0) *n_out = 0;
    return;
  }
  if (i + 1 == t.capacity || keys[i + 1] == NO_KEY) *n_out = i + 1;
  const unsigned long long* v = t.sums + 7 * (unsigned long long)slots[i];
  const unsigned long long n = v[0];
  const double cnt = __ull2double_rn(n);
  const double fden = __dmul_rn(cnt, 4294967296.0), cden = __dmul_rn(cnt, 16777216.0);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long k = (long long)((key >> (KEY_BITS * (2 - a))) & ((1ull << KEY_BITS) - 1)) - (1 << 20);
    const double pos = __dadd_rn((double)k, __ddiv_rn(__ull2double_rn(v[1 + a]), fden));
    xyz[3 * i + a] = __double2float_rn(__dadd_rn((double)t.origin[a], __dmul_rn(pos, (double)t.voxel_size)));
    const double c = __dadd_rn(__dmul_rn(__ddiv_rn(__ull2double_rn(v[4 + a]), cden), 255.0), 0.5);
    rgb[3 * i + a] = (unsigned char)floor(c);
  }
  count[i] = n < 2147483647ull ? (int)n : 2147483647;
}

// The extract's scratch: the sort's buffers of the slots' keys and indices, then the sort's temporary storage.  With a
// null base only the size is computed.
struct ExtractScratch {
  KeySlotSort pairs;
  void* temp;
  size_t temp_bytes;
  size_t total;
};

cudaError_t extract_scratch(void* base, long long cap, ExtractScratch& x) {
  ScratchCarver c(base);
  x.pairs.carve(c, cap);
  const cudaError_t e = KeySlotSort::temp_bytes(cap, x.temp_bytes);
  x.temp = c.take(x.temp_bytes, 256);
  x.total = c.size(256);
  return e;
}

}  // namespace

cudaError_t launch_ray_opacity(const float* w, long long n, int S, long long n_views, const float* blend,
                               long long blend_stride, int accumulate, float* acc, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((n + OP_RAYS - 1) / OP_RAYS);
  ray_opacity_kernel<<<blocks, OP_RAYS, 0, stream>>>(w, n, S, n / n_views, blend, blend_stride, accumulate, acc);
  return cudaGetLastError();
}

cudaError_t launch_frame_points(const LrfPointFrame& f, const LrfVoxelTable& t, cudaStream_t stream) {
  if (f.n_rays == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((f.n_rays + PT_THREADS - 1) / PT_THREADS);
  frame_points_kernel<<<blocks, PT_THREADS, 0, stream>>>(f, t);
  return cudaGetLastError();
}

cudaError_t launch_frame_colours(const LrfColourFrame& f, const float* xyz, const float* normals, long long n,
                                 unsigned long long* sums, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  frame_colours_kernel<<<(unsigned)((n + CO_THREADS - 1) / CO_THREADS), CO_THREADS, 0, stream>>>(f, xyz, normals, n,
                                                                                               sums);
  return cudaGetLastError();
}

cudaError_t launch_colour_extract(const unsigned long long* sums, long long n, unsigned char* rgb, int* count,
                                  cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  colour_extract_kernel<<<(unsigned)((n + CO_THREADS - 1) / CO_THREADS), CO_THREADS, 0, stream>>>(sums, n, rgb, count);
  return cudaGetLastError();
}

cudaError_t voxel_extract_scratch_bytes(long long cap, size_t& bytes) {
  ExtractScratch x;
  const cudaError_t e = extract_scratch(nullptr, cap, x);
  bytes = x.total;
  return e;
}

cudaError_t launch_voxel_extract(const LrfVoxelTable& t, long long min_count, float* xyz, unsigned char* rgb,
                                 int* count, long long* n_out, void* scratch, cudaStream_t stream) {
  ExtractScratch x;
  cudaError_t e = extract_scratch(scratch, t.capacity, x);
  if (e != cudaSuccess) return e;
  const unsigned blocks = (unsigned)((t.capacity + EX_THREADS - 1) / EX_THREADS);
  voxel_keys_kernel<<<blocks, EX_THREADS, 0, stream>>>(t, (unsigned long long)min_count, x.pairs.keys(),
                                                        x.pairs.slots());
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = x.pairs.sort(t.capacity, x.temp, x.temp_bytes, stream)) != cudaSuccess) return e;
  voxel_write_kernel<<<blocks, EX_THREADS, 0, stream>>>(t, x.pairs.keys(), x.pairs.slots(), xyz, rgb, count, n_out);
  return cudaGetLastError();
}

}  // namespace lrf
