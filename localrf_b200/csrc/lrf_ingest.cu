// lrf_ingest.cu -- one training frame into its slot of the frame store, from the decoded pixels of its files: the
// per-frame conversions of LocalRFDataset.read_meta (dataLoader/localrf_dataset.py:143-258) after cv2.imread, bit for
// bit (the rules are stated in include/localrf_b200.h and restated in numpy in tests/ingest_oracle.py).
//
// Launches, in order, on the caller's stream:
//   image_kernel      rgb = bgr / 255 (reduced by k in {2, 4}) into the slot, and the 8-bit grey value
//   laplacian_kernel  the 4-neighbour Laplacian of the grey image, reflect-101 borders
//   leaf_sums_kernel  } numpy's float32 pairwise sum of the Laplacian, then of its squared deviations from the mean:
//   tree_sum_kernel   } every leaf of numpy's recursion (<= 128 values, eight accumulators) is one thread's slot of
//   leaf_sums_kernel  } a 2^D-slot tree, and one CTA adds the slots back up in the recursion's order; empty slots
//   tree_sum_kernel   } (below a leaf shallower than D) pass the left value through
//   weight_kernel     loss_weight = variance (times the motion mask)
//   flow_kernel       both flows, resized as uint16, decoded and scaled
//   depth_kernel      inverse depth, resized as fp32
// Every arithmetic step that rounds is written with an explicit _rn intrinsic so that nothing is contracted to an
// FMA: the results must equal cv2 / numpy, which do not fuse these operations.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <initializer_list>

#include "../../include/localrf_b200.h"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

namespace {

constexpr int INGEST_THREADS = 256;
constexpr int TREE_THREADS = 1024;
constexpr int LEAF = 128;                // numpy's PW_BLOCKSIZE
constexpr int MAX_TREE_DEPTH = 16;

// Resize modes of one plane: 0 enlarge, 1 copy, k = 2 or 4 reduce.
int resize_mode(int ws, int hs, int w, int h) {
  if (ws == w && hs == h) return 1;
  for (int k = 2; k <= 4; k += 2)
    if (ws == k * w && hs == k * h) return k;
  return (ws <= w && hs <= h) ? 0 : -1;
}

// cv2's INTER_AREA enlargement weights along one axis: source index and the next index's weight.  The product and
// the difference each round once in double, as the host computes them: a DFMA would leave a residue of a few 1e-16
// where the weight is exactly 0 (6 -> 8 at d = 3), which a zero sample next to a large one shows in fp32.
__device__ __forceinline__ void area_weight(int d, int dst, int src, int& s, float& f) {
  const double inv_scale = (double)dst / src;
  const double scale = 1.0 / inv_scale;
  s = (int)floor(__dmul_rn((double)d, scale));
  f = __double2float_rn(__dsub_rn((double)(d + 1), __dmul_rn((double)(s + 1), inv_scale)));
  f = f <= 0.f ? 0.f : __fsub_rn(f, floorf(f));
  if (s >= src - 1) s = src - 1, f = 0.f;
}

// The area-weighted bilinear value of channel c of a [hs][stride] plane with C channels at output (x, y).
template <typename T, int C>
__device__ __forceinline__ float enlarge(const T* src, long long stride, int ws, int hs, int w, int h, int x, int y,
                                         int c) {
  int sx, sy;
  float fx, fy;
  area_weight(x, w, ws, sx, fx);
  area_weight(y, h, hs, sy, fy);
  const int sx1 = min(sx + 1, ws - 1), sy1 = min(sy + 1, hs - 1);
  const float ax = __fsub_rn(1.f, fx), ay = __fsub_rn(1.f, fy);
  const T* r0 = src + sy * stride;
  const T* r1 = src + sy1 * stride;
  const float h0 = __fadd_rn(__fmul_rn((float)r0[C * sx + c], ax), __fmul_rn((float)r0[C * sx1 + c], fx));
  const float h1 = __fadd_rn(__fmul_rn((float)r1[C * sx + c], ax), __fmul_rn((float)r1[C * sx1 + c], fx));
  return __fadd_rn(__fmul_rn(h0, ay), __fmul_rn(h1, fy));
}

// Block sum of a k x k block (k = 2: in row-major order; k = 4: each row, then the rows) times 1 / k^2.
template <typename F>
__device__ __forceinline__ float reduce_block(int k, F v) {
  if (k == 2) return __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(v(0, 0), v(0, 1)), v(1, 0)), v(1, 1)), 0.25f);
  float s = 0.f;
  for (int dy = 0; dy < 4; ++dy) {
    const float r = __fadd_rn(__fadd_rn(__fadd_rn(v(dy, 0), v(dy, 1)), v(dy, 2)), v(dy, 3));
    s = dy == 0 ? r : __fadd_rn(s, r);
  }
  return __fmul_rn(s, 0.0625f);
}

__global__ void __launch_bounds__(INGEST_THREADS) image_kernel(const LrfIngestFrame f, int k, float* rgb,
                                                               uint8_t* gray) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)f.w * f.h) return;
  const int x = (int)(p % f.w), y = (int)(p / f.w);
  int u[3];
  for (int c = 0; c < 3; ++c) {
    auto v = [&](int dy, int dx) {
      return __fdiv_rn((float)f.image[(long long)(k * y + dy) * f.image_stride + 3 * (k * x + dx) + 2 - c], 255.f);
    };
    const float r = k == 1 ? v(0, 0) : reduce_block(k, v);
    rgb[3 * p + c] = r;
    u[c] = (int)__fmul_rn(r, 255.f);                     // (img * 255).astype(uint8): r in [0, 1]
  }
  gray[p] = (uint8_t)((9798 * u[0] + 19235 * u[1] + 3735 * u[2] + (1 << 14)) >> 15);
}

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  if (i < 0) return -i;
  if (i >= n) return 2 * n - 2 - i;
  return i;
}

__global__ void __launch_bounds__(INGEST_THREADS) laplacian_kernel(const uint8_t* gray, int w, int h, float* lap) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)w * h) return;
  const int x = (int)(p % w), y = (int)(p / w);
  const int g = gray[p];
  const int s = gray[(long long)reflect101(y - 1, h) * w + x] + gray[(long long)reflect101(y + 1, h) * w + x] +
                gray[(long long)y * w + reflect101(x - 1, w)] + gray[(long long)y * w + reflect101(x + 1, w)];
  lap[p] = (float)(s - 4 * g);                            // exact, as cv2's fp32 filter is on these integers
}

// Slot i of 2^depth: numpy's pairwise sum of the leaf the bits of i select, or nothing (flag 0) when i lies below a
// leaf that ends the recursion higher up.  square: sum (x - mean)^2 instead of x, mean = stats[0].
__global__ void __launch_bounds__(INGEST_THREADS) leaf_sums_kernel(const float* x, long long n, int depth,
                                                                   bool square, const float* stats, float* sums,
                                                                   uint8_t* flags) {
  const long long i = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (i >= (1LL << depth)) return;
  long long off = 0, len = n;
  for (int d = depth - 1; d >= 0; --d) {
    if (len <= LEAF) {
      if (i & ((2LL << d) - 1)) {
        flags[i] = 0;
        return;
      }
      break;
    }
    long long n2 = len / 2;
    n2 -= n2 % 8;
    if ((i >> d) & 1) off += n2, len -= n2;
    else len = n2;
  }
  const float mean = square ? stats[0] : 0.f;
  auto val = [&](long long j) {
    const float v = x[off + j];
    if (!square) return v;
    const float d = __fsub_rn(v, mean);
    return __fmul_rn(d, d);
  };
  float s;
  if (len < 8) {
    s = -0.f;
    for (long long j = 0; j < len; ++j) s = __fadd_rn(s, val(j));
  } else {
    float r[8];
    for (int j = 0; j < 8; ++j) r[j] = val(j);
    long long j = 8;
    for (; j < len - len % 8; j += 8)
      for (int t = 0; t < 8; ++t) r[t] = __fadd_rn(r[t], val(j + t));
    s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                  __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; j < len; ++j) s = __fadd_rn(s, val(j));
  }
  sums[i] = s;
  flags[i] = 1;
}

// One CTA: the 2^depth slots added back up as the recursion pairs them (left + right, an empty right passes the
// left through), then divided by n into stats[which].
__global__ void __launch_bounds__(TREE_THREADS) tree_sum_kernel(float* sums, uint8_t* flags, int depth, long long n,
                                                                float* stats, int which) {
  __shared__ float v[TREE_THREADS];
  __shared__ uint8_t fl[TREE_THREADS];
  const long long S = 1LL << depth;
  const int active = (int)(S < TREE_THREADS ? S : TREE_THREADS);
  const long long g = S / active;                         // consecutive slots per thread, a power of two
  const int t = threadIdx.x;
  if (t < active) {
    float* s = sums + t * g;
    const uint8_t* f = flags + t * g;
    for (long long step = 1; step < g; step *= 2)
      for (long long a = 0; a < g; a += 2 * step)
        if (f[a + step]) s[a] = __fadd_rn(s[a], s[a + step]);
    v[t] = s[0];
    fl[t] = f[0];
  }
  __syncthreads();
  for (int step = 1; step < active; step *= 2) {
    if (t < active && t % (2 * step) == 0 && fl[t + step]) v[t] = __fadd_rn(v[t], v[t + step]);
    __syncthreads();
  }
  if (t == 0) stats[which] = __fdiv_rn(v[0], (float)n);
}

__global__ void __launch_bounds__(INGEST_THREADS) weight_kernel(const LrfIngestFrame f, const float* stats,
                                                                float* weight) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)f.w * f.h) return;
  const float var = stats[1];
  if (!f.mask) {
    weight[p] = var;
    return;
  }
  const int x = (int)(p % f.w), y = (int)(p / f.w);
  weight[p] = __fmul_rn(var, f.mask[(long long)y * f.mask_stride + x] > 0 ? 1.f : 0.f);
}

__global__ void __launch_bounds__(INGEST_THREADS) flow_kernel(const LrfIngestFrame f, bool enlarge_, float* fwd,
                                                              float* fwd_mask, float* bwd, float* bwd_mask) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)f.w * f.h) return;
  const int x = (int)(p % f.w), y = (int)(p / f.w);
  for (int dir = 0; dir < 2; ++dir) {
    const uint16_t* src = dir ? f.bwd_flow : f.fwd_flow;
    float* flow = dir ? bwd : fwd;
    float* mask = dir ? bwd_mask : fwd_mask;
    float e[3];
    for (int c = 0; c < 3; ++c) {
      if (enlarge_) {
        const int r = __float2int_rn(enlarge<uint16_t, 3>(src, f.flow_stride, f.wf, f.hf, f.w, f.h, x, y, c));
        e[c] = (float)min(max(r, 0), 65535);
      } else {
        e[c] = (float)src[(long long)y * f.flow_stride + 3 * x + c];
      }
    }
    for (int c = 0; c < 2; ++c)
      flow[2 * p + c] = __fmul_rn(__fdiv_rn(__fsub_rn(e[c], 32768.f), 256.f), f.flow_scale);
    mask[p] = e[2] > 32768.f ? 1.f : 0.f;
  }
}

__global__ void __launch_bounds__(INGEST_THREADS) depth_kernel(const LrfIngestFrame f, int mode, float* out) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)f.w * f.h) return;
  const int x = (int)(p % f.w), y = (int)(p / f.w);
  float d;
  if (mode == 0) {
    d = enlarge<uint16_t, 1>(f.invdepth, f.invdepth_stride, f.wd, f.hd, f.w, f.h, x, y, 0);
  } else if (mode == 1) {
    d = (float)f.invdepth[(long long)y * f.invdepth_stride + x];
  } else {
    auto v = [&](int dy, int dx) {
      return (float)f.invdepth[(long long)(mode * y + dy) * f.invdepth_stride + mode * x + dx];
    };
    d = reduce_block(mode, v);
  }
  out[p] = d;
}

// One row or column coefficient of cv2's INTER_LINEAR: f = float((d + 0.5) scale - 0.5) in double, s = floor(f),
// f -= s in float.  Each double step rounds once (no DFMA), as the host computes it.
__device__ __forceinline__ void linear_coeff(int d, double scale, int& s, float& f) {
  f = __double2float_rn(__dadd_rn(__dmul_rn(d + 0.5, scale), -0.5));
  s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
}

// cv2.resize(src, (W, H)) of a 3-channel float32 image without IPP (include/localrf_b200.h, lrf_resize_linear):
// mode 1 copies, mode 2 is the exact 2x reduction (INTER_AREA, the same block sum as image_kernel), mode 0 is the
// separable linear rule, the horizontal blend rounded to float before the vertical one.
__global__ void __launch_bounds__(INGEST_THREADS) resize_linear_kernel(const float* src, int w0, int h0,
                                                                       long long src_stride, float* dst, int W, int H,
                                                                       long long dst_stride, int mode, double scale_x,
                                                                       double scale_y) {
  const long long p = (long long)blockIdx.x * INGEST_THREADS + threadIdx.x;
  if (p >= (long long)W * H) return;
  const int x = (int)(p % W), y = (int)(p / W);
  // pixel offsets in 64 bits: a row may hold up to 2^31 - 1 pixels, so 3 x alone can pass 2^31
  float* out = dst + y * dst_stride + 3LL * x;
  if (mode == 1) {
    for (int c = 0; c < 3; ++c) out[c] = src[y * src_stride + 3LL * x + c];
    return;
  }
  if (mode == 2) {
    for (int c = 0; c < 3; ++c) {
      auto v = [&](int dy, int dx) { return src[(long long)(2 * y + dy) * src_stride + 3LL * (2LL * x + dx) + c]; };
      out[c] = reduce_block(2, v);
    }
    return;
  }
  int sx, sy;
  float fx, fy;
  linear_coeff(x, scale_x, sx, fx);
  if (sx < 0) sx = 0, fx = 0.f;
  // cv2's xmax (sx + 1 >= w0): every later column copies too.  sx + 1 and sy + 1 are not formed at the last index,
  // where a float index of 2^31 has converted to INT_MAX.
  const bool copy = sx >= w0 - 1;
  if (copy) sx = w0 - 1;
  linear_coeff(y, scale_y, sy, fy);                       // rows are not reset at the borders
  const int sy0 = min(max(sy, 0), h0 - 1), sy1 = sy >= h0 - 1 ? h0 - 1 : max(sy + 1, 0);
  const float ax = __fsub_rn(1.f, fx), ay = __fsub_rn(1.f, fy);
  const float* r0 = src + sy0 * src_stride + 3LL * sx;
  const float* r1 = src + sy1 * src_stride + 3LL * sx;
  for (int c = 0; c < 3; ++c) {
    const float h0v = copy ? r0[c] : __fadd_rn(__fmul_rn(r0[c], ax), __fmul_rn(r0[3 + c], fx));
    const float h1v = copy ? r1[c] : __fadd_rn(__fmul_rn(r1[c], ax), __fmul_rn(r1[3 + c], fx));
    out[c] = __fadd_rn(__fmul_rn(h0v, ay), __fmul_rn(h1v, fy));
  }
}

// Scratch layout (bytes): stats [2] fp32 at 0 (mean, variance), the Laplacian [n] fp32 at 16, the tree's slot sums
// [2^D] fp32, its flags [2^D] u8, the grey image [n] u8.
struct Scratch {
  float* stats;
  float* lap;
  float* sums;
  uint8_t* flags;
  uint8_t* gray;
};

Scratch carve(ScratchCarver& c, long long n, int depth) {
  const size_t S = (size_t)1 << depth;
  Scratch s;
  s.stats = c.take<float>(16, 4);
  s.lap = c.take<float>(4 * (size_t)n, 4);
  s.sums = c.take<float>(4 * S, 4);
  s.flags = c.take<uint8_t>(S, 1);
  s.gray = c.take<uint8_t>((size_t)n, 1);
  return s;
}

}  // namespace

// Depth of the slot tree: the number of halvings until every node of numpy's recursion over n values is a leaf
// (<= 128 values); -1 above MAX_TREE_DEPTH.  The node sizes of one level take few distinct values.
int ingest_tree_depth(long long n) {
  long long sizes[64];
  int m = 1, depth = 0;
  sizes[0] = n;
  for (;;) {
    long long next[64];
    int k = 0;
    bool split = false;
    for (int i = 0; i < m; ++i) {
      if (sizes[i] <= LEAF) continue;
      split = true;
      long long n2 = sizes[i] / 2;
      n2 -= n2 % 8;
      for (long long c : {n2, sizes[i] - n2}) {
        bool seen = false;
        for (int j = 0; j < k; ++j) seen |= next[j] == c;
        if (!seen && k < 64) next[k++] = c;
      }
    }
    if (!split) return depth;
    if (++depth > MAX_TREE_DEPTH) return -1;
    for (int i = 0; i < k; ++i) sizes[i] = next[i];
    m = k;
  }
}

size_t ingest_scratch_bytes(long long n_px) {
  const int depth = ingest_tree_depth(n_px);
  if (depth < 0) return 0;
  ScratchCarver c(nullptr);
  carve(c, n_px, depth);
  return c.size(8);
}

int ingest_resize_mode(int ws, int hs, int w, int h) { return resize_mode(ws, hs, w, h); }

cudaError_t launch_ingest_frame(const LrfFrameStore& st, const LrfIngestFrame& f, void* scratch,
                                cudaStream_t stream) {
  const long long n = (long long)f.w * f.h;
  const int depth = ingest_tree_depth(n);
  ScratchCarver c(scratch);
  const Scratch s = carve(c, n, depth);
  const unsigned blocks = (unsigned)((n + INGEST_THREADS - 1) / INGEST_THREADS);
  const unsigned slot_blocks = (unsigned)(((1LL << depth) + INGEST_THREADS - 1) / INGEST_THREADS);
  const long long at = f.slot * n;
  image_kernel<<<blocks, INGEST_THREADS, 0, stream>>>(f, resize_mode(f.w0, f.h0, f.w, f.h), (float*)st.rgb + 3 * at,
                                                      s.gray);
  laplacian_kernel<<<blocks, INGEST_THREADS, 0, stream>>>(s.gray, f.w, f.h, s.lap);
  for (int which = 0; which < 2; ++which) {
    leaf_sums_kernel<<<slot_blocks, INGEST_THREADS, 0, stream>>>(s.lap, n, depth, which == 1, s.stats, s.sums,
                                                                 s.flags);
    tree_sum_kernel<<<1, TREE_THREADS, 0, stream>>>(s.sums, s.flags, depth, n, s.stats, which);
  }
  weight_kernel<<<blocks, INGEST_THREADS, 0, stream>>>(f, s.stats, (float*)st.loss_weight + at);
  if (st.fwd_flow)
    flow_kernel<<<blocks, INGEST_THREADS, 0, stream>>>(f, resize_mode(f.wf, f.hf, f.w, f.h) == 0,
                                                       (float*)st.fwd_flow + 2 * at, (float*)st.fwd_mask + at,
                                                       (float*)st.bwd_flow + 2 * at, (float*)st.bwd_mask + at);
  if (st.invdepth)
    depth_kernel<<<blocks, INGEST_THREADS, 0, stream>>>(f, resize_mode(f.wd, f.hd, f.w, f.h),
                                                        (float*)st.invdepth + at);
  return cudaGetLastError();
}

cudaError_t launch_resize_linear(const float* src, int w0, int h0, long long src_stride, float* dst, int W, int H,
                                 long long dst_stride, cudaStream_t stream) {
  const int mode = (w0 == W && h0 == H) ? 1 : (w0 == 2 * W && h0 == 2 * H) ? 2 : 0;
  const double scale_x = 1.0 / ((double)W / w0), scale_y = 1.0 / ((double)H / h0);
  const long long n = (long long)W * H;
  resize_linear_kernel<<<(unsigned)((n + INGEST_THREADS - 1) / INGEST_THREADS), INGEST_THREADS, 0, stream>>>(
      src, w0, h0, src_stride, dst, W, H, dst_stride, mode, scale_x, scale_y);
  return cudaGetLastError();
}

}  // namespace lrf
