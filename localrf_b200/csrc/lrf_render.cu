// lrf_render.cu -- the fused per-ray-batch render kernel (sm_90a), streaming / warp-specialised.
//
// One launch = one (field, ray batch): ray generation -> contracted sampling -> VM density gather
// -> softplus/alpha/transmittance scan -> (floater filter) -> selection of the samples whose weight
// exceeds the threshold -> VM appearance gather -> basis+MLP -> composite -> blend / exposure /
// clamp.  Replaces TensorBase.forward (models/tensorBase.py:567-636) and the per-field body of
// LocalTensorfs.forward (local_tensorfs.py:397-497).
//
// One persistent CTA per SM, 16 warps (512 threads) in two roles that only meet through
// mbarriers and a few shared-memory counters:
//
//   producers (warps 0 .. W_CONS-1: 8)  each takes one ray at a time from a global counter (dynamic
//       scheduling: no wave quantisation of a 4096-ray batch).  March: lane = sample, 32 samples
//       per step, transmittance by a warp-shuffle product scan with a carried prefix.  Samples
//       with w > threshold go to a small per-warp queue whose entries carry their ray slot (so samples of
//       consecutive rays share a gather); every 32 of them are gathered (lane = sample: 3 planes x 4 texels
//       x 96 B + 3 lines, 72 products), split into bf16 hi/lo and written as one ROW of the current 128-row
//       A tile in shared memory (K-major 8x8 core matrices).  Rows are handed out by an atomic cursor, so
//       rays of all producers interleave in a tile; each row carries (ray slot, weight).  Every row arrives
//       once on the tile's "full" mbarrier (128 arrivals = tile ready).
//   consumers (the last two warpgroups)  per tile, one 64-row half each:
//       layer 1 (A from shared memory, basis folded into W1, K = 80) and layer 2 (A = the bias + ReLU'd
//       layer-1 accumulator re-split in registers, K = 128) as wgmma m64 bf16 MMAs, three products
//       hi*hi + hi*lo + lo*hi per K-step, fp32 accumulators in registers; layer 3 (131 -> 3) + sigmoid on
//       the CUDA cores; composite: w * rgb is added to the row's ray slot as 32-bit FIXED POINT with
//       shared-memory atomics (integer adds are associative, so results are bit-identical whatever the
//       interleaving of rows, tiles and threads); the last contributor of a ray writes its output (white
//       background, blend, accumulate, exposure, clamp) and, in a multi-GPU run, stores the finished pixel
//       into every peer's gathered buffer.  Then the tile's A buffer is released to the producers.
//
// render_kernel_t<true> (fields with positional encodings) inserts a layer 0 (basis_mat as its own product),
// builds the encoded layer-1 input in registers 64 columns at a time and streams layer 1's weight chunks by TMA.
// The weight operands are staged once per CTA by TMA bulk copies (cp.async.bulk -> UBLKCP); the sample table is read from global memory through the L1.  The launcher sets the shared-memory carveout to the
// smallest step that holds the CTA: the default build's folded-MLP layout fits the 196 KB step, which leaves
// the L1 60 KB for the texel gathers.
#include "lrf_device.cuh"
#include "lrf_launch.cuh"
#include "lrf_launchers.cuh"

namespace lrf {

constexpr int THREADS = 512;                    // 16 warps (128 registers each)
constexpr int N_CWG = 2;                        // consumer warpgroups, one 64-row half of a tile each
constexpr int N_CONS = 4 * N_CWG;               // the last warps: consumers
constexpr int W_CONS = THREADS / 32 - N_CONS;
constexpr int MAX_PROD = W_CONS;                // producer warps 0 .. W_CONS-1 (8)
constexpr int XA_LD = 33;                       // (positional encodings) floats per row of the basis-feature buffer
constexpr int NSLOT = 3;            // ray slots per producer warp
constexpr int QCAP = 64;            // per-warp queue of selected samples
constexpr int SPIN_PAD = 2048;      // polls before a blocked producer pads the open tile
constexpr unsigned SPIN_NS = 200;   // back-off of a producer waiting for a free tile: spinning takes issue slots from the gathers

// colour accumulators are 32-bit fixed point (2^-30 units, 9.3e-10: finer than an fp32 ulp of the
// sums, which are <= 1): integer adds are associative, so the rows of a ray can be composited in any
// order, by any thread, and the result is bit-identical.  (32-bit shared-memory atomics are native;
// 64-bit ones turn into contended CAS loops.)
constexpr float FIX_SCALE = 1073741824.0f;              // 2^30
constexpr float FIX_INV = 1.0f / 1073741824.0f;

struct Slot {                       // one ray in flight between a producer and the consumers
  float o[3];                       // ray origin / |d| (the gathers of queued samples read the ray from its slot)
  float nrm;
  float vd[3];
  float blend;
  unsigned int rgb[3];              // sum of w * rgb, fixed point
  float acc;
  float depth;                      // final depth of the ray (for the fused pixel exchange)
  float vterm[3];                   // (fields with view encodings) W3[:, 128:] . [vd, PE(vd)]
  long long ray;
  int pending;                      // 1 (open token) + rows submitted and not yet composited
  int state;                        // 0 free, 1 active
};

struct Ctrl {                       // CTA control block in shared memory
  unsigned long long bar_w, full[2];
  unsigned long long wrdy;          // fields with positional encodings: the streamed layer-1 weight chunk has landed
  unsigned int released;            // tiles whose A1 buffer + row metadata may be overwritten
  unsigned int cursor;              // rows handed out so far (tile = cursor >> 7)
  unsigned int prod_done;
  unsigned int n_tiles_final;
  unsigned int done;
};

struct SmemV3 {
  int prep, a1, mslot, mw, part, slots, q, alpha, ctrl, total;
  int per_prod;                     // bytes of one producer's queue (+ alpha table)
};

constexpr int PE_WBUF = (PE_RESIDENT + 1023) & ~1023;     // offset of the streamed layer-1 chunk inside the prep region
__host__ __device__ constexpr SmemV3 smem_v3(int S, bool floater, int nprod, bool pe = false) {
  SmemV3 L{};
  int off = 0;
  const int Sp = (S + 3) & ~3;
  L.prep = off;   off += pe ? PE_WBUF + 2 * PE_WC_BYTES : PREP_BYTES;
  off = (off + 1023) & ~1023;
  L.a1 = off;     off += 2 * 2 * OPER1_BYTES;          // two A1 tiles (hi + lo each)
  L.mslot = off;  off += 2 * TM;                        // per-row slot id (u8), two tiles
  L.mw = off;     off += 2 * TM * 4;                    // per-row weight
  L.part = off;   off += (pe ? N_CWG * 64 * XA_LD * 4 : 0);   // basis features of the rows a consumer warpgroup shades
  off = (off + 15) & ~15;
  L.slots = off;  off += MAX_PROD * NSLOT * (int)sizeof(Slot);
  off = (off + 15) & ~15;
  L.q = off;
  L.per_prod = QCAP * 2 + QCAP * 4 + QCAP + (floater ? Sp * 4 : 0);   // sample index, weight, slot id per entry
  L.per_prod = (L.per_prod + 15) & ~15;
  off += nprod * L.per_prod;
  L.alpha = QCAP * 7 + (16 - (QCAP * 7) % 16) % 16;     // offset of the alpha table inside a producer block
  off = (off + 15) & ~15;
  L.ctrl = off;   off += (int)sizeof(Ctrl);
  L.total = (off + 15) & ~15;
  return L;
}
// Hopper's two largest shared-memory carveout steps are 196 and 228 KB, and the SM reserves 1 KB of each CTA's
// share.  Without the floater filter the layout does not depend on S (the sample table is read from global
// memory through the L1), so the default build's CTA fits the 196 KB step for every sample table and the L1
// keeps 60 KB for the texel gathers (28 KB at the 228 KB step).
constexpr int SMEM_196K_STEP = 196 * 1024 - 1024;
static_assert(smem_v3(344, false, MAX_PROD).total <= SMEM_196K_STEP &&
              smem_v3(65535, false, MAX_PROD).total <= SMEM_196K_STEP,
              "the folded-MLP layout must fit the 196 KB carveout step");

// ---- outputs (local_tensorfs.py:467-497) --------------------------------------------------------
__device__ __forceinline__ void write_rgb(const BatchDev& B, long long r,
                                          const unsigned int* rgb_fix, float acc, float blend,
                                          float depth) {
  float c[3];
  const float bg = B.white_bg ? (1.0f - acc) : 0.0f;              // tensorBase.py:633-634
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const unsigned int v = *reinterpret_cast<const volatile unsigned int*>(rgb_fix + a);
    c[a] = (__uint2float_rn(v) * FIX_INV + bg) * blend;           // tensorBase.py:632
  }
  if (B.accumulate) {
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = B.rgb[B.rgb_stride * r + a] + c[a];
  }
  if (B.finalize) {
    const float* E = nullptr;
    if (B.exposure) E = B.exposure + 9 * (B.rays_per_view > 0 ? r / B.rays_per_view : 0);
    finalize_rgb(E, c);
  }
  float* o = B.rgb + B.rgb_stride * r;
  o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
  if (B.n_peers > 0 && B.finalize) {
    // fused pixel exchange: this ray's (r,g,b,depth) goes straight into every peer's gathered buffer
    if (B.mc_pix) {
      asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(B.mc_pix + 4 * r),
                   "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(depth)
                   : "memory");
    } else {
      const float4 v = make_float4(c[0], c[1], c[2], depth);
      for (int p = 0; p < B.n_peers; ++p) *reinterpret_cast<float4*>(B.peer_pix[p] + 4 * r) = v;
    }
  }
}

__device__ __forceinline__ void finalize_slot(const BatchDev& B, Slot* s) {
  write_rgb(B, s->ray, s->rgb, s->acc, s->blend, s->depth);
  __threadfence_block();
  *reinterpret_cast<volatile int*>(&s->state) = 0;
}

// 72 appearance products of one sample -> one row of the A1 tile (bf16 hi/lo, 9 chunks of 8)
template <bool H16>
__device__ __forceinline__ void app_row(const FieldDev& F, const float* q, unsigned char* a_hi,
                                        unsigned char* a_lo, int row) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const VmTap t = vm_tap<CA>(F.g, i, q);
#pragma unroll
    for (int c8 = 0; c8 < CA / 8; ++c8) {
      float v[8];
      vm_products<8>(t, texels<H16>(F.aplane[i]), texels<H16>(F.aline[i]), 8 * c8, v);
      store_chunk(a_hi, a_lo, row, i * (CA / 8) + c8, K1_CHUNKS, v);
    }
  }
}

struct ProdCtx {
  unsigned char* smem;
  const SmemV3* L;
  Ctrl* ctrl;
  int lane;
};

// wait until buffer (T & 1) may be rewritten for tile T: tile T-2 has been read by the tensor core
// and its row metadata by the consumers.  A monotonic counter, not an mbarrier parity: producers
// can be more than two tiles ahead of the consumers, which a 1-bit phase cannot express.
__device__ __forceinline__ void wait_tile_free(Ctrl* ctrl, unsigned int T) {
  if (T >= 2) {
    while (*reinterpret_cast<volatile unsigned int*>(&ctrl->released) + 1u < T) __nanosleep(SPIN_NS);
    __threadfence_block();
  }
}

// completes the currently open tile with invalid rows (slot 0xFF) so the consumers can drain it
__device__ __noinline__ void pad_open_tile(const ProdCtx& P) {
  unsigned int start = 0, n = 0;
  if (P.lane == 0) {
    unsigned int old = *reinterpret_cast<volatile unsigned int*>(&P.ctrl->cursor);
    for (;;) {
      const unsigned int rem = old & (TM - 1);
      if (rem == 0) { n = 0; break; }
      const unsigned int seen = atomicCAS(&P.ctrl->cursor, old, old + (TM - rem));
      if (seen == old) { start = old; n = TM - rem; break; }
      old = seen;
    }
  }
  start = __shfl_sync(0xffffffffu, start, 0);
  n = __shfl_sync(0xffffffffu, n, 0);
  if (n == 0) return;
  const unsigned int T = start >> 7;
  wait_tile_free(P.ctrl, T);
  unsigned char* mslot = P.smem + P.L->mslot + (T & 1) * TM;
  float* mw = reinterpret_cast<float*>(P.smem + P.L->mw) + (T & 1) * TM;
  const uint32_t full = smem_u32(&P.ctrl->full[T & 1]);
  for (unsigned int g = start + P.lane; g < start + n; g += 32) {
    mslot[g & (TM - 1)] = 0xFF;
    mw[g & (TM - 1)] = 0.0f;
    __threadfence_block();
    mbar_arrive(full);
  }
  __syncwarp();
}

// per-warp queue of selected samples: (sample index, weight, ray slot); entries of different rays mix
struct WarpQ {
  unsigned short* qk;
  float* qw;
  unsigned char* qs;
  int qn;
  unsigned long long n_app;
};

// gathers the first n (<= 32) queued samples (each with its own ray, read from its slot) and submits
// them as tile rows.  Their slots' `pending` counts were raised when the samples were selected.
template <bool H16>
__device__ __forceinline__ void flush_rows(const ProdCtx& P, const FieldDev& F, const Slot* slots,
                                           const WarpQ& Q, int n) {
  unsigned int start = 0;
  if (P.lane == 0) start = atomicAdd(&P.ctrl->cursor, (unsigned int)n);
  start = __shfl_sync(0xffffffffu, start, 0);
  if (P.lane < n) {
    const unsigned int g = start + P.lane, T = g >> 7;
    const int row = (int)(g & (TM - 1)), b = (int)(T & 1);
    const int k = Q.qk[P.lane], sid = Q.qs[P.lane];
    const Slot* sl = slots + sid;
    RaySm R;
    R.o[0] = sl->o[0]; R.o[1] = sl->o[1]; R.o[2] = sl->o[2];
    R.vd[0] = sl->vd[0]; R.vd[1] = sl->vd[1]; R.vd[2] = sl->vd[2];
    float p[3], q[3];
    sample_pos(F, R, __ldg(F.z + k), p, q);
    wait_tile_free(P.ctrl, T);
    unsigned char* a_hi = P.smem + P.L->a1 + b * (2 * OPER1_BYTES);
    app_row<H16>(F, q, a_hi, a_hi + OPER1_BYTES, row);
    P.smem[P.L->mslot + b * TM + row] = (unsigned char)sid;
    reinterpret_cast<float*>(P.smem + P.L->mw)[b * TM + row] = Q.qw[P.lane];
    fence_async_smem();                  // generic-proxy writes -> visible to the tensor core
    mbar_arrive(smem_u32(&P.ctrl->full[b]));
  }
  __syncwarp();
}

// appends the lanes with on == true (mask m = their ballot) to the warp's queue; flushes 32 rows when it
// holds >= 32.  The caller has already added popc(m) to the slot's pending count.
template <bool H16>
__device__ __forceinline__ void queue_push(const ProdCtx& P, const FieldDev& F, const Slot* slots,
                                           WarpQ& Q, unsigned m, bool on, int k,
                                           float wgt, int slot_id) {
  const int lane = P.lane;
  if (on) {
    const int pos = Q.qn + __popc(m & ((1u << lane) - 1u));
    Q.qk[pos] = (unsigned short)k; Q.qw[pos] = wgt; Q.qs[pos] = (unsigned char)slot_id;
  }
  Q.qn += __popc(m);
  Q.n_app += __popc(m);
  __syncwarp();
  if (Q.qn >= 32) {
    flush_rows<H16>(P, F, slots, Q, 32);
    unsigned short tk = 0; float tw = 0.0f; unsigned char ts = 0;
    if (lane < Q.qn - 32) { tk = Q.qk[32 + lane]; tw = Q.qw[32 + lane]; ts = Q.qs[32 + lane]; }
    __syncwarp();
    if (lane < Q.qn - 32) { Q.qk[lane] = tk; Q.qw[lane] = tw; Q.qs[lane] = ts; }
    Q.qn -= 32;
    __syncwarp();
  }
}

// =================================================================================================
// PE = the field has positional encodings (fea_pe > 0 or view_pe > 0): basis_mat is its own tensor-core
// product (layer 0), the consumers build the encoded layer-1 input chunk by chunk in registers, layer 1's weight
// operand is streamed by TMA in K-chunks of 64.  PE = false is the reference-default fast path (folded basis).
// H16 = the grids are stored as bfloat16 (LrfField.grid_dtype): the gathers of the producers read 16-byte
// texel pieces of 8 components; everything downstream of the gathers is the same code.
template <bool PE, bool H16 = false>
__global__ void __launch_bounds__(THREADS, 1)
render_kernel_t(const FieldDev F, const BatchDev B, const int nprod) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const bool floater = B.floater_thresh > 0.0f;
  const SmemV3 L = smem_v3(F.S, floater, nprod, PE);
  Ctrl* ctrl = reinterpret_cast<Ctrl*>(smem + L.ctrl);
  Slot* slots = reinterpret_cast<Slot*>(smem + L.slots);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = F.S;

  // ---- prologue ---------------------------------------------------------------------------------
  if (tid == 0) {
    mbar_init(smem_u32(&ctrl->bar_w), 1);
    mbar_init(smem_u32(&ctrl->full[0]), TM);
    mbar_init(smem_u32(&ctrl->full[1]), TM);
    if (PE) mbar_init(smem_u32(&ctrl->wrdy), 1);
    ctrl->cursor = 0; ctrl->prod_done = 0; ctrl->n_tiles_final = 0; ctrl->done = 0;
    ctrl->released = 0;
    constexpr uint32_t bytes = PE ? PE_RESIDENT : PREP_BYTES;
    mbar_expect_tx(smem_u32(&ctrl->bar_w), bytes);
    constexpr uint32_t CH = 32768;
    for (uint32_t o = 0; o < bytes; o += CH)
      tma_bulk_g2s(smem_u32(smem + L.prep) + o, reinterpret_cast<const char*>(F.prep) + o,
                   min(CH, bytes - o), smem_u32(&ctrl->bar_w));
  }
  for (int e = tid; e < MAX_PROD * NSLOT * (int)sizeof(Slot) / 4; e += THREADS)
    reinterpret_cast<int*>(slots)[e] = 0;
  {  // K padding 72..79 of both A1 tiles (hi and lo) is zero for the whole launch
    const float zero[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int e = tid; e < 2 * TM; e += THREADS) {
      unsigned char* a_hi = smem + L.a1 + (e / TM) * (2 * OPER1_BYTES);
      store_chunk(a_hi, a_hi + OPER1_BYTES, e % TM, K1_CHUNKS - 1, K1_CHUNKS, zero);
    }
  }
  if (B.signal_seq && B.wait_seq && tid < B.n_peers) {
    // fused pixel exchange: the peers must be done with the gathered buffer this launch overwrites
    const unsigned long long* local = B.peer_flags[B.rank] + tid;
    unsigned long long v = 0;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(local) : "memory");
    } while (v < B.wait_seq);
  }
  fence_async_smem();
  __syncthreads();

  const int prod_id = warp < W_CONS ? warp : -1;

  if (prod_id >= 0 && prod_id < nprod) {
    // ======================================= PRODUCER ============================================
    ProdCtx P{smem, &L, ctrl, lane};
    unsigned char* mine = smem + L.q + prod_id * L.per_prod;
    WarpQ Q;
    Q.qk = reinterpret_cast<unsigned short*>(mine);
    Q.qw = reinterpret_cast<float*>(mine + QCAP * 2);
    Q.qs = mine + QCAP * 6;
    Q.qn = 0; Q.n_app = 0;
    float* alpha_s = reinterpret_cast<float*>(mine + L.alpha);
    unsigned long long n_march = 0;
    int next_slot = 0;
    for (;;) {
      long long ray = 0;
      if (lane == 0) ray = (long long)atomicAdd(B.sched, 1ull);
      ray = __shfl_sync(0xffffffffu, ray, 0);
      if (ray >= B.n_rays) break;
      RaySm R;
      setup_ray(B, ray, R);
      // -- acquire a ray slot (if the consumers starve: submit what this warp holds, pad the open tile) --
      const int slot_id = prod_id * NSLOT + next_slot;
      next_slot = (next_slot + 1 == NSLOT) ? 0 : next_slot + 1;
      Slot* slot = slots + slot_id;
      for (int spins = 0;; ++spins) {
        int st = 0;
        if (lane == 0) st = *reinterpret_cast<volatile int*>(&slot->state);
        st = __shfl_sync(0xffffffffu, st, 0);
        if (st == 0) break;
        if (spins == SPIN_PAD) {
          if (Q.qn > 0) { flush_rows<H16>(P, F, slots, Q, Q.qn); Q.qn = 0; }
          pad_open_tile(P);
          spins = 0;
        }
      }
      if (lane == 0) {
        slot->o[0] = R.o[0]; slot->o[1] = R.o[1]; slot->o[2] = R.o[2]; slot->nrm = R.nrm;
        slot->vd[0] = R.vd[0]; slot->vd[1] = R.vd[1]; slot->vd[2] = R.vd[2];
        slot->blend = R.blend;
        slot->rgb[0] = slot->rgb[1] = slot->rgb[2] = 0u;
        slot->ray = ray;
        slot->pending = 1;
      }
      if (PE) {
        // view term of layer 3 (tensorBase.py:126-131): W3[:, 128:] . [vd, sin(vd 2^f), cos(vd 2^f)], d-major f-minor
        const int V = F.view_pe, nv = 3 * (1 + 2 * V), ld = FC + nv;
        float vt[3] = {0.0f, 0.0f, 0.0f};
        for (int j = lane; j < nv; j += 32) {
          float v;
          if (j < 3) v = R.vd[j];
          else {
            const int e = (j - 3) % (3 * V), d = e / V, f = e - d * V;
            const float ang = R.vd[d] * (float)(1 << f);
            v = (j - 3) < 3 * V ? sinf(ang) : cosf(ang);
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) vt[c] = fmaf(__ldg(F.w3 + c * ld + FC + j), v, vt[c]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) vt[c] = warp_sum(vt[c]);
        if (lane == 0) { slot->vterm[0] = vt[0]; slot->vterm[1] = vt[1]; slot->vterm[2] = vt[2]; }
      }
      if (lane == 0) {
        __threadfence_block();
        *reinterpret_cast<volatile int*>(&slot->state) = 1;
      }
      __syncwarp();
      float acc = 0.0f, dep = 0.0f;
      // -- march (tensorBase.py:581-615) ------------------------------------------------------------
      float carry = 1.0f, acc_p = 0.0f, dep_p = 0.0f, idx_p = 0.0f;
      int k0 = 0, marched = 0;
      float* wo = B.weights ? B.weights + (size_t)ray * S : nullptr;
      for (; k0 < S; k0 += 32) {
        const int k = k0 + lane;
        float alpha = 0.0f, fe, T, wgt;
        bool valid;
        if (k < S) {
          alpha = sample_alpha<H16>(F, R, k, S, fe, valid);
          if (valid) ++marched;
        }
        transmittance_step(alpha, k < S, lane, carry, T, wgt, [&] {
          if (k < S) {
            acc_p += wgt;
            dep_p += wgt * __ldg(F.z + k);
            idx_p += wgt * (float)k;
            if (floater) alpha_s[k] = alpha;
            else if (wo) wo[k] = wgt;
          }
        });
        if (!floater) {
          const bool on = (k < S) && (wgt > F.weight_thres);          // tensorBase.py:622
          const unsigned m = __ballot_sync(0xffffffffu, on);
          if (lane == 0 && m) atomicAdd(&slot->pending, __popc(m));
          queue_push<H16>(P, F, slots, Q, m, on, k, wgt, slot_id);
          if (carry < T_EPS) { k0 += 32; break; }                      // early ray termination
        }
      }
      if (!floater && wo)
        for (int k = k0 + lane; k < S; k += 32) wo[k] = 0.0f;          // terminated tail
      acc = warp_sum(acc_p); dep = warp_sum(dep_p);
      if (floater) {                                                   // tensorBase.py:617-620
        const float lim = warp_sum(idx_p) * B.floater_thresh;
        __syncwarp();
        float c2 = 1.0f;
        for (int kb = 0; kb < S; kb += 32) {
          const int k = kb + lane;
          float a = (k < S) ? alpha_s[k] : 0.0f;
          if ((float)k < lim) a = 0.0f;
          if (k == S - 1) a = 1.0f;
          float T, wgt;
          transmittance_step(a, k < S, lane, c2, T, wgt);
          if (k < S && wo) wo[k] = wgt;
          const bool on = (k < S) && (wgt > F.weight_thres);
          const unsigned m = __ballot_sync(0xffffffffu, on);
          if (lane == 0 && m) atomicAdd(&slot->pending, __popc(m));
          queue_push<H16>(P, F, slots, Q, m, on, k, wgt, slot_id);
        }
      }
      n_march += (unsigned long long)warp_sum((float)marched);
      // -- depth now, colour when the last row of this ray has been composited ---------------------
      if (lane == 0) {
        float dpt = __fdiv_rn(dep, R.nrm) * R.blend;                   // tensorBase.py:615
        if (B.accumulate) dpt = B.depth[B.depth_stride * ray] + dpt;
        B.depth[B.depth_stride * ray] = dpt;
        slot->acc = acc;
        slot->depth = dpt;
        __threadfence_block();
        const int old = atomicSub(&slot->pending, 1);                  // drop the open token
        if (old == 1) { __threadfence_block(); finalize_slot(B, slot); }
      }
      __syncwarp();
    }
    if (Q.qn > 0) { flush_rows<H16>(P, F, slots, Q, Q.qn); Q.qn = 0; }
    // -- the last producer completes the open tile and publishes the tile count ----------------------
    if (lane == 0 && B.stats) { atomicAdd(B.stats, n_march); atomicAdd(B.stats + 1, Q.n_app); }
    unsigned int d = 0;
    if (lane == 0) { __threadfence_block(); d = atomicAdd(&ctrl->prod_done, 1u); }
    d = __shfl_sync(0xffffffffu, d, 0);
    if (d == (unsigned int)nprod - 1) {
      pad_open_tile(P);
      if (lane == 0) {
        *reinterpret_cast<volatile unsigned int*>(&ctrl->n_tiles_final) =
            *reinterpret_cast<volatile unsigned int*>(&ctrl->cursor) >> 7;
        __threadfence_block();
        *reinterpret_cast<volatile unsigned int*>(&ctrl->done) = 1u;
      }
    }
  } else if (warp >= W_CONS) {
    // ======================================= CONSUMERS ===========================================
    const int ctid = tid - W_CONS * 32, wg = ctid >> 7, q = lane & 3;
    const float* tail = reinterpret_cast<const float*>(smem + L.prep + (PE ? PE_TAIL : PREP_TAIL));
    const float* W3_s = tail + TAIL_W3;
    const float* b3_s = tail + TAIL_B3;
    const uint32_t prep_a = smem_u32(smem + L.prep);
    const uint32_t wbuf = prep_a + PE_WBUF, wrdy = smem_u32(&ctrl->wrdy);
    const unsigned char* w1_g = reinterpret_cast<const unsigned char*>(F.prep) + PE_W1;
    const int nch = pe_chunks(F.fea_pe);
    float* xa = reinterpret_cast<float*>(smem + L.part) + wg * 64 * XA_LD;
    uint32_t wuse = 0;                                  // PE: layer-1 weight chunks consumed so far
    if (PE && ctid == 0) {                              // chunk 0 streams in under the first tile's layer 0
      mbar_expect_tx(wrdy, 2 * PE_WC_BYTES);
      tma_bulk_g2s(wbuf, w1_g, 2 * PE_WC_BYTES, wrdy);
    }
    mbar_wait(smem_u32(&ctrl->bar_w), 0);
    for (unsigned int T = 0;; ++T) {
      const int b = (int)(T & 1);
      bool stop = false;
      while (!mbar_try(smem_u32(&ctrl->full[b]), (T >> 1) & 1)) {
        if (*reinterpret_cast<volatile unsigned int*>(&ctrl->done) &&
            T >= *reinterpret_cast<volatile unsigned int*>(&ctrl->n_tiles_final)) { stop = true; break; }
      }
      if (stop) break;
      const uint32_t a1 = smem_u32(smem + L.a1 + b * (2 * OPER1_BYTES));
      const int h = wg;                                 // tile rows 64 h .. 64 h + 63
      const uint32_t a_hi = a1 + (uint32_t)h * 8u * K1_CHUNKS * 128u, a_lo = a_hi + OPER1_BYTES;
      float acc[64];
      if (PE) {
        // -- layer 0: the 27 basis features; then the encoded layer-1 input, 64 columns at a time ---------
        // x = [a, sin(a_d 2^f) (d-major, f-minor), cos(...)]   (tensorBase.py:14-21,115-125); zeros when !refine
        {
          float a0[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) a0[i] = 0.0f;
          const uint32_t sbo = (uint32_t)K1_CHUNKS * 128u;
          wgmma_fence();
          for (int ks = 0; ks < K1 / 16; ++ks) {
            const uint32_t ko = (uint32_t)ks * 256u;
            const uint64_t ah = gmma_desc(a_hi + ko, 128u, sbo), al = gmma_desc(a_lo + ko, 128u, sbo);
            const uint64_t bh = gmma_desc(prep_a + PE_B0HI + ko, 128u, sbo), bl = gmma_desc(prep_a + PE_B0LO + ko, 128u, sbo);
            wgmma_n32_ss(a0, ah, bh, ks > 0 ? 1u : 0u);
            wgmma_n32_ss(a0, ah, bl, 1u);
            wgmma_n32_ss(a0, al, bh, 1u);
          }
          wgmma_commit();
          wgmma_wait_all();
          fence_regs(a0);
          asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");   // the previous half's reads of xa are done
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              xa[wg_row(j) * XA_LD + 8 * i + 2 * q] = a0[4 * i + 2 * j];
              xa[wg_row(j) * XA_LD + 8 * i + 2 * q + 1] = a0[4 * i + 2 * j + 1];
            }
          asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        }
        const int Fp = F.fea_pe, nsin = APP_DIM * Fp;
        auto enc = [&](int j, int k) -> float {        // encoded input k of fragment row j
          const float* a = xa + wg_row(j) * XA_LD;
          if (k < APP_DIM) return a[k];
          if (B.refine && k < APP_DIM + 2 * nsin) {
            const int e = (k - APP_DIM) % nsin, d = e / Fp, f = e - d * Fp;
            const float ang = a[d] * (float)(1 << f);
            return (k - APP_DIM) < nsin ? sinf(ang) : cosf(ang);
          }
          return 0.0f;
        };
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
#pragma unroll 1
        for (int c = 0; c < nch; ++c) {
          uint32_t xh[PE_KC / 16][4], xl[PE_KC / 16][4];
#pragma unroll
          for (int ks = 0; ks < PE_KC / 16; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {               // A fragment register r: row j = r & 1, K 16 ks + 8 (r >> 1) + 2q
              const int k = c * PE_KC + 16 * ks + 8 * (r >> 1) + 2 * q;
              split2(enc(r & 1, k), enc(r & 1, k + 1), xh[ks][r], xl[ks][r]);
            }
          mbar_wait(wrdy, wuse & 1u);                   // weight chunk c is in shared memory
          const uint32_t sbo = (uint32_t)(PE_KC / 8) * 128u;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < PE_KC / 16; ++ks) {
            const uint32_t ko = (uint32_t)ks * 256u;
            const uint64_t bh = gmma_desc(wbuf + ko, 128u, sbo), bl = gmma_desc(wbuf + PE_WC_BYTES + ko, 128u, sbo);
            wgmma_n128_rs(acc, xh[ks], bh, 1u);
            wgmma_n128_rs(acc, xh[ks], bl, 1u);
            wgmma_n128_rs(acc, xl[ks], bh, 1u);
          }
          wgmma_commit();
          wgmma_wait_all();
          fence_regs(acc);
          ++wuse;
          asm volatile("bar.sync 1, %0;" ::"n"(N_CONS * 32) : "memory");   // every consumer is done with the chunk
          if (ctid == 0) {                              // the next chunk (of this tile, or chunk 0 of the next)
            mbar_expect_tx(wrdy, 2 * PE_WC_BYTES);
            tma_bulk_g2s(wbuf, w1_g + (size_t)((c + 1) % nch) * 2 * PE_WC_BYTES, 2 * PE_WC_BYTES, wrdy);
          }
        }
      } else {
        mlp_gemm_n128(acc, a_hi, a_lo, prep_a + PREP_B1HI, prep_a + PREP_B1LO, K1 / 16, K1_CHUNKS);
      }
      float sc[2][3];
      mlp_layers23(acc, tail, prep_a + (PE ? PE_B2HI : PREP_B2HI), prep_a + (PE ? PE_B2LO : PREP_B2LO), sc);
      // -- composite (tensorBase.py:632): w * rgb into the ray's fixed-point accumulators -------------
      // The quad's 2 rows x 3 channels are spread over its four lanes (all four hold the same sums): lane q
      // takes items q and q + 4 (row item / 3, channel item % 3).  Then one lane per row drops the row from
      // its ray's pending count.
      const unsigned char* mslot = smem + L.mslot + b * TM + 64 * h;
      const float* mw = reinterpret_cast<const float*>(smem + L.mw) + b * TM + 64 * h;
      const int slot0 = mslot[wg_row(0)], slot1 = mslot[wg_row(1)];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int it = q + 4 * r, j = it >= 3 ? 1 : 0, c = it - 3 * j;
        const int my_slot = j ? slot1 : slot0;
        if (it >= 6 || my_slot == 0xFF) continue;
        const float my_w = mw[wg_row(j)];
        Slot* sl = slots + my_slot;
        float v = j ? (c == 0 ? sc[1][0] : c == 1 ? sc[1][1] : sc[1][2])
                    : (c == 0 ? sc[0][0] : c == 1 ? sc[0][1] : sc[0][2]);
        if (PE) v += sl->vterm[c];
        else v += W3_s[c * W3_LD + FC] * sl->vd[0] + W3_s[c * W3_LD + FC + 1] * sl->vd[1] +
                  W3_s[c * W3_LD + FC + 2] * sl->vd[2];
        v += b3_s[c];
        v = __fdiv_rn(1.0f, 1.0f + expf(-v));
        atomicAdd(&sl->rgb[c], __float2uint_rn(my_w * v * FIX_SCALE));
      }
      __threadfence_block();
      __syncwarp();                                     // the quad's channel adds precede its rows' pending drops
      const int row_slot = q ? slot1 : slot0;
      if (q < 2 && row_slot != 0xFF) {
        Slot* sl = slots + row_slot;
        const int old = atomicSub(&sl->pending, 1);
        if (old == 1) { __threadfence_block(); finalize_slot(B, sl); }
      }
      // the A tile and its row metadata have been read: the producers may rewrite buffer b
      asm volatile("bar.sync 1, %0;" ::"n"(N_CONS * 32) : "memory");
      if (ctid == 0) {
        __threadfence_block();
        *reinterpret_cast<volatile unsigned int*>(&ctrl->released) = T + 1u;
      }
    }
    if (PE) mbar_wait(wrdy, wuse & 1u);                 // the last prefetched chunk has landed before the CTA exits
  }
  __syncthreads();
  if (B.signal_seq && tid == 0) {
    // every pixel store of this CTA is ordered before the barrier above; the last CTA of the launch
    // publishes the step to all peers (release at system scope, after a cumulative fence)
    __threadfence_system();
    const unsigned int old = atomicAdd(B.done_ctr, 1u);
    if (old == gridDim.x - 1) {
      __threadfence_system();
      for (int p = 0; p < B.n_peers; ++p) {
        unsigned long long* remote = B.peer_flags[p] + B.rank;
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(remote), "l"(B.signal_seq) : "memory");
      }
    }
  }
}

// ---- host-side launcher --------------------------------------------------------------------------
int render_threads() { return THREADS; }

// the most producer warps whose queues fit max_smem (the floater filter's alpha tables grow with S)
static int pick_nprod(int S, bool floater, int max_smem, bool pe = false) {
  for (int n = MAX_PROD; n >= 1; --n)
    if (smem_v3(S, floater, n, pe).total <= max_smem) return n;
  return 0;
}

size_t render_smem_bytes(int S, bool floater, int max_smem, bool pe) {
  const int n = pick_nprod(S, floater, max_smem, pe);
  return (size_t)smem_v3(S, floater, n ? n : 1, pe).total;
}

cudaError_t launch_render(const FieldDev& F, const BatchDev& B, int n_sms, int max_smem,
                          cudaStream_t stream) {
  const bool floater = B.floater_thresh > 0.0f;
  const bool pe = F.fea_pe > 0 || F.view_pe > 0;
  const int nprod = pick_nprod(F.S, floater, max_smem, pe);
  if (nprod < 1) return cudaErrorInvalidConfiguration;
  const size_t smem = (size_t)smem_v3(F.S, floater, nprod, pe).total;
  const int variant = pe ? 1 : (F.grid16 ? 2 : 0);   // (bf16 grids with positional encodings are refused by the ABI)
  const void* kern = variant == 1 ? (const void*)render_kernel_t<true, false>
                   : variant == 2 ? (const void*)render_kernel_t<false, true> : (const void*)render_kernel_t<false, false>;
  cudaError_t e = set_max_dynamic_smem(kern, (int)smem);
  if (e == cudaSuccess) e = set_smem_carveout(kern, (int)smem);   // the L1 gets what the CTA leaves
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(B.sched, 0, 2 * sizeof(unsigned long long), stream);   // ray counter + finished-CTA counter
  if (e != cudaSuccess) return e;
  // a CTA per SM, but never more CTAs than there are groups of 8 rays
  const unsigned int grid = cta_count(B.n_rays, 8, n_sms, 1);
  if (variant == 1) render_kernel_t<true, false><<<grid, THREADS, smem, stream>>>(F, B, nprod);
  else if (variant == 2) render_kernel_t<false, true><<<grid, THREADS, smem, stream>>>(F, B, nprod);
  else render_kernel_t<false, false><<<grid, THREADS, smem, stream>>>(F, B, nprod);
  return cudaGetLastError();
}

}  // namespace lrf
