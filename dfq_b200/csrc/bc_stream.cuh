// k_bc_stream: bias correction (dfq.py:173-293) for LARGE phases - the bandwidth-bound variant of k_bc_engine.
//
// k_bc_engine processes one tile per CTA at a time: every 18 KB row pays two CTA-wide barriers, a serial 8-way fp64
// sum and three dependent read-modify-writes by thread 0, and every element an IEEE division (MUFU.RCP + FCHK + 5 FFMA)
// and an FRND: CTA barriers and waits dominate the warp stalls and the XU pipe saturates on MUFU.RCP + FRND (2 x 4608
// quarter-rate ops per row).
//
// Here every consumer WARP owns whole tiles:
//   * one CTA per SM: 8 consumer warps + 1 producer warp, a ring of kBcStages 18 KB stages (all of the SM's shared
//     memory); per stage a `full` mbarrier (TMA transaction bytes) and an `empty` mbarrier (the consuming warp's lane 0):
//     NO CTA-wide barrier anywhere in the streaming loop;
//   * the producer's lane 0 walks the CTA's tile list (same block-cyclic order as RowPipe), waits for the stage to be
//     empty, writes the descriptor and issues the bulk copy; consumer w takes sequence numbers n = w (mod 8).  A phase
//     ends with padding SKIP items up to a multiple of 8 and then 8 END items, so every consumer sees exactly one END;
//   * a tile's rows are reduced by the warp alone (lanes over input columns, 9 taps each, warp shuffle at the end);
//     lane r requests row r's read-modify-write operands before the tile and retires them after it;
//   * the expectation vector of the current (layer, group) is cached per warp in shared memory (cols <= 512) across tiles;
//   * the row is read with 32-bit shared-memory addresses (ld.shared, no generic LD + 64-bit address arithmetic) in a
//     ROLLED column loop: the first version unrolled 16 x 9 taps x 5 variants = 23 800 SASS instructions and stalled on
//     instruction fetch;
//   * the quantization error is computed with no XU-pipe instruction:
//       - the quotient t / scale as Markstein's correction of the product with the correctly rounded reciprocal
//         (q0 = t*y, r = fma(-q0, s, t), q = fma(r, y, q0); y = __frcp_rn(s)): equal to the IEEE quotient when no
//         intermediate underflows and the mantissa of s is not all ones - both checked once per tensor (BcFastQuant::ok),
//         otherwise the plain __fdiv_rn chain runs for that tensor.  t lies in [0, max-min], q in [qmin, qmax];
//       - rint() for |t| <= 2^22 as (t + 1.5*2^23) - 1.5*2^23 (two FADDs, round-half-even like FRND);
//       - no clamp: on the tensor's own range the quotient cannot leave [qmin, qmax] before the rounding (bc_qerr_own_range).
//     tests/test_gpu_engine.py::test_bc_fast_quotient_equals_ieee_division checks codes AND quotients against __fdiv_rn
//     over thousands of scales x dense numerators including every half-integer neighbourhood.
#pragma once
#include "common.cuh"
#include "rowpipe.cuh"

namespace dfq {

// 7 consumer warps + the producer = 8 warps = two per SM sub-partition; 11 - 7 = 4 stages loading while all consumers compute.
#ifndef DFQ_BC_CONSUMERS
#define DFQ_BC_CONSUMERS 7
#endif
constexpr int kBcConsumers = DFQ_BC_CONSUMERS;
constexpr int kBcThreads = (kBcConsumers + 1) * 32;
#ifndef DFQ_BC_STAGES
#define DFQ_BC_STAGES 11
#endif
constexpr int kBcStages = DFQ_BC_STAGES;
constexpr int kBcExCols = 512;                // expectation values a consumer warp caches in shared memory (2 KB per warp)

enum { BTK_SKIP = 3, BTK_END = 4 };

struct BcFastQuant {
  float neg_min, min_v, scale, rcp, qmin, qmax;
  int ok;        // 1: the three-instruction quotient is exact for every numerator this tensor can produce
};

__device__ __forceinline__ BcFastQuant bc_fast_quant(const QuantScalars& q, int num_bits) {
  BcFastQuant f;
  f.neg_min = q.neg_min; f.min_v = q.min_v; f.scale = q.scale; f.qmin = q.qmin; f.qmax = q.qmax;
  f.rcp = __frcp_rn(q.scale);
  const unsigned bits = __float_as_uint(q.scale);
  const int e = (int)((bits >> 23) & 0xff);
  // exponent window: the residual r = t - q0*s is ~2^-24 of t and must stay normal for every t whose quotient can reach
  // 0.5 (smaller t give code 0 or qmin's neighbourhood either way): t >= s/4 -> r >= s * 2^-27.  The reciprocal must be
  // normal as well.  Mantissa all ones: the one divisor for which RN(1/s) is not close enough (Markstein).
  f.ok = (num_bits <= 16) && e >= 40 && e <= 200 && ((bits & 0x7fffffu) != 0x7fffffu) && !(q.scale != q.scale);
  return f;
}

// quantize.py:70-74 for one element, error form: Q(w) - w
template <bool FAST>
__device__ __forceinline__ float bc_qerr(float w, const BcFastQuant& f) {
  float t = __fadd_rn(w, f.neg_min);
  if (FAST) {
    const float q0 = __fmul_rn(t, f.rcp);
    const float r = __fmaf_rn(-q0, f.scale, t);
    t = __fmaf_rn(r, f.rcp, q0);
    t = fminf(fmaxf(t, f.qmin), f.qmax);
    t = __fsub_rn(__fadd_rn(t, 12582912.0f), 12582912.0f);
  } else {
    t = __fdiv_rn(t, f.scale);
    t = fminf(fmaxf(t, f.qmin), f.qmax);
    t = rintf(t);
  }
  t = __fmul_rn(t, f.scale);
  return __fsub_rn(__fadd_rn(t, f.min_v), w);
}

// scipy.stats.norm.pdf / cdf in float64 on an fp32 argument, rounded to fp32 (dfq.py:182-183)
__device__ __forceinline__ float std_pdf(float x32) {
  const double x = (double)x32;
  return (float)(exp(-x * x / 2.0) / 2.5066282746310002);   // sqrt(2*pi)
}
__device__ __forceinline__ float std_cdf(float x32) {
  // scipy.special.ndtr (cephes)
  const double x = (double)x32 * 0.70710678118654752440;
  const double z = fabs(x);
  double y;
  if (z < 0.70710678118654752440) y = 0.5 + 0.5 * erf(x);
  else { y = 0.5 * erfc(z); if (x > 0) y = 1.0 - y; }
  return (float)y;
}
// dfq.py:184 calculate_mean + :240 clamp; every op an individually rounded fp32 op as in eager PyTorch
__device__ __forceinline__ float relu_gauss_mean(float g, float b) {
  const float q = __fdiv_rn(-b, g);
  const float t1 = __fmul_rn(g, std_pdf(q));
  const float t2 = __fmul_rn(b, __fsub_rn(1.0f, std_cdf(q)));
  const float e = __fadd_rn(t1, t2);
  return e < 0.f ? 0.f : e;      // NaN stays NaN (expect[expect < 0] = 0)
}

// E[x] of one layer (dfq.py:228-278) into ex: its terms in order, each written to or (accumulate) added into its slice.
// SMEM: ex is this CTA's shared-memory copy; otherwise it lies in the arena and is accessed with .cg.  (k_bc_engine,
// k_bc_stream, and k_cle_stack's prologue of an attached correction.)
template <int THREADS, bool SMEM>
__device__ __forceinline__ void bc_expect(float* arena, const DfqBcLayer& b, const DfqExpectTerm* __restrict__ T, float* ex) {
  for (int ti = b.term_begin; ti < b.term_end; ++ti) {
    const DfqExpectTerm t = T[ti];
    for (int ch = threadIdx.x; ch < t.n; ch += THREADS) {
      const float fb = __ldcg(arena + t.bn_b_off + ch);
      const float v = t.relu ? relu_gauss_mean(__ldcg(arena + t.bn_w_off + ch), fb) : fb;
      float* d = ex + t.dst_off + ch;
      if (SMEM) *d = t.accumulate ? __fadd_rn(*d, v) : v;
      else __stcg(d, t.accumulate ? __fadd_rn(__ldcg(d), v) : v);
    }
    __syncthreads();
  }
}

// STAGES stages of kStageBytes: kBcStages for k_bc_stream and k_cle_stack (BcRing), kScanStages for the fold's scan.
template <int STAGES>
struct BcRingT {
  static constexpr int kStages = STAGES;
  unsigned char* base;
  __device__ __forceinline__ float* stage(int s) const { return (float*)(base + (size_t)s * kStageBytes); }
  uint64_t* full;      // [STAGES]
  uint64_t* empty;     // [STAGES]
  TileDesc* desc;      // [STAGES]
  __device__ void init(unsigned char* smem) {
    base = smem;
    unsigned char* p = smem + (size_t)STAGES * kStageBytes;
    full = (uint64_t*)p;
    empty = (uint64_t*)(p + 8 * STAGES);
    desc = (TileDesc*)(p + 16 * STAGES + 16);
    if (threadIdx.x == 0) {
      for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 1); desc[i].seq = -1; }
      mbar_fence_init();
    }
    __syncthreads();
  }
  // behind the ring: one expectation cache per consumer warp
  __device__ __forceinline__ float* ex_cache(int warp) const {
    return (float*)(base + ring_bytes()) + (size_t)warp * (kBcExCols + 4);
  }
  __host__ __device__ static constexpr size_t ring_bytes() { return (((size_t)STAGES * kStageBytes + 16 * STAGES + 16 + STAGES * sizeof(TileDesc)) + 127) & ~(size_t)127; }
  static constexpr size_t smem_bytes() { return ring_bytes() + (size_t)kBcConsumers * (kBcExCols + 4) * 4 + 64; }
};
using BcRing = BcRingT<kBcStages>;

// Producer lane: put item `d` at sequence number n.
template <class Ring>
__device__ __forceinline__ void bc_produce(Ring& ring, unsigned long long n, const TileDesc& d) {
  constexpr int S = Ring::kStages;
  const int s = (int)(n % S);
  if (n >= S) mbar_wait(ring.empty + s, (uint32_t)(((n / S) - 1) & 1));
  ring.desc[s] = d;
  ring.desc[s].seq = (int)n;            // before the arrive below: visible to whoever sees the phase complete
  if (d.kind == TK_BULK) {
    mbar_arrive_expect_tx(ring.full + s, (uint32_t)d.floats * 4u);
    bulk_g2s(ring.stage(s), d.gptr, (uint32_t)d.floats * 4u, ring.full + s);
  } else {
    mbar_arrive(ring.full + s);
  }
}

// Consumer side: wait for item n; returns its stage.
//
// A parity wait alone is NOT enough here.  `mbarrier.try_wait.parity p` answers "has the phase with parity p completed?" by
// comparing p with the barrier's current phase parity - which is only meaningful when the waiter is at most one phase away.
// Consumers of this ring own different stages in turn (the stage count is not a multiple of the consumer count), so the warp
// that is about to wait for use u of stage s may get there while use u-1 of that stage - another warp's item, issued 11 items
// earlier - is still LOADING: the barrier is then in phase u-1, its parity differs from u's, and try_wait returns "done" at
// once.  The warp would process the previous tile's stage a second time and arrive on `empty` a second time ("Warp
// Illegal Instruction" at the producer's next arrive, hangs, on stacks of 16-96 blocks whose loads start cold; steady-state
// runs of 1000+ blocks never hit it).  The producer therefore stamps every item with its sequence number before it arrives,
// and the consumer re-checks the stamp after every wait (and waits once more after it matched: the stamp is written before
// the producer's arrive, so by then the barrier is in the right phase).
template <class Ring>
__device__ __forceinline__ int bc_take(Ring& ring, unsigned long long n) {
  constexpr int S = Ring::kStages;
  const int s = (int)(n % S);
  const volatile int* seq = &ring.desc[s].seq;
  const uint32_t parity = (uint32_t)((n / S) & 1);
  for (;;) {                                   // common case: one hardware wait, one shared-memory compare
    mbar_wait(ring.full + s, parity);
    if (*seq == (int)n) break;                 // the stage holds MY item
    __nanosleep(64);                           // spurious "done": the barrier was still one phase behind
  }
  mbar_wait(ring.full + s, parity);            // stamp seen => the barrier is in (or past) my phase: returns when the bytes have landed
  return s;
}
template <class Ring>
__device__ __forceinline__ void bc_give_back(Ring& ring, int s, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(ring.empty + s);
}

__device__ __forceinline__ float lds_f32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}

// quantize.py:70-74 without the clamp: for a tensor quantized on ITS OWN range (always the case in bias correction,
// dfq.py:14) t = w - min lies in [0, RN(max - min)] and RN(t / scale) in [0, 255.00003] (symmetric: |q| <= 127.00002), so
// clamp_(qmin, qmax) never changes anything before the rounding.  (NaN weights propagate, as they do through torch.clamp.)
__device__ __forceinline__ float bc_qerr_own_range(float w, const BcFastQuant& f) {
  float t = __fadd_rn(w, f.neg_min);
  const float q0 = __fmul_rn(t, f.rcp);
  const float r = __fmaf_rn(-q0, f.scale, t);
  t = __fmaf_rn(r, f.rcp, q0);
  t = __fsub_rn(__fadd_rn(t, 12582912.0f), 12582912.0f);
  t = __fmul_rn(t, f.scale);
  return __fsub_rn(__fadd_rn(t, f.min_v), w);
}

// One column (kk taps at shared address `a`) of one output row.  MODE 0: XU-free arithmetic on the tensor's own range,
// 1: plain IEEE chain (per-tensor guard refused), 2: raw sum (bias absorption).
template <int MODE, int KK>
__device__ __forceinline__ float bc_col_smem(uint32_t a, int kk, const BcFastQuant& f) {
  float E = 0.f;
  if (KK == 9) {
    float w[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) w[k] = lds_f32(a + 4u * k);
#pragma unroll
    for (int k = 0; k < 9; ++k) E = __fadd_rn(E, MODE == 2 ? w[k] : (MODE == 0 ? bc_qerr_own_range(w[k], f) : bc_qerr<false>(w[k], f)));
  } else if (KK == 1) {
    const float w = lds_f32(a);
    E = __fadd_rn(E, MODE == 2 ? w : (MODE == 0 ? bc_qerr_own_range(w, f) : bc_qerr<false>(w, f)));
  } else {
    for (int k = 0; k < kk; ++k) {
      const float w = lds_f32(a + 4u * k);
      E = __fadd_rn(E, MODE == 2 ? w : (MODE == 0 ? bc_qerr_own_range(w, f) : bc_qerr<false>(w, f)));
    }
  }
  return E;
}

// One output row resident in SHARED memory: lanes over input columns (kk taps each, 36-byte lane stride for 3x3: conflict
// free), fp32 tap sum per column, fp64 dot with the expectation vector (`exs`: this warp's shared-memory copy when the
// layer has <= kBcExCols columns, else `exg` in global memory).
template <int MODE, int KK>
__device__ __forceinline__ double bc_stream_row_smem(uint32_t srow, int cols, int kk, const float* __restrict__ exs,
                                                     const float* __restrict__ exg, const BcFastQuant& f, int lane) {
  double acc = 0.0;
  const int nfull = cols >> 5;
  const uint32_t stride = 32u * 4u * (uint32_t)kk;
  uint32_t a = srow + (uint32_t)lane * 4u * (uint32_t)kk;
  if (exs) {
#pragma unroll 2
    for (int c = 0; c < nfull; ++c, a += stride)
      acc = __fma_rn((double)bc_col_smem<MODE, KK>(a, kk, f), (double)exs[lane + 32 * c], acc);
    if (lane + 32 * nfull < cols) acc = __fma_rn((double)bc_col_smem<MODE, KK>(a, kk, f), (double)exs[lane + 32 * nfull], acc);
  } else {
    for (int c = 0; c < nfull; ++c, a += stride)
      acc = __fma_rn((double)bc_col_smem<MODE, KK>(a, kk, f), (double)__ldcg(exg + lane + 32 * c), acc);
    if (lane + 32 * nfull < cols) acc = __fma_rn((double)bc_col_smem<MODE, KK>(a, kk, f), (double)__ldcg(exg + lane + 32 * nfull), acc);
  }
  return warp_sum(acc);
}

// Rows longer than a stage stay in global memory (TK_DIRECT): plain loop, L2 reads.
template <int MODE>
__device__ __forceinline__ double bc_stream_row_gmem(const float* __restrict__ row, int cols, int kk, const float* __restrict__ exg,
                                                     const BcFastQuant& f, int lane) {
  double acc = 0.0;
  for (int j = lane; j < cols; j += 32) {
    const float* p = row + (size_t)j * kk;
    float E = 0.f;
    for (int k = 0; k < kk; ++k) {
      const float w = ldg_stream1(p + k);
      E = __fadd_rn(E, MODE == 2 ? w : (MODE == 0 ? bc_qerr_own_range(w, f) : bc_qerr<false>(w, f)));
    }
    acc = __fma_rn((double)E, (double)__ldcg(exg + j), acc);
  }
  return warp_sum(acc);
}

}  // namespace dfq
