// Cross-layer equalization engine: ONE persistent cooperative kernel runs every sweep of
// dfq.py:78-117 (cross_layer_equalization) on the device, including the exit rule.
//
// Reference semantics being reproduced (file:line under /root/reference):
//   dfq.py:48-55   per-channel range of row c of W1 and of input column c of W2
//   dfq.py:58-59   s = (1/(r1+eps)) * sqrt(r1*r2+eps), clamped with Python min/max semantics
//   dfq.py:62-73   W1[c] *= s, bn_weight/bn_bias/bias[c] *= s, W2[:, c] *= 1/s
//   dfq.py:84,105-115  convergence: sum over layers of mean|W - W_prev|, exit rule
//   relation.py:20-24  Relation.S accumulates the product of per-sweep s
//
// Data-parallel restructuring (bit-identical, see DESIGN.md section 3):
//   * the reference's per-channel Python loop is independent across channels, so all ranges of a
//     relation are formed first, then all scalings;
//   * relations are visited in forward chain order, so the column scaling of relation A on layer l
//     and the row scaling of relation B on the same layer are applied in ONE pass over l
//     (v -> fl(v*inv_A[col]) -> fl(.*s_B[row])), 8 bytes of HBM traffic per weight per sweep;
//   * column ranges needed by the *next* sweep are not re-read: rounding is monotone, so after a
//     pure column scaling  max(fl(v*a)) = fl(max(v)*a)  for a > 0 (likewise min), and the running
//     column extrema are updated analytically ("derived").  Only general middle layers (both
//     column- and row-scaled with cols > 1) need fresh extrema every sweep, accumulated from the
//     rescaled tile while it still sits in shared memory.
//   * the step barrier between chain positions is a grid barrier of the persistent kernel.
#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "rowpipe.cuh"
#include "colscan.cuh"
#include "bc_stream.cuh"

namespace cg = cooperative_groups;

namespace dfq {

// CTA = 7 consumer warps (the arithmetic) + 1 producer warp (TMA loads/stores and the per-row scalar bookkeeping),
// see "warp-specialised pass" below.  kThreads / kWarps count the CONSUMERS: every tile loop and reduction strides by them.
#ifndef DFQ_CONSUMERS
#define DFQ_CONSUMERS 224
#endif
// ring geometry of THIS kernel (rowpipe.cuh's kPipeStages / kPipeCtas configure the simpler fold / bias-correction pipes)
#ifndef DFQ_CLE_STAGES
#define DFQ_CLE_STAGES 3
#endif
#ifndef DFQ_CLE_CTAS
#define DFQ_CLE_CTAS 3
#endif
constexpr int kCleStages = DFQ_CLE_STAGES;   // stages per CTA
constexpr int kCleCtas = DFQ_CLE_CTAS;       // co-resident CTAs per SM the kernel is compiled for
#ifndef DFQ_TEAMS
#define DFQ_TEAMS 1
#endif
// Consumer TEAMS: kTeams groups of kThreads threads, each working on its own tile (own named barrier, own context and
// caches), fed in turn from the one ring the producer warp fills: tile n of the CTA goes to team n % kTeams.
constexpr int kTeams = DFQ_TEAMS;
constexpr int kThreads = DFQ_CONSUMERS;      // per team
constexpr int kWarps = kThreads / 32;
constexpr int kCtaThreads = kTeams * kThreads + 32;
static_assert(kThreads % 32 == 0 && kWarps <= 8 && kTeams >= 1 && kTeams <= 8, "team geometry");
__device__ __forceinline__ int ctid() { return kTeams == 1 ? (int)threadIdx.x : (int)(threadIdx.x % kThreads); }   // thread within its team
__device__ __forceinline__ int team() { return kTeams == 1 ? 0 : (int)(threadIdx.x / kThreads); }
// a team is a virtual CTA for everything that is distributed per CTA outside the ring
__device__ __forceinline__ int vblock() { return blockIdx.x * kTeams + team(); }
__device__ __forceinline__ int vgrid() { return gridDim.x * kTeams; }
// barrier among the warps of one team only (the producer warp never joins it)
__device__ __forceinline__ void cbar() {
  if (kTeams == 1) asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory");
  else asm volatile("bar.sync %0, %1;" ::"r"(1 + team()), "n"(kThreads) : "memory");
}
#ifndef DFQ_INV_CACHE
#define DFQ_INV_CACHE 2044
#endif
constexpr int kInvCache = DFQ_INV_CACHE;    // reciprocal scales of a layer's input columns cached in shared memory
constexpr int kScanCols = (kInvCache + 4) / 2 < 1024 ? (kInvCache + 4) / 2 : 1024;   // columns a scan keeps in shared memory (aliases that cache)

// Convergence state of one GROUP of chains.  The reference's exit rule (dfq.py:81-115) is evaluated per model: one
// group.  A batch of independent models (the synthetic stack: every block is its own model) is calibrated in one
// launch with one group per model, each stopping on its own.
struct GroupState {
  double acc[3];   // rotating per-sweep accumulators of sum_l mean|dW_l|
  double diff;     // `diff` of dfq.py:81
  int count;       // `count` of dfq.py:82
  int n_sweeps;
  int done;
  int converged;
};
struct CleCtl {
  int active[2];   // groups still iterating, double-buffered by sweep parity
  double diffs[64];  // diff_tmp per sweep of group 0
  unsigned long long t_ns[32];  // %globaltimer at phase boundaries (block 0), printed when DFQ_TRACE is set
  int grid, per_sm;
  unsigned long long tile_ns[48][8];  // per-tile timeline of block 0 in the first pass (DFQ_TRACE): consumer 0-3, producer 4-7
};

#ifdef DFQ_STEP_TRACE
// debug build: per-CTA timeline of every step of sweep 2 (thread 0 of each CTA): 0 step start, 1 first tile (or END) seen,
// 2 layer context ready, 3 first tile computed, 4 first tile handed back, 5 END seen, 6 fenced (about to enter the grid
// barrier), 7 tiles consumed
__device__ unsigned long long g_step_trace[8][512][8];
#endif
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// pass tiles: contiguous chunks of rows moved by the RowPipe (rowpipe.cuh)
__host__ __device__ inline int pass_tiles(const DfqLayer& l) { return pipe_tiles(l.rows, l.cols * l.kk); }
// Everything a row pass needs to know about its layer; uniform across the CTA.
struct RowCtx {
  float* w;
  int rows, cols, kk, row_len;
  const float* inv_in;  // reciprocal scales of rel_in (applied to columns), or nullptr
  int in_gi, in_go;
  int has_out;
  const float* cmin_rd;  // column extrema of the second layer of rel_out, buffer of this sweep
  const float* cmax_rd;
  float* cmin_wr;        // next sweep's buffer (derived update), or nullptr when it is re-scanned
  float* cmax_wr;
  float *s_step, *inv_out, *s_acc, *bias, *bnw, *bnb;
  float* own_cmin_wr;    // col_mode 1: this layer's own next-sweep extrema get the row factor too
  float* own_cmax_wr;
  double inv_n;
  int first_sweep;
  int inv_cached;        // 1: inv_in[0 .. cols) of the (single) input group is cached in shared memory
};

// The column scans are rare in the sweep loop (general middle layers only): kept out of line so that their registers do
// not count against the hot rescale loop (80-register cap at 3 CTAs/SM; ptxas: 668 B -> 0 B of spills).
template <bool GLOBAL>
__device__ __noinline__ void colscan_tile_ool(const float* buf, int tid, int row0, int nrows, int J, int kk, int go, int gi,
                                             bool single_group, bool own, bool use_smem, float* smin, float* smax, float* dmin,
                                             float* dmax) {
  colscan_tile<kThreads, GLOBAL>(buf, tid, row0, nrows, J, kk, go, gi, single_group, own, use_smem, smin, smax, dmin, dmax);
}

// dfq.py:58-59 + :73.  Returns s; *inv is the factor applied to the columns of the second layer.
__device__ __forceinline__ float solve_scale(float r1, float r2, const DfqCleParams P, float* inv) {
  const float a = __frcp_rn(__fadd_rn(r1, P.eps));
  const float b = __fsqrt_rn(__fadd_rn(__fmul_rn(r1, r2), P.eps));
  const float s = __fmul_rn(a, b);
  // Python: m = min(hi, s) -> s if s < hi else hi   (NaN -> hi);  max(lo, m) -> m if m > lo else lo
  if (!(s < P.s_hi)) {
    if (P.s_hi > P.s_lo) { *inv = P.inv_hi; return P.s_hi; }
    *inv = P.inv_lo; return P.s_lo;
  }
  if (s > P.s_lo) { *inv = __frcp_rn(s); return s; }
  *inv = P.inv_lo;
  return P.s_lo;
}

__device__ __forceinline__ float range_of(float mn, float mx, int signed_mode) {
  return signed_mode ? fmaxf(fabsf(mn), fabsf(mx)) : __fsub_rn(mx, mn);
}

__device__ __forceinline__ int col_of(int e, int kk) {
  return kk == 1 ? e : (kk == 9 ? e / 9 : e / kk);
}

// CTA-wide min/max with one barrier (double-buffered scratch, see parity argument in DESIGN.md).
__device__ __forceinline__ void cta_minmax(float& mn, float& mx, float* red, int& parity) {
  mn = warp_min(mn);
  mx = warp_max(mx);
  const int w = ctid() >> 5, l = ctid() & 31;
  float* r = red + (parity & 1) * 2 * kWarps;
  parity++;
  if (l == 0) { r[w] = mn; r[kWarps + w] = mx; }
  cbar();
  float a = r[0], b = r[kWarps];
#pragma unroll
  for (int i = 1; i < kWarps; ++i) { a = fminf(a, r[i]); b = fmaxf(b, r[kWarps + i]); }
  mn = a; mx = b;
}

// Per-stage mailbox between the producer warp and the consumers for single-row tiles:
//   producer -> consumers : cmn/cmx, the column extrema of the second layer for this channel (prefetched with the tile)
//   consumers -> producer : s / inv of this sweep; the producer then does the per-channel bookkeeping (publish_row)
struct StagePub { float cmn, cmx, s, inv; int valid; int pad[3]; };

// The per-channel bookkeeping of dfq.py:62-70 + relation.py:20-24 + the derived column extrema, for ONE channel.
// All loads are issued before the first store (the stores would otherwise fence the loads one global latency apart).
// The per-channel operands of publish_row: only the row's own publisher ever writes them, so they may be requested together
// with the row's inputs, one global-memory latency before they are needed.
struct RowPub { float a0, b0, w0, w1, o0, o1; };
__device__ __forceinline__ RowPub fetch_row_pub(const RowCtx& c, const DfqCleParams P, int o) {
  RowPub q;
  const bool acc = !P.apply_only && !c.first_sweep;
  q.a0 = acc ? __ldcg(c.s_acc + o) : 1.f;
  q.b0 = __ldcg(c.bias + o);
  q.w0 = c.bnw ? __ldcg(c.bnw + o) : 0.f;
  q.w1 = c.bnb ? __ldcg(c.bnb + o) : 0.f;
  q.o0 = c.own_cmin_wr ? __ldcg(c.own_cmin_wr + o) : 0.f;
  q.o1 = c.own_cmin_wr ? __ldcg(c.own_cmax_wr + o) : 0.f;
  return q;
}
__device__ __forceinline__ void publish_row_with(const RowCtx& c, const DfqCleParams P, int o, float s, float inv, float cmn,
                                                 float cmx, const RowPub& q) {
  c.s_step[o] = s;
  __stcg(c.inv_out + o, inv);
  if (!P.apply_only) c.s_acc[o] = c.first_sweep ? s : __fmul_rn(q.a0, s);
  __stcg(c.bias + o, __fmul_rn(q.b0, s));
  if (c.bnw) __stcg(c.bnw + o, __fmul_rn(q.w0, s));
  if (c.bnb) __stcg(c.bnb + o, __fmul_rn(q.w1, s));
  if (c.cmin_wr) {  // derived column extrema of the second layer after its column scaling
    __stcg(c.cmin_wr + o, __fmul_rn(cmn, inv));
    __stcg(c.cmax_wr + o, __fmul_rn(cmx, inv));
  }
  if (c.own_cmin_wr) {  // depthwise middle layer: its single-row column is this row
    __stcg(c.own_cmin_wr + o, __fmul_rn(q.o0, s));
    __stcg(c.own_cmax_wr + o, __fmul_rn(q.o1, s));
  }
}
__device__ __forceinline__ void publish_row(const RowCtx& c, const DfqCleParams P, int o, float s, float inv, float cmn, float cmx) {
  const bool acc = !P.apply_only && !c.first_sweep;
  const float a0 = acc ? __ldcg(c.s_acc + o) : 1.f;
  const float b0 = __ldcg(c.bias + o);
  const float w0 = c.bnw ? __ldcg(c.bnw + o) : 0.f;
  const float w1 = c.bnb ? __ldcg(c.bnb + o) : 0.f;
  const float o0 = c.own_cmin_wr ? __ldcg(c.own_cmin_wr + o) : 0.f;
  const float o1 = c.own_cmin_wr ? __ldcg(c.own_cmax_wr + o) : 0.f;
  c.s_step[o] = s;
  __stcg(c.inv_out + o, inv);
  if (!P.apply_only) c.s_acc[o] = c.first_sweep ? s : __fmul_rn(a0, s);
  __stcg(c.bias + o, __fmul_rn(b0, s));
  if (c.bnw) __stcg(c.bnw + o, __fmul_rn(w0, s));
  if (c.bnb) __stcg(c.bnb + o, __fmul_rn(w1, s));
  if (c.cmin_wr) {  // derived column extrema of the second layer after its column scaling
    __stcg(c.cmin_wr + o, __fmul_rn(cmn, inv));
    __stcg(c.cmax_wr + o, __fmul_rn(cmx, inv));
  }
  if (c.own_cmin_wr) {  // depthwise middle layer: its single-row column is this row
    __stcg(c.own_cmin_wr + o, __fmul_rn(o0, s));
    __stcg(c.own_cmax_wr + o, __fmul_rn(o1, s));
  }
}

// What a row needs from global memory, fetched ahead of the row by whoever can hide the latency (producer warp for
// single-row tiles, one lane per row for a warp's batch of rows).
struct RowIn {
  float cmn, cmx;   // column extrema of the second layer for this channel (HAS_OUT)
  float u;          // the row-uniform input factor (IN_UNIFORM)
  float s_given;    // apply_only: the scale to replay
};
__device__ __forceinline__ RowIn fetch_row_in(const RowCtx& c, const DfqCleParams P, int o, bool uniform) {
  RowIn in; in.cmn = in.cmx = 0.f; in.u = 1.f; in.s_given = 1.f;
  if (c.has_out) {
    in.cmn = __ldcg(c.cmin_rd + o); in.cmx = __ldcg(c.cmax_rd + o);
    if (P.apply_only) in.s_given = __ldcg(c.s_acc + o);
  }
  if (uniform) in.u = __ldcg(c.inv_in + (o / c.in_go) * c.in_gi);
  return in;
}
// dfq.py:58-59 + :73 for one channel from its row / column extrema (or the replayed scale)
__device__ __forceinline__ float solve_row(const DfqCleParams P, const RowIn& in, float mn, float mx, float* inv) {
  if (P.apply_only) { *inv = __frcp_rn(in.s_given); return in.s_given; }
  return solve_scale(range_of(mn, mx, P.signed_mode), range_of(in.cmn, in.cmx, P.signed_mode), P, inv);
}

// How the reciprocal scales of the in-relation map onto the elements of a row (decided once per layer):
enum InMode { IN_NONE = 0, IN_UNIFORM, IN_KK1, IN_KK9, IN_GENERIC };

// Column-scale four consecutive elements e .. e+3 of a row.  `inv` points at the 1/s of this row's input group
// (shared-memory cache for IN_KK1 / IN_KK9, global memory for IN_GENERIC); `u` is the row-uniform factor (IN_UNIFORM).
template <int MODE>
__device__ __forceinline__ float4 in_scale4(float4 t, int e, const float* __restrict__ inv, float u, int kk) {
  if (MODE == IN_UNIFORM) {
    t.x = __fmul_rn(t.x, u); t.y = __fmul_rn(t.y, u); t.z = __fmul_rn(t.z, u); t.w = __fmul_rn(t.w, u);
  } else if (MODE == IN_KK1) {
    const float4 f = *(const float4*)(inv + e);            // e % 4 == 0 and the cache is 16-byte aligned
    t.x = __fmul_rn(t.x, f.x); t.y = __fmul_rn(t.y, f.y); t.z = __fmul_rn(t.z, f.z); t.w = __fmul_rn(t.w, f.w);
  } else if (MODE == IN_KK9) {
    const int q = e / 9, r = e - 9 * q;                      // four consecutive elements span at most two columns
    const float f0 = inv[q], f1 = inv[q + 1 - (r < 6 ? 1 : 0)];   // second column only when r + 3 >= 9
    t.x = __fmul_rn(t.x, f0);
    t.y = __fmul_rn(t.y, r + 1 >= 9 ? f1 : f0);
    t.z = __fmul_rn(t.z, r + 2 >= 9 ? f1 : f0);
    t.w = __fmul_rn(t.w, r + 3 >= 9 ? f1 : f0);
  } else if (MODE == IN_GENERIC) {
    t.x = __fmul_rn(t.x, __ldcg(inv + (e) / kk));
    t.y = __fmul_rn(t.y, __ldcg(inv + (e + 1) / kk));
    t.z = __fmul_rn(t.z, __ldcg(inv + (e + 2) / kk));
    t.w = __fmul_rn(t.w, __ldcg(inv + (e + 3) / kk));
  }
  return t;
}
template <int MODE>
__device__ __forceinline__ float in_scale1(float t, int e, const float* __restrict__ inv, float u, int kk) {
  if (MODE == IN_UNIFORM) return __fmul_rn(t, u);
  if (MODE == IN_KK1) return __fmul_rn(t, inv[e]);
  if (MODE == IN_KK9) return __fmul_rn(t, inv[e / 9]);
  if (MODE == IN_GENERIC) return __fmul_rn(t, __ldcg(inv + e / kk));
  return t;
}

// float4 slots a thread keeps in registers between the range reduction and the rescale (kThreads * kRowRegs * 4 >= kStageFloats)
constexpr int kRowRegs = (kStageFloats / 4 + kThreads - 1) / kThreads;
// A rescaled row is written back into its stage and the producer warp bulk-stores the tile (TMA).  (Measured alternative:
// straight from the consumers' registers with st.global - stage released right after the range reduction - was 25-40 %
// slower on the stack with every cache policy tried; DESIGN 3.1.)
// General middle layers (row- AND column-scaled, cols > 1) need their column extrema recomputed every sweep: the rescaled
// tile sits in its stage anyway, so the extrema are accumulated right there (no second read of the layer, no extra
// grid-wide phase).
constexpr int kRescanCols = 1024;   // columns a team accumulates in shared memory (more: global atomics)
constexpr size_t kTableCacheBytes = 9 * 1024;   // descriptor tables of a model this small are mirrored in shared memory
constexpr int TK_END = 3;   // sentinel tile: the pass is over for this CTA (the consumers keep no iterator of their own)
static_assert(kThreads * kRowRegs * 4 >= kStageFloats, "a single-row tile must fit the consumers' registers");

// One row resident in shared memory: [range reduction -> s] (HAS_OUT), rescale IN PLACE, accumulate |new - old|.  A row with
// a reduction is read from shared memory ONCE when it fits the registers (always for the CTA-wide single-row tiles).
// `in`: what the row needs from global memory, fetched ahead by the caller; the scale pair comes back in *s_out / *inv_out
// and the caller does (or delegates) the per-channel bookkeeping.
template <int TPR, int MODE, bool HAS_OUT>
__device__ __forceinline__ void cle_row_smem(const RowCtx& c, const DfqCleParams P, float* __restrict__ row, int o, int lane,
                                             const float* __restrict__ s_inv, float* red, int& parity, double& dacc,
                                             const RowIn& in, float* s_out, float* inv_out) {
  const int n = c.row_len, kk = c.kk;
  const bool vec = ((n & 3) == 0);
  auto put4 = [&](int i4, const float4& t) { ((float4*)row)[i4] = t; };
  auto put1 = [&](int e, float t) { row[e] = t; };
  const int n4 = n >> 2;
  const double inv_n = c.inv_n;
  const float* inv = nullptr;
  const float u = in.u;
  if (MODE == IN_KK1 || MODE == IN_KK9) inv = s_inv;
  else if (MODE == IN_GENERIC) inv = c.inv_in + (o / c.in_go) * c.in_gi;
  float s = 1.f;
  auto solve = [&](float mn, float mx) {
    if (TPR == 32) { mn = warp_min(mn); mx = warp_max(mx); }
    else cta_minmax(mn, mx, red, parity);
    float iv;
    s = solve_row(P, in, mn, mx, &iv);
    *s_out = s; *inv_out = iv;
  };
  float dsum = 0.f;
  // a row that only gets its columns scaled (no reduction to wait for) streams through the in-place loop further down:
  // holding it in registers buys nothing there and measured ~12% slower
  if (vec && n4 <= TPR * kRowRegs && HAS_OUT) {
    const float4* r4 = (const float4*)row;
    float4 v[kRowRegs];
#pragma unroll
    for (int k = 0; k < kRowRegs; ++k) {
      const int i4 = lane + k * TPR;
      v[k] = (i4 < n4) ? r4[i4] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (HAS_OUT) {
      float mn = DFQ_INF, mx = -DFQ_INF;
#pragma unroll
      for (int k = 0; k < kRowRegs; ++k) {
        const int i4 = lane + k * TPR;
        if (i4 < n4) {
          const float4 t = in_scale4<MODE>(v[k], i4 * 4, inv, u, kk);
          mn = fminf(mn, fminf(fminf(t.x, t.y), fminf(t.z, t.w)));
          mx = fmaxf(mx, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
        }
      }
      solve(mn, mx);
    }
#pragma unroll
    for (int k = 0; k < kRowRegs; ++k) {
      const int i4 = lane + k * TPR;
      if (i4 < n4) {
        float4 t = in_scale4<MODE>(v[k], i4 * 4, inv, u, kk);
        if (HAS_OUT) { t.x = __fmul_rn(t.x, s); t.y = __fmul_rn(t.y, s); t.z = __fmul_rn(t.z, s); t.w = __fmul_rn(t.w, s); }
        put4(i4, t);
        dsum += fabsf(__fsub_rn(t.x, v[k].x)) + fabsf(__fsub_rn(t.y, v[k].y)) + fabsf(__fsub_rn(t.z, v[k].z)) +
                fabsf(__fsub_rn(t.w, v[k].w));
      }
    }
  } else if (vec) {
    const float4* r4 = (const float4*)row;
    if (HAS_OUT) {
      float mn = DFQ_INF, mx = -DFQ_INF;
#pragma unroll 2
      for (int i4 = lane; i4 < n4; i4 += TPR) {
        const float4 t = in_scale4<MODE>(r4[i4], i4 * 4, inv, u, kk);
        mn = fminf(mn, fminf(fminf(t.x, t.y), fminf(t.z, t.w)));
        mx = fmaxf(mx, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
      }
      solve(mn, mx);
    }
#pragma unroll 2
    for (int i4 = lane; i4 < n4; i4 += TPR) {
      const float4 v = r4[i4];
      float4 t = in_scale4<MODE>(v, i4 * 4, inv, u, kk);
      if (HAS_OUT) { t.x = __fmul_rn(t.x, s); t.y = __fmul_rn(t.y, s); t.z = __fmul_rn(t.z, s); t.w = __fmul_rn(t.w, s); }
      put4(i4, t);
      dsum += fabsf(__fsub_rn(t.x, v.x)) + fabsf(__fsub_rn(t.y, v.y)) + fabsf(__fsub_rn(t.z, v.z)) + fabsf(__fsub_rn(t.w, v.w));
    }
  } else {
    if (HAS_OUT) {
      float mn = DFQ_INF, mx = -DFQ_INF;
      for (int e = lane; e < n; e += TPR) {
        const float t = in_scale1<MODE>(row[e], e, inv, u, kk);
        mn = fminf(mn, t); mx = fmaxf(mx, t);
      }
      solve(mn, mx);
    }
    for (int e = lane; e < n; e += TPR) {
      const float v = row[e];
      float t = in_scale1<MODE>(v, e, inv, u, kk);
      if (HAS_OUT) t = __fmul_rn(t, s);
      put1(e, t);
      dsum += fabsf(__fsub_rn(t, v));
    }
  }
  dacc += (double)dsum * inv_n;
}

// A SHORT row (<= 64 float4 / scalar items) handled by G = 1..16 lanes, 32 / G rows per warp side by side: the depthwise
// 3x3 rows of a MobileNetV2 are 9 floats and its 1x1 expansion rows 24-160 - a whole warp per row left 23-31 lanes idle and
// a warp walked through up to 73 rows of a tile one after the other (the step's critical path).
// Same arithmetic per element and the same (exact) min / max as cle_row_smem; every lane of the warp executes the
// shuffles, lanes of a group without a row (`valid` false) only skip the memory accesses.
#ifndef DFQ_SUB_ITEMS
#define DFQ_SUB_ITEMS 8      // work items a lane takes of a short row (4: twice the rows-in-flight steps, measured slower)
#endif
template <int MODE, bool HAS_OUT>
__device__ __forceinline__ void cle_row_sub(const RowCtx& c, const DfqCleParams P, float* __restrict__ row, int o, int sub, int G,
                                            bool valid, bool vec, const float* __restrict__ s_inv, double& dacc, const RowIn& in,
                                            float* s_out, float* inv_out) {
  const int n = c.row_len, kk = c.kk, n4 = n >> 2;
  const float* inv = nullptr;
  const float u = in.u;
  if (MODE == IN_KK1 || MODE == IN_KK9) inv = s_inv;
  else if (MODE == IN_GENERIC) inv = c.inv_in + (o / c.in_go) * c.in_gi;
  float s = 1.f, dsum = 0.f;
  if (HAS_OUT) {
    float mn = DFQ_INF, mx = -DFQ_INF;
    if (valid) {
      if (vec) {
        const float4* r4 = (const float4*)row;
        for (int i4 = sub; i4 < n4; i4 += G) {
          const float4 t = in_scale4<MODE>(r4[i4], i4 * 4, inv, u, kk);
          mn = fminf(mn, fminf(fminf(t.x, t.y), fminf(t.z, t.w)));
          mx = fmaxf(mx, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
        }
      } else {
        for (int e = sub; e < n; e += G) {
          const float t = in_scale1<MODE>(row[e], e, inv, u, kk);
          mn = fminf(mn, t); mx = fmaxf(mx, t);
        }
      }
    }
    for (int off = G >> 1; off; off >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    float iv;
    s = solve_row(P, in, mn, mx, &iv);
    *s_out = s; *inv_out = iv;
  }
  if (valid) {
    if (vec) {
      float4* r4 = (float4*)row;
      for (int i4 = sub; i4 < n4; i4 += G) {
        const float4 v = r4[i4];
        float4 t = in_scale4<MODE>(v, i4 * 4, inv, u, kk);
        if (HAS_OUT) { t.x = __fmul_rn(t.x, s); t.y = __fmul_rn(t.y, s); t.z = __fmul_rn(t.z, s); t.w = __fmul_rn(t.w, s); }
        r4[i4] = t;
        dsum += fabsf(__fsub_rn(t.x, v.x)) + fabsf(__fsub_rn(t.y, v.y)) + fabsf(__fsub_rn(t.z, v.z)) + fabsf(__fsub_rn(t.w, v.w));
      }
    } else {
      for (int e = sub; e < n; e += G) {
        const float v = row[e];
        float t = in_scale1<MODE>(v, e, inv, u, kk);
        if (HAS_OUT) t = __fmul_rn(t, s);
        row[e] = t;
        dsum += fabsf(__fsub_rn(t, v));
      }
    }
  }
  dacc += (double)dsum * c.inv_n;
}

// A tile of whole rows in shared memory, rescaled in place.
//   one row   : the whole team works on it; its global-memory inputs arrive in the stage mailbox and the bookkeeping is left
//               to the producer warp (mailbox again)
//   many rows : a warp per row, 32 rows per batch -- lane j fetches row j's inputs before the batch and does row j's
//               bookkeeping after it, so a batch pays TWO global-memory latencies instead of two per row
template <int MODE, bool HAS_OUT>
__device__ __forceinline__ void cle_tile_rows(const RowCtx& c, const DfqCleParams& P, float* buf, int row0, int nrows,
                                              const float* s_inv, float* red, int& parity, double& dacc, StagePub* pub) {
  const int warp = ctid() >> 5, lane = ctid() & 31;
  if (nrows == 1) {
    RowIn in;
    if (HAS_OUT && pub) { in.cmn = pub->cmn; in.cmx = pub->cmx; in.u = 1.f; in.s_given = 1.f;
                          if (MODE == IN_UNIFORM) in.u = __ldcg(c.inv_in + (row0 / c.in_go) * c.in_gi);
                          if (P.apply_only) in.s_given = __ldcg(c.s_acc + row0); }
    else in = fetch_row_in(c, P, row0, MODE == IN_UNIFORM);
    float sv = 1.f, iv = 1.f;
    cle_row_smem<kThreads, MODE, HAS_OUT>(c, P, buf, row0, ctid(), s_inv, red, parity, dacc, in, &sv, &iv);
    if (HAS_OUT && ctid() == 0) {
      if (pub) { pub->s = sv; pub->inv = iv; }
      else publish_row(c, P, row0, sv, iv, in.cmn, in.cmx);
    }
  } else {
    const int row_len = c.row_len;
    const int mine = (nrows - warp + kWarps - 1) / kWarps;       // this warp's rows: warp, warp + kWarps, ...
    const bool vec = ((row_len & 3) == 0);
    const int items = vec ? (row_len >> 2) : row_len;            // float4 / scalar work items of one row
    int G = 32;                                                  // lanes per row
    if (items <= 64) { G = 1; while (G * DFQ_SUB_ITEMS < items) G <<= 1; }   // short rows: up to DFQ_SUB_ITEMS items per lane, 32 / G rows at once
    for (int base = 0; base < mine; base += 32) {
      const int il = base + lane;
      const int ol = row0 + warp + il * kWarps;
      RowIn mine_in; mine_in.cmn = mine_in.cmx = 0.f; mine_in.u = 1.f; mine_in.s_given = 1.f;
      RowPub mine_pub; mine_pub.a0 = mine_pub.b0 = mine_pub.w0 = mine_pub.w1 = mine_pub.o0 = mine_pub.o1 = 0.f;
      if (il < mine) {
        mine_in = fetch_row_in(c, P, ol, MODE == IN_UNIFORM);
        if (HAS_OUT) mine_pub = fetch_row_pub(c, P, ol);          // in flight together with the inputs
      }
      float ks = 1.f, kinv = 1.f;
      const int nb = min(32, mine - base);
      if (G < 32) {
        const int R = 32 / G, sub = lane & (G - 1), grp = lane / G;
        for (int j = 0; j < nb; j += R) {
          const bool valid = (j + grp < nb);
          const int jj = valid ? j + grp : nb - 1;                 // lanes without a row shadow the last one (no stores)
          const int r = warp + (base + jj) * kWarps;
          RowIn in;
          in.cmn = __shfl_sync(0xffffffffu, mine_in.cmn, jj); in.cmx = __shfl_sync(0xffffffffu, mine_in.cmx, jj);
          in.u = __shfl_sync(0xffffffffu, mine_in.u, jj); in.s_given = __shfl_sync(0xffffffffu, mine_in.s_given, jj);
          float sv = 1.f, iv = 1.f;
          cle_row_sub<MODE, HAS_OUT>(c, P, buf + (size_t)r * row_len, row0 + r, sub, G, valid, vec, s_inv, dacc, in, &sv, &iv);
          // row j + g was solved by lane group g: its publisher is lane j + g
          const int src = ((lane - j) * G) & 31;
          const float ss = __shfl_sync(0xffffffffu, sv, src), ii = __shfl_sync(0xffffffffu, iv, src);
          if (lane >= j && lane < j + R && lane < nb) { ks = ss; kinv = ii; }
        }
      } else
      for (int j = 0; j < nb; ++j) {
        const int r = warp + (base + j) * kWarps;
        RowIn in;
        in.cmn = __shfl_sync(0xffffffffu, mine_in.cmn, j); in.cmx = __shfl_sync(0xffffffffu, mine_in.cmx, j);
        in.u = __shfl_sync(0xffffffffu, mine_in.u, j); in.s_given = __shfl_sync(0xffffffffu, mine_in.s_given, j);
        float sv = 1.f, iv = 1.f;
        cle_row_smem<32, MODE, HAS_OUT>(c, P, buf + (size_t)r * row_len, row0 + r, lane, s_inv, red, parity, dacc, in, &sv, &iv);
        if (lane == j) { ks = sv; kinv = iv; }
      }
      if (HAS_OUT && il < mine) publish_row_with(c, P, ol, ks, kinv, mine_in.cmn, mine_in.cmx, mine_pub);
    }
  }
}

__device__ __forceinline__ void cle_tile_smem(const RowCtx& c, const DfqCleParams P, int in_mode, float* buf, int row0, int nrows,
                                              const float* s_inv, float* red, int& parity, double& dacc, StagePub* pub) {
#define DFQ_TILE(M)                                                                            \
  if (c.has_out) cle_tile_rows<M, true>(c, P, buf, row0, nrows, s_inv, red, parity, dacc, pub); \
  else cle_tile_rows<M, false>(c, P, buf, row0, nrows, s_inv, red, parity, dacc, pub);
  switch (in_mode) {
    case IN_NONE: cle_tile_rows<IN_NONE, true>(c, P, buf, row0, nrows, s_inv, red, parity, dacc, pub); break;
    case IN_UNIFORM: DFQ_TILE(IN_UNIFORM) break;
    case IN_KK1: DFQ_TILE(IN_KK1) break;
    case IN_KK9: DFQ_TILE(IN_KK9) break;
    default: DFQ_TILE(IN_GENERIC) break;
  }
#undef DFQ_TILE
}

// Any row length / alignment: CTA per row, the row is read twice (second read is an L2 hit).
__device__ __noinline__ void cle_row_generic(const RowCtx& c, const DfqCleParams P, int o,
                                                float* red, int& parity, double& dacc) {
  float* rowp = c.w + (size_t)o * c.row_len;
  const int cbase = c.inv_in ? (o / c.in_go) * c.in_gi : 0;
  float s = 1.f;
  if (c.has_out) {
    float mn = DFQ_INF, mx = -DFQ_INF;
    for (int e = ctid(); e < c.row_len; e += kThreads) {
      float t = ldg_stream1(rowp + e);
      if (c.inv_in) t = __fmul_rn(t, __ldcg(c.inv_in + cbase + col_of(e, c.kk)));
      mn = fminf(mn, t); mx = fmaxf(mx, t);
    }
    cta_minmax(mn, mx, red, parity);
    RowIn in = fetch_row_in(c, P, o, false);
    float iv;
    s = solve_row(P, in, mn, mx, &iv);
    if (ctid() == 0) publish_row(c, P, o, s, iv, in.cmn, in.cmx);
  }
  float dsum = 0.f;
  for (int e = ctid(); e < c.row_len; e += kThreads) {
    const float u = ldg_stream1(rowp + e);
    float t = u;
    if (c.inv_in) t = __fmul_rn(t, __ldcg(c.inv_in + cbase + col_of(e, c.kk)));
    if (c.has_out) t = __fmul_rn(t, s);
    stg_stream1(rowp + e, t);
    dsum += fabsf(__fsub_rn(t, u));
  }
  dacc += (double)dsum * c.inv_n;
}

__device__ __forceinline__ void make_ctx(RowCtx& c, float* arena, const DfqLayer* L, const DfqRelation* R,
                                         int li, int sweep) {
  const DfqLayer l = L[li];
  c.w = arena + l.w_off;
  c.rows = l.rows; c.cols = l.cols; c.kk = l.kk; c.row_len = l.cols * l.kk;
  c.inv_n = 1.0 / ((double)l.rows * (double)c.row_len);
  c.first_sweep = (sweep == 0);
  const int rd = sweep & 1, wr = rd ^ 1;
  c.inv_in = nullptr; c.in_gi = 1; c.in_go = 1; c.inv_cached = 0;
  c.own_cmin_wr = c.own_cmax_wr = nullptr;
  if (l.rel_in >= 0) {
    const DfqRelation r = R[l.rel_in];
    c.inv_in = arena + r.inv_off;
    c.in_gi = r.gi; c.in_go = r.go;
    c.inv_cached = (r.groups == 1 && l.cols <= kInvCache) ? 1 : 0;
    if (l.col_mode == 1 && l.rel_out >= 0) {
      c.own_cmin_wr = arena + l.cmin_off + (size_t)wr * r.channels;
      c.own_cmax_wr = arena + l.cmax_off + (size_t)wr * r.channels;
    }
  }
  c.has_out = (l.rel_out >= 0);
  c.cmin_rd = c.cmax_rd = nullptr; c.cmin_wr = c.cmax_wr = nullptr;
  c.s_step = c.inv_out = c.s_acc = c.bnw = c.bnb = nullptr;
  c.bias = arena + l.bias_off;
  if (c.has_out) {
    const DfqRelation r = R[l.rel_out];
    const DfqLayer l2 = L[r.second];
    c.cmin_rd = arena + l2.cmin_off + (size_t)rd * r.channels;
    c.cmax_rd = arena + l2.cmax_off + (size_t)rd * r.channels;
    if (l2.col_mode != 2) {
      c.cmin_wr = arena + l2.cmin_off + (size_t)wr * r.channels;
      c.cmax_wr = arena + l2.cmax_off + (size_t)wr * r.channels;
    }
    c.s_step = arena + r.s_step_off;
    c.inv_out = arena + r.inv_off;
    c.s_acc = arena + r.s_acc_off;
    c.bnw = r.bn_w_off >= 0 ? arena + r.bn_w_off : nullptr;
    c.bnb = r.bn_b_off >= 0 ? arena + r.bn_b_off : nullptr;
  }
}

__device__ __forceinline__ void reset_cols(float* arena, const DfqLayer& l, const DfqRelation& r, int buf) {
  float* a = arena + l.cmin_off + (size_t)buf * r.channels;
  float* b = arena + l.cmax_off + (size_t)buf * r.channels;
  for (int j = ctid(); j < r.channels; j += kThreads) { __stcg(a + j, DFQ_INF); __stcg(b + j, -DFQ_INF); }
}

// Walks the pass tiles of this CTA's span in one step, skipping the layers of converged groups.  The producer thread
// keeps a second copy kCleStages-1 tiles ahead; both copies see the same `done` flags (they only change at sweep end).
struct PassIter {
  const long long* ptr; const int* step_layers; const DfqLayer* L; const GroupState* G;
  int q, q_end;
  long long q_lo, q_hi;   // tile range of task q, cached: the per-tile advance touches no global memory
  TileCursor cur;
  int q_live;   // last task whose group was checked and found still iterating (one uncached read per layer, not per tile)
  int g_seen, g_done;   // ... and per run of layers of the same group, not per layer
  // shape of the layer in hand, fetched once per layer: fill() runs in the single producer lane for EVERY tile, and a 64-byte
  // descriptor load from global memory there (an L2 latency) was what k_cle_stack waited for
  int f_q; int f_li, f_rows, f_row_len; long long f_w_off;
  __device__ __forceinline__ void settle() {
    while (cur.valid()) {
      if (cur.t >= q_hi) {
        do { ++q; } while (q + 1 < q_end && ptr[q + 1] <= cur.t);
        q_lo = ptr[q]; q_hi = ptr[q + 1];
      }
      if (G != nullptr && q != q_live) {       // (G == nullptr: a single group - it is iterating as long as the kernel runs)
        const int g = L[step_layers[q]].group;
        if (g != g_seen) { g_done = *((volatile const int*)&G[g].done); g_seen = g; }   // flags only change between sweeps
        if (g_done) { cur.seek(q_hi); continue; }
        q_live = q;
      }
      break;
    }
  }
  __device__ __forceinline__ void start(const long long* p, const int* sl, const DfqLayer* L_, const GroupState* G_, int qb, int qe) {
    ptr = p; step_layers = sl; L = L_; G = G_; q_end = qe; q_live = -1; g_seen = -1; g_done = 0; f_q = -1;
    cur.init(p[qb], p[qe]);
    q = cur.valid() ? find_task(p, qb, qe, cur.t) : qb;
    q_lo = p[q]; q_hi = (q < qe) ? p[q + 1] : p[q];
    settle();
  }
  __device__ __forceinline__ bool valid() const { return cur.valid(); }
  __device__ __forceinline__ void next() { cur.next(); settle(); }
  __device__ __forceinline__ void fill(TileDesc& d, float* arena) {
    if (q != f_q) {
      f_q = q; f_li = step_layers[q];
      const DfqLayer l = L[f_li];
      f_rows = l.rows; f_row_len = l.cols * l.kk; f_w_off = l.w_off;
    }
    const int li = f_li, row_len = f_row_len;
    const int rpt = pipe_rows_per_tile(row_len);
    d.task = li;
    d.row0 = (int)(cur.t - q_lo) * rpt;
    d.nrows = min(rpt, f_rows - d.row0);
    d.floats = d.nrows * row_len;
    d.gptr = arena + f_w_off + (size_t)d.row0 * row_len;
    if (row_len > kStageFloats) d.kind = TK_DIRECT;
    else d.kind = (((((uintptr_t)d.gptr) & 15) == 0) && ((d.floats & 3) == 0)) ? TK_BULK : TK_PLAIN;
  }
};

// ------------------------------------------------------------------------------------------------------------
// Warp-specialised pass.  Shared-memory ring of kCleStages tiles per CTA:
//   producer warp (lane 0):  for every tile  [expect_tx + cp.async.bulk load] -> prefetch the channel's column extrema into the
//                            stage mailbox -> arrive(full);  when the consumers hand a tile back (done):  per-channel bookkeeping
//                            (S, 1/s, bias, BN vectors, derived column extrema) -> cp.async.bulk store -> stage free
//   consumer warps (7):      wait(full) -> range reduction -> s -> rescale in place -> fence.proxy.async -> arrive(done)
// The consumers never wait for global-memory latency of the small vectors nor for the TMA bookkeeping, and the producer is
// off their critical path: ONE consumer barrier per tile (the block reduction).
// ------------------------------------------------------------------------------------------------------------
struct WsPipe {
  unsigned char* base;   // everything is derived from it: no pointer arrays (a runtime-indexed array would live in local memory)
  __device__ __forceinline__ float* stage(int i) const { return (float*)(base + (size_t)i * kStageBytes); }
  __device__ __forceinline__ uint64_t* full(int i) const { return (uint64_t*)(base + (size_t)kCleStages * kStageBytes) + i; }
  __device__ __forceinline__ uint64_t* done(int i) const { return (uint64_t*)(base + (size_t)kCleStages * kStageBytes + 128) + i; }
  __device__ __forceinline__ TileDesc* desc(int i) const { return (TileDesc*)(base + (size_t)kCleStages * kStageBytes + 256) + i; }
  __device__ __forceinline__ StagePub* pub(int i) const {
    return (StagePub*)(base + (size_t)kCleStages * kStageBytes + 256 + kCleStages * sizeof(TileDesc)) + i;
  }
  __device__ void init(unsigned char* smem) {
    base = smem;
    if (threadIdx.x == 0) {
      for (int i = 0; i < kCleStages; ++i) { mbar_init(full(i), 1); mbar_init(done(i), kThreads); }
      mbar_fence_init();
    }
    __syncthreads();
  }
  __host__ __device__ static constexpr size_t smem_bytes() {
    return (size_t)kCleStages * kStageBytes + 256 + kCleStages * (sizeof(TileDesc) + sizeof(StagePub)) + 64;
  }
};
static_assert(kCleStages <= 16, "barrier arrays are 128 bytes");

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// Producer WARP: issue / retire the tiles of one step.  `count` = tiles this CTA has moved since kernel start.
// One iteration retires tile m (the consumers no longer need its stage) and issues tile m + kCleStages into that stage;
// the lanes work side by side so an iteration costs ONE global-memory latency instead of their sum:
//   lane 0  bulk load of the new tile
//   lane 1  per-channel bookkeeping of tile m (publish_row: S, 1/s, bias, BN vectors, derived column extrema)
//   lane 2  prefetch of the new tile's column extrema into its mailbox
// `scan`: the initial column scan -- tiles are only loaded, no mailbox traffic.
// End of a step for the producer warp: its bulk stores have reached global memory, its bookkeeping stores are fenced.
__device__ __forceinline__ void ws_drain() {
  if ((threadIdx.x & 31) == 0) {
    bulk_wait_all();
    fence_proxy_async_all();
  }
  __threadfence();                  // lane 1's bookkeeping stores, before the grid barrier
  __syncwarp();
}

// `ahead`: tiles of this step that ws_issue_ahead() already put into the ring (pit stands behind them).  `drain` = false:
// the caller issues the next step's first loads while this step's stores are still on their way, then calls ws_drain().
__device__ __noinline__ void ws_produce(float* arena, const DfqLayer* L, const DfqRelation* R, PassIter pit, WsPipe& ws,
                           unsigned long long& count, const DfqCleParams P, int sweep, CleCtl* ctl, bool tr, bool scan,
                           int ahead = 0, bool drain = true) {
  const int lane = threadIdx.x & 31;
  const unsigned long long count0 = count;
  unsigned long long n = count + (unsigned long long)ahead, m = count;     // next tile to issue / to retire (uniform across the warp)
  RowCtx ctx;                                  // lane 1: layer being retired; lane 2: layer being issued
  int li = -1;
  int end_pending = kTeams;                    // the TK_END sentinels go last, one per consumer team
  if (lane == 0) fence_proxy_async_all();      // rows written with plain stores before the last grid barrier -> bulk loads
  for (;;) {
    const bool more = pit.valid() || end_pending > 0;
    const bool room = (n - m) < (unsigned long long)kCleStages;
    if (!(more && room) && m == n) break;
    const bool do_retire = !room || !more;
    if (do_retire) {
      const int sr = (int)(m % kCleStages);
      mbar_wait(ws.done(sr), (uint32_t)((m / kCleStages) & 1));          // the consumers are done with tile m's stage
#ifdef DFQ_TILE_TRACE
      if (tr && lane == 0 && m - count0 < 48) ctl->tile_ns[m - count0][4] = gtimer();
#endif
      if (!scan) {
        const TileDesc d = *ws.desc(sr);
        const StagePub pb = *ws.pub(sr);
        __syncwarp();                                                        // everyone holds a copy before the stage is recycled
        if (lane == 0 && d.kind == TK_BULK) {
          bulk_s2g(d.gptr, ws.stage(sr), (uint32_t)d.floats * 4u);
          bulk_commit();
          bulk_wait_read<0>();                                               // the stage may be overwritten now
        }
        if (lane == 1 && pb.valid) {
          if (d.task != li) { make_ctx(ctx, arena, L, R, d.task, sweep); li = d.task; }
          publish_row(ctx, P, d.row0, pb.s, pb.inv, pb.cmn, pb.cmx);
        }
      }
      m++;
    }
    if (more && (n - m) < (unsigned long long)kCleStages) {
      TileDesc d;
      if (pit.valid()) { pit.fill(d, arena); pit.next(); }
      else { d.gptr = nullptr; d.task = -1; d.row0 = d.floats = 0; d.kind = TK_END; d.nrows = --end_pending; }
      const int si = (int)(n % kCleStages);
      if (lane == 0) {
        *ws.desc(si) = d;
        if (d.kind == TK_BULK) {
          mbar_expect_tx(ws.full(si), (uint32_t)d.floats * 4u);
          bulk_g2s(ws.stage(si), d.gptr, (uint32_t)d.floats * 4u, ws.full(si));
        }
#ifdef DFQ_TILE_TRACE
        if (tr && n - count0 < 48) ctl->tile_ns[n - count0][6] = gtimer();
#endif
      }
      if (lane == 2) {
        StagePub pb; pb.valid = 0; pb.cmn = pb.cmx = pb.s = pb.inv = 0.f;
        if (!scan && d.nrows == 1 && (d.kind == TK_BULK || d.kind == TK_PLAIN)) {
          if (d.task != li) { make_ctx(ctx, arena, L, R, d.task, sweep); li = d.task; }
          if (ctx.has_out) { pb.cmn = __ldcg(ctx.cmin_rd + d.row0); pb.cmx = __ldcg(ctx.cmax_rd + d.row0); pb.valid = 1; }
        }
        *ws.pub(si) = pb;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(ws.full(si));   // phase completes when this arrival AND the bulk bytes have landed
      n++;
    }
    __syncwarp();
  }
  count = n;
  if (drain) ws_drain();
}

// Before the grid barrier that ends a step: start loading the first tiles of the NEXT step (the ring is empty at that
// point).  A layer's weights are only ever written in its own step, by the CTA that owns the tile (the tile -> CTA map is
// static), so these loads need nothing from the barrier; what does depend on it - 1/s of the in-relation, the column
// extrema - is read by the consumers behind it.  The mailbox of such a tile stays invalid: the consumers fetch and publish
// the row themselves.  On a MobileNetV2 the first tile used to arrive a large part of a step after the barrier (iterator
// start + L2 -> shared memory).  Returns the number of tiles issued (sequence numbers count .. count + a - 1).
__device__ __noinline__ int ws_issue_ahead(float* arena, PassIter& pit, WsPipe& ws, unsigned long long count) {
  const int lane = threadIdx.x & 31;
  int a = 0;
  for (; a < kCleStages && pit.valid(); ++a) {
    TileDesc d;
    pit.fill(d, arena);
    pit.next();
    const int si = (int)((count + (unsigned long long)a) % kCleStages);
    if (lane == 0) {
      *ws.desc(si) = d;
      if (d.kind == TK_BULK) {
        mbar_expect_tx(ws.full(si), (uint32_t)d.floats * 4u);
        bulk_g2s(ws.stage(si), d.gptr, (uint32_t)d.floats * 4u, ws.full(si));
      }
    }
    if (lane == 2) {
      StagePub pb; pb.valid = 0; pb.cmn = pb.cmx = pb.s = pb.inv = 0.f;
      *ws.pub(si) = pb;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(ws.full(si));
  }
  __syncwarp();
  return a;
}

__global__ void __launch_bounds__(kCtaThreads, kCleCtas)
k_cle_engine(float* arena, const DfqLayer* __restrict__ gL, int nL, const DfqRelation* __restrict__ gR, int nR,
             const int* __restrict__ g_step_ptr, const int* __restrict__ g_step_layers, int n_steps,
             const long long* __restrict__ g_pass_ptr,
             const long long* __restrict__ g_scan_ptr, const int* __restrict__ g_scan_layers, int n_scan,
             DfqCleParams P, CleCtl* ctl, GroupState* G, int nG, int rs_cols, const unsigned char* tbl, int tbl_bytes) {
  cg::grid_group grid = cg::this_grid();
  // per-team scratch
  __shared__ float red_all[kTeams][2 * 2 * 8];
  __shared__ double dred_all[kTeams][8];
  __shared__ RowCtx sctx_all[kTeams];
  __shared__ __align__(16) float s_inv_all[kTeams][kInvCache + 4];   // 1/s of the current layer's input columns
  struct RescanCtx { float *dmin, *dmax; int nch, go, gi; bool smem, own, single; };
  __shared__ RescanCtx rsx_all[kTeams];
  __shared__ double s_rule_diff;          // single-group exit rule, replicated per CTA: `diff`, `count` of dfq.py:81-82
  __shared__ int s_rule_count, s_rule_stop;
  if (threadIdx.x == 0) { s_rule_diff = 10.0; s_rule_count = 0; s_rule_stop = 0; }
  const int tm = threadIdx.x < kTeams * kThreads ? team() : 0;
  RescanCtx& rsx = rsx_all[tm];
  float* red = red_all[tm];
  double* dred = dred_all[tm];
  RowCtx& sctx = sctx_all[tm];
  float* s_inv = s_inv_all[tm];
  extern __shared__ __align__(128) unsigned char pipe_smem[];
  // scratch of the fused re-scan: rs_cols columns per team behind the ring, only when the problem has re-scanned layers
  // (the host sizes the dynamic shared memory; without them the CTA stays at 64 KB and the SM keeps a 60 KB L1)
  float* rs_min = (float*)(pipe_smem + ((WsPipe::smem_bytes() + 15) & ~(size_t)15)) + (size_t)tm * 2 * rs_cols;
  float* rs_max = rs_min + rs_cols;
  // the column-scan scratch aliases the reciprocal-scale cache: scans and passes never overlap
  float* smin = s_inv;
  float* smax = s_inv + kScanCols;
  static_assert(2 * kScanCols <= kInvCache + 4, "scan scratch must fit the reciprocal-scale cache");
  WsPipe ws;
  ws.init(pipe_smem);
  // A small model is latency-bound: every phase walks the descriptor tables with dependent loads.  When the whole table pack
  // fits (the host decides: tbl_bytes > 0) it is mirrored in shared memory behind the ring.  The table pointers below are pure
  // functions of kernel arguments (cheap to rematerialise, nothing held in registers across the tile loop), and derived from
  // the shared-memory base, not from the arguments: kernel pointer arguments are assumed to point to global memory.
  unsigned char* tcache = pipe_smem + ((WsPipe::smem_bytes() + 15) & ~(size_t)15) + (size_t)kTeams * 2 * rs_cols * sizeof(float);
  if (tbl_bytes > 0) {
    for (int i = threadIdx.x * 16; i < tbl_bytes; i += kCtaThreads * 16) *(int4*)(tcache + i) = *(const int4*)(tbl + i);
    __syncthreads();
  }
#define DFQ_TAB(T, g) (tbl_bytes > 0 ? (const T*)(tcache + ((const unsigned char*)(g) - tbl)) : (const T*)(g))
  const DfqLayer* L = DFQ_TAB(DfqLayer, gL);
  const DfqRelation* R = DFQ_TAB(DfqRelation, gR);
  const int* step_ptr = DFQ_TAB(int, g_step_ptr);
  const int* step_layers = DFQ_TAB(int, g_step_layers);
  const long long* pass_ptr = DFQ_TAB(long long, g_pass_ptr);
  const long long* scan_ptr = DFQ_TAB(long long, g_scan_ptr);
  const int* scan_layers = DFQ_TAB(int, g_scan_layers);
#undef DFQ_TAB
  const bool producer = threadIdx.x >= kTeams * kThreads;
  int parity = 0;
  const int warp = ctid() >> 5, lane = ctid() & 31;
  unsigned long long count = 0;     // tiles moved through the ring so far (advances identically in both roles)
  // first tile index >= c that belongs to this thread's team
  auto my_first = [&](unsigned long long c) { return c + (unsigned long long)((tm + kTeams - (int)(c % kTeams)) % kTeams); };

  int tmark = 0;
  auto mark = [&]() { if (blockIdx.x == 0 && threadIdx.x == 0 && tmark < 32) ctl->t_ns[tmark] = gtimer(); tmark++; };
  mark();
  // ---- phase 0: column extrema of every `second` layer (buffer 0) -----------------------------
  if (!producer) {
    for (int g = vblock() * kThreads + ctid(); g < nG; g += vgrid() * kThreads) G[g].diff = 10.0;   // dfq.py:81
    for (int j = ctid(); j < rs_cols; j += kThreads) { rs_min[j] = DFQ_INF; rs_max[j] = -DFQ_INF; }
    for (int li = vblock(); li < nL; li += vgrid())
      if (L[li].rel_in >= 0 && !(L[li].flags & DFQ_LAYER_COLS_READY)) reset_cols(arena, L[li], R[L[li].rel_in], 0);
  }
  grid.sync();
  {  // scan_ptr[0 .. n_scan]: pass-tile prefix over scan_layers (all `second` layers); the tiles stream through the ring
    if (producer) {
      PassIter it;
      it.start(scan_ptr, scan_layers, L, G, 0, n_scan);
      ws_produce(arena, L, R, it, ws, count, P, 0, ctl, false, true);
    } else {
      int cur_li = -1, nch = 0, J = 0, kk = 0, go = 1, gi = 1;
      bool use_smem = false, own = false, single = true;
      float *dmin = nullptr, *dmax = nullptr;
      // fold the CTA's partial extrema of the current layer into the global arrays; leave the scratch reset
      auto flush = [&]() {
        if (cur_li < 0 || !use_smem) return;
        cbar();
        colscan_flush<kThreads>(ctid(), nch, smin, smax, dmin, dmax);
        cbar();
      };
      for (int j = ctid(); j < kScanCols; j += kThreads) { smin[j] = DFQ_INF; smax[j] = -DFQ_INF; }
      cbar();
      for (count = my_first(count);; count += kTeams) {
        const int sidx = (int)(count % kCleStages);
        mbar_wait(ws.full(sidx), (uint32_t)((count / kCleStages) & 1));
        const TileDesc d = *ws.desc(sidx);
        if (d.kind == TK_END) { mbar_arrive(ws.done(sidx)); count += 1 + d.nrows; break; }   // nrows: sentinels still to come
        float* buf = ws.stage(sidx);
        if (d.kind == TK_PLAIN) {
          for (int i = ctid(); i < d.floats; i += kThreads) buf[i] = ldg_stream1(d.gptr + i);
          fence_proxy_async_smem();
          cbar();
        }
        if (d.task != cur_li) {
          flush();
          cur_li = d.task;
          const DfqLayer l = L[cur_li];
          const DfqRelation r = R[l.rel_in];
          nch = r.channels; J = l.cols; kk = l.kk; go = r.go; gi = r.gi;
          single = (r.groups == 1);
          use_smem = (nch <= kScanCols);
          own = (pipe_rows_per_tile(J * kk) == 1);
          dmin = arena + l.cmin_off; dmax = arena + l.cmax_off;    // buffer 0
        }
        if (d.kind == TK_DIRECT) {   // a row longer than a stage: straight from global memory
          colscan_tile_ool<true>(d.gptr, ctid(), d.row0, d.nrows, J, kk, go, gi, single, own, use_smem, smin, smax, dmin, dmax);
        } else {
          colscan_tile_ool<false>(buf, ctid(), d.row0, d.nrows, J, kk, go, gi, single, own, use_smem, smin, smax, dmin, dmax);
        }
        mbar_arrive(ws.done(sidx));
      }
      flush();
    }
  }
  grid.sync();
  mark();

  // single model (one convergence group): the producer warp runs one step ahead with its loads (ws_issue_ahead)
  const bool run_ahead = (nG == 1);
  PassIter it_ahead;
  int ahead = -1;                    // < 0: the iterator of the coming step has not been started
  for (int sweep = 0;; ++sweep) {
    const int slot = sweep % 3;
    for (int p = 0; p < n_steps; ++p) {
      if (producer) {
        if (ahead < 0) {
          it_ahead.start(pass_ptr, step_layers, L, nG == 1 ? nullptr : G, step_ptr[p], step_ptr[p + 1]);
          ahead = 0;
        }
        ws_produce(arena, L, R, it_ahead, ws, count, P, sweep, ctl, blockIdx.x == 0 && sweep == 0 && p == 0, false, ahead,
                   !run_ahead);
        ahead = -1;
        if (run_ahead) {
          const int pn = (p + 1 < n_steps) ? p + 1 : 0;      // (a sweep that turns out to be the last one: drained at exit)
          it_ahead.start(pass_ptr, step_layers, L, nullptr, step_ptr[pn], step_ptr[pn + 1]);
          ahead = ws_issue_ahead(arena, it_ahead, ws, count);
          ws_drain();
        }
      } else {
        double dacc = 0.0;
        int cur_g = -1;
        // sum the CTA's partial of group cur_g into that group's accumulator (one atomic)
        auto flush = [&]() {
          if (cur_g < 0) return;
          dacc = warp_sum(dacc);
          cbar();
          if (lane == 0) dred[warp] = dacc;
          cbar();
          if (ctid() == 0) {
            double t = 0.0;
#pragma unroll
            for (int i = 0; i < kWarps; ++i) t += dred[i];
            if (t != 0.0) atomicAdd(&G[cur_g].acc[slot], t);
          }
          dacc = 0.0;
        };
        int cur_li = -1, in_mode = IN_NONE;
        // fused re-scan of the layer in hand (col_mode 2): partial column extrema of its NEW rows, flushed when the layer changes
        // (its geometry lives in shared memory, written by the team leader at the layer change: the tile loop is short of registers)
        int rs_li = -1;
        auto rs_flush = [&]() {
          if (rs_li < 0) return;
          if (rsx.smem) {
            cbar();
            colscan_flush<kThreads>(ctid(), rsx.nch, rs_min, rs_max, rsx.dmin, rsx.dmax);
            cbar();
          }
          rs_li = -1;
        };
#ifdef DFQ_TILE_TRACE
        const bool tr = (blockIdx.x == 0 && threadIdx.x == 0 && sweep == 0 && p == 0);
        int trn = 0;
#define DFQ_TT(i) do { if (tr && trn < 48) ctl->tile_ns[trn][i] = gtimer(); } while (0)
#else
#define DFQ_TT(i) do { } while (0)
#endif
#ifdef DFQ_STEP_TRACE
        const bool st_tr = (sweep == 2 && threadIdx.x == 0 && p < 8 && blockIdx.x < 512);
        int st_n = 0;
#define DFQ_ST(i) do { if (st_tr && st_n == 0) g_step_trace[p][blockIdx.x][i] = gtimer(); } while (0)
        if (st_tr) { g_step_trace[p][blockIdx.x][0] = gtimer(); for (int i = 1; i < 8; ++i) g_step_trace[p][blockIdx.x][i] = 0; }
#else
#define DFQ_ST(i) do { } while (0)
#endif
        for (count = my_first(count);; count += kTeams) {
          const int sidx = (int)(count % kCleStages);
          DFQ_TT(0);
          mbar_wait(ws.full(sidx), (uint32_t)((count / kCleStages) & 1));
          DFQ_TT(1);
          DFQ_ST(1);
          // the descriptor stays in shared memory (valid until `done` is arrived): the loop is short of registers
          const volatile TileDesc& d = *ws.desc(sidx);
          // (the descriptor is read BEFORE the arrival: the producer may refill this stage for the next step right away)
          if (d.kind == TK_END) { const int rest = d.nrows; mbar_arrive(ws.done(sidx)); count += 1 + (unsigned)rest; break; }
          float* buf = ws.stage(sidx);
          if (d.kind == TK_PLAIN) {            // a tile the TMA unit cannot move: cooperative fetch
            for (int i = ctid(); i < d.floats; i += kThreads) buf[i] = ldg_stream1(d.gptr + i);
            fence_proxy_async_smem();          // the stage's next refill may be a bulk load (async proxy)
            cbar();
          }
          if (d.task != cur_li) {
            cur_li = d.task;
            const int g = L[cur_li].group;
            if (g != cur_g) { flush(); cur_g = g; }
            cbar();                              // everyone is done with the previous layer's context
            if (ctid() == 0) make_ctx(sctx, arena, L, R, cur_li, sweep);
            cbar();
            if (sctx.inv_in == nullptr) in_mode = IN_NONE;
            else if (sctx.cols == 1) in_mode = IN_UNIFORM;
            else if (sctx.inv_cached && sctx.kk == 1) in_mode = IN_KK1;
            else if (sctx.inv_cached && sctx.kk == 9) in_mode = IN_KK9;
            else in_mode = IN_GENERIC;
            if (in_mode == IN_KK1 || in_mode == IN_KK9) {
              // four loads in flight per thread: one L2 latency per 4 x kThreads columns instead of one per kThreads
              const int ncol = sctx.cols;
              const float* src = sctx.inv_in;
              for (int j0 = ctid(); j0 < ncol; j0 += 4 * kThreads) {
                float t[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) t[k] = (j0 + k * kThreads < ncol) ? __ldcg(src + j0 + k * kThreads) : 0.f;
#pragma unroll
                for (int k = 0; k < 4; ++k) if (j0 + k * kThreads < ncol) s_inv[j0 + k * kThreads] = t[k];
              }
              if (ctid() == 0) s_inv[ncol] = 1.f;
              cbar();
            }
            rs_flush();
            const DfqLayer l = L[cur_li];
            if (l.col_mode == 2 && l.rel_in >= 0) {       // accumulate into the NEXT sweep's buffer, reset one step ago
              rs_li = cur_li;
              if (ctid() == 0) {
                const DfqRelation r = R[l.rel_in];
                rsx.nch = r.channels; rsx.go = r.go; rsx.gi = r.gi;
                rsx.single = (r.groups == 1); rsx.smem = (r.channels <= rs_cols);
                rsx.own = (pipe_rows_per_tile(l.cols * l.kk) == 1);
                rsx.dmin = arena + l.cmin_off + (size_t)((sweep & 1) ^ 1) * r.channels;
                rsx.dmax = arena + l.cmax_off + (size_t)((sweep & 1) ^ 1) * r.channels;
              }
              cbar();
            }
          }
          DFQ_ST(2);
          // the re-scanned successor's next-sweep buffer is reset HERE, one step (= one grid barrier) before its pass fills it
          if (d.row0 == 0 && sctx.has_out) {
            const DfqRelation ro = R[L[cur_li].rel_out];
            if (L[ro.second].col_mode == 2) reset_cols(arena, L[ro.second], ro, (sweep & 1) ^ 1);
          }
          const RowCtx& c = sctx;
          if (d.kind == TK_DIRECT) {
            for (int r = 0; r < d.nrows; ++r) cle_row_generic(c, P, d.row0 + r, red, parity, dacc);
            if (rs_li >= 0) {
              cbar();     // the rows are final in global memory (st.cg); read them back with ld.cg
              colscan_tile_ool<true>(d.gptr, ctid(), d.row0, d.nrows, c.cols, c.kk, rsx.go, rsx.gi, rsx.single, rsx.own, rsx.smem,
                                           rs_min, rs_max, rsx.dmin, rsx.dmax);
            }
            mbar_arrive(ws.done(sidx));
          } else {
            StagePub* pub = ws.pub(sidx);
            cle_tile_smem(c, P, in_mode, buf, d.row0, d.nrows, s_inv, red, parity, dacc, pub->valid ? pub : nullptr);
            DFQ_ST(3);
            if (rs_li >= 0 || d.kind != TK_BULK) cbar();      // every row of the tile is final in the stage
            DFQ_ST(7);
            if (rs_li >= 0)
              colscan_tile_ool<false>(buf, ctid(), d.row0, d.nrows, c.cols, c.kk, rsx.go, rsx.gi, rsx.single, rsx.own, rsx.smem,
                                            rs_min, rs_max, rsx.dmin, rsx.dmax);
            if (d.kind == TK_BULK) fence_proxy_async_smem();   // my generic-proxy writes -> visible to the bulk store
            else for (int i = ctid(); i < d.floats; i += kThreads) stg_stream1(d.gptr + i, buf[i]);
            mbar_arrive(ws.done(sidx));         // hand the tile back to the producer
          }
          DFQ_TT(2);
          DFQ_ST(4);
#ifdef DFQ_STEP_TRACE
          st_n++;
#endif
#ifdef DFQ_TILE_TRACE
          trn++;
#endif
        }
#undef DFQ_TT
#ifdef DFQ_STEP_TRACE
        if (st_tr) g_step_trace[p][blockIdx.x][5] = gtimer();
#endif
        rs_flush();
        flush();
        fence_proxy_async_all();   // this pass's plain row stores -> the next pass's bulk loads (async proxy)
        __threadfence();
#ifdef DFQ_STEP_TRACE
        if (st_tr) g_step_trace[p][blockIdx.x][6] = gtimer();
#endif
#undef DFQ_ST
      }
      grid.sync();
      mark();
    }
    // ---- exit rule of dfq.py:105-115 -------------------------------------------------------------------------
    const int n = sweep + 1;
    if (nG == 1) {
      // ONE convergence group (a single model - the latency-bound case): every CTA evaluates the rule itself from the group's
      // accumulator, complete since the last step's barrier - same inputs, same decision - instead of one thread deciding and
      // a second grid barrier broadcasting it.  CTA 0 keeps the global record; the accumulator of sweep+2 is cleared here:
      // its last readers (the rule of sweep-1) passed this sweep's barriers, its next writers wait behind the next ones.
      if (threadIdx.x == 0) {
        const double diff_tmp = *((volatile double*)&G[0].acc[slot]);
        if (fabs(s_rule_diff - diff_tmp) > 1e-9) { s_rule_count = 0; s_rule_diff = diff_tmp; }
        else s_rule_count++;
        const bool cont = (s_rule_diff > P.converge_thres) && (s_rule_count < P.converge_count);
        const int cap = P.max_sweeps > 0 ? P.max_sweeps : 4096;
        const bool stop = !cont || n >= cap;
        if (blockIdx.x == 0) {
          GroupState& st = G[0];
          st.acc[(slot + 2) % 3] = 0.0;
          st.diff = s_rule_diff; st.count = s_rule_count;
          if (sweep < 64) ctl->diffs[sweep] = diff_tmp;
          if (stop) { st.n_sweeps = n; st.converged = !cont; st.done = 1; }
        }
        s_rule_stop = stop ? 1 : 0;
      }
      __syncthreads();
      if (s_rule_stop) break;
      __syncthreads();          // s_rule_stop is rewritten one sweep from now
      continue;
    }
    if (!producer) {
      for (int g = vblock() * kThreads + ctid(); g < nG; g += vgrid() * kThreads) {
        GroupState& st = G[g];
        if (st.done) continue;
        const double diff_tmp = st.acc[slot];
        st.acc[(slot + 2) % 3] = 0.0;   // last read before this sweep's final barrier, next used in sweep+2
        if (fabs(st.diff - diff_tmp) > 1e-9) { st.count = 0; st.diff = diff_tmp; }
        else st.count++;
        if (g == 0 && sweep < 64) ctl->diffs[sweep] = diff_tmp;
        const bool cont = (st.diff > P.converge_thres) && (st.count < P.converge_count);
        // safety net: the reference's loop has no bound; 4096 sweeps is ~80x what any of its models needs
        const int cap = P.max_sweeps > 0 ? P.max_sweeps : 4096;
        if (!cont || n >= cap) { st.n_sweeps = n; st.converged = !cont; st.done = 1; }
        else atomicAdd(&ctl->active[n & 1], 1);
      }
      if (blockIdx.x == 0 && threadIdx.x == 0) ctl->active[sweep & 1] = 0;   // read at the end of the previous sweep
    }
    __threadfence();
    grid.sync();
    if (*((volatile int*)&ctl->active[n & 1]) == 0) break;
  }
  // loads issued ahead for a step that never comes must have landed before the CTA's shared memory goes away
  if (producer && ahead > 0 && (threadIdx.x & 31) == 0)
    for (int a = 0; a < ahead; ++a) {
      const unsigned long long c = count + (unsigned long long)a;
      mbar_wait(ws.full((int)(c % kCleStages)), (uint32_t)((c / kCleStages) & 1));
    }
}


// ------------------------------------------------------------------------------------------------------------
// k_cle_stack: the equalization of a STACK OF TWO-LAYER CHAINS (BASELINE configs[4]; ResNet basic blocks), streaming
// variant of k_cle_engine built on the warp-autonomous ring of bc_stream.cuh.
//
// k_cle_engine keeps one tile per consumer TEAM: every first-layer row pays a CTA-wide reduction barrier and its
// bookkeeping goes through the producer warp's mailbox; with 3 stages per CTA only ~one 18 KB load per CTA is in flight
// while a tile is consumed and another one stored (the warps of the plain pipe waited for data).  Here, like k_bc_stream:
//   * one CTA per SM, kStackConsumers consumer WARPS + a producer warp, 11 stages; a warp owns whole tiles: no CTA barrier per tile;
//   * first-layer rows: two passes over the row in shared memory (min/max, then rescale in place) by the warp alone, the
//     per-channel bookkeeping of dfq.py:62-70 (publish_row) done lane-parallel - lane r retires row r - instead of by one
//     producer lane;
//   * second-layer rows: one in-place pass with the reciprocal scales of the layer's columns cached per warp;
//   * the rescaled tile leaves with a bulk store issued by the consuming warp; the stage is handed back as soon as that store
//     has READ it;
//   * same arithmetic, same exit rule per convergence group (the functions of k_cle_engine are reused): weights, S, biases
//     and BN vectors are bit-identical to the engine's; the convergence metric is summed in a different order (float64).
// Eligibility (host, dfq_cle_run): two steps; every layer either `first` only or `second` only (col_mode 0) with its column
// extrema ready (the fold's scan); ungrouped relations; rows that the TMA unit can move (multiple of 4 floats, <= a stage);
// at most kBcExCols input columns, 3x3 or 1x1 taps; not apply_only.  Everything else runs on k_cle_engine.
// ------------------------------------------------------------------------------------------------------------
// Consumer warps of k_cle_stack (of the kBcConsumers the CTA has): the pass is far from issue-bound (ncu, 7 consumers: issue
// slots 19 % busy, 45 % of the warp samples waiting for data) - what matters is how many of the 11 stages are LOADING, i.e.
// not held by a consumer.  Sequence numbers are dealt modulo this count; the other warps only join the grid barriers.
#ifndef DFQ_STACK_CONSUMERS
#define DFQ_STACK_CONSUMERS 4
#endif
constexpr int kStackConsumers = DFQ_STACK_CONSUMERS;
static_assert(kStackConsumers >= 1 && kStackConsumers <= kBcConsumers, "k_cle_stack consumer count");

__device__ __forceinline__ float4 lds_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_f4(uint32_t a, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Producer lane: this CTA's tiles of one step (layers of converged groups skipped), SKIP padding, one END per consumer.
__device__ __noinline__ void cle_stack_feed(BcRing& ring, unsigned long long& n, float* arena, PassIter it) {
  TileDesc d;
  fence_proxy_async_all();          // rows written before the last grid barrier (bulk + plain stores) -> bulk loads
  while (it.valid()) { it.fill(d, arena); bc_produce(ring, n++, d); it.next(); }
  d.gptr = nullptr; d.task = -1; d.row0 = d.nrows = d.floats = 0;
  d.kind = BTK_SKIP;
  while (n % kStackConsumers) bc_produce(ring, n++, d);
  d.kind = BTK_END;
  for (int i = 0; i < kStackConsumers; ++i) bc_produce(ring, n++, d);
}

__global__ void __launch_bounds__(kBcThreads, 1)
k_cle_stack(float* arena, const DfqLayer* __restrict__ L, int nL, const DfqRelation* __restrict__ R, int nR,
            const int* __restrict__ step_ptr, const int* __restrict__ step_layers, const long long* __restrict__ pass_ptr,
            DfqCleParams P, CleCtl* ctl, GroupState* G, int nG) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(128) unsigned char ring_smem[];
  __shared__ RowCtx wctx[kBcConsumers];
  BcRing ring;
  ring.init(ring_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool producer = (warp == kBcConsumers);
  unsigned long long n = producer ? 0 : (unsigned long long)warp;       // (warps >= kStackConsumers never use it)
  for (int g = blockIdx.x * kBcThreads + threadIdx.x; g < nG; g += gridDim.x * kBcThreads) G[g].diff = 10.0;   // dfq.py:81
  __threadfence();
  grid.sync();

  for (int sweep = 0;; ++sweep) {
    const int slot = sweep % 3;
    for (int p = 0; p < 2; ++p) {
      if (producer) {
        if (lane == 0) {
          PassIter it;
          it.start(pass_ptr, step_layers, L, G, step_ptr[p], step_ptr[p + 1]);
          cle_stack_feed(ring, n, arena, it);
        }
      } else if (warp < kStackConsumers) {
        RowCtx& c = wctx[warp];
        float* inv_s = ring.ex_cache(warp);            // reciprocal scales of the current second layer's columns (+ sentinel)
        int cur_li = -1, cur_g = -1, kk = 1;
        double dacc = 0.0;
        auto flush_metric = [&]() {
          if (cur_g >= 0) {
            const double t = warp_sum(dacc);
            if (lane == 0 && t != 0.0) atomicAdd(&G[cur_g].acc[slot], t);
          }
          dacc = 0.0;
        };
        for (;; n += kStackConsumers) {
          const int s = bc_take(ring, n);
          const TileDesc d = ring.desc[s];
          if (d.kind == BTK_END || d.kind == BTK_SKIP) {
            bc_give_back(ring, s, lane);
            if (d.kind == BTK_END) { n += kStackConsumers; break; }
            continue;
          }
          if (d.task != cur_li) {
            cur_li = d.task;
            const int g = L[cur_li].group;
            if (g != cur_g) { flush_metric(); cur_g = g; }
            __syncwarp();
            if (lane == 0) make_ctx(c, arena, L, R, cur_li, sweep);
            __syncwarp();
            kk = c.kk;
            if (c.inv_in) {
              for (int j = lane; j < c.cols; j += 32) inv_s[j] = __ldcg(c.inv_in + j);
              if (lane == 0) inv_s[c.cols] = 1.f;
              __syncwarp();
            }
          }
          const int row_len = c.row_len, n4 = row_len >> 2;
          const uint32_t sbase = smem_u32(ring.stage(s));
          const double inv_n = c.inv_n;
          RowIn mine; mine.cmn = mine.cmx = 0.f; mine.u = 1.f; mine.s_given = 1.f;
          float ks = 1.f, kinv = 1.f;
          const bool has_out = c.has_out != 0;
          if (has_out) {
            // ---- first layer of a chain: per-row range -> s -> rescale (dfq.py:48-73) --------------------------------
            if (lane < d.nrows) mine = fetch_row_in(c, P, d.row0 + lane, false);     // this lane's row: column extrema of the pair
            for (int r = 0; r < d.nrows; ++r) {
              const uint32_t a0 = sbase + (uint32_t)r * (uint32_t)row_len * 4u;
              float mn = DFQ_INF, mx = -DFQ_INF;
#pragma unroll 4
              for (int i4 = lane; i4 < n4; i4 += 32) {
                const float4 t = lds_f4(a0 + 16u * i4);
                mn = fminf(mn, fminf(fminf(t.x, t.y), fminf(t.z, t.w)));
                mx = fmaxf(mx, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
              }
              mn = warp_min(mn); mx = warp_max(mx);
              RowIn in;
              in.cmn = __shfl_sync(0xffffffffu, mine.cmn, r); in.cmx = __shfl_sync(0xffffffffu, mine.cmx, r);
              in.u = 1.f; in.s_given = 1.f;
              float iv;
              const float sv = solve_row(P, in, mn, mx, &iv);
              if (lane == r) { ks = sv; kinv = iv; }
              float dsum = 0.f;
#pragma unroll 4
              for (int i4 = lane; i4 < n4; i4 += 32) {
                const float4 v = lds_f4(a0 + 16u * i4);
                float4 t;
                t.x = __fmul_rn(v.x, sv); t.y = __fmul_rn(v.y, sv); t.z = __fmul_rn(v.z, sv); t.w = __fmul_rn(v.w, sv);
                sts_f4(a0 + 16u * i4, t);
                dsum += fabsf(__fsub_rn(t.x, v.x)) + fabsf(__fsub_rn(t.y, v.y)) + fabsf(__fsub_rn(t.z, v.z)) + fabsf(__fsub_rn(t.w, v.w));
              }
              dacc += (double)dsum * inv_n;
            }
          } else {
            // ---- second layer: columns scaled by 1/s of the relation (dfq.py:73) ------------------------------------
            for (int r = 0; r < d.nrows; ++r) {
              const uint32_t a0 = sbase + (uint32_t)r * (uint32_t)row_len * 4u;
              float dsum = 0.f;
              if (kk == 9) {
#pragma unroll 4
                for (int i4 = lane; i4 < n4; i4 += 32) {
                  const float4 v = lds_f4(a0 + 16u * i4);
                  const float4 t = in_scale4<IN_KK9>(v, i4 * 4, inv_s, 1.f, 9);
                  sts_f4(a0 + 16u * i4, t);
                  dsum += fabsf(__fsub_rn(t.x, v.x)) + fabsf(__fsub_rn(t.y, v.y)) + fabsf(__fsub_rn(t.z, v.z)) + fabsf(__fsub_rn(t.w, v.w));
                }
              } else {
#pragma unroll 4
                for (int i4 = lane; i4 < n4; i4 += 32) {
                  const float4 v = lds_f4(a0 + 16u * i4);
                  const float4 t = in_scale4<IN_KK1>(v, i4 * 4, inv_s, 1.f, 1);
                  sts_f4(a0 + 16u * i4, t);
                  dsum += fabsf(__fsub_rn(t.x, v.x)) + fabsf(__fsub_rn(t.y, v.y)) + fabsf(__fsub_rn(t.z, v.z)) + fabsf(__fsub_rn(t.w, v.w));
                }
              }
              dacc += (double)dsum * inv_n;
            }
          }
          // the rescaled tile: generic-proxy writes -> visible to the bulk store, issued by this warp
          fence_proxy_async_smem();
          __syncwarp();
          // ... and the stage goes back to the producer as soon as the store has READ it (the store itself
          // completes in the background).  Holding it until the next tile instead (tried first) left every consumer with two
          // stages and the ring with almost nothing loading.
          if (lane == 0) {
            bulk_s2g(d.gptr, ring.stage(s), (uint32_t)d.floats * 4u);
            bulk_commit();
            bulk_wait_read<0>();
            mbar_arrive(ring.empty + s);
          }
          // per-channel bookkeeping of dfq.py:62-70 (S, 1/s, bias, BN vectors, derived column extrema), lane r for row r - after
          // the stage is on its way back: a dozen dependent global accesses that the ring does not have to wait for
          if (has_out && lane < d.nrows) publish_row(c, P, d.row0 + lane, ks, kinv, mine.cmn, mine.cmx);
        }
        flush_metric();
        if (lane == 0) { bulk_wait_all(); fence_proxy_async_all(); }
        __threadfence();             // the lanes' bookkeeping stores, before the grid barrier
      }
      grid.sync();
    }
    // ---- exit rule of dfq.py:105-115, one thread per group (as in k_cle_engine) ---------------------------------------
    const int nsw = sweep + 1;
    for (int g = blockIdx.x * kBcThreads + threadIdx.x; g < nG; g += gridDim.x * kBcThreads) {
      GroupState& st = G[g];
      if (st.done) continue;
      const double diff_tmp = st.acc[slot];
      st.acc[(slot + 2) % 3] = 0.0;
      if (fabs(st.diff - diff_tmp) > 1e-9) { st.count = 0; st.diff = diff_tmp; }
      else st.count++;
      if (g == 0 && sweep < 64) ctl->diffs[sweep] = diff_tmp;
      const bool cont = (st.diff > P.converge_thres) && (st.count < P.converge_count);
      const int cap = P.max_sweeps > 0 ? P.max_sweeps : 4096;
      if (!cont || nsw >= cap) { st.n_sweeps = nsw; st.converged = !cont; st.done = 1; }
      else atomicAdd(&ctl->active[nsw & 1], 1);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) ctl->active[sweep & 1] = 0;
    __threadfence();
    grid.sync();
    if (*((volatile int*)&ctl->active[nsw & 1]) == 0) break;
  }
}

}  // namespace dfq

using namespace dfq;

extern "C" int dfq_cle_run(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                           const DfqRelation* rels, int32_t n_rels, const int32_t* step_ptr,
                           const int32_t* step_layers, int32_t n_steps, const DfqCleParams* params,
                           DfqCleResult* result, int32_t n_groups, int32_t* group_sweeps, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool trace = getenv("DFQ_TRACE") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto ms_since = [](std::chrono::steady_clock::time_point a) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
  const auto h0 = now();
  double h_valid = 0, h_occ = 0, h_upload = 0, h_launch = 0;
  DFQ_REQUIRE(arena && layers && rels && step_ptr && step_layers && params && result, "null argument");
  DFQ_REQUIRE(n_layers > 0 && n_rels > 0 && n_steps > 0 && n_groups > 0, "empty problem");
  memset(result, 0, sizeof(*result));
  // Python `while diff > thres and count < converge_count` with diff = 10, count = 0 (dfq.py:81-83)
  if (!(10.0 > params->converge_thres) || !(0 < params->converge_count)) { result->converged = 1; result->last_diff = 10.0; return 0; }

  // ---- validate descriptors, find the widest phase -----------------------------------------------
  int64_t max_tiles = 1;
  for (int i = 0; i < n_rels; ++i) {
    const DfqRelation& r = rels[i];
    DFQ_REQUIRE(r.first >= 0 && r.first < n_layers && r.second >= 0 && r.second < n_layers, "relation layer index");
    const DfqLayer& a = layers[r.first];
    const DfqLayer& b = layers[r.second];
    DFQ_REQUIRE(r.channels == a.rows, "relation.channels != rows(first)");
    DFQ_REQUIRE(r.groups >= 1 && r.groups * r.gi == r.channels && r.groups * r.go == b.rows, "relation grouping");
    DFQ_REQUIRE(r.gi == b.cols, "first.rows / groups must equal second.cols (dfq.py:29-35)");
    DFQ_REQUIRE(a.rel_out == i && b.rel_in == i, "layer/relation cross links");
    DFQ_REQUIRE(a.group == b.group, "both layers of a relation must belong to the same convergence group");
    DFQ_REQUIRE(r.s_acc_off >= 0 && r.s_step_off >= 0 && r.inv_off >= 0, "relation scratch offsets");
    DFQ_REQUIRE(b.cmin_off >= 0 && b.cmax_off >= 0, "second layer needs column range scratch");
    DFQ_REQUIRE(b.col_mode != 1 || (b.cols == 1 && r.go == 1), "col_mode 1 requires cols==1 and one row per group");
    DFQ_REQUIRE(b.col_mode != 0 || b.rel_out < 0, "col_mode 0 is for chain ends");
  }
  for (int i = 0; i < n_layers; ++i) {
    const DfqLayer& l = layers[i];
    DFQ_REQUIRE(l.rows > 0 && l.cols > 0 && l.kk > 0, "layer shape");
    DFQ_REQUIRE(l.group >= 0 && l.group < n_groups, "layer group index");
    DFQ_REQUIRE(l.w_off >= 0 && l.w_off + (int64_t)l.rows * l.cols * l.kk <= arena_floats, "weight outside arena");
    DFQ_REQUIRE(l.bias_off >= 0 && l.bias_off + l.rows <= arena_floats, "bias outside arena");
    if (l.rel_in >= 0 && l.rel_out >= 0) DFQ_REQUIRE(l.rel_in < l.rel_out, "relations must be in forward chain order");
  }
  int64_t scan_total = 0;
  for (int i = 0; i < n_layers; ++i)
    if (layers[i].rel_in >= 0 && !(layers[i].flags & DFQ_LAYER_COLS_READY)) scan_total += pass_tiles(layers[i]);
  max_tiles = std::max(max_tiles, scan_total);
  for (int p = 0; p < n_steps; ++p) {
    int64_t t = 0;
    for (int q = step_ptr[p]; q < step_ptr[p + 1]; ++q) {
      const int li = step_layers[q];
      DFQ_REQUIRE(li >= 0 && li < n_layers, "step layer index");
      const DfqLayer& l = layers[li];
      DFQ_REQUIRE(l.rel_in >= 0 || l.rel_out >= 0, "step layer without relation");
      t += pass_tiles(l);
    }
    max_tiles = std::max(max_tiles, t);
  }

  // ---- streaming variant for stacks of two-layer chains (k_cle_stack) ----------------------------------------------
  bool stack_ok = (n_steps == 2) && !params->apply_only;
  for (int i = 0; stack_ok && i < n_rels; ++i) stack_ok = rels[i].groups == 1;
  int64_t stack_tiles = 0;
  for (int p = 0; stack_ok && p < n_steps; ++p)
    for (int q = step_ptr[p]; stack_ok && q < step_ptr[p + 1]; ++q) {
      const DfqLayer& l = layers[step_layers[q]];
      const int row_len = l.cols * l.kk;
      stack_ok = (row_len % 4 == 0) && row_len <= kStageFloats && (l.w_off % 4 == 0) && (l.kk == 9 || l.kk == 1);
      if (p == 0) stack_ok = stack_ok && l.rel_in < 0 && l.rel_out >= 0;
      else stack_ok = stack_ok && l.rel_in >= 0 && l.rel_out < 0 && l.col_mode == 0 && (l.flags & DFQ_LAYER_COLS_READY) &&
                      l.cols <= kBcExCols;
      stack_tiles += pass_tiles(l);
    }
  {
    int sms_ = 0, dev_ = 0;
    DFQ_CUDA(cudaGetDevice(&dev_));
    DFQ_CUDA(cudaDeviceGetAttribute(&sms_, cudaDevAttrMultiProcessorCount, dev_));
    const bool eligible = stack_ok;
    stack_ok = eligible && stack_tiles >= (int64_t)64 * sms_;                       // large phases only: small models are latency-bound
    if (const char* e = getenv("DFQ_CLE_STACK")) stack_ok = eligible && atoi(e) != 0;   // 0: never, 1: whenever eligible (tests)
    if (stack_ok) {
      const size_t dyn_s = BcRing::smem_bytes();
      DFQ_CUDA(cudaFuncSetAttribute(k_cle_stack, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_s));
      int per_sm_s = 0;
      DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_s, k_cle_stack, kBcThreads, dyn_s));
      if (per_sm_s < 1) { set_error("k_cle_stack does not fit on an SM"); return DFQ_E_NOT_COOPERATIVE; }
      const int grid_s = (int)std::min<int64_t>((int64_t)sms_ * per_sm_s, std::max<int64_t>(1, max_tiles));
      const int n_entries_s = step_ptr[n_steps];
      std::vector<long long> pass_ptr_s(n_entries_s + 1, 0);
      for (int q = 0; q < n_entries_s; ++q) pass_ptr_s[q + 1] = pass_ptr_s[q] + pass_tiles(layers[step_layers[q]]);
      TablePack tp;
      const int iL = tp.add(layers, n_layers), iR = tp.add(rels, n_rels), iSP = tp.add(step_ptr, n_steps + 1);
      const int iSL = tp.add(step_layers, n_entries_s), iPP = tp.add(pass_ptr_s.data(), n_entries_s + 1);
      int rc;
      if ((rc = tp.upload(st))) return rc;
      DfqLayer* dL = tp.ptr<DfqLayer>(iL); DfqRelation* dR = tp.ptr<DfqRelation>(iR);
      int32_t *dSP = tp.ptr<int32_t>(iSP), *dSL = tp.ptr<int32_t>(iSL);
      long long* dPP = tp.ptr<long long>(iPP);
      CleCtl* dctl = nullptr; GroupState* dG = nullptr;
      DFQ_CUDA(cudaMallocAsync((void**)&dctl, sizeof(CleCtl), st));
      DFQ_CUDA(cudaMemsetAsync(dctl, 0, sizeof(CleCtl), st));
      DFQ_CUDA(cudaMallocAsync((void**)&dG, sizeof(GroupState) * n_groups, st));
      DFQ_CUDA(cudaMemsetAsync(dG, 0, sizeof(GroupState) * n_groups, st));
      DfqCleParams Pk = *params;
      void* args[] = {&arena, &dL, (void*)&n_layers, &dR, (void*)&n_rels, &dSP, &dSL, &dPP, &Pk, &dctl, &dG, (void*)&n_groups};
      DFQ_CUDA(cudaLaunchCooperativeKernel((void*)k_cle_stack, dim3(grid_s), dim3(kBcThreads), args, dyn_s, st));
      CleCtl h;
      std::vector<GroupState> hg(n_groups);
      ReadBack rb;
      rb.add(&h, dctl, sizeof(CleCtl));
      rb.add(hg.data(), dG, sizeof(GroupState) * n_groups);
      { const int rrc = rb.enqueue(st); if (rrc) return rrc; }
      tp.release(st);
      free_async(dctl, st); free_async(dG, st);
      DFQ_CUDA(cudaStreamSynchronize(st));
      rb.finish();
      result->n_sweeps = 0; result->converged = 1;
      for (int g = 0; g < n_groups; ++g) {
        result->n_sweeps = std::max(result->n_sweeps, hg[g].n_sweeps);
        result->converged &= hg[g].converged;
        if (group_sweeps) group_sweeps[g] = hg[g].n_sweeps;
      }
      result->last_diff = hg[0].diff;
      memcpy(result->diffs, h.diffs, sizeof(h.diffs));
      if (trace) fprintf(stderr, "[dfq_cle_run] stack variant: grid %d, sweeps %d, host ms %.3f\n", grid_s, result->n_sweeps, ms_since(h0));
      return 0;
    }
  }

  h_valid = ms_since(h0);
  int dev = 0, sms = 0, per_sm = 0, coop = 0;
  DFQ_CUDA(cudaGetDevice(&dev));
  DFQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  DFQ_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) { set_error("device does not support cooperative launch"); return DFQ_E_NOT_COOPERATIVE; }
  bool any_rescan = false;
  for (int i = 0; i < n_layers; ++i) any_rescan |= (layers[i].rel_in >= 0 && layers[i].col_mode == 2);
  int rs_cols = any_rescan ? kRescanCols : 0;
  // table mirror for small models (see the kernel); its size must be known before the occupancy query
  size_t tbl_est = 0;
  {
    const int n_entries_early = step_ptr[n_steps];
    int n_scan_est = 0;
    for (int i = 0; i < n_layers; ++i) n_scan_est += (layers[i].rel_in >= 0 && !(layers[i].flags & DFQ_LAYER_COLS_READY));
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    tbl_est = al(sizeof(DfqLayer) * n_layers) + al(sizeof(DfqRelation) * n_rels) + al(4 * (n_steps + 1)) + al(4 * n_entries_early) +
              al(8 * (n_entries_early + 1)) + al(8 * (n_scan_est + 1)) + al(4 * n_scan_est);
  }
  const bool cache_tables = tbl_est <= kTableCacheBytes;
  const size_t dyn_smem = ((WsPipe::smem_bytes() + 15) & ~(size_t)15) + (size_t)kTeams * 2 * rs_cols * sizeof(float) +
                          (cache_tables ? tbl_est : 0);
  DFQ_CUDA(cudaFuncSetAttribute(k_cle_engine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem));
  DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cle_engine, kCtaThreads, dyn_smem));
  if (per_sm < 1) { set_error("persistent kernel does not fit on an SM"); return DFQ_E_NOT_COOPERATIVE; }
  int grid = (int)std::min<int64_t>((int64_t)sms * per_sm, max_tiles);
  if (const char* e = getenv("DFQ_CLE_GRID")) grid = std::max(1, std::min(grid, atoi(e)));   // experiments: cap the grid

  h_occ = ms_since(h0);
  const int n_entries = step_ptr[n_steps];
  std::vector<long long> pass_ptr(n_entries + 1, 0);
  for (int q = 0; q < n_entries; ++q) pass_ptr[q + 1] = pass_ptr[q] + pass_tiles(layers[step_layers[q]]);
  std::vector<int32_t> scan_layers;
  std::vector<long long> scan_ptr(1, 0);
  for (int i = 0; i < n_layers; ++i)
    if (layers[i].rel_in >= 0 && !(layers[i].flags & DFQ_LAYER_COLS_READY)) {   // the others arrive with buffer 0 filled
      scan_layers.push_back(i);
      scan_ptr.push_back(scan_ptr.back() + pass_tiles(layers[i]));
    }
  int n_scan = (int)scan_layers.size();
  TablePack tp;
  const int iL = tp.add(layers, n_layers), iR = tp.add(rels, n_rels), iSP = tp.add(step_ptr, n_steps + 1);
  const int iSL = tp.add(step_layers, n_entries);
  const int iPP = tp.add(pass_ptr.data(), n_entries + 1), iSCP = tp.add(scan_ptr.data(), n_scan + 1);
  const int iSCL = tp.add(scan_layers.data(), n_scan);
  int rc;
  if ((rc = tp.upload(st))) return rc;
  DfqLayer* dL = tp.ptr<DfqLayer>(iL); DfqRelation* dR = tp.ptr<DfqRelation>(iR);
  int32_t *dSP = tp.ptr<int32_t>(iSP), *dSL = tp.ptr<int32_t>(iSL), *dSCL = tp.ptr<int32_t>(iSCL);
  long long *dPP = tp.ptr<long long>(iPP), *dSCP = tp.ptr<long long>(iSCP);
  CleCtl* dctl = nullptr;
  GroupState* dG = nullptr;
  DFQ_CUDA(cudaMallocAsync((void**)&dctl, sizeof(CleCtl), st));
  DFQ_CUDA(cudaMemsetAsync(dctl, 0, sizeof(CleCtl), st));
  DFQ_CUDA(cudaMallocAsync((void**)&dG, sizeof(GroupState) * n_groups, st));
  DFQ_CUDA(cudaMemsetAsync(dG, 0, sizeof(GroupState) * n_groups, st));
  h_upload = ms_since(h0);
  DfqCleParams P = *params;
  const unsigned char* d_tbl = tp.dev;
  int tbl_bytes = cache_tables ? (int)tp.total : 0;
  if (cache_tables && tp.total != tbl_est) { set_error("internal: table pack size mismatch"); return DFQ_E_ARG; }
  void* args[] = {&arena, &dL, (void*)&n_layers, &dR, (void*)&n_rels, &dSP, &dSL, (void*)&n_steps,
                  &dPP, &dSCP, &dSCL, (void*)&n_scan, &P, &dctl, &dG, (void*)&n_groups, &rs_cols, &d_tbl, &tbl_bytes};
  DFQ_CUDA(cudaLaunchCooperativeKernel((void*)k_cle_engine, dim3(grid), dim3(kCtaThreads), args, dyn_smem, st));
  h_launch = ms_since(h0);
  CleCtl h;
  std::vector<GroupState> hg(n_groups);
  ReadBack rb;
  rb.add(&h, dctl, sizeof(CleCtl));
  rb.add(hg.data(), dG, sizeof(GroupState) * n_groups);
  { const int rrc = rb.enqueue(st); if (rrc) return rrc; }
  tp.release(st);
  free_async(dctl, st); free_async(dG, st);
  DFQ_CUDA(cudaStreamSynchronize(st));
  rb.finish();
  result->n_sweeps = 0;
  result->converged = 1;
  for (int g = 0; g < n_groups; ++g) {
    result->n_sweeps = std::max(result->n_sweeps, hg[g].n_sweeps);
    result->converged &= hg[g].converged;
    if (group_sweeps) group_sweeps[g] = hg[g].n_sweeps;
  }
  if (trace) {
    fprintf(stderr, "[dfq_cle_run] host ms: validate %.3f occupancy %.3f upload %.3f launch %.3f done %.3f\n", h_valid, h_occ,
            h_upload, h_launch, ms_since(h0));
    fprintf(stderr, "[dfq_cle_run] grid %d (%d CTAs/SM) sweeps %d; phase ms:", grid, per_sm, result->n_sweeps);
    for (int i = 1; i < 32 && h.t_ns[i]; ++i) fprintf(stderr, " %.3f", (h.t_ns[i] - h.t_ns[i - 1]) * 1e-6);
    fprintf(stderr, "\n");
#ifdef DFQ_STEP_TRACE
    {
      static unsigned long long hs[8][512][8];
      cudaMemcpyFromSymbol(hs, g_step_trace, sizeof(hs));
      const int nb = std::min(grid, 512);
      for (int p = 0; p < std::min(n_steps, 8); ++p) {
        int last = 0, busy = 0; unsigned long long first_start = ~0ull;
        std::vector<unsigned long long> arr;
        for (int b = 0; b < nb; ++b) {
          if (hs[p][b][6] > hs[p][last][6]) last = b;
          if (hs[p][b][3]) busy++;
          first_start = std::min(first_start, hs[p][b][0]);
          arr.push_back(hs[p][b][6]);
        }
        std::sort(arr.begin(), arr.end());
        const unsigned long long* t = hs[p][last];
        auto us = [&](unsigned long long v) { return v ? (double)(v - first_start) * 1e-3 : -1.0; };
        unsigned long long next_start = ~0ull;
        if (p + 1 < std::min(n_steps, 8)) for (int b = 0; b < nb; ++b) next_start = std::min(next_start, hs[p + 1][b][0]);
        fprintf(stderr, "[step %d] busy CTAs %d/%d; last CTA %d: start %.2f firsttile %.2f ctx %.2f computed %.2f barrier %.2f handedback %.2f end %.2f fenced %.2f | median fenced %.2f | next step starts %.2f\n",
                p, busy, nb, last, us(t[0]), us(t[1]), us(t[2]), us(t[3]), us(t[7]), us(t[4]), us(t[5]), us(t[6]), us(arr[arr.size() / 2]),
                next_start != ~0ull ? us(next_start) : -1.0);
      }
    }
#endif
    if (getenv("DFQ_TRACE_TILES")) {
      const unsigned long long t0 = h.tile_ns[0][1];
      fprintf(stderr, "tile: C.wait C.ready C.done C.arrived | P.retire P.stored P.loadissued P.fullarrive  (us since first load)\n");
      for (int i = 0; i < 48; ++i) {
        fprintf(stderr, "%3d:", i);
        for (int j = 0; j < 8; ++j) fprintf(stderr, " %8.2f", h.tile_ns[i][j] ? (double)(h.tile_ns[i][j] - t0) * 1e-3 : -1.0);
        fprintf(stderr, "\n");
      }
    }
  }
  result->last_diff = hg[0].diff;
  memcpy(result->diffs, h.diffs, sizeof(h.diffs));
  return 0;
}
