// VOC average precision of SSD detections on the device: what main_ssd.py computes from the detections it writes per class
// (compute_average_precision_per_class, utils/detection/measurements.py), accumulated batch by batch.
//
//   k_map_match   one CTA per image: the image's non-difficult ground truth counted per class, then per detection (class c)
//                 the box as the reference reads it back (fl32(fl32(b + 1) - 1)), box_utils.iou_of against every ground-truth
//                 box of class c in annotation order, the first maximum (the first NaN wins), and the verdict: false
//                 positive, ignored (the maximum is on a difficult box) or a claim on the box.  A box goes to the first
//                 claiming detection in the reference's order, score descending and then row; every other claim is a
//                 false positive.  Appends the detection's sort key and verdict to the accumulation buffers.
//   k_map_curve   one CTA per class, after a stable radix sort of all accumulated detections by (class, score
//                 descending): the cumulative true and false positives, float64 precision and recall, the NaN-propagating
//                 running maximum of precision from the end, then the 11 VOC2007 maxima or the area terms at the points
//                 where recall changes.
#include <algorithm>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "box_iou.cuh"
#include "common.cuh"

namespace dfq {
namespace {

constexpr int kMatchThreads = 128;
constexpr int kCurveThreads = 256;
constexpr int kMapMaxClasses = 4096;

// The score's place in a descending order: the fp32 bits made unsigned-orderable (-0.0 folded onto +0.0), complemented;
// NaN after every number, as np.argsort(-scores) puts it.
__device__ __forceinline__ uint32_t score_desc(float v) {
  if (v != v) return 0xffffffffu;
  uint32_t u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0;
  return (u & 0x80000000u) ? u : ~(u | 0x80000000u);
}

// The ground-truth box of class c in [g0, g1) with the largest iou_of(box, gt): torch.max / torch.argmax on the CPU, the
// first NaN or else the first maximum.  -1 when the image has no box of class c.
__device__ __forceinline__ int64_t best_gt(const float4 box, int64_t c, const float4* __restrict__ gt_boxes,
                                           const int64_t* __restrict__ gt_labels, int64_t g0, int64_t g1, float* best) {
  int64_t arg = -1;
  float m = 0.f;
  for (int64_t g = g0; g < g1; ++g) {
    if (__ldg((const long long*)gt_labels + g) != c) continue;
    const float v = iou_of(box, gt_boxes[g]);
    if (arg < 0 || (m == m && (v != v || v > m))) {
      m = v;
      arg = g;
    }
  }
  *best = m;
  return arg;
}

constexpr uint8_t kPending = 3;

__global__ void __launch_bounds__(kMatchThreads) k_map_match(
    const float4* __restrict__ det_boxes, const int64_t* __restrict__ det_labels, const float* __restrict__ det_probs,
    const int64_t* __restrict__ det_off, int64_t T, const float4* __restrict__ gt_boxes,
    const int64_t* __restrict__ gt_labels, const uint8_t* __restrict__ gt_difficult, const int64_t* __restrict__ gt_off,
    int64_t G, int N, int C, double iou_threshold, unsigned long long* __restrict__ claims, uint64_t* __restrict__ keys,
    uint8_t* __restrict__ flags, unsigned long long* __restrict__ gt_count, int* __restrict__ error) {
  const int n = blockIdx.x, tid = threadIdx.x;
  const int64_t d0 = det_off[n], d1 = det_off[n + 1], g0 = gt_off[n], g1 = gt_off[n + 1];
  const bool det_ok = 0 <= d0 && d0 <= d1 && d1 <= T && (n > 0 || d0 == 0) && (n < N - 1 || d1 == T);
  const bool gt_ok = 0 <= g0 && g0 <= g1 && g1 <= G && (n > 0 || g0 == 0) && (n < N - 1 || g1 == G);
  if (!det_ok || !gt_ok) {
    if (tid == 0) atomicOr(error, (det_ok ? 0 : DFQ_MAP_ERR_DET_OFFSETS) | (gt_ok ? 0 : DFQ_MAP_ERR_GT_OFFSETS));
    return;
  }
  for (int64_t g = g0 + tid; g < g1; g += blockDim.x) {
    const int64_t l = gt_labels[g];
    if (l < 0 || l >= C) atomicOr(error, DFQ_MAP_ERR_GT_LABEL);
    else if (!gt_difficult[g]) atomicAdd(gt_count + l, 1ull);
    claims[g] = ~0ull;
  }
  __syncthreads();

  // verdicts, and a claim (score, row) on the best box where that decides
  for (int64_t t = d0 + tid; t < d1; t += blockDim.x) {
    const int64_t c = det_labels[t];
    const uint32_t sd = score_desc(det_probs[t]);
    if (c < 1 || c >= C) {
      atomicOr(error, DFQ_MAP_ERR_DET_LABEL);
      keys[t] = sd;
      flags[t] = DFQ_MAP_FP;
      continue;
    }
    keys[t] = ((uint64_t)c << 32) | sd;
    const float4 b = det_boxes[t];
    const float4 box = make_float4((b.x + 1.f) - 1.f, (b.y + 1.f) - 1.f, (b.z + 1.f) - 1.f, (b.w + 1.f) - 1.f);
    float m;
    const int64_t arg = best_gt(box, c, gt_boxes, gt_labels, g0, g1, &m);
    uint8_t f = DFQ_MAP_FP;
    if (arg >= 0 && (double)m > iou_threshold) {
      if (gt_difficult[arg]) {
        f = DFQ_MAP_IGNORED;
      } else {
        atomicMin(claims + arg, ((unsigned long long)sd << 32) | (uint32_t)(t - d0));
        f = kPending;
      }
    }
    flags[t] = f;
  }
  __syncthreads();
  for (int64_t t = d0 + tid; t < d1; t += blockDim.x) {
    if (flags[t] != kPending) continue;
    const float4 b = det_boxes[t];
    const float4 box = make_float4((b.x + 1.f) - 1.f, (b.y + 1.f) - 1.f, (b.z + 1.f) - 1.f, (b.w + 1.f) - 1.f);
    float m;
    const int64_t arg = best_gt(box, det_labels[t], gt_boxes, gt_labels, g0, g1, &m);
    const unsigned long long mine = ((unsigned long long)(keys[t] & 0xffffffffu) << 32) | (uint32_t)(t - d0);
    flags[t] = claims[arg] == mine ? DFQ_MAP_TP : DFQ_MAP_FP;
  }
}

// np.maximum: NaN in, NaN out
struct NanMax {
  __device__ __forceinline__ double operator()(double a, double b) const { return (a != a || a > b) ? a : b; }
};

// first index in [0, D) whose key's class (the upper 32 bits) is >= c
__device__ __forceinline__ int64_t class_begin(const uint64_t* __restrict__ keys, int64_t D, int c) {
  int64_t a = 0, b = D;
  while (a < b) {
    const int64_t m = (a + b) >> 1;
    if ((keys[m] >> 32) < (uint64_t)c) a = m + 1; else b = m;
  }
  return a;
}

__global__ void __launch_bounds__(kCurveThreads) k_map_curve(
    const uint64_t* __restrict__ keys, const uint8_t* __restrict__ flags, int64_t D, int C,
    const unsigned long long* __restrict__ gt_count, int use_2007, double* __restrict__ out, int64_t out_len,
    int64_t* __restrict__ term_count) {
  using Reduce = cub::BlockReduce<unsigned long long, kCurveThreads>;
  using ScanU = cub::BlockScan<unsigned long long, kCurveThreads>;
  using ScanD = cub::BlockScan<double, kCurveThreads>;
  __shared__ union {
    typename Reduce::TempStorage reduce;
    typename ScanU::TempStorage scan_u;
    typename ScanD::TempStorage scan_d;
  } tmp;
  __shared__ int64_t s_begin, s_end, s_base;
  __shared__ unsigned long long s_total;
  __shared__ double s_p[11];
  const int c = blockIdx.x + 1, tid = threadIdx.x;
  if (tid == 0) {
    s_begin = class_begin(keys, D, c);
    s_end = class_begin(keys, D, c + 1);
    int64_t base = c - 1;                        // class c' owns gt_count[c'] + 1 area terms
    for (int k = 1; k < c; ++k) base += (int64_t)gt_count[k];
    s_base = base;
  }
  if (tid < 11) s_p[tid] = 0.0;
  __syncthreads();
  const int64_t s = s_begin, n = s_end - s_begin, base = s_base;
  const double nt = (double)gt_count[c];

  // totals: true positives in the upper 32 bits, false positives in the lower
  unsigned long long sum = 0;
  for (int64_t i = s + tid; i < s + n; i += kCurveThreads) {
    const uint8_t f = flags[i];
    sum += f == DFQ_MAP_TP ? (1ull << 32) : f == DFQ_MAP_FP ? 1ull : 0ull;
  }
  sum = Reduce(tmp.reduce).Sum(sum);
  if (tid == 0) s_total = sum;
  __syncthreads();
  const unsigned long long total = s_total;
  const int64_t tp_total = (int64_t)(total >> 32), fp_total = (int64_t)(total & 0xffffffffu);

  // from the end: position i = s + n - 1 - idx; suffix sums give tp / fp at i, the scan of precision its running maximum
  unsigned long long carry_sum = 0;
  double carry_p = 0.0;                          // the 0.0 compute_average_precision appends
  double last_recall = 0.0;                      // recall at the last detection (0.0, the padded value, when there is none)
  for (int64_t base_idx = 0; base_idx < n; base_idx += kCurveThreads) {
    const int64_t idx = base_idx + tid;
    const bool valid = idx < n;
    const int64_t i = s + n - 1 - idx;
    const uint8_t f = valid ? flags[i] : DFQ_MAP_IGNORED;
    const unsigned long long inc = f == DFQ_MAP_TP ? (1ull << 32) : f == DFQ_MAP_FP ? 1ull : 0ull;
    unsigned long long suf, agg;
    ScanU(tmp.scan_u).InclusiveSum(inc, suf, agg);
    suf += carry_sum;
    const int64_t inc_tp = (int64_t)(inc >> 32), inc_fp = (int64_t)(inc & 0xffffffffu);
    const int64_t tp = tp_total - ((int64_t)(suf >> 32) - inc_tp);
    const int64_t fp = fp_total - ((int64_t)(suf & 0xffffffffu) - inc_fp);
    const double dtp = (double)tp;
    const double precision = valid ? dtp / (dtp + (double)fp) : 0.0;
    const double recall = dtp / nt, recall_prev = (double)(tp - inc_tp) / nt;
    __syncthreads();
    double pmax, pagg;
    ScanD(tmp.scan_d).InclusiveScan(precision, pmax, NanMax(), pagg);
    pmax = NanMax()(pmax, carry_p);
    if (valid) {
      if (idx == 0) last_recall = recall;
      if (use_2007) {
        for (int k = 0; k < 11; ++k) {           // np.arange(0., 1.1, 0.1)[k] is k * 0.1
          const double th = k * 0.1;
          if (recall >= th && (idx == n - 1 || !(recall_prev >= th))) s_p[k] = pmax;
        }
      } else if (inc_tp) {
        const int64_t slot = base + tp - 1;
        if (slot < out_len) out[slot] = (recall - recall_prev) * pmax;
      }
    }
    carry_sum += agg;
    carry_p = NanMax()(carry_p, pagg);
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) {
    if (use_2007) {
      for (int k = 0; k < 11; ++k) out[(int64_t)(c - 1) * 11 + k] = s_p[k];
      term_count[c] = n;
    } else {
      int64_t m = tp_total;
      if (last_recall != 1.0) {
        const int64_t slot = base + m;
        if (slot < out_len) out[slot] = (1.0 - last_recall) * 0.0;
        ++m;
      }
      term_count[c] = m;
    }
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int check_classes(int C, const char* who) {
  if (C < 2) { set_error("%s: C must be at least 2 (background and one class), got %d", who, C); return DFQ_E_ARG; }
  if (C > kMapMaxClasses) { set_error("%s: C = %d is above the limit %d", who, C, kMapMaxClasses); return DFQ_E_UNSUPPORTED; }
  return 0;
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_map_match(const float* det_boxes, const int64_t* det_labels, const float* det_probs,
                             const int64_t* det_offsets, int64_t T, const float* gt_boxes, const int64_t* gt_labels,
                             const uint8_t* gt_difficult, const int64_t* gt_offsets, int64_t G, int32_t N, int32_t C,
                             double iou_threshold, uint64_t* keys, uint8_t* flags, uint64_t* gt_count, int32_t* error,
                             void* stream) {
  const char* who = "dfq_map_match";
  if (int rc = check_classes(C, who)) return rc;
  if (N < 1 || T < 0 || G < 0) {
    set_error("%s: N must be positive and T, G non-negative, got %d, %lld, %lld", who, N, (long long)T, (long long)G);
    return DFQ_E_ARG;
  }
  if (!det_offsets || !gt_offsets || !gt_count || !error) {
    set_error("%s: det_offsets, gt_offsets, gt_count and error must be non-NULL", who);
    return DFQ_E_ARG;
  }
  if (T > 0 && (!det_boxes || !det_labels || !det_probs || !keys || !flags || !aligned16(det_boxes))) {
    set_error("%s: with detections, det_boxes (16-byte aligned), det_labels, det_probs, keys and flags must be non-NULL",
              who);
    return DFQ_E_ARG;
  }
  if (G > 0 && (!gt_boxes || !gt_labels || !gt_difficult || !aligned16(gt_boxes))) {
    set_error("%s: with ground truth, gt_boxes (16-byte aligned), gt_labels and gt_difficult must be non-NULL", who);
    return DFQ_E_ARG;
  }
  if (T > INT32_MAX) {
    set_error("%s: %lld detections in one batch, above the limit %d", who, (long long)T, INT32_MAX);
    return DFQ_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* claims = nullptr;
  if (G > 0) DFQ_CUDA(cudaMallocAsync((void**)&claims, sizeof(unsigned long long) * G, st));
  k_map_match<<<N, kMatchThreads, 0, st>>>((const float4*)det_boxes, det_labels, det_probs, det_offsets, T,
                                           (const float4*)gt_boxes, gt_labels, gt_difficult, gt_offsets, G, N, C,
                                           iou_threshold, claims, keys, flags, (unsigned long long*)gt_count, error);
  const cudaError_t e = cudaGetLastError();
  free_async(claims, st);
  DFQ_CUDA(e);
  return 0;
}

extern "C" int dfq_map_curve(const uint64_t* keys, const uint8_t* flags, int64_t D, int32_t C, const uint64_t* gt_count,
                             int32_t use_2007, double* out, int64_t out_len, int64_t* term_count, void* stream) {
  const char* who = "dfq_map_curve";
  if (int rc = check_classes(C, who)) return rc;
  if (D < 0) { set_error("%s: D must be non-negative, got %lld", who, (long long)D); return DFQ_E_ARG; }
  if (use_2007 != 0 && use_2007 != 1) { set_error("%s: use_2007 must be 0 or 1, got %d", who, use_2007); return DFQ_E_ARG; }
  if (!gt_count || !out || !term_count || (D > 0 && (!keys || !flags))) {
    set_error("%s: gt_count, out, term_count and, with detections, keys and flags must be non-NULL", who);
    return DFQ_E_ARG;
  }
  const int64_t need = use_2007 ? 11ll * (C - 1) : (int64_t)C;
  if (out_len < need) {
    set_error("%s: out holds %lld values, at least %lld are needed", who, (long long)out_len, (long long)need);
    return DFQ_E_ARG;
  }
  if (D > INT32_MAX) {
    set_error("%s: %lld detections, above the limit %d", who, (long long)D, INT32_MAX);
    return DFQ_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint64_t* sorted_keys = nullptr;
  uint8_t* sorted_flags = nullptr;
  void* tmp = nullptr;
  cudaError_t e = cudaSuccess;
  if (D > 0) {
    int end_bit = 33;                            // the class in bits 32 .. end_bit - 1
    while ((1 << (end_bit - 32)) < C) ++end_bit;
    size_t tmp_bytes = 0;
    DFQ_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, sorted_keys, flags, sorted_flags, (int)D, 0,
                                             end_bit, st));
    DFQ_CUDA(cudaMallocAsync((void**)&sorted_keys, sizeof(uint64_t) * D, st));
    e = cudaMallocAsync((void**)&sorted_flags, D, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&tmp, tmp_bytes, st);
    if (e == cudaSuccess)
      e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, sorted_keys, flags, sorted_flags, (int)D, 0, end_bit, st);
  }
  if (e == cudaSuccess) {
    k_map_curve<<<C - 1, kCurveThreads, 0, st>>>(sorted_keys, sorted_flags, D, C, (const unsigned long long*)gt_count,
                                                 use_2007, out, out_len, term_count);
    e = cudaGetLastError();
  }
  free_async(tmp, st);
  free_async(sorted_flags, st);
  free_async(sorted_keys, st);
  DFQ_CUDA(e);
  return 0;
}
