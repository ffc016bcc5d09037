// Stand-alone tensor kernels of the C ABI (activations, module forward, API-level helpers) and the
// library's host-side plumbing.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <mutex>
#include <unordered_map>

#include <cooperative_groups.h>

#include "common.cuh"

namespace dfq {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (int)e;
}
int sm_count() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}
int coop_grid(const void* kernel, const char* kernel_name, int threads, size_t dyn_smem, int64_t max_tiles, int* grid) {
  int dev = 0, sms = 0, per_sm = 0;
  DFQ_CUDA(cudaGetDevice(&dev));
  DFQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (dyn_smem > 0) DFQ_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem));
  DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, dyn_smem));
  if (per_sm < 1) { set_error("%s does not fit on an SM", kernel_name); return DFQ_E_NOT_COOPERATIVE; }
  *grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sms * per_sm, max_tiles));
  return 0;
}

namespace {
struct Slot { unsigned char* host = nullptr; unsigned char* dev = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool used = false; };
// One ring per device: a slot's event belongs to the device it was created on and is recorded on that device's streams
// only, and each device's default pool is tuned once.
struct SlotRing { Slot slots[4]; int next = 0; bool pool_tuned = false; };
std::unordered_map<int, SlotRing> g_rings;
std::mutex g_slot_mu;
}  // namespace

// word-wise copy between device memory and mapped page-locked host memory (either direction), a few KB to a few hundred KB
__global__ void k_copy_words(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t nwords) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
static int launch_copy_words(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  const size_t nwords = bytes / 4;
  if (nwords == 0) return 0;
  const int blocks = (int)std::min<size_t>(64, (nwords + 255) / 256);
  k_copy_words<<<blocks, 256, 0, st>>>((uint32_t*)dst, (const uint32_t*)src, nwords);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

namespace {
struct RbSlot { unsigned char* host = nullptr; unsigned char* dev = nullptr; size_t cap = 0; bool busy = false; };
RbSlot g_rb[4];
std::mutex g_rb_mu;
}  // namespace

int ReadBack::enqueue(cudaStream_t st) {
  {
    std::lock_guard<std::mutex> lk(g_rb_mu);
    for (int i = 0; i < 4 && slot < 0; ++i) if (!g_rb[i].busy) { slot = i; g_rb[i].busy = true; }
  }
  if (slot < 0) {   // more than four read-backs in flight (concurrent host threads): the copy engine will do
    for (int i = 0; i < n; ++i) DFQ_CUDA(cudaMemcpyAsync(items[i].host, items[i].dev, items[i].bytes, cudaMemcpyDeviceToHost, st));
    return 0;
  }
  RbSlot& sl = g_rb[slot];
  if (sl.cap < total) {
    if (sl.host) cudaFreeHost(sl.host);
    sl.host = nullptr; sl.cap = 0;
    const size_t cap = std::max<size_t>(total, 256 << 10);
    DFQ_CUDA(cudaHostAlloc((void**)&sl.host, cap, cudaHostAllocMapped));
    DFQ_CUDA(cudaHostGetDevicePointer((void**)&sl.dev, sl.host, 0));
    sl.cap = cap;
  }
  mapped = sl.host;
  for (int i = 0; i < n; ++i) {
    const int rc = launch_copy_words(sl.dev + items[i].off, items[i].dev, items[i].bytes, st);
    if (rc) return rc;
  }
  return 0;
}

void ReadBack::finish() {
  if (slot < 0) return;
  for (int i = 0; i < n; ++i) memcpy(items[i].host, mapped + items[i].off, items[i].bytes);
  std::lock_guard<std::mutex> lk(g_rb_mu);
  g_rb[slot].busy = false;
  slot = -1;
}

void ReadBack::abandon() {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(g_rb_mu);
  g_rb[slot].busy = false;
  slot = -1;
}

int TablePack::upload(cudaStream_t st) {
  dev = nullptr;
  if (total == 0) return 0;
  int d = 0;
  DFQ_CUDA(cudaGetDevice(&d));
  std::lock_guard<std::mutex> lk(g_slot_mu);
  SlotRing& ring = g_rings[d];
  if (!ring.pool_tuned) {   // keep freed descriptor blocks in the default pool instead of returning them to the OS at every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, d) == cudaSuccess) {
      unsigned long long thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    ring.pool_tuned = true;
  }
  Slot& sl = ring.slots[ring.next];
  ring.next = (ring.next + 1) % 4;
  if (sl.used) DFQ_CUDA(cudaEventSynchronize(sl.ev));
  sl.used = false;
  if (sl.cap < total) {
    if (sl.host) cudaFreeHost(sl.host);
    sl.host = nullptr; sl.cap = 0;
    const size_t cap = std::max<size_t>(total, 1 << 20);
    DFQ_CUDA(cudaHostAlloc((void**)&sl.host, cap, cudaHostAllocMapped));
    DFQ_CUDA(cudaHostGetDevicePointer((void**)&sl.dev, sl.host, 0));
    sl.cap = cap;
  }
  if (!sl.ev) DFQ_CUDA(cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming));
  for (int i = 0; i < n; ++i)
    if (items[i].bytes) memcpy(sl.host + items[i].off, items[i].src, items[i].bytes);
  DFQ_CUDA(cudaMallocAsync((void**)&dev, total, st));
  int rc = launch_copy_words(dev, sl.dev, total, st);
  if (rc == 0) {
    const cudaError_t e = cudaEventRecord(sl.ev, st);
    if (e == cudaSuccess) { sl.used = true; return 0; }
    rc = cuda_fail(e, "cudaEventRecord(sl.ev, st)");
  }
  // the copy may be in flight without an event to wait on: let it finish before the slot is reused, then free the block
  cudaStreamSynchronize(st);
  release(st);
  return rc;
}

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
// floats per thread of one (sample, split) work item of the per-sample statistics, and of one k_minmax thread
constexpr int kItemFloats = 16;
// dfq_range_rows: rows longer than this get a CTA each, shorter ones a warp
constexpr int kRangeCtaRow = 2048;

// grid-stride min/max of a flat tensor, 4 independent 128-bit loads in flight per thread
__device__ __forceinline__ void flat_minmax(const float* __restrict__ x, int64_t n, int64_t start, int64_t stride,
                                            float& mn, float& mx) {
  if ((((uintptr_t)x) & 15) == 0) {
    const float4* x4 = (const float4*)x;
    const int64_t n4 = n >> 2;
    int64_t i = start;
    for (; i + 3 * stride < n4; i += 4 * stride) {
      const float4 a = ldg_stream(x4 + i), b = ldg_stream(x4 + i + stride);
      const float4 c = ldg_stream(x4 + i + 2 * stride), d = ldg_stream(x4 + i + 3 * stride);
      mn = fminf(mn, fminf(fminf(fminf(a.x, a.y), fminf(a.z, a.w)), fminf(fminf(b.x, b.y), fminf(b.z, b.w))));
      mn = fminf(mn, fminf(fminf(fminf(c.x, c.y), fminf(c.z, c.w)), fminf(fminf(d.x, d.y), fminf(d.z, d.w))));
      mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)), fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w))));
      mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(c.x, c.y), fmaxf(c.z, c.w)), fmaxf(fmaxf(d.x, d.y), fmaxf(d.z, d.w))));
    }
    for (; i < n4; i += stride) minmax4(mn, mx, ldg_stream(x4 + i));
    for (int64_t j = (n4 << 2) + start; j < n; j += stride) { const float v = x[j]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
  } else {
    for (int64_t j = start; j < n; j += stride) { const float v = x[j]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
  }
}

__global__ void k_init2(float* out2, int64_t pairs) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < pairs; i += (int64_t)gridDim.x * blockDim.x) {
    out2[2 * i] = DFQ_INF; out2[2 * i + 1] = -DFQ_INF;
  }
}

__global__ void __launch_bounds__(kThreads) k_minmax(const float* __restrict__ x, int64_t n, float* out2) {
  __shared__ float red[2 * kWarps];
  float mn = DFQ_INF, mx = -DFQ_INF;
  flat_minmax(x, n, blockIdx.x * (int64_t)kThreads + threadIdx.x, (int64_t)gridDim.x * kThreads, mn, mx);
  block_minmax<kThreads>(mn, mx, red);
  if (threadIdx.x == 0) { atomic_min_f(out2, mn); atomic_max_f(out2 + 1, mx); }
}

// x viewed as [batch, per]; blockIdx.y = sample, blockIdx.x = split of the sample.  scratch[2*b] pairs.
__global__ void __launch_bounds__(kThreads) k_sample_minmax(const float* __restrict__ x, int64_t per, float* scratch) {
  __shared__ float red[2 * kWarps];
  const float* xs = x + (int64_t)blockIdx.y * per;
  float mn = DFQ_INF, mx = -DFQ_INF;
  flat_minmax(xs, per, blockIdx.x * (int64_t)kThreads + threadIdx.x, (int64_t)gridDim.x * kThreads, mn, mx);
  block_minmax<kThreads>(mn, mx, red);
  if (threadIdx.x == 0) { atomic_min_f(scratch + 2 * blockIdx.y, mn); atomic_max_f(scratch + 2 * blockIdx.y + 1, mx); }
}

// mean over the batch of the per-sample extrema (quantize.py:106-107: .min(-1)[0].mean()); summed in
// float64 in sample order and rounded once to fp32.
__global__ void k_batch_mean(const float* __restrict__ scratch, int64_t batch, float* out2) {
  __shared__ double sm[2][32];
  double a = 0.0, b = 0.0;
  for (int64_t i = threadIdx.x; i < batch; i += blockDim.x) { a += (double)scratch[2 * i]; b += (double)scratch[2 * i + 1]; }
  a = warp_sum(a); b = warp_sum(b);
  if ((threadIdx.x & 31) == 0) { sm[0][threadIdx.x >> 5] = a; sm[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s0 = 0, s1 = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s0 += sm[0][i]; s1 += sm[1][i]; }
    out2[0] = (float)(s0 / (double)batch);
    out2[1] = (float)(s1 / (double)batch);
  }
}

__global__ void k_observer_update(float* rmin, float* rmax, const float* __restrict__ stat2, int mode, double momentum) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (mode == 1) {
      // Python min()/max() on 0-d tensors (quantize.py:106-107): the smaller / larger value
      rmin[0] = fminf(rmin[0], stat2[0]);
      rmax[0] = fmaxf(rmax[0], stat2[1]);
    } else {
      // running.mul_(1 - m).add_(value * m) (quantize.py:112-113), separately rounded; 1 - m is formed in double from the
      // Python float, like the reference's scalar
      const float om = (float)(1.0 - momentum), m = (float)momentum;
      rmin[0] = __fadd_rn(__fmul_rn(rmin[0], om), __fmul_rn(stat2[0], m));
      rmax[0] = __fadd_rn(__fmul_rn(rmax[0], om), __fmul_rn(stat2[1], m));
    }
  }
}

// Scalar prologue when min/max are fp32 0-d TENSORS in the reference (quantize.py:24-35 then :49-66 on
// tensors): the same formulas evaluated with fp32 tensor ops.  recip = a CUDA tensor divided by a
// Python scalar is a multiply by the fp32 reciprocal in PyTorch eager.
__device__ inline QuantScalars quant_scalars_f32(float mn, float mx, int num_bits, int symmetric, bool recip) {
  QuantScalars q;
  float scale;
  if (symmetric) {
    q.qmin = -ldexpf(1.0f, num_bits - 1);
    q.qmax = ldexpf(1.0f, num_bits - 1) - 1.0f;
    mx = fabsf(mx); mn = fabsf(mn);
    if (mx < mn) mx = mn;
    scale = recip ? __fmul_rn(mx, __frcp_rn(q.qmax)) : __fdiv_rn(mx, q.qmax);
    mn = 0.f;
  } else {
    q.qmin = 0.f;
    q.qmax = (float)(ldexp(1.0, num_bits) - 1.0);
    const float d = __fsub_rn(mx, mn);
    scale = recip ? __fmul_rn(d, __frcp_rn(q.qmax)) : __fdiv_rn(d, q.qmax);
  }
  if (1e-8f > scale) scale = 1e-8f;
  q.neg_min = -mn; q.min_v = mn; q.scale = scale; q.inv_scale = (float)(1.0 / (double)scale);
  return q;
}

template <bool RECIP, bool DEV_RANGE, bool ERR>
__global__ void __launch_bounds__(kThreads)
k_quant(const float* __restrict__ x, float* __restrict__ y, int64_t n, QuantScalars qs, const float* __restrict__ min_ptr,
        const float* __restrict__ max_ptr, int num_bits, int symmetric, int prologue, float* __restrict__ codes) {
  QuantScalars q = qs;
  if (DEV_RANGE) {
    if (prologue == 0) q = quant_scalars((double)min_ptr[0], (double)max_ptr[0], num_bits, symmetric);
    else q = quant_scalars_f32(min_ptr[0], max_ptr[0], num_bits, symmetric, prologue == 2);
  }
  const int64_t start = blockIdx.x * (int64_t)kThreads + threadIdx.x, stride = (int64_t)gridDim.x * kThreads;
  const bool al = ((((uintptr_t)x) | ((uintptr_t)y) | ((uintptr_t)codes)) & 15) == 0;
  if (al) {
    const int64_t n4 = n >> 2;
    for (int64_t i = start; i < n4; i += stride) {
      const float4 v = ldg_stream((const float4*)x + i);
      float4 c;
      float4 r = fake_quant4<RECIP>(v, q, &c);
      if (ERR) { r.x = __fsub_rn(r.x, v.x); r.y = __fsub_rn(r.y, v.y); r.z = __fsub_rn(r.z, v.z); r.w = __fsub_rn(r.w, v.w); }
      stg_stream((float4*)y + i, r);
      if (codes) stg_stream((float4*)codes + i, c);
    }
    for (int64_t j = (n4 << 2) + start; j < n; j += stride) {
      float c; float r = fake_quant<RECIP>(x[j], q, &c);
      if (ERR) r = __fsub_rn(r, x[j]);
      y[j] = r; if (codes) codes[j] = c;
    }
  } else {
    for (int64_t j = start; j < n; j += stride) {
      const float v = x[j];
      float c; float r = fake_quant<RECIP>(v, q, &c);
      if (ERR) r = __fsub_rn(r, v);
      y[j] = r; if (codes) codes[j] = c;
    }
  }
}


// ------------------------------------------------------------------------------------------------------------------
// Fused activation observer + fake quantization: ONE launch for QuantMeasure.forward (quantize.py:102-119) and for the
// per-forward weight / bias quantization of the Quant* / Q* layers (quantize.py:24-35,194-203).
//
//   phase 1  per-sample min/max of x viewed as [batch, per]: the (sample, split) work items are dealt to the CTAs of a
//            persistent cooperative grid; every item leaves one (min, max) pair in `scratch` (plain stores, no init)
//   -------- grid barrier ---------------------------------------------------------------------------------------
//   phase 2  EVERY CTA reduces the splits and takes the batch mean the same way (float64, sample order: bit-identical
//            everywhere), derives the running-statistics update and the quantization range from the OLD running values it
//            read before the barrier; block 0 alone writes the updated running_min / running_max back
//   phase 3  fake-quantize x -> y with that range (second read of x: an L2 hit for activation-sized tensors)
//
// flags: OBS_UPDATE  running = (min(running_min, stat_min), max(running_max, stat_max))        quantize.py:103-107
//        OBS_EMA     running = running*(1-m) + stat*m (after OBS_UPDATE), range = the batch stat quantize.py:109-113
//        OBS_OWN     no running buffers: range = the statistic itself (weights: batch 1 = per-tensor min/max)
//        otherwise   range = the (updated) running values                                        quantize.py:115-119
enum { OBS_UPDATE = 1, OBS_EMA = 2, OBS_OWN = 4 };

template <bool RECIP>
__global__ void __launch_bounds__(kThreads)
k_observe_quant(const float* __restrict__ x, float* __restrict__ y, int64_t batch, int64_t per, int splits,
                float* running_min, float* running_max, float* __restrict__ scratch, float* stat_out, int flags, double momentum,
                int num_bits, int symmetric, int prologue) {
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  __shared__ float red[2 * kWarps];
  __shared__ float s_range[2];
  // the running statistics as they are BEFORE this call (block 0 overwrites them after the barrier)
  float old_min = 0.f, old_max = 0.f;
  if (!(flags & OBS_OWN)) { old_min = __ldcg(running_min); old_max = __ldcg(running_max); }
  const int64_t chunk = (per + splits - 1) / splits;
  const int64_t items = batch * splits;
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int64_t b = it / splits, sp = it - b * splits;
    const int64_t lo = sp * chunk, hi = min(per, lo + chunk);
    float mn = DFQ_INF, mx = -DFQ_INF;
    if (hi > lo) flat_minmax(x + b * per + lo, hi - lo, threadIdx.x, kThreads, mn, mx);
    __syncthreads();
    block_minmax<kThreads>(mn, mx, red);
    if (threadIdx.x == 0) { __stcg(scratch + 2 * it, mn); __stcg(scratch + 2 * it + 1, mx); }
  }
  __threadfence();
  grid.sync();
  if (threadIdx.x < 32) {
    // batch mean of the per-sample extrema: float64, sample order, one rounding (as k_batch_mean); lanes over samples
    double a = 0.0, c = 0.0;
    for (int64_t b = threadIdx.x; b < batch; b += 32) {
      float mn = DFQ_INF, mx = -DFQ_INF;
      for (int sp = 0; sp < splits; ++sp) {
        mn = fminf(mn, __ldcg(scratch + 2 * (b * splits + sp))); mx = fmaxf(mx, __ldcg(scratch + 2 * (b * splits + sp) + 1));
      }
      a += (double)mn; c += (double)mx;
    }
    // fixed-shape tree over the 32 lanes: identical in every CTA
    a = warp_sum(a); c = warp_sum(c);
    if (threadIdx.x == 0) {
      const float st_min = (float)(a / (double)batch), st_max = (float)(c / (double)batch);
      float r_min = old_min, r_max = old_max, q_min, q_max;
      if (flags & OBS_OWN) { q_min = st_min; q_max = st_max; }
      else {
        if (flags & OBS_UPDATE) { r_min = fminf(r_min, st_min); r_max = fmaxf(r_max, st_max); }
        if (flags & OBS_EMA) {
          const float om = (float)(1.0 - momentum), m = (float)momentum;
          r_min = __fadd_rn(__fmul_rn(r_min, om), __fmul_rn(st_min, m));
          r_max = __fadd_rn(__fmul_rn(r_max, om), __fmul_rn(st_max, m));
          q_min = st_min; q_max = st_max;
        } else { q_min = r_min; q_max = r_max; }
        if (blockIdx.x == 0) { __stcg(running_min, r_min); __stcg(running_max, r_max); }
      }
      if (blockIdx.x == 0 && stat_out) { stat_out[0] = st_min; stat_out[1] = st_max; }
      s_range[0] = q_min; s_range[1] = q_max;
    }
  }
  __syncthreads();
  QuantScalars q;
  if (prologue == 0) q = quant_scalars((double)s_range[0], (double)s_range[1], num_bits, symmetric);
  else q = quant_scalars_f32(s_range[0], s_range[1], num_bits, symmetric, prologue == 2);
  const int64_t n = batch * per;
  const int64_t start = blockIdx.x * (int64_t)kThreads + threadIdx.x, stride = (int64_t)gridDim.x * kThreads;
  if (((((uintptr_t)x) | ((uintptr_t)y)) & 15) == 0) {
    const int64_t n4 = n >> 2;
    for (int64_t i = start; i < n4; i += stride) {
      stg_stream((float4*)y + i, fake_quant4<RECIP>(ldg_stream((const float4*)x + i), q));
    }
    for (int64_t j = (n4 << 2) + start; j < n; j += stride) y[j] = fake_quant<RECIP>(x[j], q);
  } else {
    for (int64_t j = start; j < n; j += stride) y[j] = fake_quant<RECIP>(x[j], q);
  }
}

// one warp per row (short rows) or one CTA per row
__global__ void __launch_bounds__(kThreads)
k_range_rows(const float* __restrict__ w, int64_t rows, int64_t row_len, float* out_min, float* out_max, int cta_row) {
  __shared__ float red[2 * kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (cta_row) {
    for (int64_t o = blockIdx.x; o < rows; o += gridDim.x) {
      float mn = DFQ_INF, mx = -DFQ_INF;
      flat_minmax(w + o * row_len, row_len, threadIdx.x, kThreads, mn, mx);
      __syncthreads();
      block_minmax<kThreads>(mn, mx, red);
      if (threadIdx.x == 0) { out_min[o] = mn; out_max[o] = mx; }
    }
  } else {
    for (int64_t o = blockIdx.x * (int64_t)kWarps + warp; o < rows; o += (int64_t)gridDim.x * kWarps) {
      float mn = DFQ_INF, mx = -DFQ_INF;
      flat_minmax(w + o * row_len, row_len, lane, 32, mn, mx);
      mn = warp_min(mn); mx = warp_max(mx);
      if (lane == 0) { out_min[o] = mn; out_max[o] = mx; }
    }
  }
}

// W[O, J, kk]; tile = 32 rows of one group; positions strided over the CTA; global float atomics
__global__ void __launch_bounds__(kThreads)
k_range_cols(const float* __restrict__ w, int64_t O, int64_t J, int64_t kk, int64_t groups, float* out_min, float* out_max) {
  const int64_t go = O / groups, row_len = J * kk;
  const int64_t nb = (go + 31) / 32, nt = groups * nb;
  for (int64_t t = blockIdx.x; t < nt; t += gridDim.x) {
    const int64_t g = t / nb, b = t - g * nb;
    const int64_t r0 = g * go + b * 32, r1 = min(r0 + 32, (g + 1) * go);
    for (int64_t p = threadIdx.x; p < row_len; p += kThreads) {
      float mn = DFQ_INF, mx = -DFQ_INF;
      const float* q = w + r0 * row_len + p;
#pragma unroll 8
      for (int64_t r = r0; r < r1; ++r, q += row_len) { const float v = ldg_stream1(q); mn = fminf(mn, v); mx = fmaxf(mx, v); }
      const int64_t j = p / kk;
      atomic_min_f(out_min + g * J + j, mn);
      atomic_max_f(out_max + g * J + j, mx);
    }
  }
}

__global__ void __launch_bounds__(kThreads)
k_abs_diff_sum(const float* __restrict__ a, const float* __restrict__ b, int64_t n, double inv_n, double* out) {
  __shared__ double sm[kWarps];
  double acc = 0.0;
  const int64_t start = blockIdx.x * (int64_t)kThreads + threadIdx.x, stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = start; i < n; i += stride) acc += (double)fabsf(__fsub_rn(a[i], b[i]));
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < kWarps; ++i) t += sm[i];
    atomicAdd(out, t * inv_n);
  }
}

__global__ void k_fill(float* p, int64_t n, float v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

__global__ void __launch_bounds__(kThreads) k_clamp(float* x, int64_t n, float lo, float hi) {
  const int64_t start = blockIdx.x * (int64_t)kThreads + threadIdx.x, stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = start; i < n; i += stride) x[i] = clamp_keep(x[i], lo, hi);
}

static int flat_grid(int64_t n, int per_thread) {
  const int64_t want = (n + (int64_t)kThreads * per_thread - 1) / ((int64_t)kThreads * per_thread);
  const int cap = std::max(1, sm_count()) * 8;
  return (int)std::max<int64_t>(1, std::min<int64_t>(want, cap));
}

}  // namespace dfq

using namespace dfq;

extern "C" int dfq_abi_version(void) { return DFQ_ABI_VERSION; }
extern "C" const char* dfq_last_error(void) { return g_err; }

extern "C" int dfq_device_info(int* sm, int* engine_ctas) {
  int dev = 0, sms = 0;
  DFQ_CUDA(cudaGetDevice(&dev));
  DFQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (sm) *sm = sms;
  if (engine_ctas) *engine_ctas = sms * 2;
  return 0;
}

extern "C" int dfq_struct_size(int which) {
  switch (which) {
    case 0: return (int)sizeof(DfqLayer);
    case 1: return (int)sizeof(DfqRelation);
    case 2: return (int)sizeof(DfqCleParams);
    case 3: return (int)sizeof(DfqCleResult);
    case 4: return (int)sizeof(DfqFold);
    case 5: return (int)sizeof(DfqExpectTerm);
    case 6: return (int)sizeof(DfqBcLayer);
    case 7: return (int)sizeof(DfqQuantTask);
    case 8: return (int)sizeof(DfqI8Conv);
    case 9: return (int)sizeof(DfqI8Epilogue);
    case 10: return (int)sizeof(DfqI8Pool);
    case 11: return (int)sizeof(DfqI8Resize);
    case 12: return (int)sizeof(DfqI8Affine);
    case 13: return (int)sizeof(DfqI8AffineEpilogue);
    case 14: return (int)sizeof(DfqI8AffineObserve);
    case 15: return (int)sizeof(DfqI8AffineLayout);
    case 16: return (int)sizeof(DfqI8AffineResize);
    case 17: return (int)sizeof(DfqI8AffineRows);
    case 18: return (int)sizeof(DfqSsdNms);
    case 19: return (int)sizeof(DfqSegArgmax);
    case 21: return (int)sizeof(DfqPreImage);
    case 22: return (int)sizeof(DfqPreResample);
    case 23: return (int)sizeof(DfqJpegImage);
    case 24: return (int)sizeof(DfqJpegSegment);
    case 25: return (int)sizeof(DfqJpegDecode);
    case 26: return (int)sizeof(DfqJpegHuff);
    case 27: return (int)sizeof(DfqJpegTables);
    case 28: return (int)sizeof(DfqAbsorb);
    case 29: return (int)sizeof(DfqPngImage);
    case 30: return (int)sizeof(DfqPngDecode);
    default: return -1;
  }
}

extern "C" int dfq_minmax(const float* x, int64_t n, float* out2, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && out2 && n > 0, "bad argument");
  k_init2<<<1, 32, 0, st>>>(out2, 1);
  k_minmax<<<flat_grid(n, kItemFloats), kThreads, 0, st>>>(x, n, out2);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_quant_dequant(const float* x, float* y, int64_t n, float min_value, double scale, float qmin,
                                 float qmax, int div_mode, float* codes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && y && n > 0, "bad argument");
  QuantScalars q;
  q.neg_min = -min_value; q.min_v = min_value; q.scale = (float)scale; q.inv_scale = (float)(1.0 / scale);
  q.qmin = qmin; q.qmax = qmax;
  const int grid = flat_grid(n, 8);
  if (div_mode) k_quant<true, false, false><<<grid, kThreads, 0, st>>>(x, y, n, q, nullptr, nullptr, 0, 0, 0, codes);
  else          k_quant<false, false, false><<<grid, kThreads, 0, st>>>(x, y, n, q, nullptr, nullptr, 0, 0, 0, codes);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_quant_dequant_dev(const float* x, float* y, int64_t n, const float* min_ptr, const float* max_ptr,
                                     int num_bits, int symmetric, int div_mode, int prologue, float* codes,
                                     void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && y && min_ptr && max_ptr && n > 0 && num_bits >= 1 && num_bits <= 32, "bad argument");
  DFQ_REQUIRE(prologue >= 0 && prologue <= 2, "prologue must be 0, 1 or 2");
  QuantScalars q{};
  const int grid = flat_grid(n, 8);
  // a tensor divisor (prologue 1/2) is always a true division in PyTorch, on CPU and on CUDA
  if (div_mode && prologue == 0)
    k_quant<true, true, false><<<grid, kThreads, 0, st>>>(x, y, n, q, min_ptr, max_ptr, num_bits, symmetric, prologue, codes);
  else
    k_quant<false, true, false><<<grid, kThreads, 0, st>>>(x, y, n, q, min_ptr, max_ptr, num_bits, symmetric, prologue, codes);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_quant_error(const float* w, float* eps, int64_t n, const float* minmax2, int num_bits, int symmetric,
                               void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(w && eps && minmax2 && n > 0, "bad argument");
  QuantScalars q{};
  k_quant<false, true, true><<<flat_grid(n, 8), kThreads, 0, st>>>(w, eps, n, q, minmax2, minmax2 + 1, num_bits, symmetric, 0, nullptr);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_act_minmax_per_sample(const float* x, int64_t batch, int64_t per_sample, float* out2,
                                         float* scratch_2b, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && out2 && scratch_2b && batch > 0 && per_sample > 0, "bad argument");
  DFQ_REQUIRE(batch <= 65535, "batch too large for one launch");
  k_init2<<<(int)std::min<int64_t>(64, (batch + 255) / 256), 256, 0, st>>>(scratch_2b, batch);
  const int sms = std::max(1, sm_count());
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>((per_sample + kThreads * kItemFloats - 1) / (kThreads * kItemFloats),
                                                           std::max<int64_t>(1, (int64_t)sms * 8 / batch)));
  k_sample_minmax<<<dim3(splits, (unsigned)batch), kThreads, 0, st>>>(x, per_sample, scratch_2b);
  k_batch_mean<<<1, 256, 0, st>>>(scratch_2b, batch, out2);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_observer_update(float* running_min, float* running_max, const float* stat2, int mode, double momentum,
                                   void* stream) {
  DFQ_REQUIRE(running_min && running_max && stat2 && (mode == 1 || mode == 2), "bad argument");
  k_observer_update<<<1, 32, 0, (cudaStream_t)stream>>>(running_min, running_max, stat2, mode, momentum);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}


extern "C" int dfq_observe_quant(const float* x, float* y, int64_t batch, int64_t per_sample, float* running_min,
                                 float* running_max, float* stat_out2, int flags, double momentum, int num_bits, int symmetric,
                                 int div_mode, int prologue, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(x && y && batch > 0 && per_sample > 0, "bad argument");
  DFQ_REQUIRE((flags & OBS_OWN) || (running_min && running_max), "running statistics required unless OBS_OWN");
  DFQ_REQUIRE((flags & (OBS_UPDATE | OBS_EMA | OBS_OWN)) != 0, "nothing to observe: use dfq_quant_dequant_dev");
  DFQ_REQUIRE(num_bits >= 1 && num_bits <= 32 && prologue >= 0 && prologue <= 2, "num_bits / prologue");
  static int per_sm_recip = 0, per_sm_div = 0;
  // a tensor divisor (prologue 1/2) is always a true division, as in dfq_quant_dequant_dev
  const bool recip = div_mode && prologue == 0;
  int& per_sm = recip ? per_sm_recip : per_sm_div;
  const void* fn = recip ? (const void*)k_observe_quant<true> : (const void*)k_observe_quant<false>;
  if (per_sm == 0) DFQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kThreads, 0));
  if (per_sm < 1) { set_error("k_observe_quant does not fit on an SM"); return DFQ_E_NOT_COOPERATIVE; }
  const int sms = std::max(1, sm_count());
  const int64_t n = batch * per_sample;
  // enough CTAs to fill the machine for big tensors, few for small ones (a grid barrier costs with the grid size)
  int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)sms * std::min(per_sm, 4), (n + (int64_t)kThreads * kItemFloats - 1) / ((int64_t)kThreads * kItemFloats)));
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>((per_sample + kThreads * kItemFloats - 1) / (kThreads * kItemFloats), std::max<int64_t>(1, grid / batch)));
  float* scratch = nullptr;
  DFQ_CUDA(cudaMallocAsync((void**)&scratch, sizeof(float) * 2 * (size_t)batch * splits, st));
  void* args[] = {(void*)&x, (void*)&y, (void*)&batch, (void*)&per_sample, (void*)&splits, (void*)&running_min, (void*)&running_max,
                  (void*)&scratch, (void*)&stat_out2, (void*)&flags, (void*)&momentum, (void*)&num_bits, (void*)&symmetric, (void*)&prologue};
  cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kThreads), args, 0, st);
  cudaFreeAsync(scratch, st);
  if (e != cudaSuccess) return cuda_fail(e, "cudaLaunchCooperativeKernel(k_observe_quant)");
  return 0;
}

extern "C" int dfq_range_rows(const float* w, int64_t rows, int64_t row_len, float* out_min, float* out_max, void* stream) {
  DFQ_REQUIRE(w && out_min && out_max && rows > 0 && row_len > 0, "bad argument");
  const int cta_row = row_len > kRangeCtaRow;
  const int64_t want = cta_row ? rows : (rows + kWarps - 1) / kWarps;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)std::max(1, sm_count()) * 8));
  k_range_rows<<<grid, kThreads, 0, (cudaStream_t)stream>>>(w, rows, row_len, out_min, out_max, cta_row);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_range_cols(const float* w, int64_t O, int64_t J, int64_t kk, int64_t groups, float* out_min,
                              float* out_max, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(w && out_min && out_max && O > 0 && J > 0 && kk > 0 && groups > 0 && O % groups == 0, "bad argument");
  const int64_t C = groups * J;
  k_fill<<<(int)std::min<int64_t>(std::max(1, sm_count()), (C + 255) / 256), 256, 0, st>>>(out_min, C, INFINITY);
  k_fill<<<(int)std::min<int64_t>(std::max(1, sm_count()), (C + 255) / 256), 256, 0, st>>>(out_max, C, -INFINITY);
  const int64_t nt = groups * ((O / groups + 31) / 32);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(nt, (int64_t)std::max(1, sm_count()) * 8));
  k_range_cols<<<grid, kThreads, 0, st>>>(w, O, J, kk, groups, out_min, out_max);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_mean_abs_diff(const float* a, const float* b, int64_t n, double* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DFQ_REQUIRE(a && b && out && n > 0, "bad argument");
  DFQ_CUDA(cudaMemsetAsync(out, 0, sizeof(double), st));
  k_abs_diff_sum<<<flat_grid(n, 8), kThreads, 0, st>>>(a, b, n, 1.0 / (double)n, out);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dfq_clamp(float* x, int64_t n, float lo, float hi, void* stream) {
  DFQ_REQUIRE(x && n > 0, "bad argument");
  k_clamp<<<flat_grid(n, 8), kThreads, 0, (cudaStream_t)stream>>>(x, n, lo, hi);
  DFQ_CUDA(cudaGetLastError());
  return 0;
}
