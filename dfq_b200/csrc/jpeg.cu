// JPEG decoding on the device, bit for bit as libjpeg-turbo decodes with its defaults (what Pillow and OpenCV run):
// baseline sequential Huffman streams, 8-bit, gray or YCbCr 4:4:4 / 4:2:2 / 4:2:0, one interleaved scan, any restart
// interval, for a batch of images of mixed sizes and samplings.
//
//   k_jpeg_huff    one thread per restart interval (the whole scan when the stream has none): it walks the bits of its
//                  segment - byte stuffing, the DC predictors from zero, the tables' 9-bit lookahead and libjpeg's
//                  maxcode walk for longer codes - and stores each block's int16 coefficients in natural order into a
//                  zeroed workspace.  Reads stay inside the segment (past its end the reader shifts in zeros, as libjpeg
//                  does, and counts them); an invalid code, a run past coefficient 63 or bits taken past the end stop
//                  the segment and are recorded in the error word.  A warp thus holds up to 32 independent walkers.
//   k_jpeg_idct    8 threads per block: dequantisation and the islow IDCT (CONST_BITS 13, PASS1_BITS 2, pass 1 down the
//                  columns into shared memory, pass 2 along the rows) with the arithmetic of libjpeg-turbo's SIMD
//                  jsimd_idct_islow: 16-bit dequantisation and lane sums, pass 1 saturated to int16 (or its 16-bit
//                  DC-only shortcut), the output saturated to 0 .. 255; one uint8 plane per component, padded to whole
//                  MCUs.
//   k_jpeg_color   one thread per output pixel: h2v1 / h2v2 "fancy" upsampling (the triangle filter, edges replicated
//                  at the downsampled width and height; plain replication when the chroma plane is at most 2 wide, as
//                  jinit_upsampler chooses), then ycc_rgb_convert's 16-bit fixed-point tables, written HWC RGB into
//                  the image's place in the blob, which dfq_pre_resample reads as it reads host-decoded pixels.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace dfq {
namespace {

constexpr int kSegThreads = 64;
constexpr int kIdctThreads = 256;          // 8 per block: 32 blocks per CTA
constexpr int kTileW = 32, kTileH = 8;

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Per image, formed by the entry from the descriptors: where its coefficients, planes, blocks and colour tiles start.
struct JpegWork {
  int64_t coef;                  // int16 elements into the coefficient workspace
  int64_t plane[3];              // bytes into the plane workspace
  int64_t block0, tile0;         // first global block (k_jpeg_idct) and colour tile (k_jpeg_color)
  int32_t pw[3];                 // plane widths
  int32_t _pad;
};

__device__ __forceinline__ int ny_of(const DfqJpegImage& im) { return im.ncomp == 3 ? im.hs * im.vs : 1; }
__device__ __forceinline__ int bpm_of(const DfqJpegImage& im) { return ny_of(im) + (im.ncomp == 3 ? 2 : 0); }

// The largest i < n with key(i) <= v: the image a global block or tile belongs to.
template <typename F>
__device__ __forceinline__ int owner(int n, int64_t v, F key) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (key(mid) <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- entropy decoding ----------------------------------------------------------------------------------------------------
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t buf = 0;              // next bits, MSB first
  int cnt = 0;                   // valid bits in buf
  int pad = 0;                   // zero bytes shifted in past the end
  __device__ __forceinline__ void fill() {
    while (cnt <= 56) {
      uint32_t b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF && p < end) ++p;                 // FF 00: a stuffed FF
      } else {
        ++pad;
      }
      buf |= (uint64_t)b << (56 - cnt);
      cnt += 8;
    }
  }
  __device__ __forceinline__ void skip(int n) { buf <<= n; cnt -= n; }
  __device__ __forceinline__ int bits(int n) {
    const int v = n ? (int)(buf >> (64 - n)) : 0;
    skip(n);
    return v;
  }
};

// HUFF_DECODE: the 9-bit lookahead, then the maxcode walk over lengths 10 .. 16.  -1 for an invalid code.
__device__ __forceinline__ int huff_decode(BitReader& br, const DfqJpegHuff& h) {
  const uint32_t pk = (uint32_t)(br.buf >> 48);
  const uint32_t e = h.look[pk >> 7];
  if (e) {
    br.skip(e >> 8);
    return e & 255;
  }
  for (int l = 10; l <= 16; ++l) {
    const int code = pk >> (16 - l);
    if (code <= h.maxcode[l]) {
      br.skip(l);
      const int i = code + h.valoff[l];
      return i >= 0 && i < 256 ? h.vals[i] : -1;
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

__global__ void __launch_bounds__(kSegThreads) k_jpeg_huff(const DfqJpegSegment* __restrict__ segs, int nseg,
                                                           const DfqJpegImage* __restrict__ ims,
                                                           const JpegWork* __restrict__ work,
                                                           const uint8_t* __restrict__ blob, int16_t* __restrict__ coef,
                                                           unsigned long long* err, unsigned long long call) {
  const int s = blockIdx.x * kSegThreads + threadIdx.x;
  if (s >= nseg) return;
  const DfqJpegSegment sg = segs[s];
  const DfqJpegImage im = ims[sg.image];
  const DfqJpegTables* T = (const DfqJpegTables*)(blob + im.tables);
  BitReader br{blob + sg.begin, blob + sg.end};
  const int ny = ny_of(im), bpm = bpm_of(im);
  int16_t* out = coef + work[sg.image].coef + (int64_t)sg.mcu0 * bpm * 64;
  int pred0 = 0, pred1 = 0, pred2 = 0;                             // scalars, not an array: no local memory
  int fail = 0;
  for (int m = 0; m < sg.mcus && !fail; ++m) {
    for (int b = 0; b < bpm; ++b, out += 64) {
      const int c = b < ny ? 0 : b - ny + 1;
      br.fill();
      const int t = huff_decode(br, T->dc[c]);
      if (t < 0 || t > 15) { fail = DFQ_JPEG_BAD_CODE; break; }
      int& pred = c == 0 ? pred0 : c == 1 ? pred1 : pred2;
      pred = (int)((unsigned)pred + (unsigned)(t ? extend(br.bits(t), t) : 0));      // libjpeg's wrapping sum
      out[0] = (int16_t)pred;
      for (int k = 1; k < 64; ++k) {
        br.fill();
        const int rs = huff_decode(br, T->ac[c]);
        if (rs < 0) { fail = DFQ_JPEG_BAD_CODE; break; }
        const int r = rs >> 4, sz = rs & 15;
        if (sz) {
          k += r;
          if (k > 63) { fail = DFQ_JPEG_BAD_RUN; break; }
          out[kZigzag[k]] = (int16_t)extend(br.bits(sz), sz);
        } else {
          if (r != 15) break;                          // EOB
          k += 15;                                     // ZRL
        }
      }
      if (!fail && br.pad > 8) fail = DFQ_JPEG_SHORT_SCAN;   // every buffered bit is past the end
      if (fail) break;
    }
  }
  if (!fail && br.pad * 8 > br.cnt) fail = DFQ_JPEG_SHORT_SCAN;   // bits were taken past the end
  if (fail) {
    atomicMin(err, (call << 32) | (unsigned long long)sg.image);
    atomicOr(err + 1, (unsigned long long)fail);
  }
}

// ---- jsimd_idct_islow -------------------------------------------------------------------------------------------------------
// libjpeg-turbo's SIMD islow IDCT (what Pillow and OpenCV run on x86), not the C jidctint.c: the arithmetic of its 16-bit
// lanes is part of the output once a block reconstructs outside 0 .. 255.
constexpr int F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633, F1_501 = 12299,
              F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;

__device__ __forceinline__ int lo16(int v) { return (int)(int16_t)(uint16_t)(unsigned)v; }     // a 16-bit lane's wrap
__device__ __forceinline__ unsigned mul(int a, int c) { return (unsigned)a * (unsigned)c; }

// One 1-D pass on the int16 values x[0..7] (index = frequency), results before the descale in o[0..7] (index = position),
// modulo 2^32 as the lanes form them: x0 + x4, x0 - x4, x7 + x3 and x5 + x1 wrap in 16 bits (paddw / psubw), every other
// sum is taken in 32 bits from pmaddwd products with the constant pairs below.
__device__ __forceinline__ void idct_1d(const int* x, unsigned* o) {
  const unsigned tmp3 = mul(x[2], F0_541 + F0_765) + mul(x[6], F0_541);
  const unsigned tmp2 = mul(x[2], F0_541) + mul(x[6], F0_541 - F1_847);
  const unsigned tmp0 = mul(lo16(x[0] + x[4]), 8192), tmp1 = mul(lo16(x[0] - x[4]), 8192);   // << CONST_BITS
  const unsigned t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  const int z3 = lo16(x[7] + x[3]), z4 = lo16(x[5] + x[1]);
  const unsigned y3 = mul(z3, F1_175 - F1_961) + mul(z4, F1_175), y4 = mul(z3, F1_175) + mul(z4, F1_175 - F0_390);
  const unsigned a0 = mul(x[7], F0_298 - F0_899) + mul(x[1], -F0_899) + y3;
  const unsigned a3 = mul(x[7], -F0_899) + mul(x[1], F1_501 - F0_899) + y4;
  const unsigned a1 = mul(x[5], F2_053 - F2_562) + mul(x[3], -F2_562) + y4;
  const unsigned a2 = mul(x[5], -F2_562) + mul(x[3], F3_072 - F2_562) + y3;
  o[0] = t10 + a3; o[7] = t10 - a3; o[1] = t11 + a2; o[6] = t11 - a2;
  o[2] = t12 + a1; o[5] = t12 - a1; o[3] = t13 + a0; o[4] = t13 - a0;
}

// DESCALE(, n) as paddd + psrad: the rounding constant added modulo 2^32, then an arithmetic shift.
__device__ __forceinline__ int descale(unsigned v, int n) { return (int)(v + (1u << (n - 1))) >> n; }

// The output limit: packssdw + packsswb saturate to -128 .. 127, then paddb adds CENTERJSAMPLE.
__device__ __forceinline__ uint32_t idct_limit(int v) { return (uint32_t)(min(max(v, -128), 127) + 128); }

__global__ void __launch_bounds__(kIdctThreads) k_jpeg_idct(const DfqJpegImage* __restrict__ ims,
                                                            const JpegWork* __restrict__ work, int n, int64_t nblocks,
                                                            const uint8_t* __restrict__ blob,
                                                            const int16_t* __restrict__ coef, uint8_t* __restrict__ planes) {
  __shared__ int ws[kIdctThreads / 8][64];
  const int64_t blk = ((int64_t)blockIdx.x * kIdctThreads + threadIdx.x) >> 3;
  const int t = threadIdx.x & 7, lb = threadIdx.x >> 3;
  const bool live = blk < nblocks;
  int i = 0, comp = 0;
  int64_t b = 0, bx = 0, by = 0;
  int x[8];
  unsigned o[8];
  bool ac = false;
  if (live) {
    i = owner(n, blk, [&](int k) { return work[k].block0; });
    const DfqJpegImage& im = ims[i];
    b = blk - work[i].block0;
    const int ny = ny_of(im), bpm = bpm_of(im);
    const int64_t m = b / bpm;
    const int r = (int)(b % bpm);
    const int64_t mx = m % im.mcux, my = m / im.mcux;
    if (r < ny) {
      bx = mx * (ny == 1 ? 1 : im.hs) + r % im.hs;
      by = my * (ny == 1 ? 1 : im.vs) + r / im.hs;
    } else {
      comp = r - ny + 1;
      bx = mx;
      by = my;
    }
    const int32_t* q = ((const DfqJpegTables*)(blob + im.tables))->q[comp];
    const int16_t* cb = coef + work[i].coef + b * 64;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      x[k] = lo16((int)cb[k * 8 + t] * q[k * 8 + t]);              // DEQUANTIZE: pmullw keeps the low 16 bits
      ac |= k > 0 && cb[k * 8 + t] != 0;
    }
  }
  // Pass 1's shortcut is taken per block, when the coefficients of rows 1 .. 7 are all zero (its 8 threads' votes).
  const bool dc_only = ((__ballot_sync(0xffffffffu, ac) >> (threadIdx.x & 24)) & 0xFF) == 0;
  if (live) {
    if (dc_only) {
#pragma unroll
      for (int k = 0; k < 8; ++k) ws[lb][k * 8 + t] = lo16(x[0] * 4);                 // psllw by PASS1_BITS
    } else {
      idct_1d(x, o);
#pragma unroll
      for (int k = 0; k < 8; ++k) ws[lb][k * 8 + t] = min(max(descale(o[k], 11), -32768), 32767);   // packssdw
    }
  }
  __syncwarp();                                                   // a block's 8 threads share a warp
  if (!live) return;
#pragma unroll
  for (int k = 0; k < 8; ++k) x[k] = ws[lb][t * 8 + k];
  idct_1d(x, o);
  uint32_t lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    lo |= idct_limit(descale(o[k], 18)) << (8 * k);               // DESCALE(, CONST_BITS + PASS1_BITS + 3)
    hi |= idct_limit(descale(o[k + 4], 18)) << (8 * k);
  }
  uint8_t* dst = planes + work[i].plane[comp] + (by * 8 + t) * work[i].pw[comp] + bx * 8;
  *(uint2*)dst = make_uint2(lo, hi);
}

// ---- upsampling and colour conversion ---------------------------------------------------------------------------------------
// The chroma sample of output pixel (x, y) as libjpeg-turbo's upsampler gives it; p is the plane, pw its width.
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ p, int pw, int x, int y, const DfqJpegImage& im) {
  if (im.hs == 1) return p[(int64_t)y * pw + x];
  const int dw = (im.W + 1) >> 1, ci = x >> 1;
  const int cy = im.vs == 2 ? y >> 1 : y;
  const uint8_t* row = p + (int64_t)cy * pw;
  if (dw <= 2) return row[ci];                                   // h2v1_upsample / h2v2_upsample
  const int cn = (x & 1) ? min(ci + 1, dw - 1) : max(ci - 1, 0);
  if (im.vs == 1) return (x & 1) ? (3 * row[ci] + row[cn] + 2) >> 2 : (3 * row[ci] + row[cn] + 1) >> 2;
  const int dh = (im.H + 1) >> 1;
  const uint8_t* near = p + (int64_t)((y & 1) ? min(cy + 1, dh - 1) : max(cy - 1, 0)) * pw;
  const int cs = 3 * row[ci] + near[ci], cs2 = 3 * row[cn] + near[cn];
  return (x & 1) ? (3 * cs + cs2 + 7) >> 4 : (3 * cs + cs2 + 8) >> 4;
}

__global__ void __launch_bounds__(kTileW * kTileH) k_jpeg_color(const DfqJpegImage* __restrict__ ims,
                                                                const JpegWork* __restrict__ work, int n,
                                                                const uint8_t* __restrict__ planes, uint8_t* __restrict__ blob) {
  const int i = owner(n, blockIdx.x, [&](int k) { return work[k].tile0; });
  const DfqJpegImage im = ims[i];
  const JpegWork& w = work[i];
  const int64_t tile = blockIdx.x - w.tile0;
  const int tiles_x = (im.W + kTileW - 1) / kTileW;
  const int x = (int)(tile % tiles_x) * kTileW + threadIdx.x % kTileW, y = (int)(tile / tiles_x) * kTileH + threadIdx.x / kTileW;
  if (x >= im.W || y >= im.H) return;
  const int Y = planes[w.plane[0] + (int64_t)y * w.pw[0] + x];
  uint8_t* o = blob + im.dst + ((int64_t)y * im.W + x) * 3;
  if (im.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int cb = chroma(planes + w.plane[1], w.pw[1], x, y, im) - 128;
  const int cr = chroma(planes + w.plane[2], w.pw[2], x, y, im) - 128;
  // build_ycc_rgb_table: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414) at SCALEBITS 16, ONE_HALF rounding
  const int r = Y + ((91881 * cr + 32768) >> 16);
  const int g = Y + ((-22554 * cb + 32768 + -46802 * cr) >> 16);
  const int bl = Y + ((116130 * cb + 32768) >> 16);
  o[0] = (uint8_t)min(max(r, 0), 255);
  o[1] = (uint8_t)min(max(g, 0), 255);
  o[2] = (uint8_t)min(max(bl, 0), 255);
}

bool in_blob(int64_t off, int64_t bytes, int64_t align, int64_t blob) {
  return off >= 0 && off % align == 0 && bytes >= 0 && bytes <= blob - off;
}

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_jpeg_decode(const DfqJpegDecode* d, const DfqJpegImage* images, const DfqJpegSegment* segs, void* blob,
                               uint64_t* error, void* stream) {
  if (!d || !images || !segs || !blob || !error) {
    set_error("dfq_jpeg_decode: d, images, segs, blob and error must be non-NULL");
    return DFQ_E_ARG;
  }
  if (d->n < 1 || d->n > 65535 || d->nseg < 1 || d->blob_bytes < 1 || d->call >= (1ull << 31)) {
    set_error("dfq_jpeg_decode: n must be in 1 .. 65535, nseg and blob_bytes at least 1, call below 2^31 (n %d, nseg %d, "
              "blob %lld)", d->n, d->nseg, (long long)d->blob_bytes);
    return DFQ_E_ARG;
  }
  if ((uintptr_t)blob % 8 || (uintptr_t)error % 8) {
    set_error("dfq_jpeg_decode: blob and error must be 8-byte aligned");
    return DFQ_E_ARG;
  }
  const int64_t B = d->blob_bytes;
  std::vector<JpegWork> work(d->n);
  std::vector<int64_t> next(d->n, 0);
  int64_t coefs = 0, plane_bytes = 0, blocks = 0, tiles = 0;
  for (int i = 0; i < d->n; ++i) {
    const DfqJpegImage& m = images[i];
    const bool geo = m.H >= 1 && m.W >= 1 && m.H <= 65535 && m.W <= 65535 &&
                     (m.ncomp == 1 ? m.hs == 1 && m.vs == 1
                                   : m.ncomp == 3 && ((m.hs == 1 && m.vs == 1) || (m.hs == 2 && (m.vs == 1 || m.vs == 2)))) &&
                     m.mcux == (m.W + 8 * m.hs - 1) / (8 * m.hs) && m.mcuy == (m.H + 8 * m.vs - 1) / (8 * m.vs);
    if (!geo || !in_blob(m.tables, sizeof(DfqJpegTables), 8, B) || !in_blob(m.dst, (int64_t)m.H * m.W * 3, 1, B)) {
      set_error("dfq_jpeg_decode: image %d: %d x %d, %d components, sampling %dx%d, %d x %d MCUs: unsupported or "
                "inconsistent geometry, or its tables or output outside the %lld-byte blob or misaligned", i, m.H, m.W,
                m.ncomp, m.hs, m.vs, m.mcux, m.mcuy, (long long)B);
      return DFQ_E_ARG;
    }
    JpegWork& w = work[i];
    const int64_t mcus = (int64_t)m.mcux * m.mcuy, ny = m.ncomp == 3 ? m.hs * m.vs : 1;
    w.coef = coefs;
    w.block0 = blocks;
    w.tile0 = tiles;
    w.pw[0] = m.mcux * 8 * m.hs;
    w.plane[0] = plane_bytes;
    plane_bytes += (int64_t)w.pw[0] * m.mcuy * 8 * m.vs;
    for (int c = 1; c < 3; ++c) {
      w.pw[c] = m.ncomp == 3 ? m.mcux * 8 : 0;
      w.plane[c] = plane_bytes;
      plane_bytes += (int64_t)w.pw[c] * m.mcuy * 8;
    }
    const int64_t nb = mcus * (ny + (m.ncomp == 3 ? 2 : 0));
    blocks += nb;
    coefs += nb * 64;
    tiles += (int64_t)((m.W + kTileW - 1) / kTileW) * ((m.H + kTileH - 1) / kTileH);
  }
  for (int s = 0; s < d->nseg; ++s) {
    const DfqJpegSegment& g = segs[s];
    const bool ok = g.image >= 0 && g.image < d->n && g.begin >= 0 && g.begin <= g.end && g.end <= B && g.mcus >= 1 &&
                    g.mcu0 == next[g.image] &&
                    g.mcus <= (int64_t)images[g.image].mcux * images[g.image].mcuy - g.mcu0;
    if (!ok) {
      set_error("dfq_jpeg_decode: segment %d (image %d, bytes %lld .. %lld, MCUs %d + %d): outside the blob, or not the "
                "next MCUs of its image", s, g.image, (long long)g.begin, (long long)g.end, g.mcu0, g.mcus);
      return DFQ_E_ARG;
    }
    next[g.image] += g.mcus;
  }
  for (int i = 0; i < d->n; ++i)
    if (next[i] != (int64_t)images[i].mcux * images[i].mcuy) {
      set_error("dfq_jpeg_decode: the segments of image %d cover %lld of its %lld MCUs", i, (long long)next[i],
                (long long)images[i].mcux * images[i].mcuy);
      return DFQ_E_ARG;
    }
  if (tiles > INT32_MAX) {
    set_error("dfq_jpeg_decode: %lld colour tiles: above 2^31 - 1", (long long)tiles);
    return DFQ_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int16_t* coef = nullptr;
  uint8_t* planes = nullptr;
  DFQ_CUDA(cudaMallocAsync((void**)&coef, coefs * sizeof(int16_t), st));
  DFQ_CUDA(cudaMallocAsync((void**)&planes, plane_bytes, st));
  DFQ_CUDA(cudaMemsetAsync(coef, 0, coefs * sizeof(int16_t), st));
  TablePack tp;
  const int iI = tp.add(images, d->n), iS = tp.add(segs, d->nseg), iW = tp.add(work.data(), d->n);
  if (int rc = tp.upload(st)) return rc;
  const DfqJpegImage* dim = tp.ptr<DfqJpegImage>(iI);
  const JpegWork* dw = tp.ptr<JpegWork>(iW);
  k_jpeg_huff<<<(d->nseg + kSegThreads - 1) / kSegThreads, kSegThreads, 0, st>>>(
      tp.ptr<DfqJpegSegment>(iS), d->nseg, dim, dw, (const uint8_t*)blob, coef, (unsigned long long*)error, d->call);
  k_jpeg_idct<<<(unsigned)((blocks * 8 + kIdctThreads - 1) / kIdctThreads), kIdctThreads, 0, st>>>(
      dim, dw, d->n, blocks, (const uint8_t*)blob, coef, planes);
  k_jpeg_color<<<(unsigned)tiles, kTileW * kTileH, 0, st>>>(dim, dw, d->n, planes, (uint8_t*)blob);
  DFQ_CUDA(cudaGetLastError());
  tp.release(st);
  cudaFreeAsync(coef, st);
  cudaFreeAsync(planes, st);
  return 0;
}
