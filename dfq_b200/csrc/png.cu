// PNG label decoding on the device, bit for bit as Pillow's Image.open reads 8-bit palette and gray streams: zlib's
// inflate, fed by Pillow one scanline at a time, then Pillow's scanline filters (one byte per pixel).
//
//   k_png_inflate   one warp per image.  All 32 lanes hold the same 64-bit bit buffer and decode the same symbol, so
//                   control flow stays uniform; the warp builds each block's code tables in shared memory (a 9-bit
//                   lookahead, the canonical walk for longer codes) with zlib's checks on the code sets, lanes copy
//                   stored blocks in parallel, lane 0 writes literals, and a match of length L at distance D is written
//                   by the whole warp: lane l writes bytes i = l, l + 32, ... from out[p - D + i mod D], which were all
//                   written before the match, so overlapping matches (D < L) need no serial loop.  The filtered
//                   scanlines go to the image's work room.  Once the image is full, the stream is read on up to the first
//                   symbol that would write, as zlib reads it with no output room left: block headers, code sets,
//                   end-of-block codes and a length's distance code are still checked, and the Adler-32 after the final
//                   block is compared (the warp sums it as per-lane partial sums).
//   k_png_unfilter  one warp per image, rows in order: None and Up across lanes, Sub as a mod-256 warp prefix scan,
//                   Average and Paeth (a serial dependency along the row) by one lane; written to dst, where
//                   dfq_pre_resample reads a label.  The work room stays intact: distances refer to filtered bytes.
#include "common.cuh"

namespace dfq {
namespace {

constexpr int kLook = 9;                                  // lookahead bits
constexpr unsigned kFull = 0xffffffffu;

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// One code: look[bits] = (length << 9 | symbol) for codes of up to kLook bits, 0 otherwise; count[] and the symbols in
// canonical order (sym[]) for the walk over longer codes.
struct Huff {
  uint16_t look[1 << kLook];
  uint16_t sym[288];
  int count[16];
  int start[16], next[16], first[16];
  int maxlen;
};

// Builds h from lens[0 .. n) (warp-collective).  0, or -1 for an over-subscribed set, or an incomplete one unless
// `single` and it is one code of one bit (or, for distances, no code at all), as zlib's inflate_table decides.
__device__ int build(Huff& h, const uint8_t* lens, int n, bool single, int lane) {
  if (lane < 16) h.count[lane] = 0;
  for (int i = lane; i < (1 << kLook) / 2; i += 32) ((uint32_t*)h.look)[i] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32)
    if (lens[s]) atomicAdd(&h.count[lens[s]], 1);
  __syncwarp();
  int left = 1, maxlen = 0;
  for (int l = 1; l < 16; ++l) {
    left = (left << 1) - h.count[l];
    if (left < 0) break;
    if (h.count[l]) maxlen = l;
  }
  if (lane == 0) h.maxlen = maxlen;                     // decode() reads it even for a set with no code
  __syncwarp();
  if (left < 0) return -1;
  if (maxlen == 0) return single ? 0 : -1;
  if (left > 0 && !(single && maxlen == 1)) return -1;
  if (lane == 0) {
    int code = 0, off = 0;
    for (int l = 1; l < 16; ++l) {
      code = (code + h.count[l - 1] * (l > 1)) << 1;
      h.first[l] = code;
      h.start[l] = h.next[l] = off;
      off += h.count[l];
    }
  }
  __syncwarp();
  const unsigned lt = (1u << lane) - 1;
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const int l = s < n ? lens[s] : 0;
    const unsigned same = __match_any_sync(kFull, l);
    const int rank = __popc(same & lt);
    if (l) {
      const int pos = h.next[l] + rank;
      h.sym[pos] = (uint16_t)s;
      if (l <= kLook) {
        const unsigned rev = __brev((unsigned)(h.first[l] + pos - h.start[l])) >> (32 - l);
        for (unsigned k = rev; k < (1u << kLook); k += 1u << l) h.look[k] = (uint16_t)(l << 9 | s);
      }
    }
    __syncwarp();
    if (l && rank == 0) h.next[l] += __popc(same);
    __syncwarp();
  }
  return 0;
}

// The next symbol of bb (LSB first); *used its length, or the code's longest length with -1 for an invalid code.
__device__ __forceinline__ int decode(const Huff& h, uint64_t bb, int* used) {
  const int e = h.look[bb & ((1 << kLook) - 1)];
  if (e) {
    *used = e >> 9;
    return e & 511;
  }
  int code = 0, first = 0, index = 0;                     // puff's canonical walk
  for (int len = 1; len < 16; ++len) {
    code |= (int)(bb >> (len - 1)) & 1;
    const int count = h.count[len];
    if (code - count < first) {
      *used = len;
      return h.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  *used = max(h.maxlen, 1);
  return -1;
}

// The stream's bits, LSB first.  ip runs on past iend, where zero bytes are shifted in; over() says bits were taken
// from them.
struct Bits {
  const uint8_t* blob;
  int64_t ip, iend;
  uint64_t bb;
  int bc;
  __device__ __forceinline__ void fill() {
    while (bc <= 56) {
      const uint64_t b = ip < iend ? blob[ip] : 0;
      ++ip;
      bb |= b << bc;
      bc += 8;
    }
  }
  __device__ __forceinline__ unsigned take(int n) {
    const unsigned v = (unsigned)(bb & ((1ull << n) - 1));
    bb >>= n;
    bc -= n;
    return v;
  }
  __device__ __forceinline__ int64_t real() const { return (int64_t)bc - 8 * max(ip - iend, (int64_t)0); }
  __device__ __forceinline__ bool over() const { return real() < 0; }
  __device__ __forceinline__ int64_t byte_pos() {           // drop to a byte boundary: the next unread byte
    take(bc & 7);
    return ip - bc / 8;
  }
};

enum { kEnd = 0, kFullStop = 1, kOut = 2 };               // the final block ended; a symbol would write; input ran out

__device__ __forceinline__ void report(unsigned long long* err, unsigned long long call, int image, int why) {
  atomicMin(err, (call << 32) | (unsigned long long)image);
  atomicOr(err + 1, (unsigned long long)why);
}

__global__ void __launch_bounds__(32) k_png_inflate(const DfqPngImage* __restrict__ ims, uint8_t* blob,
                                                    unsigned long long* err, unsigned long long call) {
  __shared__ Huff lit, dist;
  __shared__ uint8_t lens[320];
  const int lane = threadIdx.x, img = blockIdx.x;
  const DfqPngImage im = ims[img];
  const int64_t T = (int64_t)im.H * (im.W + 1);
  uint8_t* out = blob + im.work;               // read back by other lanes: coherent loads
  Bits r{blob, im.src + 2, im.src_end, 0, 0};
  int64_t pos = 0;
  int fail = 0, status = kEnd;
  bool fixed = false;
  for (bool final = false; !final && !fail;) {
    r.fill();
    final = r.take(1);
    const int type = r.take(2);
    if (r.over()) { status = kOut; break; }
    if (type == 0) {
      int64_t q = r.byte_pos();
      if (q + 4 > im.src_end) { status = kOut; break; }
      const int len = blob[q] | blob[q + 1] << 8, nlen = blob[q + 2] | blob[q + 3] << 8;
      if (len != (~nlen & 0xFFFF)) { fail = DFQ_PNG_STORED_LEN; break; }
      q += 4;
      const int64_t avail = min((int64_t)len, im.src_end - q), w = min(avail, T - pos);
      for (int64_t i = lane; i < w; i += 32) out[pos + i] = blob[q + i];
      pos += w;
      r.ip = q + len;
      r.bb = 0;
      r.bc = 0;
      __syncwarp();
      if (w < len) { status = pos == T ? kFullStop : kOut; break; }
      continue;
    }
    if (type == 3) { fail = DFQ_PNG_BAD_BLOCK; break; }
    if (type == 1) {
      if (!fixed) {
        for (int s = lane; s < 320; s += 32) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
        __syncwarp();
        build(lit, lens, 288, false, lane);
        build(dist, lens + 288, 32, false, lane);
        fixed = true;
      }
    } else {
      fixed = false;
      r.fill();
      const int hlit = r.take(5) + 257, hdist = r.take(5) + 1, hclen = r.take(4) + 4;
      if (r.over()) { status = kOut; break; }
      if (hlit > 286 || hdist > 30) { fail = DFQ_PNG_BAD_CODESET; break; }
      if (lane < 19) lens[lane] = 0;
      __syncwarp();
      for (int k = 0; k < hclen; ++k) {
        r.fill();
        const int v = r.take(3);
        if (lane == 0) lens[kClOrder[k]] = (uint8_t)v;
      }
      if (r.over()) { status = kOut; break; }
      __syncwarp();
      if (build(dist, lens, 19, false, lane)) { fail = DFQ_PNG_BAD_CODESET; break; }
      __syncwarp();
      int i = 0, prev = 0;
      const int total = hlit + hdist;
      while (i < total) {
        r.fill();
        int used;
        const int s = decode(dist, r.bb, &used);
        if (s < 0) {
          if (r.real() < used) status = kOut; else fail = DFQ_PNG_BAD_CODESET;
          break;
        }
        r.take(used);
        int rep = 1, v = s;
        if (s == 16) {
          if (i == 0) { fail = DFQ_PNG_BAD_CODESET; break; }
          rep = 3 + r.take(2);
          v = prev;
        } else if (s == 17) {
          rep = 3 + r.take(3);
          v = 0;
        } else if (s == 18) {
          rep = 11 + r.take(7);
          v = 0;
        }
        if (r.over()) { status = kOut; break; }
        if (i + rep > total) { fail = DFQ_PNG_BAD_CODESET; break; }
        __syncwarp();                                      // the code-length table is read above, lens written below
        for (int k = lane; k < rep; k += 32) lens[i + k] = (uint8_t)v;
        i += rep;
        prev = v;
      }
      if (fail || status == kOut) break;
      __syncwarp();
      if (lens[256] == 0 || build(lit, lens, hlit, true, lane) || build(dist, lens + hlit, hdist, true, lane)) {
        fail = DFQ_PNG_BAD_CODESET;
        break;
      }
    }
    __syncwarp();
    for (;;) {
      r.fill();
      int used;
      int s = decode(lit, r.bb, &used);
      if (s < 0) {
        if (r.real() < used) status = kOut; else fail = DFQ_PNG_BAD_CODE;
        break;
      }
      r.take(used);
      if (r.over()) { status = kOut; break; }
      if (s < 256) {
        if (pos == T) { status = kFullStop; break; }
        if (lane == 0) out[pos] = (uint8_t)s;
        ++pos;
        continue;
      }
      if (s == 256) break;
      if (s >= 286) { fail = DFQ_PNG_BAD_CODE; break; }
      s -= 257;
      const int L = kLenBase[s] + r.take(kLenExtra[s]);
      if (r.over()) { status = kOut; break; }
      const int ds = decode(dist, r.bb, &used);
      if (ds < 0) {
        if (r.real() < used) status = kOut; else fail = DFQ_PNG_BAD_CODE;
        break;
      }
      r.take(used);
      if (r.over()) { status = kOut; break; }
      if (ds >= 30) { fail = DFQ_PNG_BAD_CODE; break; }
      const int D = kDistBase[ds] + r.take(kDistExtra[ds]);
      if (r.over()) { status = kOut; break; }
      if (pos == T) { status = kFullStop; break; }
      if (D > pos) { fail = DFQ_PNG_FAR; break; }
      const int w = (int)min((int64_t)L, T - pos);
      uint8_t* dst = out + pos;
      const uint8_t* src = dst - D;
      __syncwarp();                                        // lane 0's literals are read below
      for (int k = lane; k < w; k += 32) dst[k] = src[D >= w ? k : k % D];
      pos += w;
      __syncwarp();
      if (w < L) { status = kFullStop; break; }           // zlib leaves with the rest of the match pending
    }
    if (status != kEnd) break;
  }
  // The final block ended: with the image, or at the end of an earlier row (Pillow then keeps the rows that came and
  // leaves the others zero, when the whole trailer is there).  Anywhere else the stream is short.
  const bool rows_end = status == kEnd && pos > 0 && pos % (im.W + 1) == 0;
  if (!fail && pos < T && !rows_end) fail = DFQ_PNG_SHORT;
  if (!fail && status == kEnd) {                           // its Adler-32 over the pos bytes written
    const int64_t q = r.byte_pos();
    if (q + 4 <= im.src_end) {
      __syncwarp();
      unsigned long long s1 = 0, s2 = 0;
      for (int64_t i = lane, j = 0; i < pos; i += 32, ++j) {
        const unsigned d = out[i];
        s1 += d;
        s2 += (unsigned long long)(pos - i) * d;
        if ((j & 0xFFFF) == 0xFFFF) s2 %= 65521;             // 2^16 terms below 2^39 each: no overflow
      }
      s1 %= 65521;
      s2 %= 65521;
      for (int o = 16; o; o >>= 1) {
        s1 += __shfl_xor_sync(kFull, s1, o);
        s2 += __shfl_xor_sync(kFull, s2, o);
      }
      const unsigned a = (unsigned)((1 + s1) % 65521), b = (unsigned)((pos % 65521 + s2) % 65521);
      const unsigned want = (unsigned)blob[q] << 24 | (unsigned)blob[q + 1] << 16 | (unsigned)blob[q + 2] << 8 | blob[q + 3];
      if ((b << 16 | a) != want) fail = DFQ_PNG_ADLER;
    } else if (pos < T) {
      fail = DFQ_PNG_SHORT;                                  // Pillow waits for the rest of the trailer: truncated
    }
  }
  // Rows the stream did not reach are zero scanlines of filter None: zero labels, as Pillow leaves them, and no filter
  // byte the walk never wrote for k_png_unfilter to trip on when the image failed.
  for (int64_t i = pos + lane; i < T; i += 32) out[i] = 0;
  if (fail && lane == 0) report(err, call, img, fail);
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(32) k_png_unfilter(const DfqPngImage* __restrict__ ims, uint8_t* blob,
                                                     unsigned long long* err, unsigned long long call) {
  const int lane = threadIdx.x, img = blockIdx.x;
  const DfqPngImage im = ims[img];
  const int W = im.W;
  for (int y = 0; y < im.H; ++y) {
    // no __restrict__: up is the row this warp wrote last, which a non-coherent load could miss
    const uint8_t* row = blob + im.work + (int64_t)y * (W + 1);
    uint8_t* cur = blob + im.dst + (int64_t)y * W;
    const uint8_t* up = y ? cur - W : nullptr;
    const int t = row[0];
    ++row;
    if (t > 4) {
      if (lane == 0) report(err, call, img, DFQ_PNG_BAD_FILTER);
      return;
    }
    if (t == 0 || t == 2) {
      for (int x = lane; x < W; x += 32) cur[x] = (uint8_t)(row[x] + (t == 2 && up ? up[x] : 0));
    } else if (t == 1) {
      unsigned carry = 0;
      for (int base = 0; base < W; base += 32) {
        const int x = base + lane;
        unsigned v = x < W ? row[x] : 0;
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned u = __shfl_up_sync(kFull, v, o);
          if (lane >= o) v += u;
        }
        v += carry;
        if (x < W) cur[x] = (uint8_t)v;
        carry = __shfl_sync(kFull, v, 31);
      }
    } else if (lane == 0) {
      int a = 0, c = 0;
      for (int x = 0; x < W; ++x) {
        const int b = up ? up[x] : 0;
        a = (row[x] + (t == 3 ? (a + b) >> 1 : paeth(a, b, c))) & 255;
        cur[x] = (uint8_t)a;
        c = b;
      }
    }
    __syncwarp();
  }
}

bool inside(int64_t off, int64_t bytes, int64_t blob) { return off >= 0 && bytes >= 0 && bytes <= blob - off; }
bool apart(int64_t a, int64_t an, int64_t b, int64_t bn) { return a + an <= b || b + bn <= a; }

}  // namespace
}  // namespace dfq

using namespace dfq;

extern "C" int dfq_png_decode(const DfqPngDecode* d, const DfqPngImage* images, void* blob, uint64_t* error, void* stream) {
  if (!d || !images || !blob || !error) {
    set_error("dfq_png_decode: d, images, blob and error must be non-NULL");
    return DFQ_E_ARG;
  }
  if (d->n < 1 || d->n > 65535 || d->blob_bytes < 1 || d->call >= (1ull << 31)) {
    set_error("dfq_png_decode: n must be in 1 .. 65535, blob_bytes at least 1, call below 2^31 (n %d, blob %lld)", d->n,
              (long long)d->blob_bytes);
    return DFQ_E_ARG;
  }
  if ((uintptr_t)error % 8) {
    set_error("dfq_png_decode: error must be 8-byte aligned");
    return DFQ_E_ARG;
  }
  const int64_t B = d->blob_bytes;
  for (int i = 0; i < d->n; ++i) {
    const DfqPngImage& m = images[i];
    const int64_t px = (int64_t)m.H * m.W, T = px + m.H, S = m.src_end - m.src;
    const bool ok = m.H >= 1 && m.W >= 1 && px <= INT32_MAX && S >= 2 && inside(m.src, S, B) && inside(m.work, T, B) &&
                    inside(m.dst, px, B) && apart(m.src, S, m.work, T) && apart(m.src, S, m.dst, px) &&
                    apart(m.work, T, m.dst, px);
    if (!ok) {
      set_error("dfq_png_decode: image %d: %d x %d, stream %lld .. %lld, work %lld, output %lld: unsupported size, or a "
                "stream shorter than its header, or a region outside the %lld-byte blob or overlapping another", i, m.H,
                m.W, (long long)m.src, (long long)m.src_end, (long long)m.work, (long long)m.dst, (long long)B);
      return DFQ_E_ARG;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  TablePack tp;
  const int iI = tp.add(images, d->n);
  if (int rc = tp.upload(st)) return rc;
  const DfqPngImage* dim = tp.ptr<DfqPngImage>(iI);
  k_png_inflate<<<d->n, 32, 0, st>>>(dim, (uint8_t*)blob, (unsigned long long*)error, d->call);
  k_png_unfilter<<<d->n, 32, 0, st>>>(dim, (uint8_t*)blob, (unsigned long long*)error, d->call);
  DFQ_CUDA(cudaGetLastError());
  tp.release(st);
  return 0;
}
