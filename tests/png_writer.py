"""A PNG and DEFLATE writer for tests: every choice an encoder makes is explicit here, so streams that Pillow and OpenCV never
write (a filter per row, stored blocks of any length, fixed blocks, hand-chosen code lengths up to 15 bits, single-code
distance trees, matches of any length and distance, IDATs split anywhere) can be built and, where needed, broken on
purpose.  Test infrastructure only.

A block is ("stored", data), ("fixed", symbols) or ("dynamic", symbols[, lit_lengths, dist_lengths]); symbols are literal
byte values and (length, distance) pairs, the end-of-block code is added.  zlib(blocks) is the whole zlib stream.
"""
import heapq
import struct
import zlib as _zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


class Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, n):                                   # Huffman codes go MSB first
        self.put(int("{:0{}b}".format(c, n)[::-1], 2) if n else 0, n)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def bytes(self):
        self.align()
        return bytes(self.out)


def canonical(lengths):
    """The canonical codes of a length list (0 = unused)."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = []
    for l in lengths:
        out.append(nxt[l] if l else 0)
        if l:
            nxt[l] += 1
    return out


def huffman_lengths(freq, limit):
    """Huffman code lengths of freq, at most `limit` bits (frequencies halved until they fit); one used symbol gets 1 bit."""
    freq = list(freq)
    while True:
        used = [i for i, f in enumerate(freq) if f]
        lengths = [0] * len(freq)
        if len(used) == 1:
            lengths[used[0]] = 1
            return lengths
        if not used:
            return lengths
        heap = [(freq[i], i, [i]) for i in used]
        heapq.heapify(heap)
        k = len(freq)
        while len(heap) > 1:
            fa, _, a = heapq.heappop(heap)
            fb, _, b = heapq.heappop(heap)
            for s in a + b:
                lengths[s] += 1
            heapq.heappush(heap, (fa + fb, k, a + b))
            k += 1
        if max(lengths) <= limit:
            return lengths
        freq = [(f + 1) // 2 if f else 0 for f in freq]


def _len_code(L):
    for c in range(28, -1, -1):
        if L >= LEN_BASE[c] and (c != 28 or L == 258):
            if c == 28 or L - LEN_BASE[c] < (1 << LEN_EXTRA[c]):
                return c
    raise ValueError(L)


def _dist_code(D):
    for c in range(29, -1, -1):
        if D >= DIST_BASE[c]:
            return c
    raise ValueError(D)


def _emit(bw, symbols, lc, ll, dc, dl):
    for s in symbols:
        if isinstance(s, tuple):
            L, D = s
            c = _len_code(L)
            bw.code(lc[257 + c], ll[257 + c])
            bw.put(L - LEN_BASE[c], LEN_EXTRA[c])
            c = _dist_code(D)
            bw.code(dc[c], dl[c])
            bw.put(D - DIST_BASE[c], DIST_EXTRA[c])
        else:
            bw.code(lc[s], ll[s])
    bw.code(lc[256], ll[256])


def _rle(lengths):
    """The code-length alphabet's run-length coding of lengths: [(symbol, extra bits value, extra bit count)]."""
    out, i = [], 0
    while i < len(lengths):
        v, run = lengths[i], 1
        while i + run < len(lengths) and lengths[i + run] == v:
            run += 1
        take = run
        if v == 0 and run >= 3:
            take = min(run, 138)
            out.append((18, take - 11, 7) if take >= 11 else (17, take - 3, 3))
        elif v and run >= 4:
            out.append((v, 0, 0))
            take = 1 + min(run - 1, 6)
            out.append((16, take - 4, 2))
        else:
            take = 1
            out.append((v, 0, 0))
        i += take
    return out


def block(bw, kind, payload, final, lit_lengths=None, dist_lengths=None):
    bw.put(final, 1)
    if kind == "stored":
        bw.put(0, 2)
        bw.align()
        n = len(payload)
        bw.put(n, 16)
        bw.put(n ^ 0xFFFF, 16)
        for b in payload:
            bw.put(b, 8)
        return
    if kind == "fixed":
        bw.put(1, 2)
        _emit(bw, payload, canonical(FIXED_LIT), FIXED_LIT, canonical(FIXED_DIST + [5, 5]), FIXED_DIST + [5, 5])
        return
    lf, df = [0] * 286, [0] * 30
    lf[256] = 1
    for s in payload:
        if isinstance(s, tuple):
            lf[257 + _len_code(s[0])] += 1
            df[_dist_code(s[1])] += 1
        else:
            lf[s] += 1
    ll = list(lit_lengths) if lit_lengths is not None else huffman_lengths(lf, 15)
    dl = list(dist_lengths) if dist_lengths is not None else huffman_lengths(df, 15)
    if not any(dl):
        dl = [0] * 30
        dl[0] = 1
    hlit = max(257, max(i for i, l in enumerate(ll) if l) + 1)
    hdist = max(1, max(i for i, l in enumerate(dl) if l) + 1)
    seq = _rle(ll[:hlit] + dl[:hdist])
    cf = [0] * 19
    for s, _, _ in seq:
        cf[s] += 1
    cl = huffman_lengths(cf, 7)
    if sum(1 for l in cl if l) == 1:                       # a code-length code must be complete: give it a second symbol
        cl[next(i for i in range(19) if not cl[i])] = 1
    cc = canonical(cl)
    hclen = max(4, max(k + 1 for k in range(19) if cl[CL_ORDER[k]]))
    bw.put(2, 2)
    bw.put(hlit - 257, 5)
    bw.put(hdist - 1, 5)
    bw.put(hclen - 4, 4)
    for k in range(hclen):
        bw.put(cl[CL_ORDER[k]], 3)
    for s, v, n in seq:
        bw.code(cc[s], cl[s])
        bw.put(v, n)
    _emit(bw, payload, canonical(ll), ll, canonical(dl), dl)


def deflate(blocks):
    bw = Bits()
    for k, b in enumerate(blocks):
        block(bw, b[0], b[1], k == len(blocks) - 1, *b[2:])
    return bw.bytes()


def zlib(blocks, data=None, header=b"\x78\x9c", adler=None):
    """A zlib stream: the header, the blocks and the Adler-32 of data (or the given adler; b"" for none)."""
    body = deflate(blocks)
    if adler is None:
        adler = struct.pack(">I", _zlib.adler32(data))
    return header + body + adler


def lz77(data, max_len=258, window=32768):
    """Greedy LZ77 symbols of data (hash chains on 3 bytes)."""
    data = bytes(data)
    out, i, heads = [], 0, {}
    while i < len(data):
        best, bd = 0, 0
        if i + 3 <= len(data):
            for j in reversed(heads.get(data[i:i + 3], [])[-64:]):
                if i - j > window:
                    break
                L = 0
                while L < max_len and i + L < len(data) and data[j + L] == data[i + L]:
                    L += 1
                if L > best:
                    best, bd = L, i - j
        if best >= 3:
            for k in range(i, i + best):
                heads.setdefault(data[k:k + 3], []).append(k)
            out.append((best, bd))
            i += best
        else:
            heads.setdefault(data[i:i + 3], []).append(i)
            out.append(data[i])
            i += 1
    return out


def inflate_symbols(symbols):
    """The bytes that symbols stand for."""
    out = bytearray()
    for s in symbols:
        if isinstance(s, tuple):
            for _ in range(s[0]):
                out.append(out[-s[1]])
        else:
            out.append(s)
    return bytes(out)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def filter_rows(img, filters):
    """The filtered scanlines of a uint8 [H, W] image, row r with filter filters[r % len(filters)] (0 .. 4)."""
    img = np.asarray(img, np.int32)
    H, W = img.shape
    out = bytearray()
    for r in range(H):
        f = filters[r % len(filters)]
        prev = img[r - 1] if r else np.zeros(W, np.int32)
        cur = img[r]
        left = np.concatenate([[0], cur[:-1]])
        ul = np.concatenate([[0], prev[:-1]])
        if f == 0:
            pred = np.zeros(W, np.int32)
        elif f == 1:
            pred = left
        elif f == 2:
            pred = prev
        elif f == 3:
            pred = (left + prev) // 2
        else:
            pred = np.array([_paeth(int(a), int(b), int(c)) for a, b, c in zip(left, prev, ul)], np.int32)
        out.append(f)
        out += ((cur - pred) % 256).astype(np.uint8).tobytes()
    return bytes(out)


def chunk(cid, body, crc=None):
    c = _zlib.crc32(cid + body) if crc is None else crc
    return struct.pack(">I", len(body)) + cid + body + struct.pack(">I", c & 0xFFFFFFFF)


def ihdr(H, W, depth=8, ctype=0, comp=0, filt=0, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ctype, comp, filt, interlace))


def png(H, W, stream, ctype=0, depth=8, split=None, palette=True, extra=b"", iend=True, **kw):
    """A PNG of one zlib stream: IDATs of `split` bytes each (None: one IDAT; a list: those cut points)."""
    if split is None:
        parts = [stream]
    elif isinstance(split, int):
        parts = [stream[k:k + split] for k in range(0, len(stream), split)] or [b""]
    else:
        cuts = [0] + list(split) + [len(stream)]
        parts = [stream[a:b] for a, b in zip(cuts, cuts[1:])]
    out = SIG + ihdr(H, W, depth, ctype, **kw) + extra
    if ctype == 3 and palette:
        out += chunk(b"PLTE", bytes((np.arange(256 * 3) * 7 % 256).astype(np.uint8)))
    out += b"".join(chunk(b"IDAT", p) for p in parts)
    return out + (chunk(b"IEND", b"") if iend else b"")


def image_png(img, filters=(0,), blocks=None, ctype=0, **kw):
    """A PNG of the uint8 [H, W] image: its rows filtered, then `blocks(raw)` (default: one dynamic block of lz77 symbols)."""
    img = np.asarray(img, np.uint8)
    raw = filter_rows(img, filters)
    bl = blocks(raw) if blocks is not None else [("dynamic", lz77(raw))]
    return png(img.shape[0], img.shape[1], zlib(bl, raw), ctype=ctype, **kw)
