"""A baseline JPEG writer for the decoder's tests: it takes quantised coefficient blocks per component and writes the
stream, so tests can reach coefficients, Huffman tables and marker layouts that Pillow and OpenCV never write.  Test
infrastructure only.

    w = write([y, cb, cr], height=17, width=5, sampling="420", qtables=[q0, q1])
    w.data                      # the stream's bytes
    w.lengths[(1, 0)]           # the code lengths the scan used from AC table 0

Planes are int arrays [block rows, block columns, 64] in natural order, padded to whole MCUs: the luma plane is
[mcuy * vs, mcux * hs] blocks, each chroma plane [mcuy, mcux].  Entry [..., 0] is the block's DC value (not the
difference); the writer codes the differences, restarting them at every restart interval, so any DC value whose
differences stay within 15 bits can be written.  Byte stuffing and the 1-bit padding before each marker are libjpeg's.
Component k uses quantisation table min(k, len(qtables) - 1) and Huffman tables min(k, 1).
"""
import dataclasses
import heapq

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])        # zigzag index -> natural index
SAMPLING = {"gray": (1, 1), "444": (1, 1), "422": (2, 1), "420": (2, 2)}


@dataclasses.dataclass
class Written:
    data: bytes
    lengths: dict          # (class, table) -> set of the code lengths the scan used
    symbols: dict          # (class, table) -> set of the symbols the scan used
    intervals: int         # restart intervals in the scan
    tables: dict           # (class, table) -> (counts, vals) as written


def _category(v):
    return int(abs(int(v))).bit_length()


def _bits(v, s):
    """The s low bits that code v in category s (negative values as v - 1, as JPEG's EXTEND undoes)."""
    return (v if v >= 0 else v + (1 << s) - 1) & ((1 << s) - 1)


def _symbols(planes, layout, mcux, mcuy, ri):
    """Per MCU block: (component, [(symbol, extra bits value, extra bits count)]) in scan order; DC as a difference."""
    total = mcux * mcuy
    step = ri or total
    out = []
    for m in range(total):
        if m % step == 0:
            pred = [0, 0, 0]
        my, mx = divmod(m, mcux)
        for c, dy, dx, hs, vs in layout:
            blk = planes[c][my * vs + dy, mx * hs + dx]
            diff = int(blk[0]) - pred[c]
            pred[c] = int(blk[0])
            s = _category(diff)
            if s > 15:
                raise ValueError("DC difference %d does not fit 15 bits" % diff)
            syms = [((0, s), _bits(diff, s), s)]
            zz = [int(v) for v in np.asarray(blk)[ZIGZAG[1:]]]
            last = max([k for k, v in enumerate(zz) if v] or [-1])
            run = 0
            for k in range(last + 1):
                if zz[k] == 0:
                    run += 1
                    continue
                while run > 15:
                    syms.append(((1, 0xF0), 0, 0))
                    run -= 16
                s = _category(zz[k])
                if s > 15:
                    raise ValueError("AC coefficient %d does not fit 15 bits" % zz[k])
                syms.append(((1, run << 4 | s), _bits(zz[k], s), s))
                run = 0
            if last < 62:
                syms.append(((1, 0x00), 0, 0))                    # EOB
            out.append((m, c, syms))
    return out


def optimal_table(freq, maxlen=16):
    """(counts, vals) of a length-limited Huffman table for {symbol: frequency}, as jpeg_gen_optimal_table builds it: a
    reserved pseudo-symbol keeps the all-ones code out, and the lengths are folded down to maxlen (Annex K.3)."""
    items = [(f, s) for s, f in freq.items() if f] + [(0.5, 256)]
    if len(items) > (1 << maxlen):
        raise ValueError("%d symbols do not fit codes of %d bits" % (len(items) - 1, maxlen))
    heap = [(f, k, [s]) for k, (f, s) in enumerate(items)]
    heapq.heapify(heap)
    size = {s: 0 for _, s in items}
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            size[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    bits = [0] * 64
    for s, l in size.items():
        bits[l] += 1
    for i in range(63, maxlen, -1):                           # adjust_bits, for any limit
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = maxlen
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                              # drop the pseudo-symbol
    order = sorted((s for _, s in items if s != 256), key=lambda s: (size[s], s))   # by unfolded length, as libjpeg
    counts = bits[1:17]
    return bytes(counts), bytes(order)


def codes(counts, vals):
    """{symbol: (code, length)} of a table, as the canonical (Annex C) assignment gives them."""
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(counts[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        self.acc = (self.acc << n) | v
        self.n += n
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 255
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)                            # byte stuffing
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)    # pad with 1-bits, as libjpeg's flush_bits


def _seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)


def _dqt(tables):
    body = bytearray()
    for tq, (t, bits16) in tables:
        body.append((1 if bits16 else 0) << 4 | tq)
        z = np.asarray(t, np.int64)[ZIGZAG]
        body += b"".join(int(v).to_bytes(2, "big") for v in z) if bits16 else bytes(int(v) for v in z)
    return _seg(0xDB, body)


def _dht(tables):
    body = bytearray()
    for (tc, th), (counts, vals) in tables:
        body += bytes([tc << 4 | th]) + bytes(counts) + bytes(vals)
    return _seg(0xC4, body)


def write(planes, *, height, width, sampling="gray", qtables, qbits=8, huff=None, maxlen=16, ri=0, sof=0xC0, ids=None,
          group=True, tables_after_sof=False, redefine=False, extras=False, fill=0, seed=0):
    """The baseline stream of the quantised blocks in planes (see the module docstring).

    qbits: 8 or 16 (the DQT precision; 16-bit tables take values up to 65535).  huff: {(class, table): (counts, vals)}
    for explicit tables, otherwise each table is built from the scan's symbol statistics with codes of at most maxlen
    bits.  ri: the DRI interval (0: none).  sof: 0xC0 or 0xC1.  ids: the component ids (default 1, 2, 3).  group: all
    tables of a kind in one DQT / DHT segment, else one segment per table.  tables_after_sof: the tables between SOF and
    SOS.  redefine: first define every table with other contents, then again before SOS.  extras: APP1 and COM segments
    between the others, with seeded payloads.  fill: FF fill bytes before every RSTn and before EOI."""
    hs, vs = SAMPLING[sampling]
    nc = 1 if sampling == "gray" else 3
    assert len(planes) == nc and sof in (0xC0, 0xC1)
    mcux, mcuy = -(-width // (8 * hs)), -(-height // (8 * vs))
    assert planes[0].shape[:2] == (mcuy * vs, mcux * hs), planes[0].shape
    for p in planes[1:]:
        assert p.shape[:2] == (mcuy, mcux), p.shape
    ids = list(ids or [1, 2, 3][:nc])
    layout = [(0, dy, dx, hs, vs) for dy in range(vs) for dx in range(hs)] + [(c, 0, 0, 1, 1) for c in range(1, nc)]
    hsel = [min(c, 1) for c in range(nc)]
    qsel = [min(c, len(qtables) - 1) for c in range(nc)]
    blocks = _symbols(planes, layout, mcux, mcuy, ri)
    huff = dict(huff or {})
    for tc in (0, 1):
        for th in sorted(set(hsel)):
            if (tc, th) not in huff:
                freq = {}
                for _, c, syms in blocks:
                    for (k, s), _, _ in syms:
                        if k == tc and hsel[c] == th:
                            freq[s] = freq.get(s, 0) + 1
                huff[(tc, th)] = optimal_table(freq or {0: 1}, maxlen)
    code = {k: codes(*v) for k, v in huff.items()}
    lengths, symbols = {k: set() for k in huff}, {k: set() for k in huff}
    bw = _Bits()
    scan = bytearray()
    step = ri or mcux * mcuy
    g = np.random.default_rng(seed)
    prev = 0
    for m, c, syms in blocks:
        if m != prev and m % step == 0:
            bw.flush()
            scan += bw.out + b"\xff" * fill + bytes([0xFF, 0xD0 + (m // step - 1) % 8])
            bw.out = bytearray()
        prev = m
        for (k, s), v, n in syms:
            key = (k, hsel[c])
            if s not in code[key]:
                raise ValueError("symbol 0x%02X is not in %s table %d" % (s, "DC AC".split()[k], hsel[c]))
            cw, cl = code[key][s]
            lengths[key].add(cl)
            symbols[key].add(s)
            bw.put(cw, cl)
            if n:
                bw.put(v, n)
    bw.flush()
    scan += bw.out + b"\xff" * fill

    qt = [(tq, (qtables[tq], qbits == 16)) for tq in sorted(set(qsel))]
    ht = sorted(huff.items())
    junk_q = [(tq, ([255 - k % 200 for k in range(64)], False)) for tq, _ in qt]
    junk_h = [(k, (bytes([0, 1] + [1] * 14), bytes(range(15)))) for k, _ in ht]

    def tables(q, h):
        segs = [_dqt(q)] if group else [_dqt([t]) for t in q]
        segs += [_dht(h)] if group else [_dht([t]) for t in h]
        return segs

    def extra():
        if not extras:
            return []
        return [_seg(0xE1, b"test\0" + g.integers(0, 256, int(g.integers(0, 40))).astype(np.uint8).tobytes()),
                _seg(0xFE, g.integers(0, 256, int(g.integers(1, 40))).astype(np.uint8).tobytes())]

    frame = bytearray([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([nc])
    for c in range(nc):
        h, v = (hs, vs) if c == 0 else (1, 1)
        frame += bytes([ids[c], h << 4 | v, qsel[c]])
    sos = bytearray([nc])
    for c in range(nc):
        sos += bytes([ids[c], hsel[c] << 4 | hsel[c]])
    sos += bytes([0, 63, 0])
    out = [b"\xff\xd8", _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")] + extra()
    if redefine:
        out += tables(junk_q, junk_h) + extra()
    if not tables_after_sof:
        out += tables(qt, ht) + extra()
    if ri:
        out.append(_seg(0xDD, ri.to_bytes(2, "big")))
    out += [_seg(sof, frame)] + extra()
    if tables_after_sof:
        out += tables(qt, ht) + extra()
    out += [_seg(0xDA, sos), bytes(scan), b"\xff\xd9"]
    return Written(b"".join(out), lengths, symbols, -(-mcux * mcuy // step), dict(huff))
