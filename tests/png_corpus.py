"""Seeded PNG label streams for the PNG decoder's tests: what Pillow writes for VOC-like palette labels at every compression
level, what cv2.imwrite writes for gray labels under every deflate strategy, and streams of tests/png_writer.py that
reach every path of the inflate and unfilter kernels.  corpus() returns [(name, bytes)]; pillow(b) is the reference."""
import io

import cv2
import numpy as np
from PIL import Image

import png_writer as W


def pillow(data):
    return np.array(Image.open(io.BytesIO(data)))


def voc_label(h, w, seed):
    """A VOC-like label map: a few class blobs with 255 borders on a background of 0, mostly flat."""
    g = np.random.default_rng(seed)
    a = np.zeros((h, w), np.uint8)
    yy, xx = np.mgrid[:h, :w]
    for _ in range(int(g.integers(1, 5))):
        cy, cx = g.integers(0, h), g.integers(0, w)
        ry, rx = g.integers(max(h // 8, 1), max(h // 3, 2)), g.integers(max(w // 8, 1), max(w // 3, 2))
        d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
        a[d <= 1.15] = 255
        a[d <= 1.0] = int(g.integers(1, 21))
    return a


def pil_p(a, **kw):
    b = io.BytesIO()
    im = Image.frombytes("P", (a.shape[1], a.shape[0]), a.tobytes())
    im.putpalette(list(range(256)) * 3)
    im.save(b, "PNG", **kw)
    return b.getvalue()


def cv_gray(a, params=()):
    ok, buf = cv2.imencode(".png", a, list(params))
    assert ok
    return buf.tobytes()


STRATEGIES = ["DEFAULT", "FILTERED", "HUFFMAN_ONLY", "RLE", "FIXED"]


def _noise(h, w, seed, levels=6):
    g = np.random.default_rng(seed)
    return (g.integers(0, levels, (h, w)) * (250 // levels)).astype(np.uint8)


def writer_streams(big=True):
    out = []
    img = _noise(9, 13, 1)
    for f in range(5):
        out.append(("filter%d" % f, W.image_png(img, filters=(f,))))
    out.append(("filters_per_row", W.image_png(_noise(15, 11, 2), filters=(0, 1, 2, 3, 4, 4, 3, 2, 1))))
    tie = np.array([[10, 20, 10, 20], [20, 10, 20, 10], [10, 10, 20, 20], [15, 15, 15, 15]], np.uint8)  # pa = pb = pc ties
    out.append(("paeth_ties", W.image_png(np.tile(tie, (3, 5)), filters=(4,))))
    out.append(("paeth_flat", W.image_png(np.full((6, 7), 200, np.uint8), filters=(4,))))
    raw = W.filter_rows(_noise(300, 250, 3), (0,))              # 75,300 bytes: one full stored block and more
    out.append(("stored_65535", W.png(300, 250, W.zlib([("stored", b""), ("stored", raw[:65535]), ("stored", b""),
                                                        ("stored", raw[65535:])], raw))))
    r2 = W.filter_rows(img, (1,))
    out.append(("fixed", W.png(9, 13, W.zlib([("fixed", W.lz77(r2))], r2))))
    out.append(("fixed_dynamic_stored", W.png(9, 13, W.zlib([("fixed", list(r2[:30])), ("dynamic", W.lz77(r2[30:70])),
                                                              ("stored", r2[70:90]), ("fixed", W.lz77(r2[90:]))], r2))))
    out.append(("literals_only", W.png(9, 13, W.zlib([("dynamic", list(r2))], r2))))
    # one distance code only: a single-code distance tree of one bit
    flat = np.full((8, 40), 7, np.uint8)
    rf = W.filter_rows(flat, (0,))
    out.append(("single_distance_code", W.png(8, 40, W.zlib([("dynamic", [0, 7, (39, 1)] * 8)], rf))))
    # length 258 at distance 32,768 and overlapping matches at every distance 1 .. 33 (bytes 0 .. 4: any can be a filter)
    head = bytes(np.random.default_rng(4).integers(0, 5, 32768, dtype=np.uint8))
    syms, Wd = list(head) + [(258, 32768)] + [(3 + 7 * D, D) for D in range(1, 34)], 256
    n = 32768 + 258 + sum(3 + 7 * D for D in range(1, 34))
    syms += [0] * ((-n) % (Wd + 1))
    body = W.inflate_symbols(syms)
    out.append(("long_far_overlapping", W.png(len(body) // (Wd + 1), Wd, W.zlib([("dynamic", syms)], body))))
    # 15-bit codes: literal lengths 1 .. 15, 15 over 16 symbols (a complete code)
    lit = [0] * 286
    used = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 256, 257, 258]
    for s, l in zip(used, list(range(1, 16)) + [15]):
        lit[s] = l
    a15 = np.array([[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 0, 0, 0]] * 3, np.uint8)
    r15 = W.filter_rows(a15, (0,))
    syms15 = list(r15[:20]) + [(3, 17), (4, 17)] + list(r15[27:])
    assert W.inflate_symbols(syms15) == r15
    dist = [0] * 30
    dist[8] = 1
    dist[0] = 1
    out.append(("codes_15_bits", W.png(3, 16, W.zlib([("dynamic", syms15, lit, dist)], r15))))
    # IDATs split at every byte of a small stream, and zero-length IDATs
    small = W.zlib([("dynamic", W.lz77(r2))], r2)
    for cut in range(1, len(small)):
        out.append(("split_at_%d" % cut, W.png(9, 13, small, split=[cut])))
    out.append(("split_every_byte", W.png(9, 13, small, split=1)))
    out.append(("zero_length_idats", W.png(9, 13, small, split=[0, 0, 5, 5, 5, len(small), len(small)])))
    for h, w in ((1, 1), (1, 37), (41, 1), (1, 300), (300, 1)):
        out.append(("size_%dx%d" % (h, w), W.image_png(_noise(h, w, h * 7 + w), filters=(0, 1, 2, 3, 4))))
    if big:
        out.append(("size_4000x3000", pil_p(voc_label(3000, 4000, 5))))
        out.append(("size_4000x3000_cv", cv_gray(_noise(3000, 4000, 6, 3))))
    # streams that are odd but taken: no Adler-32, half of it, bytes after it, more data than the image
    r3 = W.filter_rows(img, (2,))
    out.append(("no_adler", W.png(9, 13, W.zlib([("fixed", list(r3))], r3, adler=b""))))
    out.append(("half_adler", W.png(9, 13, W.zlib([("fixed", list(r3))], r3)[:-2])))
    out.append(("after_adler", W.png(9, 13, W.zlib([("fixed", list(r3))], r3) + b"\x00\xff\x13")))
    out.append(("more_data_bad_adler", W.png(9, 13, W.zlib([("fixed", list(r3) + [1, 2, (5, 3)])], r3, adler=b"\0\0\0\0"))))
    out.append(("no_iend", W.png(9, 13, W.zlib([("fixed", list(r3))], r3), iend=False)))
    out.append(("bad_idat_crc", _bad_idat_crc(W.png(9, 13, W.zlib([("fixed", list(r3))], r3)))))
    out.append(("palette_writer", W.image_png(img, filters=(4,), ctype=3)))
    out.append(("gray_trns", W.image_png(img, extra=W.chunk(b"tRNS", b"\x00\x05"))))
    return out


def _bad_idat_crc(b):
    i = b.index(b"IDAT")
    n = int.from_bytes(b[i - 4:i], "big")
    bb = bytearray(b)
    bb[i + 4 + n] ^= 0xFF
    return bytes(bb)


def corpus(big=True):
    out = []
    for h, w in ((375, 500), (500, 333), (281, 500), (7, 5)):
        a = voc_label(h, w, h * w)
        for lvl in (0, 1, 6, 9):
            out.append(("pil_%dx%d_l%d" % (h, w, lvl), pil_p(a, compress_level=lvl)))
        out.append(("pil_%dx%d_opt" % (h, w), pil_p(a, optimize=True)))
        for s in STRATEGIES:
            out.append(("cv_%dx%d_%s" % (h, w, s), cv_gray(a, [cv2.IMWRITE_PNG_STRATEGY,
                                                                getattr(cv2, "IMWRITE_PNG_STRATEGY_" + s)])))
        out.append(("cv_%dx%d_l9" % (h, w), cv_gray(_noise(h, w, h), [cv2.IMWRITE_PNG_COMPRESSION, 9])))
    return out + writer_streams(big)


# ---- corrupt streams: (name, bytes, DFQ_PNG_* reason); each is one Pillow rejects ------------------------------------------
def _fixed_raw(bw, raw):
    lc = W.canonical(W.FIXED_LIT)
    for x in raw:
        bw.code(lc[x], W.FIXED_LIT[x])
    return lc


def _fixed_then(raw, tail, final=1):
    """A fixed block with raw's literals, then tail(bw, lit_codes) appended before its end; zero-padded stream."""
    bw = W.Bits()
    bw.put(final, 1)
    bw.put(1, 2)
    lc = _fixed_raw(bw, raw)
    tail(bw, lc)
    return b"\x78\x9c" + bw.bytes() + b"\0" * 6


def corrupt_streams():
    from dfq_b200 import _lib
    img = _noise(5, 8, 9)
    raw = W.filter_rows(img, (0,))
    H, Wd = img.shape

    def mk(stream):
        return W.png(H, Wd, stream)

    out = []
    bw = W.Bits(); bw.put(1, 1); bw.put(3, 2)
    out.append(("block_type_3", mk(b"\x78\x9c" + bw.bytes() + b"\0" * 8), _lib.PNG_BAD_BLOCK))
    bw = W.Bits(); bw.put(1, 1); bw.put(2, 2); bw.put(0, 5); bw.put(0, 5); bw.put(15, 4)
    for _ in range(19):
        bw.put(1, 3)                                          # 19 codes of one bit: over-subscribed
    out.append(("codelength_oversubscribed", mk(b"\x78\x9c" + bw.bytes() + b"\0" * 8), _lib.PNG_BAD_CODESET))
    bw = W.Bits(); bw.put(1, 1); bw.put(2, 2); bw.put(30, 5); bw.put(0, 5); bw.put(0, 4)
    out.append(("hlit_287", mk(b"\x78\x9c" + bw.bytes() + b"\0" * 8), _lib.PNG_BAD_CODESET))
    lit = W.huffman_lengths([1] * 256 + [0] + [1] * 29, 15)     # no end-of-block code
    out.append(("no_end_of_block", mk(_dyn_header_only(lit)), _lib.PNG_BAD_CODESET))
    out.append(("literal_286", mk(_fixed_then(raw[:7], lambda bw, lc: bw.code(lc[286], 8))), _lib.PNG_BAD_CODE))
    out.append(("distance_30", mk(_fixed_then(raw[:7], lambda bw, lc: (bw.code(lc[257], 7), bw.code(30, 5)))),
                _lib.PNG_BAD_CODE))
    out.append(("too_far_back", mk(_fixed_then(raw[:3], lambda bw, lc: (bw.code(lc[257], 7), bw.code(3, 5)))),
                _lib.PNG_FAR))
    bw = W.Bits(); bw.put(1, 1); bw.put(0, 2); bw.align(); bw.put(len(raw), 16); bw.put(len(raw), 16)
    out.append(("stored_nlen", mk(b"\x78\x9c" + bw.bytes() + raw), _lib.PNG_STORED_LEN))
    out.append(("short", mk(W.zlib([("fixed", list(raw[:-1]))], raw[:-1])), _lib.PNG_SHORT))
    out.append(("short_cut", mk(W.zlib([("stored", raw)], raw)[:len(raw) // 2]), _lib.PNG_SHORT))
    bad = bytearray(raw)
    bad[(Wd + 1) * 3] = 5
    out.append(("filter_5", mk(W.zlib([("fixed", list(bad))], bytes(bad))), _lib.PNG_BAD_FILTER))
    out.append(("adler", mk(W.zlib([("fixed", list(raw))], raw, adler=b"\0\0\0\1")), _lib.PNG_ADLER))
    big = np.zeros((1000, 1000), np.uint8)
    rb = W.filter_rows(big, (0,))
    out.append(("adler_1000x1000", W.png(1000, 1000, W.zlib([("dynamic", [0] + [(258, 1)] * 3879 + [(217, 1)])], rb,
                                                             adler=b"\0\0\0\1")), _lib.PNG_ADLER))
    # past the last row: what zlib still reads with no output room left
    out.append(("after_end_eob_then_type_3", mk(_fixed_then(raw, lambda bw, lc: (bw.code(lc[256], 7), bw.put(1, 1),
                                                                                  bw.put(3, 2)), final=0)), _lib.PNG_BAD_BLOCK))
    out.append(("after_end_literal_286", mk(_fixed_then(raw, lambda bw, lc: bw.code(lc[286], 8))), _lib.PNG_BAD_CODE))
    out.append(("after_end_length_bad_distance", mk(_fixed_then(raw, lambda bw, lc: (bw.code(lc[257], 7),
                                                                                      bw.code(31, 5)))), _lib.PNG_BAD_CODE))
    out.append(("after_end_stored_nlen", mk(_fixed_then(raw, lambda bw, lc: (bw.code(lc[256], 7), bw.put(0, 1), bw.put(0, 2),
                                                                             bw.align(), bw.put(5, 16), bw.put(5, 16)),
                                                        final=0)), _lib.PNG_STORED_LEN))
    out.append(("after_end_hlit_287", mk(_fixed_then(raw, lambda bw, lc: (bw.code(lc[256], 7), bw.put(1, 1), bw.put(2, 2),
                                                                          bw.put(30, 5), bw.put(0, 5), bw.put(0, 4)),
                                                     final=0)), _lib.PNG_BAD_CODESET))
    return out + [(n, d, why) for n, d, why in _rows_end() if why is not True]


def _dyn_header_only(lit):
    bw = W.Bits()
    W.block(bw, "dynamic", [], 1, lit, [1] + [0] * 29)
    return b"\x78\x9c" + bw.bytes() + b"\0" * 8


def accepted_edges():
    """Streams past the last row that zlib stops reading before anything wrong: (name, bytes), each equal to Pillow."""
    img = _noise(5, 8, 9)
    raw = W.filter_rows(img, (0,))
    H, Wd = img.shape
    return [("after_end_literal_then_garbage", W.png(H, Wd, _fixed_then(raw, lambda bw, lc: (bw.code(lc[7], 8),
                                                                                            bw.put(0x7FFF, 15))))),
            ("after_end_length_far_distance", W.png(H, Wd, _fixed_then(raw, lambda bw, lc: (bw.code(lc[257], 7),
                                                                                           bw.code(29, 5), bw.put(0, 13)))))] \
        + _match_across_end() + [(n, d) for n, d, ok in _rows_end() if ok is True]


def _match_across_end():
    """A match that runs past the last byte, then the final end-of-block and the Adler-32 of every byte the stream holds
    (and the same with garbage in place of the trailer): zlib writes what fits and stops there."""
    raw = W.filter_rows(np.full((2, 4), 3, np.uint8), (0,))
    syms = list(raw[:8]) + [(5, 1)]
    s = W.zlib([("fixed", syms)], W.inflate_symbols(syms))
    return [("match_across_end", W.png(2, 4, s)), ("match_across_end_then_garbage", W.png(2, 4, s[:-4] + b"\xff" * 5))]


def _rows_end():
    """(name, bytes, taken) of whole streams that end at the end of a row before the last: Pillow keeps the rows that came
    and leaves the rest zero when the whole, right Adler-32 follows; it refuses them without it."""
    from dfq_b200 import _lib
    out = []
    img = (np.arange(12).reshape(3, 4) * 9 + 1).astype(np.uint8)
    raw = W.filter_rows(img, (0, 1))
    for k in (1, 2):
        r = raw[:5 * k]
        full = W.zlib([("fixed", list(r))], r)
        out.append(("rows_end_%d_of_3" % k, W.png(3, 4, full), True))
        out.append(("rows_end_%d_of_3_no_trailer" % k, W.png(3, 4, full[:-4]), _lib.PNG_SHORT))
        out.append(("rows_end_%d_of_3_half_trailer" % k, W.png(3, 4, full[:-2]), _lib.PNG_SHORT))
        out.append(("rows_end_%d_of_3_bad_adler" % k, W.png(3, 4, W.zlib([("fixed", list(r))], r, adler=b"\0\0\0\1")),
                    _lib.PNG_ADLER))
    out.append(("rows_end_0_of_3", W.png(3, 4, W.zlib([("fixed", [])], b"")), _lib.PNG_SHORT))
    big = (np.arange(300 * 200).reshape(300, 200) % 7 * 30).astype(np.uint8)
    rb = W.filter_rows(big, (0, 2, 4))[:201 * 150]
    out.append(("rows_end_150_of_300", W.png(300, 200, W.zlib([("dynamic", W.lz77(rb))], rb)), True))
    return out
