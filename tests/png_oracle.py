"""A host oracle of the PNG label decode: Python's zlib inflating with no more output room than the image (zlib then
reads on up to the first symbol that would write, as it does for Pillow, which feeds it one row at a time), then the
five scanline filters in numpy.  Test infrastructure only; tests/test_png_host.py pins it to Pillow."""
import struct
import zlib

import numpy as np

from dfq_b200 import _lib

_REASONS = [("invalid block type", _lib.PNG_BAD_BLOCK), ("invalid code lengths set", _lib.PNG_BAD_CODESET),
            ("invalid bit length repeat", _lib.PNG_BAD_CODESET), ("too many length", _lib.PNG_BAD_CODESET),
            ("missing end-of-block", _lib.PNG_BAD_CODESET), ("invalid literal/lengths set", _lib.PNG_BAD_CODESET),
            ("invalid distances set", _lib.PNG_BAD_CODESET), ("invalid literal/length code", _lib.PNG_BAD_CODE),
            ("invalid distance code", _lib.PNG_BAD_CODE), ("too far back", _lib.PNG_FAR),
            ("invalid stored block lengths", _lib.PNG_STORED_LEN), ("incorrect data check", _lib.PNG_ADLER)]


def inflate(stream, H, W):
    """(the H x (W + 1) filtered bytes of the stream, 0) or (None, the DFQ_PNG_* reason).  A stream that ends whole (its
    Adler-32 checked) at the end of an earlier row gives its rows and zeros, as Pillow keeps the rest of its image zero."""
    T = H * (W + 1)
    d = zlib.decompressobj()
    try:
        raw = d.decompress(bytes(stream), T)
    except zlib.error as e:
        return None, next((why for k, why in _REASONS if k in str(e)), -1)
    if len(raw) < T and d.eof and raw and len(raw) % (W + 1) == 0:
        raw += bytes(T - len(raw))
    return (raw, 0) if len(raw) == T else (None, _lib.PNG_SHORT)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def unfilter(raw, H, W):
    """(uint8 [H, W], 0) or (None, DFQ_PNG_BAD_FILTER)."""
    f = np.frombuffer(raw, np.uint8).reshape(H, W + 1)
    out = np.zeros((H, W), np.uint8)
    prev = np.zeros(W, np.int64)
    for y in range(H):
        t, row = int(f[y, 0]), f[y, 1:].astype(np.int64)
        if t > 4:
            return None, _lib.PNG_BAD_FILTER
        if t == 0:
            cur = row
        elif t == 2:
            cur = row + prev
        elif t == 1:
            cur = np.cumsum(row)
        else:
            cur, a, c = np.zeros(W, np.int64), 0, 0
            for x in range(W):
                b = int(prev[x])
                a = (int(row[x]) + ((a + b) >> 1 if t == 3 else _paeth(a, b, c))) & 255
                cur[x], c = a, b
        cur = cur & 255
        out[y], prev = cur, cur
    return out, 0


def decode(data):
    """np.array(Image.open(BytesIO(data))) for the streams the device decoder takes; ValueError for a corrupt one."""
    pos, H, W, parts = 8, None, None, []
    while pos + 8 <= len(data):
        n, cid = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        pos += 12 + n
        if cid == b"IHDR":
            W, H = struct.unpack(">II", body[:8])
        elif cid == b"IDAT":
            parts.append(body)
        elif parts or cid == b"IEND":
            break
    raw, why = inflate(b"".join(parts), H, W)
    if why:
        raise ValueError("corrupt stream (reason %d)" % why)
    img, why = unfilter(raw, H, W)
    if why:
        raise ValueError("corrupt stream (reason %d)" % why)
    return img
