"""JPEG decoding on the GPU, bit for bit what Pillow's Image.open(...).convert("RGB") and OpenCV's cv2.imdecode + cvtColor
give: both run libjpeg-turbo with the slow-integer IDCT, "fancy" chroma upsampling and the fixed-point YCbCr -> RGB tables,
all integer arithmetic that csrc/jpeg.cu repeats step for step.

Baseline sequential Huffman JPEGs (SOF0 / SOF1) with 8-bit samples, 1 component (gray, replicated into RGB as
convert("RGB") does) or 3 (YCbCr 4:4:4, 4:2:2 or 4:2:0) in one interleaved scan, with any restart interval.  The headers
are parsed here and every unsupported stream is refused by name before any launch; the compressed bytes, the Huffman
and quantisation tables travel to the device with the rest of the batch in one host-to-device copy.

    for items in loader:                 # workers return open(path, "rb").read(); probe() routes odd files to PIL
        x = preprocess.imagenet(items)   # bytes and decoded arrays may be mixed in one batch
    jpeg.check()                         # once per epoch: raises for an entropy-coded segment found corrupt on the device

decode() returns the pixels for users who want them.  Nothing here synchronises with the host except check().
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools
import struct

import numpy as np
import torch

from . import _lib

__all__ = ["probe", "decode", "check", "Probe"]

_ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                    7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                    31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
_SOF_REFUSED = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "differential (hierarchical)",
                0xC6: "differential progressive", 0xC7: "differential lossless", 0xC9: "arithmetic-coded",
                0xCA: "arithmetic-coded progressive", 0xCB: "arithmetic-coded lossless",
                0xCC: "arithmetic-coded (DAC marker)", 0xCD: "arithmetic-coded differential",
                0xCE: "arithmetic-coded differential progressive", 0xCF: "arithmetic-coded differential lossless"}
_SAMPLING = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0"}
_ERRORS = {_lib.JPEG_BAD_CODE: "invalid Huffman code", _lib.JPEG_BAD_RUN: "coefficient run past 63",
           _lib.JPEG_SHORT_SCAN: "scan ends before its last MCU"}


class Refused(Exception):
    """A stream the device decoder does not take; str() is the reason."""


@dataclasses.dataclass(frozen=True)
class Probe:
    """Header facts of one JPEG.  supported is False with the refusal's reason when the device decoder would refuse it (the
    other fields are then None where the header did not give them).  sampling: "gray", "4:4:4", "4:2:2" or "4:2:0";
    orientation: the EXIF orientation tag, 1 when there is none."""
    supported: bool
    reason: str | None
    height: int | None = None
    width: int | None = None
    components: int | None = None
    sampling: str | None = None
    restart_interval: int | None = None
    orientation: int = 1


class _Jpeg:
    """One parsed stream: what the batch packing needs.  shape is the decoded image's (H, W, 3)."""
    __slots__ = ("data", "shape", "ncomp", "hs", "vs", "mcux", "mcuy", "tables", "segments", "orientation", "ri")


# ---- header parsing ----------------------------------------------------------------------------------------------------
def _parse(data) -> _Jpeg:
    if not isinstance(data, (bytes, bytearray, memoryview)):
        raise Refused("not bytes (%s)" % type(data).__name__)
    b = bytes(data) if not isinstance(data, bytes) else data
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise Refused("not a JPEG (no SOI marker)")
    pos, q, huff, frame, ri, jfif, adobe, orient = 2, {}, {}, None, 0, False, None, 1
    while True:
        if pos >= n or b[pos] != 0xFF:
            raise Refused("truncated or corrupt header at byte %d" % pos)
        while pos < n and b[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise Refused("truncated data (header ends at byte %d)" % pos)
        m = b[pos]
        pos += 1
        if m == 0xD9:
            raise Refused("no scan before EOI")
        if m == 0xDC:
            raise Refused("DNL marker (height defined after the scan)")
        if m in _SOF_REFUSED:
            raise Refused("%s JPEG (SOF%d)" % (_SOF_REFUSED[m], m - 0xC0) if m != 0xCC else _SOF_REFUSED[m])
        if m == 0x01 or 0xD0 <= m <= 0xD8:
            raise Refused("unexpected marker 0x%02X in the header" % m)
        if pos + 2 > n:
            raise Refused("truncated data (header ends at byte %d)" % pos)
        ln = (b[pos] << 8) | b[pos + 1]
        if ln < 2 or pos + ln > n:
            raise Refused("truncated data (a 0x%02X segment of %d bytes at byte %d)" % (m, ln, pos))
        body = b[pos + 2:pos + ln]
        pos += ln
        if m == 0xDB:
            _dqt(body, q)
        elif m == 0xC4:
            _dht(body, huff)
        elif m in (0xC0, 0xC1):
            frame = _sof(body)
        elif m == 0xDD:
            if len(body) < 2:
                raise Refused("corrupt DRI segment")
            ri = (body[0] << 8) | body[1]
        elif m == 0xE0:
            jfif = jfif or body[:5] == b"JFIF\0"
        elif m == 0xEE:
            if body[:5] == b"Adobe" and len(body) >= 12:
                adobe = body[11]
        elif m == 0xE1:
            if body[:6] == b"Exif\0\0":
                orient = _exif_orientation(body[6:])
        elif m == 0xDA:
            if frame is None:
                raise Refused("SOS before the frame header")
            return _scan(b, body, pos, frame, q, huff, ri, jfif, adobe, orient)
        # APPn, COM and anything else with a length: skipped


def _dqt(body, q):
    i = 0
    while i < len(body):
        pq, tq = body[i] >> 4, body[i] & 15
        size = 128 if pq else 64
        if pq > 1 or tq > 3 or i + 1 + size > len(body):
            raise Refused("corrupt DQT segment")
        vals = np.frombuffer(body[i + 1:i + 1 + size], ">u2" if pq else np.uint8).astype(np.int32)
        t = np.zeros(64, np.int32)
        t[_ZIGZAG] = vals
        q[tq] = t
        i += 1 + size


def _dht(body, huff):
    i = 0
    while i < len(body):
        if i + 17 > len(body):
            raise Refused("corrupt DHT segment")
        tc, th = body[i] >> 4, body[i] & 15
        counts = bytes(body[i + 1:i + 17])
        total = sum(counts)
        if tc > 1 or th > 3 or total > 256 or i + 17 + total > len(body):
            raise Refused("corrupt DHT segment")
        vals = bytes(body[i + 17:i + 17 + total])
        huff[(tc, th)] = (counts, vals)
        i += 17 + total


def _sof(body):
    if len(body) < 6:
        raise Refused("corrupt SOF segment")
    P, H, W, nc = body[0], (body[1] << 8) | body[2], (body[3] << 8) | body[4], body[5]
    if P != 8:
        raise Refused("%d-bit samples (only 8-bit)" % P)
    if H == 0:
        raise Refused("DNL marker (height defined after the scan)")
    if W == 0:
        raise Refused("zero width")
    if nc not in (1, 3):
        raise Refused("%d components (only 1, gray, or 3, YCbCr%s)" % (nc, "; CMYK / YCCK" if nc == 4 else ""))
    if len(body) < 6 + 3 * nc:
        raise Refused("corrupt SOF segment")
    comps = [(body[6 + 3 * k], body[7 + 3 * k] >> 4, body[7 + 3 * k] & 15, body[8 + 3 * k]) for k in range(nc)]
    if len({c[0] for c in comps}) != nc or any(not (1 <= c[1] <= 4 and 1 <= c[2] <= 4) or c[3] > 3 for c in comps):
        raise Refused("corrupt SOF segment")
    return H, W, comps


def _exif_orientation(t):
    """The orientation tag (0x0112) of IFD0, 1 when absent or unreadable."""
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        return 1
    e = "<" if t[:2] == b"II" else ">"
    ifd = struct.unpack(e + "I", t[4:8])[0]
    if ifd + 2 > len(t):
        return 1
    for k in range(struct.unpack(e + "H", t[ifd:ifd + 2])[0]):
        o = ifd + 2 + 12 * k
        if o + 12 > len(t):
            return 1
        tag, typ = struct.unpack(e + "HH", t[o:o + 4])
        if tag == 0x0112 and typ == 3:
            return struct.unpack(e + "H", t[o + 8:o + 10])[0]
    return 1


def _scan(b, body, start, frame, q, huff, ri, jfif, adobe, orient):
    H, W, comps = frame
    nc = len(comps)
    if nc == 3:
        if not jfif and adobe == 0:
            raise Refused("Adobe transform 0 (RGB-coded, not YCbCr)")
        if not jfif and adobe is None and [c[0] for c in comps] == [82, 71, 66]:
            raise Refused("RGB-coded (component ids R, G, B)")
        if (comps[0][1], comps[0][2]) not in _SAMPLING or any((c[1], c[2]) != (1, 1) for c in comps[1:]):
            raise Refused("sampling %s (only 4:4:4, 4:2:2 and 4:2:0)" % "/".join("%dx%d" % (c[1], c[2]) for c in comps))
    ns = body[0] if body else 0
    if len(body) < 4 + 2 * ns or ns != nc or [body[1 + 2 * k] for k in range(ns)] != [c[0] for c in comps]:
        raise Refused("more than one scan (the first scan does not hold every component in frame order)")
    Ss, Se, A = body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns]
    if Ss != 0 or Se != 63 or A != 0:
        raise Refused("corrupt SOS segment (spectral selection %d..%d, approximation %d)" % (Ss, Se, A))
    sel = [(body[2 + 2 * k] >> 4, body[2 + 2 * k] & 15) for k in range(ns)]
    for c, (td, ta) in zip(comps, sel):
        if c[3] not in q:
            raise Refused("missing table (quantisation table %d)" % c[3])
        if (0, td) not in huff or (1, ta) not in huff:
            raise Refused("missing table (Huffman table DC %d / AC %d)" % (td, ta))
    j = _Jpeg()
    j.data, j.shape, j.ncomp, j.orientation, j.ri = b, (H, W, 3), nc, orient, ri
    j.hs, j.vs = (comps[0][1], comps[0][2]) if nc == 3 else (1, 1)
    j.mcux, j.mcuy = -(-W // (8 * j.hs)), -(-H // (8 * j.vs))
    key = tuple((q[c[3]].tobytes(), huff[(0, td)], huff[(1, ta)]) for c, (td, ta) in zip(comps, sel))
    j.tables = _tables(key)
    j.segments = _segments(b, start, j.mcux * j.mcuy, ri)
    return j


def _segments(b, start, total, ri):
    """[(begin, end)] of the restart intervals' entropy-coded bytes, the RSTn and fill bytes excluded: a marker scan of the
    whole scan, which must end in EOI."""
    a = np.frombuffer(b, np.uint8)[start:]
    ff = np.flatnonzero(a[:-1] == 0xFF)
    nxt = a[ff + 1]
    marks = ff[(nxt != 0) & (nxt != 0xFF)]
    intervals = -(-total // ri) if ri else 1
    segs, lo = [], start
    for p in marks.tolist():
        m = int(a[p + 1])
        end = p
        while end > 0 and a[end - 1] == 0xFF:                # fill bytes before the marker
            end -= 1
        if 0xD0 <= m <= 0xD7:
            if not ri or m != 0xD0 + len(segs) % 8 or len(segs) + 1 >= intervals:
                raise Refused("corrupt scan (RST%d where restart interval %d of %d ends)" % (m - 0xD0, len(segs) + 1, intervals))
            segs.append((lo, start + end))
            lo = start + p + 2
            continue
        if m == 0xD9:
            segs.append((lo, start + end))
            if len(segs) != intervals:
                raise Refused("truncated data (%d of %d restart intervals before EOI)" % (len(segs), intervals))
            return segs
        if m == 0xDC:
            raise Refused("DNL marker (height defined after the scan)")
        raise Refused("more than one scan (marker 0x%02X after the first)" % m)
    raise Refused("truncated data (no EOI after the scan)")


# ---- device tables ---------------------------------------------------------------------------------------------------------
_HUFF_DT, _TABLES_DT = _lib.JPEG_HUFF_DT, _lib.JPEG_TABLES_DT


def _huff(counts, vals, dc):
    """libjpeg's jpeg_make_d_derived_tbl: maxcode / valoffset per code length and a 9-bit lookahead (len << 8 | symbol)."""
    t = np.zeros((), _HUFF_DT)
    t["maxcode"][:] = -1
    code, k = 0, 0
    for l in range(1, 17):
        if counts[l - 1]:
            t["valoff"][l] = k - code
            code += counts[l - 1]
            k += counts[l - 1]
            t["maxcode"][l] = code - 1
            if code >= (1 << l):                      # libjpeg: no code may be all ones, so the last must stay below
                raise Refused("bad Huffman table (full at length %d: a code of all ones)" % l)
        code <<= 1
    t["maxcode"][17] = 0xFFFFF
    t["vals"][:len(vals)] = np.frombuffer(vals, np.uint8)
    if dc and any(v > 15 for v in vals):
        raise Refused("bad Huffman table (DC category above 15)")
    code, k = 0, 0
    for l in range(1, 10):
        for _ in range(counts[l - 1]):
            lo = code << (9 - l)
            t["look"][lo:lo + (1 << (9 - l))] = (l << 8) | vals[k]
            code += 1
            k += 1
        code <<= 1
    return t


@functools.lru_cache(maxsize=256)
def _tables(key):
    """The DfqJpegTables block of one (quantisation, DC, AC) table triple per component; streams from one encoder share
    it, and the batch packing places a shared block once."""
    t = np.zeros(1, _TABLES_DT)
    for c, (qb, dc, ac) in enumerate(key):
        t["q"][0, c] = np.frombuffer(qb, np.int32)
        t["dc"][0, c] = _huff(*dc, True)
        t["ac"][0, c] = _huff(*ac, False)
    a = t.view(np.uint8)
    a.setflags(write=False)
    return a


# ---- public interface ------------------------------------------------------------------------------------------------------
def probe(data) -> Probe:
    """Header facts of one JPEG, or the reason the device decoder would refuse it; never raises."""
    try:
        j = _parse(data)
    except Refused as e:
        return Probe(False, str(e))
    return Probe(True, None, j.shape[0], j.shape[1], j.ncomp, _SAMPLING[(j.hs, j.vs)] if j.ncomp == 3 else "gray",
                 j.ri, j.orientation)


def parse(items, what="images"):
    """Each bytes item parsed (a DfqError names the first refused one); other items are returned as they are."""
    out = []
    for i, a in enumerate(items):
        if isinstance(a, (bytes, bytearray, memoryview)):
            try:
                a = _parse(a)
            except Refused as e:
                raise _lib.DfqError("%s[%d]: %s" % (what, i, e)) from None
        out.append(a)
    return out


def decode(items) -> list:
    """uint8 [H, W, 3] device tensors, one per JPEG of items (a list of bytes), each equal to Pillow's
    np.asarray(Image.open(BytesIO(b)).convert("RGB")).  One host-to-device copy, and no host synchronisation; a corrupt
    entropy-coded segment is reported by the next check().  The tensors are views of one device block."""
    from . import preprocess
    if isinstance(items, (bytes, bytearray, memoryview)) or not hasattr(items, "__len__") or len(items) == 0:
        raise _lib.DfqError("decode takes a non-empty list of JPEG bytes")
    js = parse(items, "items")
    for i, j in enumerate(js):
        if not isinstance(j, _Jpeg):
            raise _lib.DfqError("items[%d] is %s, not JPEG bytes" % (i, type(j).__name__))
    stage = preprocess._Stage()
    batch = _Batch(stage)
    ks = [batch.add(j) for j in js]
    blob = stage.upload(batch.extra)
    batch.launch(blob)
    return [blob[batch.dst(k):batch.dst(k) + j.shape[0] * j.shape[1] * 3].view(j.shape) for k, j in zip(ks, js)]


def check(device=None) -> None:
    """Wait for the device decodes enqueued so far on device (default: every device used) and raise DfqError for the first
    corrupt entropy-coded segment found since the last check().  The image's pixels are unspecified; the rest of its batch
    is decoded."""
    devs = [torch.device(device)] if device is not None else list(_state)
    for dev in devs:
        st = _state.get(dev)
        if st is None:
            continue
        w = st["word"].cpu().tolist()
        calls = st["calls"]
        st["word"].copy_(torch.tensor(_CLEAR), non_blocking=False)
        st["calls"] = 0
        if w[0] != _CLEAR[0]:
            call, image = w[0] >> 32, w[0] & 0xFFFFFFFF
            why = ", ".join(v for k, v in _ERRORS.items() if w[1] & k) or "error 0x%x" % w[1]
            raise _lib.DfqError("jpeg: corrupt entropy-coded data in image %d of decode call %d of %d since the last "
                                "check() on %s: %s" % (image, call + 1, calls, dev, why))


# ---- batch packing and launch ---------------------------------------------------------------------------------------------
_CLEAR = [(1 << 63) - 1, 0]
_state = {}       # device -> {"word": int64 [2] (first corrupt (call << 32 | image), reason bits), "calls": decodes since check}


class _Batch:
    """The JPEGs of one batch placed in a staging block: their bytes and tables in the copied part, their pixels in
    `extra` bytes that only the device block has, past the copied ones."""

    def __init__(self, stage):
        self.stage, self.images, self.segs, self.extra, self.pending = stage, [], [], 0, []

    def add(self, j):
        """Place j; returns its index in the batch."""
        data = np.frombuffer(j.data, np.uint8)
        base = self.stage.place(data)
        k = len(self.images)
        step = j.ri if j.ri else j.mcux * j.mcuy
        for s, (lo, hi) in enumerate(j.segments):
            self.segs.append((base + lo, base + hi, k, s * step, min(step, j.mcux * j.mcuy - s * step)))
        self.pending.append(self.extra)
        self.extra += (j.shape[0] * j.shape[1] * 3 + 63) // 64 * 64
        self.images.append((j, self.stage.table(j.tables)))
        return k

    def dst(self, k):
        """Byte offset of image k's pixels in the device block, once the batch's last segment is placed."""
        return self.stage.total + self.pending[k]

    def launch(self, blob):
        lib = _lib.load()
        im = np.zeros(len(self.images), _lib.JPEG_IMAGE_DT)
        for k, (j, tab) in enumerate(self.images):
            im[k]["dst"], im[k]["tables"] = self.dst(k), tab
            im[k]["H"], im[k]["W"] = j.shape[:2]
            im[k]["ncomp"], im[k]["hs"], im[k]["vs"], im[k]["mcux"], im[k]["mcuy"] = j.ncomp, j.hs, j.vs, j.mcux, j.mcuy
        sg = np.zeros(len(self.segs), _lib.JPEG_SEGMENT_DT)
        if self.segs:
            a = np.array(self.segs, np.int64)
            sg["begin"], sg["end"], sg["image"], sg["mcu0"], sg["mcus"] = a.T
        dev = blob.device
        st = _state.get(dev)
        if st is None:
            st = _state[dev] = {"word": torch.tensor(_CLEAR, dtype=torch.int64, device=dev), "calls": 0}
        p = np.zeros(1, _lib.JPEG_DECODE_DT)
        p["n"], p["nseg"], p["blob_bytes"], p["call"] = len(self.images), len(self.segs), blob.numel(), st["calls"]
        st["calls"] += 1
        _lib.check(lib.dfq_jpeg_decode(_lib.table_ptr(p), _lib.table_ptr(im), _lib.table_ptr(sg),
                                       C.c_void_p(blob.data_ptr()), C.c_void_p(st["word"].data_ptr()),
                                       _lib.stream_ptr()), "dfq_jpeg_decode")
