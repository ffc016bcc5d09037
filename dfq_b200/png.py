"""PNG label decoding on the GPU, bit for bit what np.array(Image.open(BytesIO(b))) gives for segmentation labels.

Non-interlaced streams of 8-bit palette indices (colour type 3: VOC's SegmentationClass, the palette never applied) or
8-bit gray (colour type 0: SegmentationClassAug, cv2.imwrite) come back from Pillow as a uint8 HW array, which is what
preprocess.voc_segmentation takes as labels.  The chunks are walked here, with Pillow's CRC check on every chunk before the
first IDAT, and every other stream is refused by name before any launch; the IDAT payloads are joined into one zlib stream
that travels to the device with the rest of the batch in one host-to-device copy, and csrc/png.cu inflates and unfilters
it there.

    for images, labels in loader:                               # workers return open(path, "rb").read() for both
        x, y = preprocess.voc_segmentation(images, labels)      # JPEG and PNG bytes, mixed with arrays if need be
    png.check()                                                 # once per epoch: raises for a stream found corrupt

decode() returns the labels for users who want them.  Nothing here synchronises with the host except check().
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import struct
import zlib

import numpy as np
import torch

from . import _lib

__all__ = ["probe", "parse", "decode", "check", "Probe"]

_SIG = b"\x89PNG\r\n\x1a\n"
MAX_PIXELS = 89478485              # PIL.Image.MAX_IMAGE_PIXELS: Pillow warns above it and refuses above twice it
_COLOUR = {0: "gray", 2: "RGB", 3: "palette", 4: "gray+alpha", 6: "RGBA"}
_ERRORS = {_lib.PNG_BAD_BLOCK: "invalid block type", _lib.PNG_BAD_CODESET: "invalid code-length, literal/length or "
           "distance code set", _lib.PNG_BAD_CODE: "invalid literal/length or distance code",
           _lib.PNG_FAR: "distance too far back", _lib.PNG_STORED_LEN: "stored block length mismatch",
           _lib.PNG_SHORT: "stream ends before the last row", _lib.PNG_BAD_FILTER: "filter type above 4",
           _lib.PNG_ADLER: "Adler-32 mismatch"}


class Refused(Exception):
    """A stream the device decoder does not take; str() is the reason."""


@dataclasses.dataclass(frozen=True)
class Probe:
    """Header facts of one PNG.  supported is False with the refusal's reason when the device decoder would refuse it (the
    other fields are then None where the header did not give them).  colour_type: 0 gray or 3 palette for supported
    streams."""
    supported: bool
    reason: str | None
    height: int | None = None
    width: int | None = None
    colour_type: int | None = None


class _Png:
    """One parsed stream: what the batch packing needs.  shape is the decoded label's (H, W); stream the joined IDAT
    payloads (the zlib stream, its header included) as a uint8 array."""
    __slots__ = ("shape", "colour_type", "stream")


# ---- chunk walk ----------------------------------------------------------------------------------------------------------
def _ihdr(body):
    if len(body) != 13:
        raise Refused("corrupt header chunk (IHDR of %d bytes)" % len(body))
    W, H, depth, ctype, comp, filt, interlace = struct.unpack(">IIBBBBB", body)
    if W == 0 or H == 0 or W > 2 ** 31 - 1 or H > 2 ** 31 - 1:
        raise Refused("corrupt header chunk (%d x %d)" % (H, W))
    if ctype in (2, 4, 6):
        raise Refused("%s (colour type %d): only 8-bit palette or gray labels" % (_COLOUR[ctype], ctype))
    if ctype not in (0, 3) or depth not in ((1, 2, 4, 8, 16) if ctype == 0 else (1, 2, 4, 8)):
        raise Refused("corrupt header chunk (colour type %d at bit depth %d)" % (ctype, depth))
    if depth == 16:
        raise Refused("16-bit samples")
    if depth < 8:
        raise Refused("%s below 8 bits (%d-bit)" % ("gray" if ctype == 0 else "palette", depth))
    if comp != 0:
        raise Refused("compression method %d (only 0)" % comp)
    if filt != 0:
        raise Refused("filter method %d (only 0)" % filt)
    if interlace:
        raise Refused("interlaced (Adam7)" if interlace == 1 else "corrupt header chunk (interlace method %d)" % interlace)
    if H * W > MAX_PIXELS:
        raise Refused("%d x %d: more pixels than Pillow's decompression-bomb limit (%d)" % (H, W, MAX_PIXELS))
    return H, W, ctype


def _parse(data) -> _Png:
    if not isinstance(data, (bytes, bytearray, memoryview)):
        raise Refused("not bytes (%s)" % type(data).__name__)
    b = bytes(data) if not isinstance(data, bytes) else data
    n = len(b)
    if b[:8] != _SIG:
        raise Refused("not a PNG (no PNG signature)")
    pos, head, idat, run = 8, None, [], 0              # run: 0 before the IDATs, 1 in them, 2 after them
    while pos < n:
        if pos + 8 > n:
            if run:
                break                                      # Pillow stops at a cut-off chunk header after the IDATs
            raise Refused("truncated (a chunk header at byte %d)" % pos)
        length, cid = struct.unpack(">I4s", b[pos:pos + 8])
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in cid):
            raise Refused("corrupt chunk type %r at byte %d" % (cid, pos))
        if length > 2 ** 31 - 1 or pos + 12 + length > n:
            raise Refused("truncated (a %s chunk of %d bytes at byte %d)" % (cid.decode(), length, pos))
        body = b[pos + 8:pos + 8 + length]
        crc = struct.unpack(">I", b[pos + 8 + length:pos + 12 + length])[0]
        if not run and cid != b"IDAT" and crc != zlib.crc32(cid + body):
            raise Refused("corrupt header chunk (bad CRC in %s)" % cid.decode())
        pos += 12 + length
        if head is None:
            if cid != b"IHDR":
                raise Refused("corrupt header chunk (%s before IHDR)" % cid.decode())
            head = _ihdr(body)
        elif cid == b"IDAT":
            if run == 2:
                raise Refused("IDATs are not consecutive")
            run = 1
            idat.append(body)
        elif cid == b"IEND":
            break
        elif cid == b"acTL" and not run:
            raise Refused("APNG (acTL chunk)")
        elif cid == b"IHDR":
            raise Refused("corrupt header chunk (a second IHDR)")
        elif run == 1:
            run = 2
    if head is None:
        raise Refused("truncated (no IHDR)")
    if not run:
        raise Refused("no IDAT")
    stream = b"".join(idat)
    if len(stream) < 2:
        raise Refused("corrupt zlib header (a stream of %d bytes)" % len(stream))
    cmf, flg = stream[0], stream[1]
    if (cmf << 8 | flg) % 31 or cmf & 15 != 8 or cmf >> 4 > 7:
        raise Refused("corrupt zlib header (%02X %02X)" % (cmf, flg))
    if flg & 0x20:
        raise Refused("preset dictionary (zlib FDICT)")
    p = _Png()
    p.shape, p.colour_type = head[:2], head[2]
    p.stream = np.frombuffer(stream, np.uint8)
    return p


# ---- public interface ------------------------------------------------------------------------------------------------------
def probe(data) -> Probe:
    """Header facts of one PNG, or the reason the device decoder would refuse it; never raises."""
    try:
        p = _parse(data)
    except Refused as e:
        return Probe(False, str(e))
    return Probe(True, None, p.shape[0], p.shape[1], p.colour_type)


def parse(items, what="labels"):
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
    """uint8 [H, W] device tensors, one per PNG of items (a list of bytes), each equal to np.array(Image.open(BytesIO(b))).
    One host-to-device copy, and no host synchronisation; a corrupt stream is reported by the next check().  The tensors
    are views of one device block."""
    from . import preprocess
    if isinstance(items, (bytes, bytearray, memoryview)) or not hasattr(items, "__len__") or len(items) == 0:
        raise _lib.DfqError("decode takes a non-empty list of PNG bytes")
    ps = parse(items, "items")
    for i, p in enumerate(ps):
        if not isinstance(p, _Png):
            raise _lib.DfqError("items[%d] is %s, not PNG bytes" % (i, type(p).__name__))
    _lib.require_cuda()
    stage = preprocess._Stage()
    batch = _Batch(stage)
    ks = [batch.add(p) for p in ps]
    blob = stage.upload(batch.extra)
    batch.launch(blob)
    return [blob[batch.dst(k):batch.dst(k) + p.shape[0] * p.shape[1]].view(p.shape) for k, p in zip(ks, ps)]


def check(device=None) -> None:
    """Wait for the device decodes enqueued so far on device (default: every device used) and raise DfqError for the first
    corrupt stream found since the last check().  That image's label is unspecified; the rest of its batch is decoded.  The
    reasons name every fault found in that image: a row with a bad filter type can precede a fault in the compressed data."""
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
            raise _lib.DfqError("png: corrupt compressed data in image %d of decode call %d of %d since the last check() "
                                "on %s: %s" % (image, call + 1, calls, dev, why))


# ---- batch packing and launch ---------------------------------------------------------------------------------------------
_CLEAR = [(1 << 63) - 1, 0]
_state = {}       # device -> {"word": int64 [2] (first corrupt (call << 32 | image), reason bits), "calls": decodes since check}


def _round(n):
    return (n + 63) // 64 * 64


class _Batch:
    """The PNGs of one batch placed in a staging block: their zlib streams in the copied part; their filtered scanlines
    and labels in `extra` bytes that only the device block has, from `base` past the copied ones (room other decoders of
    the batch place before it)."""

    def __init__(self, stage):
        self.stage, self.images, self.extra, self.base = stage, [], 0, 0

    def add(self, p):
        """Place p; returns its index in the batch."""
        H, W = p.shape
        src = self.stage.place(p.stream)
        work = self.extra
        dst = work + _round(H * (W + 1))
        self.extra = dst + _round(H * W)
        self.images.append((p, src, work, dst))
        return len(self.images) - 1

    def dst(self, k):
        """Byte offset of image k's label in the device block, once the batch's last segment is placed."""
        return self.stage.total + self.base + self.images[k][3]

    def launch(self, blob):
        lib = _lib.load()
        im = np.zeros(len(self.images), _lib.PNG_IMAGE_DT)
        at = self.stage.total + self.base
        for k, (p, src, work, dst) in enumerate(self.images):
            im[k]["src"], im[k]["src_end"] = src, src + p.stream.nbytes
            im[k]["work"], im[k]["dst"] = at + work, at + dst
            im[k]["H"], im[k]["W"] = p.shape
        dev = blob.device
        st = _state.get(dev)
        if st is None:
            st = _state[dev] = {"word": torch.tensor(_CLEAR, dtype=torch.int64, device=dev), "calls": 0}
        d = np.zeros(1, _lib.PNG_DECODE_DT)
        d["n"], d["blob_bytes"], d["call"] = len(self.images), blob.numel(), st["calls"]
        st["calls"] += 1
        _lib.check(lib.dfq_png_decode(_lib.table_ptr(d), _lib.table_ptr(im), C.c_void_p(blob.data_ptr()),
                                      C.c_void_p(st["word"].data_ptr()), _lib.stream_ptr()), "dfq_png_decode")
