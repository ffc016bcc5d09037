"""tests/fakelib_preprocess.py's stand-in, extended by a host twin of dfq_jpeg_decode with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.jpeg and dfq_b200.preprocess through it inside a test, so the JPEG
batch packing (the compressed bytes, the table blocks, the restart-interval segments, the decoded images' places in the
blob) runs without a GPU.  The twin walks each segment's bits from the blob with the blob's DfqJpegTables the way
k_jpeg_huff does, then hands the coefficients to tests/jpeg_oracle.py's IDCT, upsampling and colour conversion, so its
output equals Pillow's only if the host path packed the batch right.
"""
import ctypes as C

import numpy as np

import fakelib_preprocess
import jpeg_oracle as O
from dfq_b200 import _lib
from fakelib import _table, _val
from fakelib_preprocess import E_ARG, _bytes


def _walk(data, mcus, comp_of_block, T, coef, at):
    """k_jpeg_huff on one segment: returns 0 or the error reason.  coef: [blocks, 64] natural order, from block `at`."""
    buf = bytearray()
    i = 0
    while i < len(data):                                 # byte stuffing, as the kernel's reader skips it
        buf.append(data[i])
        i += 2 if data[i] == 0xFF else 1
    nbits = len(buf) * 8
    buf += bytes(8)
    pos, pred = 0, [0, 0, 0]

    def peek(n):
        b = pos >> 3
        return (int.from_bytes(buf[b:b + 4], "big") >> (32 - (pos & 7) - n)) & ((1 << n) - 1)

    def symbol(h):
        nonlocal pos
        pk = peek(16)
        e = int(h["look"][pk >> 7])
        if e:
            pos += e >> 8
            return e & 255
        for l in range(10, 17):
            code = pk >> (16 - l)
            if code <= h["maxcode"][l]:
                pos += l
                return int(h["vals"][code + h["valoff"][l]])
        return -1

    def extend(s):
        nonlocal pos
        v = peek(s)
        pos += s
        return v if v >= (1 << (s - 1)) else v - (1 << s) + 1

    for _ in range(mcus):
        for c in comp_of_block:
            t = symbol(T["dc"][c])
            if t < 0 or t > 15:
                return _lib.JPEG_BAD_CODE
            pred[c] = (pred[c] + (extend(t) if t else 0) + 2 ** 31) % 2 ** 32 - 2 ** 31
            coef[at, 0] = (pred[c] + 32768) % 65536 - 32768
            k = 1
            while k < 64:
                rs = symbol(T["ac"][c])
                if rs < 0:
                    return _lib.JPEG_BAD_CODE
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    if k > 63:
                        return _lib.JPEG_BAD_RUN
                    coef[at, O.ZIGZAG[k]] = extend(s)
                elif r == 15:
                    k += 15
                else:
                    break
                k += 1
            at += 1
            if pos > nbits + 64:
                return _lib.JPEG_SHORT_SCAN
    return _lib.JPEG_SHORT_SCAN if pos > nbits else 0


class FakeJpegLib(fakelib_preprocess.FakePreprocessLib):
    def __init__(self, real):
        super().__init__(real)
        self.jpeg_descriptors = None    # the last dfq_jpeg_decode call's (images, segments, DfqJpegDecode)

    def dfq_jpeg_decode(self, d_p, im_p, seg_p, blob_p, err_p, stream):
        self.calls.append("dfq_jpeg_decode")
        d_p, im_p, seg_p, blob_p, err_p = (int(_val(v) or 0) for v in (d_p, im_p, seg_p, blob_p, err_p))
        if not (d_p and im_p and seg_p and blob_p and err_p):
            return self._refuse("NULL pointer")
        d = _table(d_p, 1, _lib.JPEG_DECODE_DT)[0].copy()
        n, nseg, B = int(d["n"]), int(d["nseg"]), int(d["blob_bytes"])
        if not (1 <= n <= 65535 and nseg >= 1 and B >= 1 and int(d["call"]) < 2 ** 31):
            return self._refuse("bad sizes")
        ims = _table(im_p, n, _lib.JPEG_IMAGE_DT).copy()
        segs = _table(seg_p, nseg, _lib.JPEG_SEGMENT_DT).copy()
        TB = _lib.JPEG_TABLES_DT.itemsize
        for m in ims:
            H, W, nc, hs, vs = (int(m[k]) for k in ("H", "W", "ncomp", "hs", "vs"))
            geo = (nc == 1 and hs == vs == 1) or (nc == 3 and (hs, vs) in ((1, 1), (2, 1), (2, 2)))
            geo = geo and 1 <= H <= 65535 and 1 <= W <= 65535 and m["mcux"] == -(-W // (8 * hs)) and m["mcuy"] == -(-H // (8 * vs))
            if not (geo and 0 <= m["tables"] and m["tables"] % 8 == 0 and m["tables"] + TB <= B and 0 <= m["dst"]
                    and m["dst"] + H * W * 3 <= B):
                return self._refuse("image geometry, tables or output")
        nxt = np.zeros(n, np.int64)
        for g in segs:
            i = int(g["image"])
            if not (0 <= i < n and 0 <= g["begin"] <= g["end"] <= B and g["mcus"] >= 1 and g["mcu0"] == nxt[i]
                    and g["mcu0"] + g["mcus"] <= ims[i]["mcux"] * ims[i]["mcuy"]):
                return self._refuse("segment")
            nxt[i] += g["mcus"]
        if (nxt != ims["mcux"].astype(np.int64) * ims["mcuy"]).any():
            return self._refuse("segments do not cover the MCUs")
        if blob_p % 8 or err_p % 8:
            return self._refuse("misaligned pointer")
        self.jpeg_descriptors = (ims, segs, d)
        blob = _bytes(blob_p, B)
        err = np.ctypeslib.as_array((C.c_int64 * 2).from_address(err_p))
        for i, m in enumerate(ims):
            H, W, nc, hs, vs, mx, my = (int(m[k]) for k in ("H", "W", "ncomp", "hs", "vs", "mcux", "mcuy"))
            T = np.frombuffer(blob[m["tables"]:m["tables"] + TB].tobytes(), _lib.JPEG_TABLES_DT)[0]
            layout = [0] * (hs * vs) + ([1, 2] if nc == 3 else [])
            coef = np.zeros((mx * my * len(layout), 64), np.int64)
            for g in segs[segs["image"] == i]:
                why = _walk(blob[g["begin"]:g["end"]].tobytes(), int(g["mcus"]), layout, T, coef,
                            int(g["mcu0"]) * len(layout))
                if why:
                    err[0] = min(int(err[0]), (int(d["call"]) << 32) | i)
                    err[1] |= why
            cm = coef.reshape(my, mx, len(layout), 64)
            planes = [cm[:, :, :hs * vs].reshape(my, mx, vs, hs, 64).transpose(0, 2, 1, 3, 4).reshape(my * vs, mx * hs, 64)]
            planes += [cm[:, :, hs * vs + k] for k in range(nc - 1)]
            planes = [p * T["q"][c][None, None, :] for c, p in enumerate(planes)]
            rgb = O.reconstruct(H, W, hs, vs, planes)
            blob[m["dst"]:m["dst"] + H * W * 3] = rgb.reshape(-1)
        return 0


def install(monkeypatch):
    """fakelib_preprocess.install() with the JPEG twin; the CPU stands in for the device while it is active."""
    from dfq_b200 import jpeg
    real = _lib.load()
    fakelib_preprocess.install(monkeypatch)
    fake = FakeJpegLib(real)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(jpeg, "_state", {})
    return fake
