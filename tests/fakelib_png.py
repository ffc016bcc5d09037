"""tests/fakelib_jpeg.py's stand-in, extended by a host twin of dfq_png_decode with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.png, dfq_b200.jpeg and dfq_b200.preprocess through it inside a test,
so the PNG batch packing (the joined zlib streams, the work rooms and labels past the copied bytes, their offsets in the
descriptors) runs without a GPU.  The twin inflates each stream from the blob with tests/png_oracle.py into its work
room and unfilters it into its output, so the labels equal Pillow's only if the host path packed the batch right.
"""
import ctypes as C

import numpy as np

import fakelib_jpeg
import png_oracle as O
from dfq_b200 import _lib
from fakelib import _table, _val
from fakelib_preprocess import _bytes


class FakePngLib(fakelib_jpeg.FakeJpegLib):
    def __init__(self, real):
        super().__init__(real)
        self.png_descriptors = None     # the last dfq_png_decode call's (images, DfqPngDecode)

    def dfq_png_decode(self, d_p, im_p, blob_p, err_p, stream):
        self.calls.append("dfq_png_decode")
        d_p, im_p, blob_p, err_p = (int(_val(v) or 0) for v in (d_p, im_p, blob_p, err_p))
        if not (d_p and im_p and blob_p and err_p):
            return self._refuse("NULL pointer")
        d = _table(d_p, 1, _lib.PNG_DECODE_DT)[0].copy()
        n, B = int(d["n"]), int(d["blob_bytes"])
        if not (1 <= n <= 65535 and B >= 1 and int(d["call"]) < 2 ** 31) or err_p % 8:
            return self._refuse("bad sizes")
        ims = _table(im_p, n, _lib.PNG_IMAGE_DT).copy()

        def inside(off, size):
            return 0 <= off and 0 <= size <= B - off

        def apart(a, an, b, bn):
            return a + an <= b or b + bn <= a

        for m in ims:
            H, W, src, S, work, dst = (int(m[k]) for k in ("H", "W", "src", "src_end", "work", "dst"))
            S -= src
            px, T = H * W, H * (W + 1)
            if not (H >= 1 and W >= 1 and px < 2 ** 31 and S >= 2 and inside(src, S) and inside(work, T)
                    and inside(dst, px) and apart(src, S, work, T) and apart(src, S, dst, px) and apart(work, T, dst, px)):
                return self._refuse("image geometry, stream, work room or output")
        self.png_descriptors = (ims, d)
        blob = _bytes(blob_p, B)
        err = np.ctypeslib.as_array((C.c_int64 * 2).from_address(err_p))
        for i, m in enumerate(ims):
            H, W = int(m["H"]), int(m["W"])
            raw, why = O.inflate(blob[m["src"]:m["src_end"]].tobytes(), H, W)
            if not why:
                blob[m["work"]:m["work"] + H * (W + 1)] = np.frombuffer(raw, np.uint8)
                img, why = O.unfilter(raw, H, W)
            if why:
                err[0] = min(int(err[0]), (int(d["call"]) << 32) | i)
                err[1] |= why
                continue
            blob[m["dst"]:m["dst"] + H * W] = img.reshape(-1)
        return 0


def install(monkeypatch):
    """fakelib_jpeg.install() with the PNG twin; the CPU stands in for the device while it is active."""
    from dfq_b200 import png
    real = _lib.load()
    fakelib_jpeg.install(monkeypatch)
    fake = FakePngLib(real)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(png, "_state", {})
    return fake
