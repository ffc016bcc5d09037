"""Oracle of the pixel-major fp32 epilogue (dfq_i8_conv_nhwc) and its host twin  --  TEST INFRASTRUCTURE.

i8_rows restates what the per-layer path computes for one detection head: the dequantizing epilogue, the pass-throughs as
one clamp that keeps NaN (tests/int8_residual_oracle.py's i8_epilogue_value without a residual), then
`permute(0, 2, 3, 1).contiguous()` flattened per image.  FakeLayoutLib adds the host twin of the entry, with its refusals, to
tests/int8_upsample_oracle.py's FakeUpsampleLib.
"""
import numpy as np

import fakelib
import int8_residual_oracle as RO
import int8_upsample_oracle as UO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import E_UNSUPPORTED, _geometry

f32 = np.float32
E_ARG = UO.E_ARG


def i8_rows(y, pre=RO.NONE, post=RO.NONE):
    """[N, OH * OW * O]: the clamped fp32 output y [N, O, OH, OW] laid out pixel-major per image."""
    v = RO.i8_epilogue_value(np.asarray(y, f32), None, pre, post)
    return np.ascontiguousarray(v.transpose(0, 2, 3, 1)).reshape(v.shape[0], -1)


class FakeLayoutLib(UO.FakeUpsampleLib):
    def dfq_i8_conv_nhwc(self, xq_p, wq_p, dq_p, b_p, e_p, off, img_stride, g_p, stream):
        self.calls.append("dfq_i8_conv_nhwc")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        e = _table(e_p, 1, _lib.I8_EPILOGUE_DT)[0]
        off, stride = int(_val(off)), int(_val(img_stride))
        r_p, y_p, yq_p = int(e["residual"]), int(e["y"]), int(e["yq"])
        N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
        ext = OH * OW * O_
        xq_p, nx = int(_val(xq_p)), N * g["H"] * g["W"] * g["Cpad"]
        if not y_p or y_p % 4 or r_p or yq_p or not RO._ordered(e["pre_lo"], e["pre_hi"]) or \
                not RO._ordered(e["post_lo"], e["post_hi"]) or off < 0 or stride < off + ext or \
                RO._overlap(xq_p, nx, y_p + 4 * off, 4 * ((N - 1) * stride + ext)):
            return E_ARG
        y = np.empty(N * ext, f32)
        rc = self.dfq_i8_conv(xq_p, wq_p, dq_p, b_p, y.ctypes.data, None, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        rows = i8_rows(y.reshape(N, O_, OH, OW), (e["pre_lo"], e["pre_hi"]), (e["post_lo"], e["post_hi"]))
        out = _floats(y_p, (N - 1) * stride + off + ext)
        for n in range(N):
            out[n * stride + off:n * stride + off + ext] = rows[n]
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins up to the pixel-major epilogue's: returns the fake dfq_b200._lib.load() hands
    out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeLayoutLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
