"""Oracle of the requantizing int8 epilogue (dfq_i8_conv_requant) and its host twin  --  TEST INFRASTRUCTURE.

i8_requantize restates, on top of tests/int8_oracle.py, what the per-layer path computes between two chained layers: the
dequantizing epilogue, the activation as one clamp that keeps NaN (torch's relu / hardtanh), and the quantizer at the next
layer's scale.  FakeChainLib adds the host twin of dfq_i8_conv_requant to tests/fakelib_int8.py's FakeInt8Lib.
"""
import numpy as np

import fakelib
import fakelib_int8
import int8_oracle as I8
from dfq_b200 import _lib
from fakelib import _floats, _val
from fakelib_int8 import E_UNSUPPORTED, _array, _geometry

f32 = np.float32
E_ARG = -1            # DFQ_E_ARG


def i8_clamp(v, lo, hi):
    """v < lo ? lo : (v > hi ? hi : v) in fp32: a NaN stays NaN."""
    v, lo, hi = np.asarray(v, f32), f32(lo), f32(hi)
    return np.where(v < lo, lo, np.where(v > hi, hi, v)).astype(f32)


def i8_requantize(acc, act_scale, w_scale, bias, out_scale, lo, hi):
    """The next layer's codes [N, O, ...] from the int32 sums: i8_dequant, the clamp (lo, hi), i8_quantize at out_scale."""
    return I8.i8_quantize(i8_clamp(I8.i8_dequant(acc, act_scale, w_scale, bias), lo, hi), f32(out_scale))


def to_nhwc_codes(codes):
    """[N, O, H, W] codes -> [N, H, W, round_up(O, 16)] with zero pad channels, the layout dfq_i8_conv_requant writes."""
    N, O_, H, W = codes.shape
    out = np.zeros((N, H, W, (O_ + 15) // 16 * 16), np.int8)
    out[..., :O_] = codes.transpose(0, 2, 3, 1)
    return out


class FakeChainLib(fakelib_int8.FakeInt8Lib):
    def dfq_i8_conv_requant(self, xq_p, wq_p, dq_p, b_p, yq_p, out_scale, lo, hi, g_p, stream):
        self.calls.append("dfq_i8_conv_requant")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        s, lo, hi = f32(_val(out_scale)), f32(_val(lo)), f32(_val(hi))
        if np.isnan(lo) or np.isnan(hi) or lo > hi or not np.isfinite(s) or s < 0 or int(_val(yq_p)) % 16:
            return E_ARG
        N, O_ = g["N"], g["O"]
        OH, OW = g["OH"], g["OW"]
        y = np.empty(N * O_ * OH * OW, f32)
        rc = self.dfq_i8_conv(xq_p, wq_p, dq_p, b_p, y.ctypes.data, None, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        codes = I8.i8_quantize(i8_clamp(y.reshape(N, O_, OH, OW), lo, hi), s)
        out = to_nhwc_codes(codes)
        _array(yq_p, out.size, np.int8)[...] = out.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins and dfq_i8_conv_requant's: returns the fake dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeChainLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
