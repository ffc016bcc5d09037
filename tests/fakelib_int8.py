"""tests/fakelib.py's oracle-backed stand-in for libdfq_sm90.so, extended by host twins of the int8 entries
(dfq_i8_quantize_nhwc, dfq_i8_pack_weights, dfq_i8_conv) computed by tests/int8_oracle.py.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so the host path of dfq_b200.int8 (packing
plan, scale choice, module swap) runs without a GPU.
"""
import ctypes as C

import numpy as np

import fakelib
import int8_oracle as I8
from dfq_b200 import _lib
from fakelib import _floats, _table, _val

f32 = np.float32
E_UNSUPPORTED = -2    # DFQ_E_UNSUPPORTED


def _array(ptr, n, dtype):
    return np.frombuffer((C.c_char * (int(n) * np.dtype(dtype).itemsize)).from_address(int(_val(ptr))), dtype=dtype)


def _geometry(g_p):
    """The DfqI8Conv as a dict, or None for a grouping the library refuses."""
    g = _table(g_p, 1, _lib.I8_CONV_DT)[0]
    g = {k: int(g[k]) for k in _lib.I8_CONV_DT.names}
    return g if g["groups"] == 1 or g["groups"] == g["C"] == g["O"] else None


class FakeInt8Lib(fakelib.FakeLib):
    def dfq_i8_quantize_nhwc(self, x_p, q_p, N, Cn, H, W, Cpad, scale, stream):
        self.calls.append("dfq_i8_quantize_nhwc")
        x = _floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W)
        q = _array(q_p, N * H * W * Cpad, np.int8).reshape(N, H, W, Cpad)
        q[...] = 0
        q[..., :Cn] = I8.i8_quantize(x, f32(_val(scale))).transpose(0, 2, 3, 1)
        return 0

    def dfq_i8_pack_weights(self, w_p, ws_p, out_p, g_p, stream):
        self.calls.append("dfq_i8_pack_weights")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        O_, Cn, taps, Cp = g["O"], g["C"], g["kh"] * g["kw"], g["Cpad"]
        codes = I8.i8_quantize(_floats(w_p, O_ * (Cn // g["groups"]) * taps).reshape(O_, -1, taps),
                               _floats(ws_p, O_).reshape(-1, 1, 1))
        if g["groups"] == 1:
            out = _array(out_p, O_ * taps * Cp, np.int8).reshape(O_, taps, Cp)
            out[...] = 0
            out[:, :, :Cn] = codes.transpose(0, 2, 1)
        else:
            out = _array(out_p, taps * Cp, np.int8).reshape(taps, Cp)
            out[...] = 0
            out[:, :Cn] = codes[:, 0, :].T
        return 0

    def dfq_i8_conv(self, xq_p, wq_p, dq_p, b_p, y_p, acc_p, g_p, stream):
        self.calls.append("dfq_i8_conv")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        N, Cn, H, W, O_, kh, kw, Cp = (g[k] for k in ("N", "C", "H", "W", "O", "kh", "kw", "Cpad"))
        xq = _array(xq_p, N * H * W * Cp, np.int8).reshape(N, H, W, Cp)[..., :Cn].transpose(0, 3, 1, 2)
        if g["groups"] == 1:
            wq = _array(wq_p, O_ * kh * kw * Cp, np.int8).reshape(O_, kh, kw, Cp)[..., :Cn].transpose(0, 3, 1, 2)
        else:
            wq = _array(wq_p, kh * kw * Cp, np.int8).reshape(kh, kw, Cp)[..., :Cn].transpose(2, 0, 1)[:, None]
        acc = I8.i8_conv(xq, wq, (g["stride_h"], g["stride_w"]), (g["pad_h"], g["pad_w"]), (g["dil_h"], g["dil_w"]),
                         g["groups"])
        dq = _floats(dq_p, O_).reshape(1, -1, 1, 1)
        bias = (_floats(b_p, O_) if _val(b_p) else np.zeros(O_, f32)).reshape(1, -1, 1, 1)
        y = _floats(y_p, acc.size).reshape(acc.shape)
        y[...] = (acc.astype(f32) * dq).astype(f32) + bias
        if _val(acc_p):
            _array(acc_p, acc.size, np.int32)[...] = acc.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins: returns the fake the patched dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeInt8Lib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
