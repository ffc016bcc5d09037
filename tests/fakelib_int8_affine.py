"""tests/fakelib_int8.py's stand-in for libdfq_sm90.so, extended by host twins of the affine int8 entries
(dfq_i8_affine_quantize, dfq_i8_affine_pack, dfq_i8_affine_conv) computed by tests/int8_affine_oracle.py.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so the host path of
dfq_b200.int8.convert_affine (plan, weight-grid search, refusals, module swap) runs without a GPU.
"""
import math

import numpy as np

import fakelib
import fakelib_int8
import int8_affine_oracle as A
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import _array, _geometry

f32 = np.float32
E_ARG, E_UNSUPPORTED = -1, -2


def _refused(g, bits):
    if g is None or bits > 8:
        return E_UNSUPPORTED
    if bits < 1:
        return E_ARG
    return E_UNSUPPORTED if g["kh"] * g["kw"] * (g["C"] // g["groups"]) >= 131072 else 0


class FakeAffineLib(fakelib_int8.FakeInt8Lib):
    def dfq_i8_affine_quantize(self, x_p, q_p, S_p, N, Cn, H, W, Cpad, act_min, act_max, bits, stream):
        self.calls.append("dfq_i8_affine_quantize")
        if not 1 <= bits <= 8:
            return E_UNSUPPORTED if bits > 8 else E_ARG
        lo, hi = _val(act_min), _val(act_max)
        _, ma, fa, ra, _ = A.act_scalars(lo, hi, bits)
        if not all(math.isfinite(v) for v in (lo, hi, fa, ra)):
            return E_ARG
        q, S = A.act_codes(_floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W), lo, hi, bits)
        out = _array(q_p, N * H * W * Cpad, np.int8).reshape(N, H, W, Cpad)
        out[...] = 0
        out[..., :Cn] = q.transpose(0, 2, 3, 1)
        _array(S_p, N * H * W, np.int32)[...] = S.reshape(-1)
        return 0

    def dfq_i8_affine_pack(self, w_p, w_min, w_scale, bits, out_p, table_p, nbad_p, g_p, stream):
        self.calls.append("dfq_i8_affine_pack")
        g = _geometry(g_p)
        rc = _refused(g, bits)
        if rc:
            return rc
        mn, s = _val(w_min), _val(w_scale)
        if not (math.isfinite(mn) and math.isfinite(s) and s > 0):
            return E_ARG
        O_, Cn, kh, kw, Cp = g["O"], g["C"], g["kh"], g["kw"], g["Cpad"]
        Cg = Cn // g["groups"]
        codes, bad = A.weight_codes(_floats(w_p, O_ * Cg * kh * kw).reshape(O_, Cg, kh, kw), mn, s, bits)
        if g["groups"] == 1:
            out = _array(out_p, O_ * kh * kw * Cp, np.int8).reshape(O_, kh, kw, Cp)
            out[...] = 0
            out[..., :Cn] = codes.transpose(0, 2, 3, 1)
            _array(table_p, O_ * (kh + 1) * (kw + 1), np.int32)[...] = A.tap_table(codes).reshape(-1)
        else:
            out = _array(out_p, kh * kw * Cp, np.int8).reshape(kh * kw, Cp)
            out[...] = 0
            out[:, :Cn] = codes.reshape(Cn, kh * kw).T
        _array(nbad_p, 1, np.int32)[0] = bad
        return 0

    def dfq_i8_affine_conv(self, xq_p, S_p, wq_p, table_p, k_p, b_p, y_p, acc_p, g_p, stream):
        self.calls.append("dfq_i8_affine_conv")
        g = _geometry(g_p)
        rc = _refused(g, 8)
        if rc:
            return rc
        k = _table(k_p, 1, _lib.I8_AFFINE_DT)[0]
        k = tuple(float(k[f]) for f in ("kP", "kA", "kW", "kN"))
        if not all(math.isfinite(v) for v in k):
            return E_ARG
        N, Cn, H, W, O_, kh, kw, Cp = (g[key] for key in ("N", "C", "H", "W", "O", "kh", "kw", "Cpad"))
        xq = _array(xq_p, N * H * W * Cp, np.int8).reshape(N, H, W, Cp)[..., :Cn].transpose(0, 3, 1, 2)
        if g["groups"] == 1:
            wq = _array(wq_p, O_ * kh * kw * Cp, np.int8).reshape(O_, kh, kw, Cp)[..., :Cn].transpose(0, 3, 1, 2)
        else:
            wq = _array(wq_p, kh * kw * Cp, np.int8).reshape(kh, kw, Cp)[..., :Cn].transpose(2, 0, 1)[:, None]
        P, Ax, Wv, Nv = A.terms(xq, wq, (g["stride_h"], g["stride_w"]), (g["pad_h"], g["pad_w"]),
                                (g["dil_h"], g["dil_w"]), g["groups"])
        bias = _floats(b_p, O_) if _val(b_p) else None
        y = _floats(y_p, P.size).reshape(P.shape)
        y[...] = A.epilogue(P, Ax, Wv, Nv, k, bias)
        if _val(acc_p):
            _array(acc_p, P.size, np.int32)[...] = P.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 and affine twins: returns the fake the patched dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeAffineLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
