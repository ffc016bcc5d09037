"""tests/fakelib_int8.py's stand-in extended by host twins of dfq_i8_pack_codes, dfq_i8_unpack_codes and dfq_i8_plane_mean
(the rule of ncnn_oracle.plane_mean), with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so ncnn.load / ncnn.write run their host
path (parsing, refusals, module construction, the files written) without a GPU.
"""
import numpy as np

import fakelib
import fakelib_int8
import ncnn_oracle
from dfq_b200 import _lib
from fakelib import _floats, _val
from fakelib_int8 import _array, _geometry

E_ARG = -1


class FakeNcnnLib(fakelib_int8.FakeInt8Lib):
    def _refuse(self, who, rc, msg):
        self.error = "%s: %s" % (who, msg)
        return rc

    def dfq_last_error(self):
        return getattr(self, "error", "").encode()

    def _layout(self, g_p, who, a_p, b_p):
        g = _geometry(g_p)
        if g is None:
            return None, fakelib_int8.E_UNSUPPORTED
        if not _val(a_p) or not _val(b_p):
            return None, self._refuse(who, E_ARG, "null pointer")
        return g, 0

    def dfq_i8_pack_codes(self, codes_p, out_p, g_p, stream):
        who = "dfq_i8_pack_codes"
        self.calls.append(who)
        g, rc = self._layout(g_p, who, codes_p, out_p)
        if rc:
            return rc
        O_, Cn, taps, Cp = g["O"], g["C"], g["kh"] * g["kw"], g["Cpad"]
        codes = _array(codes_p, O_ * (Cn // g["groups"]) * taps, np.int8).reshape(O_, -1, taps)
        if g["groups"] == 1:
            out = _array(out_p, O_ * taps * Cp, np.int8).reshape(O_, taps, Cp)
            out[...] = 0
            out[:, :, :Cn] = codes.transpose(0, 2, 1)
        else:
            out = _array(out_p, taps * Cp, np.int8).reshape(taps, Cp)
            out[...] = 0
            out[:, :Cn] = codes[:, 0, :].T
        return 0

    def dfq_i8_unpack_codes(self, packed_p, codes_p, g_p, stream):
        who = "dfq_i8_unpack_codes"
        self.calls.append(who)
        g, rc = self._layout(g_p, who, packed_p, codes_p)
        if rc:
            return rc
        O_, Cn, taps, Cp = g["O"], g["C"], g["kh"] * g["kw"], g["Cpad"]
        codes = _array(codes_p, O_ * (Cn // g["groups"]) * taps, np.int8).reshape(O_, -1, taps)
        if g["groups"] == 1:
            codes[...] = _array(packed_p, O_ * taps * Cp, np.int8).reshape(O_, taps, Cp)[:, :, :Cn].transpose(0, 2, 1)
        else:
            codes[:, 0, :] = _array(packed_p, taps * Cp, np.int8).reshape(taps, Cp)[:, :Cn].T
        return 0

    def dfq_i8_plane_mean(self, x_p, y_p, yq_p, N, Cn, P, divide, out_scale, stream):
        who = "dfq_i8_plane_mean"
        self.calls.append(who)
        if not _val(x_p):
            return self._refuse(who, E_ARG, "null input")
        if not _val(y_p) and not _val(yq_p):
            return self._refuse(who, E_ARG, "no output requested (y and yq are both NULL)")
        if N <= 0 or Cn <= 0 or P <= 0:
            return self._refuse(who, E_ARG, "empty dimension")
        if divide not in (0, 1):
            return self._refuse(who, E_ARG, "divide must be 0 or 1")
        s = np.float32(_val(out_scale))
        if _val(yq_p) and not (np.isfinite(s) and s >= 0):
            return self._refuse(who, E_ARG, "out_scale must be finite and non-negative when yq is written")
        v = ncnn_oracle.plane_mean(_floats(x_p, N * Cn * P).reshape(N, Cn, P), bool(divide))
        if _val(y_p):
            _floats(y_p, N * Cn)[...] = v.reshape(-1)
        if _val(yq_p):
            cp = (Cn + 15) // 16 * 16
            q = _array(yq_p, N * cp, np.int8).reshape(N, cp)
            q[...] = 0
            q[:, :Cn] = ncnn_oracle.q8(v, s)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 and ncnn twins: returns the fake the patched dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeNcnnLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
