"""tests/fakelib_int8_affine.py's stand-in for libdfq_sm90.so, extended by the host twin of dfq_i8_affine_conv_fused
computed by tests/int8_affine_chain_oracle.py, with the entry's refusals.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so dfq_b200.int8.chain_affine's graph rules
and its chained layers run without a GPU (with torch told that CPU tensors are on the GPU).
"""
import math

import numpy as np

import fakelib
import fakelib_int8_affine
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A
from dfq_b200 import _lib
from fakelib import _floats, _table
from fakelib_int8 import _array, _geometry
from fakelib_int8_affine import E_ARG, E_UNSUPPORTED

f32 = np.float32


def _ordered(lo, hi):
    return not (np.isnan(lo) or np.isnan(hi)) and lo <= hi


def _overlap(a, na, b, nb):
    return bool(a and b and a < b + nb and b < a + na)


class FakeAffineChainLib(fakelib_int8_affine.FakeAffineLib):
    def dfq_i8_affine_conv_fused(self, xq_p, S_p, wq_p, table_p, k_p, b_p, e_p, g_p, stream):
        self.calls.append("dfq_i8_affine_conv_fused")
        g = _geometry(g_p)
        e = _table(e_p, 1, _lib.I8_AFFINE_EPILOGUE_DT)[0]
        r_p, y_p, yq_p, s_p = (int(e[f]) for f in ("residual", "y", "yq", "S"))
        bits = int(e["out_bits"])
        if g is not None and yq_p and bits > 8:
            return E_UNSUPPORTED
        pre, post = (f32(e["pre_lo"]), f32(e["pre_hi"])), (f32(e["post_lo"]), f32(e["post_hi"]))
        out_ok = True
        if yq_p and bits >= 1:
            _, _, fa, ra, _ = A.act_scalars(e["out_min"], e["out_max"], bits)
            out_ok = all(math.isfinite(float(v)) for v in (e["out_min"], e["out_max"], fa, ra))
        if g is not None:
            N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
            n, nq, ns = 4 * N * O_ * OH * OW, N * OH * OW * ((O_ + 15) // 16 * 16), 4 * N * OH * OW
            if not (y_p or yq_p) or (s_p and not yq_p) or yq_p % 16 or r_p % 4 or y_p % 4 or s_p % 4 or \
                    not _ordered(*pre) or not _ordered(*post) or (yq_p and (bits < 1 or not out_ok)) or \
                    any(_overlap(a, na, b, nb) for (a, na), (b, nb) in (
                        ((r_p, n), (y_p, n)), ((r_p, n), (yq_p, nq)), ((r_p, n), (s_p, ns)), ((y_p, n), (yq_p, nq)),
                        ((y_p, n), (s_p, ns)), ((yq_p, nq), (s_p, ns)))):
                return E_ARG
        P = np.empty(N * O_ * OH * OW if g is not None else 1, np.int32)
        y = np.empty(P.size, f32)
        rc = self.dfq_i8_affine_conv(xq_p, S_p, wq_p, table_p, k_p, b_p, y.ctypes.data, P.ctypes.data, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        r = _floats(r_p, n // 4).reshape(N, O_, OH, OW).copy() if r_p else None
        v = AC.epilogue_value(y.reshape(N, O_, OH, OW), r, pre, post)
        if y_p:
            _floats(y_p, n // 4)[...] = v.reshape(-1)
        if yq_p:
            q, S = A.act_codes(v, e["out_min"], e["out_max"], bits)
            _array(yq_p, nq, np.int8)[...] = AC.to_nhwc(q).reshape(-1)
            if s_p:
                _array(s_p, ns // 4, np.int32)[...] = S.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8, affine and affine-epilogue twins: returns the fake dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeAffineChainLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
