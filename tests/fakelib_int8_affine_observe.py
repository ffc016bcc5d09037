"""tests/fakelib_int8_affine_chain.py's stand-in for libdfq_sm90.so, extended by the host twin of
dfq_i8_affine_conv_observed computed by tests/int8_affine_observe_oracle.py, with the entry's refusals.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so chain_affine's observer rules and the
chained layers run without a GPU.  QuantMeasure runs in its CUDA mode (reciprocal multiply), as the epilogue does.
"""
import math

import numpy as np

import fakelib_int8_affine_chain
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A
import int8_affine_observe_oracle as AO
from dfq_b200 import _lib
from fakelib import _floats, _table
from fakelib_int8 import _array, _geometry
from fakelib_int8_affine import E_ARG, E_UNSUPPORTED

f32 = np.float32


def _observer(lo, hi, bits):
    """(rc, (lo, hi, bits) | None) of one observer of DfqI8AffineObserve."""
    if bits < 0:
        return E_ARG, None
    if bits > 8:
        return E_UNSUPPORTED, None
    if bits == 0:
        return 0, None
    _, _, fa, ra, _ = A.act_scalars(lo, hi, bits)
    if not all(math.isfinite(float(v)) for v in (lo, hi, fa, ra)):
        return E_ARG, None
    return 0, (f32(lo), f32(hi), int(bits))


class FakeAffineObserveLib(fakelib_int8_affine_chain.FakeAffineChainLib):
    def dfq_i8_affine_conv_observed(self, xq_p, S_p, wq_p, table_p, k_p, b_p, e_p, o_p, g_p, stream):
        self.calls.append("dfq_i8_affine_conv_observed")
        g = _geometry(g_p)
        e = _table(e_p, 1, _lib.I8_AFFINE_EPILOGUE_DT)[0]
        o = _table(o_p, 1, _lib.I8_AFFINE_OBSERVE_DT)[0]
        r_p, y_p, yq_p, s_p = (int(e[f]) for f in ("residual", "y", "yq", "S"))
        rc_o, obs = _observer(o["obs_min"], o["obs_max"], int(o["obs_bits"]))
        rc_r, res = _observer(o["res_min"], o["res_max"], int(o["res_bits"]))
        # everything dfq_i8_affine_conv_fused refuses first, with scratch outputs: nothing is written on a refusal
        if g is not None:
            N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
            n, nq, ns = N * O_ * OH * OW, N * OH * OW * ((O_ + 15) // 16 * 16), N * OH * OW
        else:
            n = nq = ns = 1
        y_s, q_s, s_s = np.empty(n, f32), np.empty(nq + 16, np.int8), np.empty(ns, np.int32)
        q_addr = (q_s.ctypes.data + 15) // 16 * 16
        e2 = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
        e2[0] = e
        e2[0]["y"], e2[0]["yq"], e2[0]["S"] = (y_s.ctypes.data if y_p else 0), (q_addr if yq_p else 0), \
            (s_s.ctypes.data if s_p else 0)
        e2[0]["residual"] = 0
        rc = super().dfq_i8_affine_conv_fused(xq_p, S_p, wq_p, table_p, k_p, b_p, e2.ctypes.data, g_p, stream)
        self.calls.pop()
        if rc == 0 and (r_p % 4 or any(fakelib_int8_affine_chain._overlap(r_p, 4 * n, a, na) for a, na in (
                (y_p, 4 * n), (yq_p, nq), (s_p, 4 * ns)))):
            rc = E_ARG
        rc = rc or rc_o or rc_r
        if rc == 0 and ((res is not None and not r_p) or (obs is None and res is None)):
            rc = E_ARG
        if rc:
            return rc
        P = np.empty(n, np.int32)
        y = np.empty(n, f32)
        self.dfq_i8_affine_conv(xq_p, S_p, wq_p, table_p, k_p, b_p, y.ctypes.data, P.ctypes.data, g_p, stream)
        self.calls.pop()
        pre, post = (f32(e["pre_lo"]), f32(e["pre_hi"])), (f32(e["post_lo"]), f32(e["post_hi"]))
        r = _floats(r_p, n).reshape(N, O_, OH, OW).copy() if r_p else None
        v = AO.observed_value(y.reshape(N, O_, OH, OW), r, pre, post, obs, res, gpu_nan=False)
        if y_p:
            _floats(y_p, n)[...] = v.reshape(-1)
        if yq_p:
            q, S = A.act_codes(v, e["out_min"], e["out_max"], int(e["out_bits"]))
            _array(yq_p, nq, np.int8)[...] = AC.to_nhwc(q).reshape(-1)
            if s_p:
                _array(s_p, ns, np.int32)[...] = S.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib_int8_affine_chain.install() with the observed-epilogue twin, QuantMeasure in its CUDA (reciprocal) mode."""
    import dfq_b200.utils.quantize as q
    fakelib_int8_affine_chain.install(monkeypatch, sqrt_fn)
    fake = FakeAffineObserveLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(q, "_dev_f32", lambda x: (x.contiguous(), False))
    return fake
