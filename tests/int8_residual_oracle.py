"""Oracle of the residual int8 epilogue (dfq_i8_conv_fused) and its host twin  --  TEST INFRASTRUCTURE.

i8_epilogue restates, on top of tests/int8_oracle.py and tests/int8_chain_oracle.py, what the per-layer path computes from a
convolution to the tensor after a residual block's add: the dequantizing epilogue, the pass-throughs before the add as one
clamp that keeps NaN, the fp32 add, the pass-throughs after it, then the fp32 value and its codes at the next layer's scale.
FakeResidualLib adds the host twin of dfq_i8_conv_fused to tests/int8_chain_oracle.py's FakeChainLib.
"""
import numpy as np

import fakelib
import int8_chain_oracle as CO
import int8_oracle as I8
from dfq_b200 import _lib
from fakelib import _floats, _table
from fakelib_int8 import E_UNSUPPORTED, _array, _geometry

f32 = np.float32
E_ARG = CO.E_ARG
NONE = (-np.inf, np.inf)


GPU_NAN = np.array(0x7FFFFFFF, np.uint32).view(f32)    # the NaN an H100 fp32 add returns, whatever NaN goes in


def i8_epilogue_value(y, r=None, pre=NONE, post=NONE, gpu_nan=False):
    """The fp32 value after the add: clamp(clamp(y, *pre) + r, *post) in fp32, r broadcast-free ([N, O, ...] like y).
    gpu_nan: a NaN sum is GPU_NAN, as on the GPU (numpy keeps the NaN operand's payload, as torch does on the CPU)."""
    v = CO.i8_clamp(y, *pre)
    if r is not None:
        assert np.shape(r) == np.shape(v)
        with np.errstate(over="ignore", invalid="ignore"):
            v = (v + np.asarray(r, f32)).astype(f32)
        if gpu_nan:
            v = np.where(np.isnan(v), GPU_NAN, v).astype(f32)
    return CO.i8_clamp(v, *post)


def i8_epilogue(acc, act_scale, w_scale, bias, r=None, pre=NONE, post=NONE, out_scale=None, gpu_nan=True):
    """(fp32 value [N, O, ...], codes [N, O, ...] at out_scale or None) from the int32 sums."""
    v = i8_epilogue_value(I8.i8_dequant(acc, act_scale, w_scale, bias), r, pre, post, gpu_nan)
    return v, (None if out_scale is None else I8.i8_quantize(v, f32(out_scale)))


def _ordered(lo, hi):
    return not (np.isnan(lo) or np.isnan(hi)) and lo <= hi


def _overlap(a, na, b, nb):
    return bool(a and b and a < b + nb and b < a + na)


class FakeResidualLib(CO.FakeChainLib):
    def dfq_i8_conv_fused(self, xq_p, wq_p, dq_p, b_p, e_p, g_p, stream):
        self.calls.append("dfq_i8_conv_fused")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        e = _table(e_p, 1, _lib.I8_EPILOGUE_DT)[0]
        r_p, y_p, yq_p = int(e["residual"]), int(e["y"]), int(e["yq"])
        s = f32(e["out_scale"])
        N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
        n = N * O_ * OH * OW
        nq = N * OH * OW * ((O_ + 15) // 16 * 16)
        if not (y_p or yq_p) or yq_p % 16 or r_p % 4 or y_p % 4 or not _ordered(e["pre_lo"], e["pre_hi"]) or \
                not _ordered(e["post_lo"], e["post_hi"]) or (yq_p and not (np.isfinite(s) and s >= 0)) or \
                _overlap(r_p, 4 * n, y_p, 4 * n) or _overlap(r_p, 4 * n, yq_p, nq) or _overlap(y_p, 4 * n, yq_p, nq):
            return E_ARG
        y = np.empty(n, f32)
        rc = self.dfq_i8_conv(xq_p, wq_p, dq_p, b_p, y.ctypes.data, None, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        r = _floats(r_p, n).reshape(N, O_, OH, OW).copy() if r_p else None
        v = i8_epilogue_value(y.reshape(N, O_, OH, OW), r, (e["pre_lo"], e["pre_hi"]), (e["post_lo"], e["post_hi"]))
        if y_p:
            _floats(y_p, n)[...] = v.reshape(-1)
        if yq_p:
            _array(yq_p, nq, np.int8)[...] = CO.to_nhwc_codes(I8.i8_quantize(v, s)).reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins, dfq_i8_conv_requant's and dfq_i8_conv_fused's: returns the fake
    dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeResidualLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
