"""Oracle of the int8 max pool (dfq_i8_maxpool) and of the channel-slice epilogue (dfq_i8_conv_slice), and their host twins
--  TEST INFRASTRUCTURE.

i8_maxpool restates torch's CUDA max_pool2d (from -inf, taps row-major, the running max replaced when v > max or v is NaN)
and the byte-wise max of codes; FakePoolCatLib adds the host twins of the two entries to tests/int8_residual_oracle.py's
FakeResidualLib.
"""
import numpy as np

import fakelib
import int8_chain_oracle as CO
import int8_oracle as I8
import int8_residual_oracle as RO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import E_UNSUPPORTED, _array, _geometry

f32 = np.float32
E_ARG = CO.E_ARG


def pool_extent(n, k, p, s, d, ceil_mode):
    o = (n + 2 * p - d * (k - 1) - 1 + (s - 1 if ceil_mode else 0)) // s + 1
    return o - 1 if ceil_mode and (o - 1) * s >= n + p else o


def _taps(H, W, OH, OW, k, s, p, d):
    """(ih [OH], iw [OW], valid rows, valid cols) per tap (r, c), row-major."""
    for r in range(k[0]):
        ih = np.arange(OH) * s[0] - p[0] + r * d[0]
        for c in range(k[1]):
            iw = np.arange(OW) * s[1] - p[1] + c * d[1]
            yield ih, iw, (ih >= 0) & (ih < H), (iw >= 0) & (iw < W)


def i8_maxpool(x, k, s, p, d, ceil_mode):
    """torch's max_pool2d of fp32 x [N, C, H, W] (NaN wins and stays; the first of tied values is kept)."""
    x = np.asarray(x, f32)
    N, Cn, H, W = x.shape
    OH, OW = pool_extent(H, k[0], p[0], s[0], d[0], ceil_mode), pool_extent(W, k[1], p[1], s[1], d[1], ceil_mode)
    m = np.full((N, Cn, OH, OW), -np.inf, f32)
    for ih, iw, vh, vw in _taps(H, W, OH, OW, k, s, p, d):
        v = x[:, :, np.clip(ih, 0, H - 1)][:, :, :, np.clip(iw, 0, W - 1)]
        upd = ((v > m) | np.isnan(v)) & vh[:, None] & vw[None, :]
        m = np.where(upd, v, m).astype(f32)
    return m


def i8_maxpool_codes(xq, C, k, s, p, d, ceil_mode):
    """The byte-wise max of int8 NHWC codes [N, H, W, Cpad]; a window with no tap inside gives -127 (pad channels 0)."""
    N, H, W, Cp = xq.shape
    OH, OW = pool_extent(H, k[0], p[0], s[0], d[0], ceil_mode), pool_extent(W, k[1], p[1], s[1], d[1], ceil_mode)
    m = np.full((N, OH, OW, Cp), -128, np.int16)
    for ih, iw, vh, vw in _taps(H, W, OH, OW, k, s, p, d):
        v = xq[:, np.clip(ih, 0, H - 1)][:, :, np.clip(iw, 0, W - 1)].astype(np.int16)
        ok = (vh[:, None] & vw[None, :])[None, :, :, None]
        m = np.where(ok, np.maximum(m, v), m)
    empty = m == -128
    m[empty & (np.arange(Cp) < C)] = -127
    m[empty & (np.arange(Cp) >= C)] = 0
    return m.astype(np.int8)


def _overlap(a, na, b, nb):
    return bool(a and b and a < b + nb and b < a + na)


class FakePoolCatLib(RO.FakeResidualLib):
    def dfq_i8_conv_slice(self, xq_p, wq_p, dq_p, b_p, e_p, coff, cstride, g_p, stream):
        self.calls.append("dfq_i8_conv_slice")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        e = _table(e_p, 1, _lib.I8_EPILOGUE_DT)[0]
        coff, cstride = int(_val(coff)), int(_val(cstride))
        r_p, y_p, yq_p = int(e["residual"]), int(e["y"]), int(e["yq"])
        s = f32(e["out_scale"])
        N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
        cpad, px = (O_ + 15) // 16 * 16, N * OH * OW
        n = N * O_ * OH * OW
        ext = (yq_p + coff, (px - 1) * cstride + cpad)
        if not yq_p or yq_p % 16 or r_p % 4 or y_p % 4 or not RO._ordered(e["pre_lo"], e["pre_hi"]) or \
                not RO._ordered(e["post_lo"], e["post_hi"]) or not (np.isfinite(s) and s >= 0) or coff < 0 or \
                cstride <= 0 or coff % 16 or cstride % 16 or coff + cpad > cstride or _overlap(r_p, 4 * n, *ext) or \
                _overlap(y_p, 4 * n, *ext) or _overlap(r_p, 4 * n, y_p, 4 * n):
            return E_ARG
        y = np.empty(n, f32)
        rc = self.dfq_i8_conv(xq_p, wq_p, dq_p, b_p, y.ctypes.data, None, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        r = _floats(r_p, n).reshape(N, O_, OH, OW).copy() if r_p else None
        v = RO.i8_epilogue_value(y.reshape(N, O_, OH, OW), r, (e["pre_lo"], e["pre_hi"]), (e["post_lo"], e["post_hi"]))
        if y_p:
            _floats(y_p, n)[...] = v.reshape(-1)
        out = _array(yq_p, px * cstride, np.int8).reshape(px, cstride)
        out[:, coff:coff + cpad] = CO.to_nhwc_codes(I8.i8_quantize(v, s)).reshape(px, cpad)
        return 0

    def dfq_i8_maxpool(self, xq_p, x_p, y_p, yq_p, out_scale, g_p, stream):
        self.calls.append("dfq_i8_maxpool")
        g = _table(g_p, 1, _lib.I8_POOL_DT)[0]
        g = {k: int(g[k]) for k in _lib.I8_POOL_DT.names}
        N, Cn, H, W, Cp = g["N"], g["C"], g["H"], g["W"], g["Cpad"]
        k, s, p, d = (g["kh"], g["kw"]), (g["stride_h"], g["stride_w"]), (g["pad_h"], g["pad_w"]), (g["dil_h"], g["dil_w"])
        ceil = bool(g["ceil_mode"])
        xq_p, x_p, y_p, yq_p = (int(_val(v) or 0) for v in (xq_p, x_p, y_p, yq_p))
        sc = f32(_val(out_scale))
        ok = min(N, Cn, H, W, *k, *s, *d) > 0 and min(p) >= 0 and g["ceil_mode"] in (0, 1) and \
            all(p[i] <= k[i] // 2 and p[i] <= (d[i] * (k[i] - 1) + 1) // 2 for i in (0, 1)) and Cp >= Cn and Cp % 16 == 0
        ok = ok and (g["OH"], g["OW"]) == (pool_extent(H, k[0], p[0], s[0], d[0], ceil),
                                          pool_extent(W, k[1], p[1], s[1], d[1], ceil)) and min(g["OH"], g["OW"]) > 0
        ok = ok and (bool(xq_p) != bool(x_p))
        OH, OW = g["OH"], g["OW"]
        if ok and xq_p:
            ok = bool(yq_p) and not y_p and xq_p % 16 == 0 and yq_p % 16 == 0
        elif ok:
            ok = bool(y_p or yq_p) and yq_p % 16 == 0 and x_p % 4 == 0 and y_p % 4 == 0 and \
                (not yq_p or (np.isfinite(sc) and sc >= 0))
        if not ok:
            return E_ARG
        if xq_p:
            xq = _array(xq_p, N * H * W * Cp, np.int8).reshape(N, H, W, Cp)
            _array(yq_p, N * OH * OW * Cp, np.int8)[...] = i8_maxpool_codes(xq, Cn, k, s, p, d, ceil).reshape(-1)
            return 0
        y = i8_maxpool(_floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W), k, s, p, d, ceil)
        if y_p:
            _floats(y_p, y.size)[...] = y.reshape(-1)
        if yq_p:
            q = np.zeros((N, OH, OW, Cp), np.int8)
            q[..., :Cn] = I8.i8_quantize(y, sc).transpose(0, 2, 3, 1)
            _array(yq_p, q.size, np.int8)[...] = q.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins, the residual epilogue's, the slice epilogue's and the max pool's: returns the
    fake dfq_b200._lib.load() hands out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakePoolCatLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
