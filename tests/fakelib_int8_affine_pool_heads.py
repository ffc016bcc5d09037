"""tests/fakelib_int8_affine_layout.py's stand-in for libdfq_sm90.so, extended by the host twins of dfq_i8_affine_maxpool
and dfq_i8_affine_conv_rows (tests/int8_affine_pool_heads_oracle.py) with their refusals.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so chain_affine's pool and head rules run
without a GPU.
"""
import numpy as np

import fakelib_int8_affine_layout
import int8_affine_pool_heads_oracle as AP
import int8_pool_cat_oracle as PO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import E_UNSUPPORTED, _array, _geometry
from fakelib_int8_affine import E_ARG

f32 = np.float32


class FakeAffinePoolLib(fakelib_int8_affine_layout.FakeAffineLayoutLib):
    def dfq_i8_affine_maxpool(self, xq_p, x_p, y_p, yq_p, S_p, out_min, out_max, out_bits, g_p, stream):
        self.calls.append("dfq_i8_affine_maxpool")
        g = _table(g_p, 1, _lib.I8_POOL_DT)[0]
        g = {k: int(g[k]) for k in _lib.I8_POOL_DT.names}
        N, Cn, H, W, Cp = g["N"], g["C"], g["H"], g["W"], g["Cpad"]
        k, s, p, d = (g["kh"], g["kw"]), (g["stride_h"], g["stride_w"]), (g["pad_h"], g["pad_w"]), (g["dil_h"], g["dil_w"])
        ceil = bool(g["ceil_mode"])
        xq_p, x_p, y_p, yq_p, S_p = (int(_val(v) or 0) for v in (xq_p, x_p, y_p, yq_p, S_p))
        out = (f32(_val(out_min)), f32(_val(out_max)), int(_val(out_bits)))
        ok = min(N, Cn, H, W, *k, *s, *d) > 0 and min(p) >= 0 and g["ceil_mode"] in (0, 1) and \
            all(p[i] <= k[i] // 2 and p[i] <= (d[i] * (k[i] - 1) + 1) // 2 for i in (0, 1)) and Cp >= Cn and Cp % 16 == 0
        ok = ok and (g["OH"], g["OW"]) == (PO.pool_extent(H, k[0], p[0], s[0], d[0], ceil),
                                          PO.pool_extent(W, k[1], p[1], s[1], d[1], ceil)) and min(g["OH"], g["OW"]) > 0
        ok = ok and bool(xq_p) != bool(x_p) and (not S_p or yq_p) and S_p % 4 == 0
        if ok and xq_p:
            ok = bool(yq_p) and not y_p and xq_p % 16 == 0 and yq_p % 16 == 0
        elif ok:
            ok = bool(y_p or yq_p) and yq_p % 16 == 0 and x_p % 4 == 0 and y_p % 4 == 0
            if ok and yq_p:
                if out[2] > 8:
                    return E_UNSUPPORTED
                lo, hi = float(out[0]), float(out[1])
                scale = max((hi - lo) / (2. ** out[2] - 1), 1e-8) if out[2] >= 1 else np.nan
                ok = out[2] >= 1 and np.isfinite(lo) and np.isfinite(hi) and np.isfinite(f32(scale)) and \
                    np.isfinite(f32(1 / scale))
        if not ok:
            return E_ARG
        OH, OW = g["OH"], g["OW"]
        if xq_p:
            q, S = AP.maxpool_codes(_array(xq_p, N * H * W * Cp, np.int8).reshape(N, H, W, Cp), Cn, k, s, p, d, ceil)
        else:
            y, q, S = AP.maxpool_fp32(_floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W), k, s, p, d, ceil,
                                      out if yq_p else None)
            if y_p:
                _floats(y_p, y.size)[...] = y.reshape(-1)
            if q is not None:
                q = np.concatenate([q, np.zeros(q.shape[:3] + (Cp - q.shape[3],), np.int8)], -1)
        if yq_p:
            _array(yq_p, N * OH * OW * Cp, np.int8)[...] = q.reshape(-1)
        if S_p:
            _array(S_p, N * OH * OW, np.int32)[...] = S.reshape(-1)
        return 0


    def dfq_i8_affine_conv_rows(self, xq_p, S_p, wq_p, table_p, k_p, b_p, r_p, g_p, stream):
        self.calls.append("dfq_i8_affine_conv_rows")
        g = _geometry(g_p)
        if g is None:
            return E_UNSUPPORTED
        r = _table(r_p, 1, _lib.I8_AFFINE_ROWS_DT)[0]
        N, O_, OH, OW = g["N"], g["O"], g["OH"], g["OW"]
        y_p, off, stride = int(r["y"]), int(r["off"]), int(r["img_stride"])
        ext = OH * OW * O_
        bits = [int(r["obs_bits"]), int(r["tail_bits"])]
        if any(b > 8 for b in bits):
            return E_UNSUPPORTED
        if not y_p or y_p % 4 or off < 0 or stride < off + ext or any(b < 0 for b in bits) or \
                not all(np.isfinite(r[f]) or f.endswith(("lo", "hi")) for f in ("obs_min", "obs_max", "tail_min", "tail_max")) \
                or np.isnan([r["pre_lo"], r["pre_hi"], r["post_lo"], r["post_hi"]]).any() or r["pre_lo"] > r["pre_hi"] or \
                r["post_lo"] > r["post_hi"]:
            return E_ARG
        y = np.zeros(N * O_ * OH * OW, f32)
        rc = self.dfq_i8_affine_conv(xq_p, S_p, wq_p, table_p, k_p, b_p, y.ctypes.data, None, g_p, stream)
        self.calls.pop()                                        # the inner call is part of this one
        if rc:
            return rc
        obs = (f32(r["obs_min"]), f32(r["obs_max"]), bits[0]) if bits[0] else None
        tail = (f32(r["tail_min"]), f32(r["tail_max"]), bits[1]) if bits[1] else None
        v = AP.rows_value(y.reshape(N, O_, OH, OW), (r["pre_lo"], r["pre_hi"]), (r["post_lo"], r["post_hi"]), obs, tail)
        out = _floats(y_p, (N - 1) * stride + off + ext)
        for n in range(N):
            out[n * stride + off:n * stride + off + ext] = v[n].transpose(1, 2, 0).reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib_int8_affine_layout.install() with the affine max pool's and head rows' twins."""
    fakelib_int8_affine_layout.install(monkeypatch, sqrt_fn)
    fake = FakeAffinePoolLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
