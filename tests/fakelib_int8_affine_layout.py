"""tests/fakelib_int8_affine_observe.py's stand-in for libdfq_sm90.so, extended by host twins of dfq_i8_affine_conv_layout
(the layer on the codes padded with the pad code, computed by the observed / fused twins, then written into the slice) and
dfq_i8_affine_upsample_bilinear (torch's CPU bilinear upsample, the oracle's observer and quantizer), with the layout's
refusals.

Test infrastructure only: `install()` routes dfq_b200 through it inside a test, so chain_affine's pad and concatenation
rules run without a GPU.
"""
import numpy as np
import torch
import torch.nn.functional as F

import fakelib_int8_affine_observe
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A
import int8_affine_observe_oracle as AO
from dfq_b200 import _lib
from fakelib import _floats, _table
from fakelib_int8 import _array, _geometry
from fakelib_int8_affine import E_ARG

f32 = np.float32


def _aligned(n, dtype):
    """A 16-byte aligned numpy scratch array of n elements."""
    raw = np.zeros(n * np.dtype(dtype).itemsize + 16, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + n * np.dtype(dtype).itemsize].view(dtype)


class FakeAffineLayoutLib(fakelib_int8_affine_observe.FakeAffineObserveLib):
    def dfq_i8_affine_conv_layout(self, xq_p, S_p, wq_p, table_p, k_p, b_p, e_p, o_p, l_p, g_p, stream):
        self.calls.append("dfq_i8_affine_conv_layout")
        g = _geometry(g_p)
        lay = {k: int(v) for k, v in zip(_lib.I8_AFFINE_LAYOUT_DT.names, _table(l_p, 1, _lib.I8_AFFINE_LAYOUT_DT)[0])}
        e = _table(e_p, 1, _lib.I8_AFFINE_EPILOGUE_DT)[0]
        cpad = (g["O"] + 15) // 16 * 16
        if lay["coff"] < 0 or lay["cstride"] <= 0 or lay["coff"] % 16 or lay["cstride"] % 16 or \
                lay["coff"] + cpad > lay["cstride"] or lay["S_accumulate"] not in (0, 1) or lay["pad_code_on"] not in (0, 1) \
                or (lay["pad_code_on"] and not -128 <= lay["pad_code"] <= 127):
            return E_ARG
        N, Cn, H, W, Cp = g["N"], g["C"], g["H"], g["W"], g["Cpad"]
        xq = _array(xq_p, N * H * W * Cp, np.int8).reshape(N, H, W, Cp)
        g2 = _table(g_p, 1, _lib.I8_CONV_DT).copy()
        if lay["pad_code_on"]:
            t, l = g["pad_h"], g["pad_w"]
            xp = _aligned(N * (H + 2 * t) * (W + 2 * l) * Cp, np.int8).reshape(N, H + 2 * t, W + 2 * l, Cp)
            xp[..., :Cn] = lay["pad_code"]
            xp[:, t:t + H, l:l + W] = xq
            g2[0]["H"], g2[0]["W"], g2[0]["pad_h"], g2[0]["pad_w"] = H + 2 * t, W + 2 * l, 0, 0
        else:
            xp = xq
        Sp = np.ascontiguousarray(xp[..., :Cn].astype(np.int32).sum(-1))
        OH, OW, O_ = g["OH"], g["OW"], g["O"]
        pixels = N * OH * OW
        q_t, s_t = _aligned(pixels * cpad, np.int8), np.zeros(pixels, np.int32)
        e2 = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
        e2[0] = e
        yq_p, s_p = int(e["yq"]), int(e["S"])
        e2[0]["yq"], e2[0]["S"] = (q_t.ctypes.data if yq_p else 0), (s_t.ctypes.data if s_p else 0)
        args = (xp.ctypes.data, Sp.ctypes.data, wq_p, table_p, k_p, b_p, e2.ctypes.data)
        if o_p:
            rc = self.dfq_i8_affine_conv_observed(*args, o_p, g2.ctypes.data, stream)
        else:
            rc = self.dfq_i8_affine_conv_fused(*args, g2.ctypes.data, stream)
        self.calls.pop()
        if rc:
            return rc
        if yq_p:
            rows = _array(yq_p, (pixels - 1) * lay["cstride"] + lay["coff"] + cpad, np.int8)
            for m in range(pixels):
                start = m * lay["cstride"] + lay["coff"]
                rows[start:start + cpad] = q_t[m * cpad:(m + 1) * cpad]
        if s_p:
            S = _array(s_p, pixels, np.int32)
            S[...] = S + s_t if lay["S_accumulate"] else s_t
        return 0

    def dfq_i8_affine_upsample_bilinear(self, x_p, yq_p, S_p, g_p, stream):
        self.calls.append("dfq_i8_affine_upsample_bilinear")
        g = _table(g_p, 1, _lib.I8_AFFINE_RESIZE_DT)[0]
        N, Cn, H, W, OH, OW = (int(g[k]) for k in ("N", "C", "H", "W", "OH", "OW"))
        coff, cstride = int(g["coff"]), int(g["cstride"])
        cpad = (Cn + 15) // 16 * 16
        if coff % 16 or cstride % 16 or coff + cpad > cstride or not x_p or not yq_p:
            return E_ARG
        x = torch.from_numpy(_floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W).copy())
        v = F.interpolate(x, size=(OH, OW), mode="bilinear", align_corners=bool(g["align_corners"])).numpy()
        obs = (f32(g["obs_min"]), f32(g["obs_max"]), int(g["obs_bits"])) if int(g["obs_bits"]) else None
        v = AO.observed_value(v, None, (f32(g["pre_lo"]), f32(g["pre_hi"])), (f32(g["post_lo"]), f32(g["post_hi"])), obs,
                              None, gpu_nan=False)
        q, S = A.act_codes(v, g["out_min"], g["out_max"], int(g["out_bits"]))
        rows = _array(yq_p, N * OH * OW * cstride, np.int8).reshape(N * OH * OW, cstride)
        rows[:, coff:coff + cpad] = AC.to_nhwc(q).reshape(N * OH * OW, -1)[:, :cpad]
        if S_p:
            out = _array(S_p, N * OH * OW, np.int32)
            out[...] = out + S.reshape(-1)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib_int8_affine_observe.install() with the layout and upsample twins."""
    fakelib_int8_affine_observe.install(monkeypatch, sqrt_fn)
    fake = FakeAffineLayoutLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
