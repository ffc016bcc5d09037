"""Oracle of the int8 bilinear upsample (dfq_i8_upsample_bilinear) and its host twin  --  TEST INFRASTRUCTURE.

i8_upsample_bilinear restates torch's CUDA upsample_bilinear2d_out_frame<float, float> for a contiguous NCHW input and a
given size, operation for operation as its sm_90 SASS (torch 2.11, compiled with contraction on) computes it:

    scale  = align_corners ? fp32(in - 1) / fp32(out - 1) (0 when out == 1) : fp32(in) / fp32(out)     on the host
    src    = align_corners ? fl(dst * scale) : fma(fl(dst + 0.5), scale, -0.5), then src < 0 ? 0 : src
    i      = trunc(src),  l1 = fl(src - i),  l0 = fl(1 - l1),  the second tap i + 1 only while i < in - 1
    row(h) = fma(w_l0, x[h, w_i], fl(w_l1 * x[h, w_i + w_p]))                 for h = h_i and h_i + h_p
    y      = fma(h_l0, row(h_i), fl(h_l1 * row(h_i + h_p)))

and a plain copy when the size does not change.  fma32 rounds a * b + c once: the product of two fp32 numbers is exact in
float64, the float64 sum is corrected to round-to-odd from its exact two-sum error, and rounding that to fp32 is then the
correctly rounded result (53 >= 24 + 2 bits), which fma32_exact checks against exact rationals.  A NaN the arithmetic makes
is the H100's canonical NaN; the copy keeps x's bits.  FakeUpsampleLib adds the host twin of the entry to
tests/int8_pool_cat_oracle.py's FakePoolCatLib.
"""
from fractions import Fraction

import numpy as np

import fakelib
import int8_chain_oracle as CO
import int8_oracle as I8
import int8_pool_cat_oracle as PO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import _array
from int8_residual_oracle import GPU_NAN

f32 = np.float32
E_ARG = CO.E_ARG


def fma32(a, b, c):
    """fp32 fma(a, b, c) = a * b + c rounded once to nearest even, elementwise (broadcasting)."""
    a, b, c = np.broadcast_arrays(*(np.asarray(v, f32) for v in (a, b, c)))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)                 # exact: 24 + 24 significant bits
        cd = c.astype(np.float64)
        s = p + cd
        bp = s - cd
        e = (p - bp) + (cd - (s - bp))                                  # two-sum: s + e == p + cd exactly
        odd = (s.view(np.int64) & 1) == 1
        fix = np.isfinite(s) & (e != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(f32)


def _round_f32(q):
    """The fp32 number nearest the rational q (ties to even; beyond the largest finite fp32, infinity)."""
    if q == 0:
        return f32(0)
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    quantum = Fraction(2) ** (max(e, -126) - 23)
    n = q / quantum
    r = n.numerator // n.denominator
    rem = n - r
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and r % 2):
        r += 1
    v = r * quantum
    return f32(sign * np.inf) if v >= Fraction(2) ** 128 else f32(sign * float(v))


def fma32_exact(a, b, c):
    """fma(a, b, c) of finite fp32 scalars through exact rationals (a zero result compares by value only)."""
    return _round_f32(Fraction(float(f32(a))) * Fraction(float(f32(b))) + Fraction(float(f32(c))))


def bilinear_scale(n_in, n_out, align_corners):
    if align_corners:
        return f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0)
    return f32(n_in) / f32(n_out)


def _axis(n_out, n_in, align_corners):
    """(i0, i1, l0, l1) per destination index of one axis."""
    scale = bilinear_scale(n_in, n_out, align_corners)
    d = np.arange(n_out).astype(f32)
    if align_corners:
        src = (d * scale).astype(f32)
    else:
        src = fma32((d + f32(0.5)).astype(f32), scale, f32(-0.5))
        src = np.where(src < 0, f32(0), src).astype(f32)
    i0 = src.astype(np.int64)                                           # src >= 0: truncation
    i1 = i0 + (i0 < n_in - 1)
    l1 = (src - i0.astype(f32)).astype(f32)
    return i0, i1, (f32(1) - l1).astype(f32), l1


def i8_upsample_bilinear(x, OH, OW, align_corners):
    """torch's F.interpolate(x, size=(OH, OW), mode='bilinear', align_corners=...) of fp32 x [N, C, H, W] on the GPU."""
    x = np.asarray(x, f32)
    N, Cn, H, W = x.shape
    if (H, W) == (OH, OW):
        return x.copy()
    h0, h1, hl0, hl1 = _axis(OH, H, align_corners)
    w0, w1, wl0, wl1 = _axis(OW, W, align_corners)
    with np.errstate(all="ignore"):
        def row(h):
            xr = x[:, :, h]
            return fma32(wl0, xr[:, :, :, w0], (wl1 * xr[:, :, :, w1]).astype(f32))
        a, b = row(h0), row(h1)
        y = fma32(hl0[:, None], a, (hl1[:, None] * b).astype(f32))
    return np.where(np.isnan(y), GPU_NAN, y).astype(f32)


def i8_upsample_codes(y, out_scale, lo=-np.inf, hi=np.inf):
    """q(clamp(y, lo, hi), out_scale) as int8 NHWC [N, OH, OW, round_up(C, 16)] with zero pad channels."""
    return CO.to_nhwc_codes(I8.i8_quantize(CO.i8_clamp(y, lo, hi), f32(out_scale)))


class FakeUpsampleLib(PO.FakePoolCatLib):
    def dfq_i8_upsample_bilinear(self, x_p, y_p, yq_p, g_p, stream):
        self.calls.append("dfq_i8_upsample_bilinear")
        g = _table(g_p, 1, _lib.I8_RESIZE_DT)[0]
        N, Cn, H, W, OH, OW, ac, coff, cstride = (int(g[k]) for k in _lib.I8_RESIZE_DT.names[:9])
        s, lo, hi = f32(g["out_scale"]), f32(g["lo"]), f32(g["hi"])
        x_p, y_p, yq_p = (int(_val(v) or 0) for v in (x_p, y_p, yq_p))
        cpad, px = (Cn + 15) // 16 * 16, N * OH * OW
        ext = (yq_p + coff if yq_p else 0, (px - 1) * cstride + cpad)
        nx, ny = 4 * N * Cn * H * W, 4 * px * Cn
        if not x_p or min(N, Cn, H, W, OH, OW) <= 0 or ac not in (0, 1) or coff < 0 or cstride <= 0 or coff % 16 or \
                cstride % 16 or coff + cpad > cstride or not (y_p or yq_p) or yq_p % 16 or x_p % 4 or y_p % 4 or \
                (yq_p and not (np.isfinite(s) and s >= 0)) or not PO.RO._ordered(lo, hi) or \
                PO._overlap(x_p, nx, y_p, ny) or PO._overlap(x_p, nx, *ext) or PO._overlap(y_p, ny, *ext):
            return E_ARG
        y = i8_upsample_bilinear(_floats(x_p, N * Cn * H * W).reshape(N, Cn, H, W), OH, OW, bool(ac))
        if y_p:
            _floats(y_p, y.size)[...] = y.reshape(-1)
        if yq_p:
            out = _array(yq_p, px * cstride, np.int8).reshape(px, cstride)
            out[:, coff:coff + cpad] = i8_upsample_codes(y, s, lo, hi).reshape(px, cpad)
        return 0


def install(monkeypatch, sqrt_fn=None):
    """fakelib.install() with the int8 twins up to the bilinear upsample's: returns the fake dfq_b200._lib.load() hands
    out."""
    fakelib.install(monkeypatch, sqrt_fn)
    fake = FakeUpsampleLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
