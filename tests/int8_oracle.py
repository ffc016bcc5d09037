"""Integer oracle of int8 execution (dfq_b200.int8, dfq_i8_* in libdfq_sm90.so)  --  TEST INFRASTRUCTURE.

ncnn's dequantizing int8 convolution with the scales of the table convert_ncnn.py:178-201 writes, restated in numpy:
symmetric codes clamp(round_half_away(fp32(v * s)), -127, 127), exact integer sums, and the two separately rounded fp32 ops of
the epilogue.  Every fp32 op here is a correctly rounded IEEE op, so results compare bit for bit with the GPU.
"""
from typing import Optional

import numpy as np

f32 = np.float32


def i8_quantize(v: np.ndarray, s) -> np.ndarray:
    """int8 codes clamp(round_half_away(fp32(v * s)), -127, 127); `s` is a scalar or broadcasts against v.

    A NaN product (a NaN input, inf * 0, 0 * inf) gives -127: the kernel's fminf(fmaxf(NaN, -127), 127) is -127, and so is
    ncnn's float2int8 (a C cast of the rounded value, then the clamp) on x86.  +-inf products clamp to +-127."""
    with np.errstate(over="ignore", invalid="ignore"):
        p = (np.asarray(v, f32) * np.asarray(s, f32)).astype(np.float64)   # fp32 product, widened exactly
        r = np.sign(p) * np.floor(np.abs(p) + 0.5)                         # exact in float64 for every fp32 p
    r = np.where(np.isnan(r), -127.0, r)                                   # never numpy's undefined NaN -> int8 cast
    return np.clip(r, -127, 127).astype(np.int8)


def i8_conv(xq: np.ndarray, wq: np.ndarray, stride=(1, 1), padding=(0, 0), dilation=(1, 1), groups=1) -> np.ndarray:
    """Exact int64 sums of codes xq [N, C, H, W] * wq [O, C/groups, kh, kw] (zero padding): im2col + matmul.

    The matmul runs in float64, which is exact here: every product and partial sum is an integer below
    127 * 127 * K << 2**53.  Depthwise layers (groups == C == O) sum tap by tap in int32 instead, so a large batch does not
    need the im2col copy."""
    N, Cn, H, W = xq.shape
    O, Cg, kh, kw = wq.shape
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    assert 127 * 127 * Cg * kh * kw < 2 ** 53
    OH = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1
    OW = (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    if Cg == 1 and groups == Cn == O:                                                 # depthwise: one MAC per tap
        xp = np.zeros((N, Cn, H + 2 * ph, W + 2 * pw), np.int32)
        xp[:, :, ph:ph + H, pw:pw + W] = xq
        acc = np.zeros((N, O, OH, OW), np.int32)                                      # |acc| <= 127^2 * taps < 2^31
        for r in range(kh):
            for s in range(kw):
                acc += xp[:, :, r * dh: r * dh + sh * (OH - 1) + 1: sh, s * dw: s * dw + sw * (OW - 1) + 1: sw] * \
                    wq[:, 0, r, s].astype(np.int32).reshape(1, -1, 1, 1)
        return acc.astype(np.int64)
    xp = np.zeros((N, Cn, H + 2 * ph, W + 2 * pw), np.float64)
    xp[:, :, ph:ph + H, pw:pw + W] = xq
    cols = np.stack([xp[:, :, r * dh: r * dh + sh * (OH - 1) + 1: sh, s * dw: s * dw + sw * (OW - 1) + 1: sw]
                     for r in range(kh) for s in range(kw)], axis=2)                    # [N, C, taps, OH, OW]
    cols = cols.reshape(N, groups, Cg * kh * kw, OH * OW)
    wm = wq.astype(np.float64).reshape(groups, O // groups, Cg * kh * kw)
    acc = np.einsum("gok,ngkp->ngop", wm, cols, optimize=True) if groups > 1 else np.matmul(wm[0], cols[:, 0])
    return np.rint(acc).astype(np.int64).reshape(N, O, OH, OW)


def i8_dequant(acc: np.ndarray, act_scale, w_scale: np.ndarray, bias: Optional[np.ndarray] = None) -> np.ndarray:
    """y = fp32(fp32_rn(acc) * dq[o]) + bias[o] with dq[o] = fp32(1 / fp32(a * w_s[o])) (0 where a * w_s[o] is 0);
    acc is [N, O, ...].  No bias adds +0.0, as the kernel does."""
    den = f32(act_scale) * np.asarray(w_scale, f32)
    dq = np.where(den == 0, f32(0), f32(1) / np.where(den == 0, f32(1), den)).astype(f32)
    shape = (1, -1) + (1,) * (acc.ndim - 2)
    y = (acc.astype(f32) * dq.reshape(shape)).astype(f32)
    b = np.zeros(dq.shape, f32) if bias is None else np.asarray(bias, f32)
    return (y + b.reshape(shape)).astype(f32)
