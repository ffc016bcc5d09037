"""Integer oracle of the affine int8 scheme (dfq_i8_affine_* in libdfq_sm90.so, dfq_b200.int8.convert_affine)  --  TEST
INFRASTRUCTURE.

The reference's asymmetric per-tensor min / max quantization restated in numpy: the activation codes with QuantMeasure's
fp32 ops, their per-pixel sums S, the weight codes recovered from fake-quantized weights, the per-output-channel prefix
tables of tap sums and the double epilogue y = fp32(kP P + kA A + kW Wv + kN Nv) + bias in the kernels' op order.  Every
op is a correctly rounded IEEE op (numpy never contracts), so results compare bit for bit with the GPU.
"""
import numpy as np

import int8_oracle as I8
from oracle import dfq_oracle as D

f32, f64 = np.float32, np.float64


def act_scalars(running_min, running_max, num_bits):
    """(neg_min, ma, fa, r_a, qmax) in fp32: QuantMeasure's eval-mode scalars on CUDA - the double prologue of
    dfq_oracle.quant_scalars, fa = fp32(scale), r_a = fp32(1 / scale) formed in double (div_ as a reciprocal multiply)."""
    _, qmax, mn, scale = D.quant_scalars(num_bits, float(f32(running_min)), float(f32(running_max)))
    with np.errstate(over="ignore"):
        return f32(-mn), f32(mn), f32(scale), f32(1.0 / scale), f32(qmax)


def act_codes(x, running_min, running_max, num_bits):
    """(q' int8 [N, C, H, W], S int32 [N, H, W]): q' = rint(clamp(fp32(fp32(x + (-ma)) * r_a), 0, qmax)) - 128 (NaN -> code
    -128, where the fake quantization outputs NaN) and S = the sum of q' over the channels."""
    neg, _, _, ra, qmax = act_scalars(running_min, running_max, num_bits)
    with np.errstate(over="ignore", invalid="ignore"):
        t = ((np.asarray(x, f32) + neg).astype(f32) * ra).astype(f32)
        t = np.where(np.isnan(t), f32(0), np.minimum(np.maximum(t, f32(0)), qmax))
    q = (np.rint(t).astype(np.int32) - 128).astype(np.int8)
    return q, q.astype(np.int32).sum(axis=1)


def act_dequant(q, running_min, running_max, num_bits):
    """fp32(fp32((q' + 128) * fa) + ma): what the fake quantization outputs for the code."""
    _, ma, fa, _, _ = act_scalars(running_min, running_max, num_bits)
    with np.errstate(over="ignore", invalid="ignore"):
        return ((q.astype(f32) + f32(128)) * fa).astype(f32) + ma


def fake_quant(x, running_min, running_max, num_bits):
    """The repo's oracle of QuantMeasure's eval-mode output on CUDA (dfq_oracle.quantize, reciprocal mode)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return D.quantize(x, num_bits, float(f32(running_min)), float(f32(running_max)), div_mode="recip")


def weight_codes(w_hat, w_min, w_scale, num_bits):
    """(q' int8 of w_hat's shape, n_bad): q = clamp(rint(fp32(fp32(w - w_min) / w_scale)), 0, qmax), stored q - 128; n_bad
    = the weights with fp32(fp32(q * w_scale) + w_min) != w, bit for bit."""
    w = np.asarray(w_hat, f32)
    mn, s, qmax = f32(w_min), f32(w_scale), f32(2. ** num_bits - 1.)
    with np.errstate(over="ignore", invalid="ignore"):
        t = np.rint(((w - mn).astype(f32) / s).astype(f32))
        q = np.where(np.isnan(t), f32(0), np.minimum(np.maximum(t, f32(0)), qmax))
        back = ((q * s).astype(f32) + mn).astype(f32)
    bad = int(np.count_nonzero(back.view(np.int32) != w.view(np.int32)))
    return (q.astype(np.int32) - 128).astype(np.int8), bad


def fake_quant_weights(w, num_bits):
    """quantize_targ_layer's fake quantization of one weight tensor on CUDA (its own min / max, reciprocal mode)."""
    return D.quantize(np.asarray(w, f32), num_bits, div_mode="recip")


def tap_table(wq):
    """[O, kh + 1, kw + 1] int32: T[o, r, s] = sum of wq[o] (shifted codes [O, C/groups, kh, kw]) over taps r' < r, s' < s."""
    tap = wq.astype(np.int64).sum(axis=1)
    T = np.zeros((wq.shape[0], wq.shape[2] + 1, wq.shape[3] + 1), np.int64)
    T[:, 1:, 1:] = tap.cumsum(1).cumsum(2)
    return T.astype(np.int32)


def constants(ma, fa, mw, fw):
    """(kP, kA, kW, kN) in double: ma' = ma + 128 fa, mw' = mw + 128 fw, kP = fa fw, kA = fa mw', kW = ma' fw, kN = ma' mw'."""
    ma, fa, mw, fw = float(ma), float(fa), float(mw), float(fw)
    ma2, mw2 = ma + 128. * fa, mw + 128. * fw
    return fa * fw, fa * mw2, ma2 * fw, ma2 * mw2


def terms(xq, wq, stride=(1, 1), padding=(0, 0), dilation=(1, 1), groups=1):
    """(P, A, Wv, Nv) int64 [N, O, OH, OW] over the in-image taps: P = sum q'x q'w, A = sum q'x, Wv = sum q'w, Nv = their
    count times C / groups.  Each is a convolution of codes or ones with zero padding (int8_oracle.i8_conv)."""
    geo = (stride, padding, dilation, groups)
    ones_x, ones_w = np.ones(xq.shape, np.int8), np.ones(wq.shape, np.int8)
    return (I8.i8_conv(xq, wq, *geo), I8.i8_conv(xq, ones_w, *geo), I8.i8_conv(ones_x, wq, *geo),
            I8.i8_conv(ones_x, ones_w, *geo))


def epilogue(P, A, Wv, Nv, k, bias=None):
    """y = fp32(((kP P + kA A) + kW Wv) + kN Nv) + bias[o], every product and sum a double op; no bias adds +0.0."""
    kP, kA, kW, kN = (f64(v) for v in k)
    t = kP * P.astype(f64)
    t = t + kA * A.astype(f64)
    t = t + kW * Wv.astype(f64)
    t = t + kN * Nv.astype(f64)
    b = np.zeros(P.shape[1], f32) if bias is None else np.asarray(bias, f32)
    return t.astype(f32) + b.reshape((1, -1) + (1,) * (P.ndim - 2))


def conv(x, running_min, running_max, act_bits, w_hat, w_min, w_scale, w_bits, bias=None, stride=(1, 1), padding=(0, 0),
         dilation=(1, 1), groups=1):
    """(P, y) of an affine layer from its fp32 input and fake-quantized weights."""
    xq, _ = act_codes(x, running_min, running_max, act_bits)
    wq, bad = weight_codes(w_hat, w_min, w_scale, w_bits)
    assert bad == 0
    _, ma, fa, _, _ = act_scalars(running_min, running_max, act_bits)
    P, A, Wv, Nv = terms(xq, wq, stride, padding, dilation, groups)
    return P, epilogue(P, A, Wv, Nv, constants(ma, fa, w_min, w_scale), bias)
