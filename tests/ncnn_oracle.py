"""Oracle of ncnn's plane mean (dfq_i8_plane_mean, ncnn.PlaneMean)  --  TEST INFRASTRUCTURE.

The rule is a reading of ncnn's reduction.cpp (Reduction MEAN, coeff 1) and pooling.cpp (Pooling global average) of the
era of the reference's model; no ncnn build was available to confirm it:
    sum = 0.f;  for p in 0 .. P - 1: sum = fp32(sum + x[p])          sequential, every add rounded to fp32
    Reduction MEAN:          fp32(sum * fp32(1.f / P))
    Pooling global average:  fp32(sum / P)
and the consumer's codes are int8_oracle.i8_quantize of that value (roundf, clamp +-127, NaN -> -127).
"""
import numpy as np

import int8_oracle as I8

f32 = np.float32


def plane_mean(x, divide):
    """fp32 [N, C] of x fp32 [N, C, P]: the sequential sum over P, column by column (numpy's fp32 add rounds each step),
    then the layer's final op."""
    x = np.asarray(x, f32)
    s = np.zeros(x.shape[:2], f32)
    with np.errstate(over="ignore", invalid="ignore"):
        for p in range(x.shape[2]):
            s = (s + x[:, :, p]).astype(f32)
        P = f32(x.shape[2])
        return (s / P).astype(f32) if divide else (s * (f32(1) / P)).astype(f32)


def q8(v, s):
    return I8.i8_quantize(v, s)
