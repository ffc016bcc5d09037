"""Oracle of the affine residual epilogue (dfq_i8_affine_conv_fused)  --  TEST INFRASTRUCTURE.

On top of tests/int8_affine_oracle.py: what the per-layer affine path computes from a convolution to the next layer's
input - the double epilogue y = fp32(kP P + kA A + kW Wv + kN Nv) + bias, the pass-throughs before a residual add as one
clamp that keeps NaN, the fp32 add, the pass-throughs after it - and then the codes and per-pixel sums
dfq_i8_affine_quantize gives that fp32 value at the consumer's range and bits.
"""
import numpy as np

import int8_affine_oracle as A
import int8_residual_oracle as RO

f32 = np.float32
NONE = RO.NONE


def epilogue_value(y, r=None, pre=NONE, post=NONE, gpu_nan=False):
    """clamp(clamp(y, *pre) + r, *post) in fp32 (r None: no add).  gpu_nan: every NaN is the one an H100 fp32 add returns
    (the epilogue's NaNs all come out of the bias or residual add)."""
    v = RO.i8_epilogue_value(y, r, pre, post)
    return np.where(np.isnan(v), RO.GPU_NAN, v).astype(f32) if gpu_nan else v


def fused(P, Ax, Wv, Nv, k, bias=None, r=None, pre=NONE, post=NONE, out=None, gpu_nan=True):
    """(v fp32 [N, O, OH, OW], codes int8 [N, O, OH, OW] | None, S int32 [N, OH, OW] | None) of the epilogue from the four
    integer terms (int8_affine_oracle.terms); out = the consumer's (act_min, act_max, act_bits), None: no codes."""
    v = epilogue_value(A.epilogue(P, Ax, Wv, Nv, k, bias), r, pre, post, gpu_nan)
    if out is None:
        return v, None, None
    q, S = A.act_codes(v, *out)
    return v, q, S


def to_nhwc(q):
    """[N, O, H, W] codes -> [N, H, W, round_up(O, 16)], pad channels 0: the layout the epilogue writes."""
    N, O_, H, W = q.shape
    out = np.zeros((N, H, W, (O_ + 15) // 16 * 16), np.int8)
    out[..., :O_] = q.transpose(0, 2, 3, 1)
    return out
