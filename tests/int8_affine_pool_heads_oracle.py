"""Oracle of the affine int8 max pool (dfq_i8_affine_maxpool) and of the affine detection-head rows
(dfq_i8_affine_conv_rows)  --  TEST INFRASTRUCTURE.

Codes mode is the byte-wise max of shifted codes over the taps inside the input, -128 (torch's -inf) for a window without
one; fp32 mode is tests/int8_pool_cat_oracle.py's restatement of torch's CUDA max_pool2d followed by the quantizer oracle
of dfq_i8_affine_quantize (tests/int8_affine_oracle.py act_codes).  S is the codes' sum over the real channels.  The rows
are the layer's value through clamp, the operand's observer, clamp and the tail observer (tests/int8_affine_observe_oracle.py),
permuted pixel-major into a slice of each image's floats.
"""
import numpy as np

import int8_affine_chain_oracle as AC
import int8_affine_observe_oracle as AO
import int8_affine_oracle as A
import int8_pool_cat_oracle as PO


def maxpool_codes(xq, C, k, s, p, d, ceil_mode):
    """(codes int8 [N, OH, OW, Cpad], S int32 [N, OH, OW]) of shifted codes xq int8 NHWC [N, H, W, Cpad]: the max over
    the window's taps inside the input; -128 in the real channels and 0 in the pad channels of a window without one."""
    N, H, W, Cp = xq.shape
    OH, OW = PO.pool_extent(H, k[0], p[0], s[0], d[0], ceil_mode), PO.pool_extent(W, k[1], p[1], s[1], d[1], ceil_mode)
    m = np.full((N, OH, OW, Cp), -128, np.int16)
    seen = np.zeros((OH, OW), bool)
    for ih, iw, vh, vw in PO._taps(H, W, OH, OW, k, s, p, d):
        v = xq[:, np.clip(ih, 0, H - 1)][:, :, np.clip(iw, 0, W - 1)].astype(np.int16)
        ok = vh[:, None] & vw[None, :]
        m = np.where(ok[None, :, :, None], np.maximum(m, v), m)
        seen |= ok
    m[:, ~seen, C:] = 0
    q = m.astype(np.int8)
    return q, q[..., :C].astype(np.int32).sum(-1)


def maxpool_fp32(x, k, s, p, d, ceil_mode, out=None):
    """(y fp32 [N, C, OH, OW], codes int8 [N, OH, OW, round_up(C, 16)] | None, S | None) of fp32 x: torch's max_pool2d and,
    with out = (act_min, act_max, act_bits), the codes and sums dfq_i8_affine_quantize gives y."""
    y = PO.i8_maxpool(x, k, s, p, d, ceil_mode)
    if out is None:
        return y, None, None
    q, S = A.act_codes(y, *out)
    return y, AC.to_nhwc(q), S


def rows_value(y, pre, post, obs=None, tail=None):
    """fq(clamp(fq(clamp(y, pre), obs), post), tail) of the layer's fp32 NCHW value y (obs / tail None: off)."""
    v = AO.observed_value(y, None, pre, post, obs, None, gpu_nan=False)
    return v if tail is None else AO.fq(v, tail)


def write_rows(out, v, off):
    """Place v [N, O, OH, OW] pixel-major at floats [off, off + OH * OW * O) of each image of out [N, ...]."""
    flat = out.reshape(out.shape[0], -1)
    n = v[0].size
    flat[:, off:off + n] = np.asarray(v).transpose(0, 2, 3, 1).reshape(v.shape[0], n)
    return out
