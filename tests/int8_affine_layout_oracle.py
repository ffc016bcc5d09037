"""Integer oracle of dfq_i8_affine_conv_layout's pad code  --  TEST INFRASTRUCTURE.

A zero F.pad in front of an affine layer quantizes its zeros to the code z' of +0.0 at the layer's input range.  The
folded layer must compute, bit for bit, the layer with padding 0 on the codes padded with z': these helpers form both
sides from tests/int8_affine_oracle.py's pieces.
"""
import numpy as np

import int8_affine_oracle as A

f32 = np.float32


def zero_code(running_min, running_max, num_bits):
    """z' = the shifted code act_codes gives +0.0 at this range."""
    q, _ = A.act_codes(np.zeros((1, 1, 1, 1), f32), running_min, running_max, num_bits)
    return int(q.reshape(-1)[0])


def pad_codes(xq, pad, z):
    """codes [N, C, H, W] padded by pad = (t, l) rows / columns on each side with the code z."""
    t, l = pad
    return np.pad(xq, ((0, 0), (0, 0), (t, t), (l, l)), constant_values=np.int8(z))


def folded_conv(x, act, w_hat, w_min, w_scale, w_bits, bias, pad, stride, dilation, groups):
    """y of the layer on F.pad(x) (padding 0), from the codes padded with z' (act = (min, max, bits))."""
    xq, _ = A.act_codes(x, *act)
    xq = pad_codes(xq, pad, zero_code(*act))
    wq, bad = A.weight_codes(w_hat, w_min, w_scale, w_bits)
    assert bad == 0
    _, ma, fa, _, _ = A.act_scalars(*act)
    terms = A.terms(xq, wq, stride, (0, 0), dilation, groups)
    return A.epilogue(*terms, A.constants(ma, fa, w_min, w_scale), bias)


def folded_terms_direct(xq, wq, pad, z, stride, dilation, groups):
    """(P, A, Wv, Nv) of the padded input by a direct loop over every tap: what the kernels' corrections must give."""
    t, l = pad
    N, C, H, W = xq.shape
    O, Cg, kh, kw = wq.shape
    OH = (H + 2 * t - dilation[0] * (kh - 1) - 1) // stride[0] + 1
    OW = (W + 2 * l - dilation[1] * (kw - 1) - 1) // stride[1] + 1
    out = [np.zeros((N, O, OH, OW), np.int64) for _ in range(4)]
    for o in range(O):
        cs = range(C) if groups == 1 else [o]
        w = wq[o].astype(np.int64)
        for oh in range(OH):
            for ow in range(OW):
                for r in range(kh):
                    for s in range(kw):
                        ih, iw = oh * stride[0] - t + r * dilation[0], ow * stride[1] - l + s * dilation[1]
                        inside = 0 <= ih < H and 0 <= iw < W
                        for j, c in enumerate(cs):
                            xv = xq[:, c, ih, iw].astype(np.int64) if inside else np.full(N, z, np.int64)
                            wv = w[j if groups == 1 else 0, r, s]
                            out[0][:, o, oh, ow] += xv * wv
                            out[1][:, o, oh, ow] += xv
                            out[2][:, o, oh, ow] += wv
                            out[3][:, o, oh, ow] += 1
    return out
