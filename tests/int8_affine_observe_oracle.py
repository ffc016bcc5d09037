"""Oracle of the observed affine epilogue (dfq_i8_affine_conv_observed)  --  TEST INFRASTRUCTURE.

On top of tests/int8_affine_chain_oracle.py: the per-layer path of the reference's evaluation state from a convolution to
the tensor after a residual add whose operands replace_op()'s patched add quantizes - the double epilogue, the clamp before
the add, QuantMeasure's eval-mode fake quantization of the fused operand (obs) and of the residual (res), the fp32 add, the
clamp after it - and the codes and per-pixel sums of the consumer's quantizer.  torch_value is the same chain with
QuantMeasure itself, for the comparisons on the device.
"""
import numpy as np

import int8_affine_oracle as A
import int8_residual_oracle as RO

f32 = np.float32
NONE = RO.NONE


def _clamp(v, lo, hi):
    lo, hi = f32(lo), f32(hi)
    return np.where(v < lo, lo, np.where(v > hi, hi, v)).astype(f32)


def fq(v, o):
    """QuantMeasure's output for v at o = (running_min, running_max, num_bits) on a CUDA tensor: NaN stays NaN, +-inf
    saturate."""
    lo, hi, bits = o
    return np.asarray(A.fake_quant(np.asarray(v, f32), lo, hi, bits), f32)


def observed_value(y, r=None, pre=NONE, post=NONE, obs=None, res=None, gpu_nan=True):
    """clamp(fq(clamp(y, pre), obs) + fq(r, res), post) in fp32; obs / res None: that observer is off; r None: no add."""
    v = _clamp(np.asarray(y, f32), *pre)
    if obs is not None:
        v = fq(v, obs)
    if r is not None:
        rv = np.asarray(r, f32)
        if res is not None:
            rv = fq(rv, res)
        with np.errstate(invalid="ignore", over="ignore"):
            v = (v + rv).astype(f32)
    v = _clamp(v, *post)
    return np.where(np.isnan(v), RO.GPU_NAN, v).astype(f32) if gpu_nan else v


def observed(P, Ax, Wv, Nv, k, bias=None, r=None, pre=NONE, post=NONE, out=None, obs=None, res=None, gpu_nan=True):
    """(v fp32 [N, O, OH, OW], codes int8 | None, S int32 | None) of the epilogue from the four integer terms."""
    v = observed_value(A.epilogue(P, Ax, Wv, Nv, k, bias), r, pre, post, obs, res, gpu_nan)
    if out is None:
        return v, None, None
    q, S = A.act_codes(v, *out)
    return v, q, S


def _measure(o, device):
    from dfq_b200.utils.quantize import QuantMeasure
    q = QuantMeasure(num_bits=int(o[2])).to(device).eval()
    q.running_min.fill_(float(f32(o[0])))
    q.running_max.fill_(float(f32(o[1])))
    return q


def torch_value(y, r=None, pre=NONE, post=NONE, obs=None, res=None):
    """The per-layer path in torch: torch.clamp-free clamps that keep NaN, QuantMeasure modules as the observers, the
    fp32 add."""
    import torch

    def clamp(t, lo, hi):
        t = torch.where(t < lo, torch.full_like(t, lo), t)
        return torch.where(t > hi, torch.full_like(t, hi), t)
    with torch.no_grad():
        v = clamp(y, *pre)
        if obs is not None:
            v = _measure(obs, y.device)(v)
        if r is not None:
            v = v + (_measure(res, r.device)(r) if res is not None else r)
        return clamp(v, *post)
