"""Int8 execution of calibrated Conv2d / Linear layers on the H100.

The reference's end product is "true int8 inference": convert_ncnn.py:109-201 writes the weight and activation scales
(128 / max|.|) of a calibrated model into an ncnn table and ncnn's runtime then executes the model in int8 on a CPU.  This
module runs the same dequantizing int8 convolution on the GPU (include/dfq_b200.h, dfq_i8_*), one layer at a time:

    q(v, s) = clamp(round_half_away(fp32(v * s)), -127, 127)       activations: scale a, weights: w_s[o]
    y       = fp32(fp32_rn(sum q(x) q(w)) * dq[o]) + bias[o],       dq[o] = fp32(1 / fp32(a * w_s[o]))

Each converted layer takes and returns fp32 NCHW like the module it replaces; ReLU, residual adds, pooling and whatever
else sits between target layers stay in torch (ncnn keeps its elementwise ops in fp32 too).  Dense layers (groups == 1,
Linear as a 1x1 convolution) run on the tensor cores; depthwise layers (groups == C == O) on the CUDA cores; any other
grouping is refused.  There is no CPU fallback.

Order of the calibration steps, as in convert_ncnn.py: BN fold, equalization (and bias correction, if used), activation
ranges (set_quant_minmax or update_stat), then convert_to_int8 - BEFORE quantize_targ_layer, whose fake-quantized weights
are not the fp32 weights the int8 codes are made from.  The observers replace_op() installs for functional ops are not used:
tensors between converted layers stay fp32.

convert_affine executes the reference's own quantization instead (asymmetric per-tensor min / max, dfq_i8_affine_*): called
AFTER quantize_targ_layer and the activation ranges, it recovers the weight codes from the fake-quantized weights (of a
QConv2d / QuantConv2d layer: the weights its forward quantizes on the GPU, the --distill_range and --trainable states) and
computes each layer from integer sums, equal to the fake-quantized layer up to fp32 rounding.  chain_affine carries its codes
between layers; in the reference's evaluation state (replace_op() active with a CustomTensorOP) it replays the functional-op
observers into its graph and runs those on a producer's path in that producer's epilogue (dfq_i8_affine_conv_observed), so it
computes what the per-layer model computes under the patched ops.  chain_affine(concat=True, fold_pads=True) also folds zero
pads into the convolutions after them as pad codes and has the producers and bilinear upsamples of channel concatenations
write the consumer's codes directly (dfq_i8_affine_conv_layout, dfq_i8_affine_upsample_bilinear), and
chain_affine(pools=True) carries the codes through max pools (dfq_i8_affine_maxpool).

save / load write a chained model of either scheme to one file and rebuild it, in any process, from dfq_b200 alone
(dfq_b200/int8_io.py).
"""
import collections
import ctypes as C
import dataclasses
import operator
import os
import sys
from typing import NamedTuple, Optional, Tuple

import numpy as np
import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, engine, export

_f32 = np.float32


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _pair(v):
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def dequant_scales(act_scale, w_scale):
    """dq[o] = fp32(1 / fp32(a * w_s[o])); 0 where a * w_s[o] is 0 (a zero range quantizes to codes 0)."""
    den = _f32(act_scale) * np.asarray(w_scale, _f32)
    return np.where(den == 0, _f32(0), _f32(1) / np.where(den == 0, _f32(1), den)).astype(_f32)


def check_scale(what, scale, layer):
    """Refuse an activation or weight scale (128 / range) that is not a finite, non-negative fp32 number.  A range below about
    3.8e-37 gives a scale that is inf in fp32, and inf * 0 would quantize every zero input to NaN and then to -127."""
    s = np.asarray(scale, np.float64).reshape(-1)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        s32 = s.astype(_f32)
        bad = ~np.isfinite(s32) | (s32 < 0)
        if bad.any():
            i = int(np.argmax(bad))
            raise _lib.DfqError("layer %s: %s scale %g%s (range 128 / scale = %g) is not a finite non-negative fp32 number"
                                % (layer, what, float(s[i]), " of channel %d" % i if s.size > 1 else "", 128. / s[i]))


class Epilogue(NamedTuple):
    """The residual epilogue of a chained layer (dfq_i8_conv_fused): v = clamp(dequant, *pre); v = v + r when `residual`
    (forward(x, r)); v = clamp(v, *post); then the codes of v at out_scale (None: no codes) and / or v in fp32 (`fp32`).
    Both clamps keep NaN, (-inf, inf) is none."""
    out_scale: Optional[float] = None
    pre: Tuple[float, float] = (-float("inf"), float("inf"))
    post: Tuple[float, float] = (-float("inf"), float("inf"))
    residual: bool = False
    fp32: bool = False


def _ordered(lo, hi, what="activation"):
    lo, hi = _f32(lo), _f32(hi)
    if np.isnan(lo) or np.isnan(hi) or lo > hi:
        raise _lib.DfqError("%s bounds (%g, %g) must be ordered and not NaN" % (what, lo, hi))
    return float(lo), float(hi)


def _channel_slice(out_slice, channels, who):
    """(coff, cstride) of channels [coff, coff + round_up(channels, 16)) of an int8 NHWC tensor of cstride channels (a
    concatenation's codes), or DfqError naming `who` when the slice is not 16-aligned inside it."""
    coff, cstride = (int(v) for v in out_slice)
    if coff < 0 or coff % 16 or cstride % 16 or coff + (channels + 15) // 16 * 16 > cstride:
        raise _lib.DfqError("%s: channel slice (%d, %d) is not 16-aligned inside its tensor" % (who, coff, cstride))
    return coff, cstride


def _zero_padding_refusal(conv, who=""):
    """The DfqError refusing an nn.Conv2d whose padding is not numeric zero padding (all the int8 kernels compute), its
    text prefixed by `who`; None when it is."""
    if conv.padding_mode == "zeros" and not isinstance(conv.padding, str):
        return None
    return _lib.DfqError("%sint8 execution supports numeric zero padding only (padding=%r, padding_mode=%r)"
                         % (who, conv.padding, conv.padding_mode))


class _ConvLayer(nn.Module):
    """What the two schemes' convolution layers share: the shape of the convolution, its geometry table, the copies
    `chained` makes and the checks of `run`."""

    codes_in = False
    epilogue = None
    out_slice = None
    layer_name = None
    _copied = ("out_channels", "in_channels", "groups", "kernel_size", "stride", "padding", "dilation", "cpad")

    def __init__(self, weight, stride, padding, dilation, groups):
        super().__init__()
        O, Cg, kh, kw = weight.shape
        self.out_channels, self.in_channels, self.groups = int(O), int(Cg) * int(groups), int(groups)
        self.kernel_size, self.stride, self.padding, self.dilation = (int(kh), int(kw)), _pair(stride), _pair(padding), _pair(dilation)
        self.cpad = (self.in_channels + 15) // 16 * 16

    def _geometry(self, N, H, W, stride=None, padding=None):
        (sh, sw), (ph, pw), (dh, dw) = stride or self.stride, padding or self.padding, self.dilation
        kh, kw = self.kernel_size
        g = np.zeros(1, _lib.I8_CONV_DT)
        for k, v in dict(N=N, C=self.in_channels, H=H, W=W, O=self.out_channels, kh=kh, kw=kw, stride_h=sh, stride_w=sw,
                         pad_h=ph, pad_w=pw, dil_h=dh, dil_w=dw, groups=self.groups,
                         OH=(H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, OW=(W + 2 * pw - dw * (kw - 1) - 1) // sw + 1,
                         Cpad=self.cpad).items():
            g[0][k] = v
        return g

    def _pack_geometry(self):
        # geometry of a 1-pixel image: the packers only read O, C, kh, kw, groups and Cpad
        kh, kw = self.kernel_size
        return self._geometry(1, (kh - 1) * self.dilation[0] + 1, (kw - 1) * self.dilation[1] + 1, stride=(1, 1),
                              padding=(0, 0))

    def _who(self):
        return self.layer_name or "%s(%d, %d, kernel_size=%s)" % (type(self).__name__, self.in_channels, self.out_channels,
                                                                  self.kernel_size)

    @classmethod
    def _build(cls, attrs, buffers):
        """A module of this class with the given attributes on the given buffers, nothing packed: the one route by which
        chained copies (_copy) and loaded layers (int8.load) are made."""
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        for k, v in attrs.items():
            setattr(new, k, v)
        for k, b in buffers.items():
            new.register_buffer(k, b)
        return new

    def _copy(self, codes_in, name):
        """A new module of the same class on the same buffers, with the attributes in _copied, codes_in and name."""
        return self._build(dict({k: getattr(self, k) for k in self._copied}, codes_in=bool(codes_in), layer_name=name),
                           self._buffers)

    def _check_residual(self, residual):
        if (residual is not None) != bool(self.epilogue and self.epilogue.residual):
            raise _lib.DfqError("layer %s: %s" % (self._who(), "takes a residual input" if residual is None else
                                                    "takes no residual input"))

    def _check_out(self, out):
        if out is not None and self.out_slice is None:
            raise _lib.DfqError("layer %s: takes no output tensor" % self._who())

    def out_extent(self, x):
        """OH * OW * C_out: the floats one image of input x (fp32 NCHW, or the codes of a codes_in layer - the affine
        scheme's (codes, S) pair) gives."""
        if isinstance(x, tuple):
            x = x[0]
        H, W = (x.shape[1], x.shape[2]) if self.codes_in else (x.shape[2], x.shape[3])
        g = self._geometry(1, int(H), int(W))
        return int(g[0]["OH"]) * int(g[0]["OW"]) * self.out_channels

    def _rows_out(self, out, off, N, OH, OW, dev):
        """(out, off) of a rows-mode layer: `out` checked to hold this layer's rows at `off` of each image, or a new
        [N, OH * OW, C_out] tensor and 0."""
        n = OH * OW * self.out_channels
        if out is None:
            return torch.empty((N, OH * OW, self.out_channels), dtype=torch.float32, device=dev), 0
        if not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.dim() < 2 or out.shape[0] != N or \
                out.device != dev or not out.is_contiguous():
            raise _lib.DfqError("layer %s: the rows' tensor must be contiguous fp32 [%d, ...] on %s, got %s" % (
                self._who(), N, dev, "%s %s on %s" % (out.dtype, list(out.shape), out.device)
                if isinstance(out, torch.Tensor) else type(out).__name__))
        if not 0 <= off <= out[0].numel() - n:
            raise _lib.DfqError("layer %s: rows [%d, %d) do not fit in the %d floats of an image"
                                % (self._who(), off, off + n, out[0].numel()))
        return out, off

    def _output_geometry(self, N, H, W):
        """(geometry, OH, OW) of an input [N, *, H, W], or DfqError when it is smaller than the kernel."""
        g = self._geometry(N, H, W)
        OH, OW = int(g[0]["OH"]), int(g[0]["OW"])
        if OH <= 0 or OW <= 0:
            raise _lib.DfqError("int8 layer: input %dx%d is smaller than the kernel" % (H, W))
        return g, OH, OW

    def _residual(self, r, shape, dev):
        """The residual r, checked to be fp32 `shape` on dev, contiguous; None when r is."""
        if r is None:
            return None
        if not isinstance(r, torch.Tensor) or r.dtype != torch.float32 or not r.is_cuda or tuple(r.shape) != shape or \
                r.device != dev:
            raise _lib.DfqError("layer %s: the residual must be fp32 %s on %s, got %s" % (
                self._who(), list(shape), dev, "%s %s on %s" % (r.dtype, list(r.shape), r.device)
                if isinstance(r, torch.Tensor) else type(r).__name__))
        return r.contiguous()

    def _linear_forward(self, x):
        """forward of the Linear layers: x [..., in_features] as the 1x1 convolution of [B, I, 1, 1]."""
        lead = x.shape[:-1]
        y, _ = self.run(x.reshape(-1, self.in_channels, 1, 1))
        return y.reshape(*lead, self.out_channels)


class _Int8Layer(_ConvLayer):
    """Packed int8 weights, dq and bias of one layer on the device; forward quantizes the input and convolves.

    Execution modes, set only on the copies chain_int8 makes (`chained`): `codes_in` - the input is already int8 NHWC codes
    [N, H, W, cpad] at this layer's act_scale; `requant` = (out_scale, lo, hi) - the output is the next layer's int8 NHWC
    codes (dfq_i8_conv_requant) instead of fp32 NCHW; `epilogue` - the residual epilogue (dfq_i8_conv_fused, see Epilogue);
    `rows` - the clamped fp32 output pixel-major, a detection head's rows of its concatenation (dfq_i8_conv_nhwc).
    A layer convert_to_int8 made takes and returns fp32 only."""

    requant = None
    rows = False
    _copied = _ConvLayer._copied + ("act_scale",)
    _modes = ("codes_in", "layer_name", "requant", "epilogue", "out_slice", "rows")     # what chained() sets

    def __init__(self, weight, bias, act_scale, w_scale, stride=1, padding=0, dilation=1, groups=1):
        super().__init__(weight, stride, padding, dilation, groups)
        O, _, kh, kw = weight.shape
        check_scale("activation", act_scale, self._who())
        check_scale("weight", w_scale, self._who())
        self.act_scale = float(_f32(act_scale))
        depthwise = self.groups == self.in_channels == self.out_channels and self.groups > 1
        if self.groups != 1 and not depthwise:
            raise _lib.DfqError("int8 execution supports groups == 1 or depthwise (groups == C_in == C_out), got groups=%d "
                                "C_in=%d C_out=%d" % (self.groups, self.in_channels, self.out_channels))
        dev = engine._default_device()
        w_scale = np.broadcast_to(np.asarray(w_scale, _f32), (O,)).copy()
        taps = kh * kw
        self.register_buffer("weight_codes", torch.zeros((taps * self.cpad,) if depthwise else (O * taps * self.cpad,),
                                                         dtype=torch.int8, device=dev))
        self.register_buffer("w_scale", torch.from_numpy(w_scale).to(dev))
        self.register_buffer("dq", torch.from_numpy(dequant_scales(self.act_scale, w_scale)).to(dev))
        b = torch.zeros(O) if bias is None else bias.detach().float()
        self.register_buffer("bias", b.to(dev).contiguous())
        lib = _lib.load()
        if weight.dtype == torch.int8:                          # codes, packed verbatim (Int8Conv2d.from_codes)
            w = weight.detach().to(dev).contiguous()
            with _lib.launch(w, self.weight_codes) as st:
                _lib.check(lib.dfq_i8_pack_codes(_ptr(w), _ptr(self.weight_codes), _lib.table_ptr(self._pack_geometry()),
                                                 st), "dfq_i8_pack_codes")
            return
        w = weight.detach().float().to(dev).contiguous()
        with _lib.launch(w, self.weight_codes) as st:
            _lib.check(lib.dfq_i8_pack_weights(_ptr(w), _ptr(self.w_scale), _ptr(self.weight_codes),
                                               _lib.table_ptr(self._pack_geometry()), st), "dfq_i8_pack_weights")

    def unpack_codes(self):
        """The int8 weight codes [O, C/groups, kh, kw] of the packed layer (dfq_i8_unpack_codes), on its device."""
        kh, kw = self.kernel_size
        codes = torch.empty((self.out_channels, self.in_channels // self.groups, kh, kw), dtype=torch.int8,
                            device=self.weight_codes.device)
        with _lib.launch(self.weight_codes, codes) as st:
            _lib.check(_lib.load().dfq_i8_unpack_codes(_ptr(self.weight_codes), _ptr(codes),
                                                       _lib.table_ptr(self._pack_geometry()), st),
                       "dfq_i8_unpack_codes (layer %s)" % self._who())
        return codes

    def chained(self, codes_in=False, requant=None, epilogue=None, name=None, out_slice=None, rows=False, sums=False):
        """A new module of the same class on the same packed buffers (weight_codes, dq, bias, w_scale), in the given execution
        mode: codes_in - take int8 NHWC codes; requant = (out_scale, lo, hi) - return the next layer's codes; epilogue - an
        Epilogue: the residual epilogue (not together with requant); out_slice = (coff, cstride), with requant - write the
        codes into channels [coff, coff + round_up(C_out, 16)) of an int8 NHWC tensor [N, OH, OW, cstride] (a channel
        concatenation, dfq_i8_conv_slice), given as forward(x, out=...) or made when out is None; rows - the fp32 output
        pixel-major (dfq_i8_conv_nhwc): forward(x, out=y, off=off) writes permute(0, 2, 3, 1) of it as OH * OW * C_out floats
        at y[n].view(-1)[off:] of a contiguous fp32 y [N, ...] (a detection head's slice of its [N, R, k] concatenation), or
        returns a new [N, OH * OW, C_out] tensor when out is None; the clamps come from an fp32-only epilogue without
        residual (none: no clamp), and rows excludes requant.  name: the layer's name in error messages.  sums: the affine
        scheme's per-pixel code sums (_AffineInt8Layer.chained); ncnn codes have none, so it changes nothing here.  self
        is not modified."""
        new = self._copy(codes_in, name)
        if requant is not None and epilogue is not None:
            raise _lib.DfqError("layer %s: requant and epilogue are two output modes; give one" % new._who())
        if requant is not None:
            s, lo, hi = requant
            check_scale("output", s, "%s -> next layer" % type(self).__name__)
            lo, hi = _ordered(lo, hi, "activation")
            requant = (float(_f32(s)), lo, hi)
        new.requant = requant
        if epilogue is not None:
            e = Epilogue(*epilogue)
            if e.out_scale is None and not e.fp32:
                raise _lib.DfqError("layer %s: the epilogue returns neither codes nor fp32" % new._who())
            if e.out_scale is not None:
                check_scale("output", e.out_scale, "%s -> next layer" % new._who())
            epilogue = Epilogue(None if e.out_scale is None else float(_f32(e.out_scale)), _ordered(*e.pre, what="pre-add"),
                                _ordered(*e.post, what="post-add"), bool(e.residual), bool(e.fp32))
        new.epilogue = epilogue
        if out_slice is not None:
            if requant is None:
                raise _lib.DfqError("layer %s: a channel slice needs requant" % new._who())
            out_slice = _channel_slice(out_slice, self.out_channels, "layer %s" % new._who())
        new.out_slice = out_slice
        if rows:
            if requant is not None or out_slice is not None or \
                    (epilogue is not None and (epilogue.out_scale is not None or epilogue.residual)):
                raise _lib.DfqError("layer %s: pixel-major fp32 rows exclude codes and a residual" % new._who())
            new.epilogue = epilogue or Epilogue(fp32=True)
        new.rows = bool(rows)
        return new

    def run(self, x, with_acc=False, residual=None, out=None, off=0):
        """(y, acc | None) for x [N, C, H, W] fp32 on the GPU; acc = the int32 sums before the epilogue.  In the chained modes
        x is int8 codes [N, H, W, cpad] (codes_in) and y int8 codes [N, OH, OW, round_up(C_out, 16)] (requant).  With an
        epilogue, y is the codes, the fp32 output, or (codes, fp32 output) when it returns both, and `residual` is the fp32
        tensor [N, C_out, OH, OW] the epilogue adds (exactly that shape, no broadcasting, on x's device).  With out_slice, y
        is `out` (int8 [N, OH, OW, cstride] on x's device) or a new such tensor, its slice written.  With rows, y is `out`
        with this layer's rows written at `off` of each image, or a new [N, OH * OW, C_out] tensor (see chained)."""
        if not x.is_cuda or not self.dq.is_cuda:
            raise _lib.DfqError("int8 layers run on the GPU only (no CPU fallback): input on %s, layer on %s"
                                % (x.device, self.dq.device))
        if x.device != self.dq.device:
            raise _lib.DfqError("layer %s is on %s, its input on %s: an int8 layer runs on its own device"
                                % (self._who(), self.dq.device, x.device))
        if self.codes_in:
            if x.dtype != torch.int8 or x.dim() != 4 or x.shape[3] != self.cpad:
                raise _lib.DfqError("chained int8 layer expects int8 codes [N, H, W, %d], got %s %s"
                                    % (self.cpad, x.dtype, tuple(x.shape)))
            N, H, W, _ = x.shape
        elif x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != self.in_channels:
            raise _lib.DfqError("int8 layer expects fp32 [N, %d, H, W], got %s %s" % (self.in_channels, x.dtype, tuple(x.shape)))
        else:
            N, _, H, W = x.shape
        if (self.requant is not None or self.epilogue is not None) and with_acc:
            raise _lib.DfqError("a requantizing int8 layer does not return its int32 sums")
        self._check_residual(residual)
        x = x.contiguous()
        g, OH, OW = self._output_geometry(N, H, W)
        lib = _lib.load()
        if self.codes_in:
            xq = x
        else:
            xq = torch.empty(N * H * W * self.cpad, dtype=torch.int8, device=x.device)
            with _lib.launch(x, self.dq) as st:
                _lib.check(lib.dfq_i8_quantize_nhwc(_ptr(x), _ptr(xq), N, self.in_channels, H, W, self.cpad,
                                                    C.c_float(self.act_scale), st), "dfq_i8_quantize_nhwc")
        if self.rows:
            return self._run_rows(xq, out, off, g, N, OH, OW), None
        if self.epilogue is not None:
            return self._run_fused(xq, residual, g, N, OH, OW), None
        self._check_out(out)
        if self.out_slice is not None:
            return self._run_slice(xq, out, g, N, OH, OW), None
        if self.requant is not None:
            s, lo, hi = self.requant
            yq = torch.empty((N, OH, OW, (self.out_channels + 15) // 16 * 16), dtype=torch.int8, device=x.device)
            with _lib.launch(xq, self.weight_codes) as st:
                _lib.check(lib.dfq_i8_conv_requant(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias), _ptr(yq),
                                                   C.c_float(s), C.c_float(lo), C.c_float(hi), _lib.table_ptr(g), st),
                           "dfq_i8_conv_requant")
            return yq, None
        y = torch.empty((N, self.out_channels, OH, OW), dtype=torch.float32, device=x.device)
        acc = torch.empty(y.shape, dtype=torch.int32, device=x.device) if with_acc else None
        with _lib.launch(xq, self.weight_codes) as st:
            _lib.check(lib.dfq_i8_conv(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias), _ptr(y), _ptr(acc),
                                       _lib.table_ptr(g), st), "dfq_i8_conv")
        return y, acc

    def _run_slice(self, xq, out, g, N, OH, OW):
        (s, lo, hi), (coff, cstride) = self.requant, self.out_slice
        shape = (N, OH, OW, cstride)
        if out is None:
            out = torch.empty(shape, dtype=torch.int8, device=xq.device)
        elif not isinstance(out, torch.Tensor) or out.dtype != torch.int8 or tuple(out.shape) != shape or \
                out.device != xq.device or not out.is_contiguous():
            raise _lib.DfqError("layer %s: the concatenation's codes must be contiguous int8 %s on %s, got %s" % (
                self._who(), list(shape), xq.device, "%s %s on %s" % (out.dtype, list(out.shape), out.device)
                if isinstance(out, torch.Tensor) else type(out).__name__))
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0, 0, out.data_ptr(), s, lo, hi, -_INF, _INF)
        with _lib.launch(xq, self.weight_codes, out) as st:
            _lib.check(_lib.load().dfq_i8_conv_slice(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias),
                                                     _lib.table_ptr(d), coff, cstride, _lib.table_ptr(g), st),
                       "dfq_i8_conv_slice (layer %s)" % self._who())
        return out

    def _run_rows(self, xq, out, off, g, N, OH, OW):
        e = self.epilogue
        out, off = self._rows_out(out, off, N, OH, OW, xq.device)
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0, out.data_ptr(), 0, 0.0) + e.pre + e.post
        with _lib.launch(xq, self.weight_codes, out) as st:
            _lib.check(_lib.load().dfq_i8_conv_nhwc(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias),
                                                    _lib.table_ptr(d), int(off), out[0].numel(), _lib.table_ptr(g),
                                                    st), "dfq_i8_conv_nhwc (layer %s)" % self._who())
        return out

    def _run_fused(self, xq, r, g, N, OH, OW):
        e = self.epilogue
        shape = (N, self.out_channels, OH, OW)
        r = self._residual(r, shape, xq.device)
        yq = None if e.out_scale is None else \
            torch.empty((N, OH, OW, (self.out_channels + 15) // 16 * 16), dtype=torch.int8, device=xq.device)
        y = torch.empty(shape, dtype=torch.float32, device=xq.device) if e.fp32 else None
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0 if r is None else r.data_ptr(), 0 if y is None else y.data_ptr(), 0 if yq is None else yq.data_ptr(),
                0.0 if e.out_scale is None else e.out_scale) + e.pre + e.post
        lib = _lib.load()
        with _lib.launch(xq, self.weight_codes, r, y, yq) as st:
            _lib.check(lib.dfq_i8_conv_fused(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias),
                                             _lib.table_ptr(d), _lib.table_ptr(g), st),
                       "dfq_i8_conv_fused (layer %s)" % self._who())
        return (yq, y) if yq is not None and y is not None else (y if yq is None else yq)


class Int8Conv2d(_Int8Layer):
    """nn.Conv2d executed in int8 (zero padding; groups == 1 or depthwise)."""

    @classmethod
    def from_conv(cls, conv: nn.Conv2d, act_scale, w_scale):
        err = _zero_padding_refusal(conv)
        if err is not None:
            raise err
        return cls(conv.weight, conv.bias, act_scale, w_scale, conv.stride, conv.padding, conv.dilation, conv.groups)

    @classmethod
    def from_codes(cls, codes, bias, act_scale, w_scale, stride=1, padding=0, dilation=1, groups=1):
        """The layer of int8 weight codes [O, C/groups, kh, kw] (an ncnn model file's, ncnn.load), packed verbatim
        (dfq_i8_pack_codes) rather than re-derived from fp32 weights; bias [O] or None, w_scale a scalar or [O]."""
        codes = torch.as_tensor(np.ascontiguousarray(codes, np.int8))
        if codes.dim() != 4:
            raise _lib.DfqError("int8 weight codes must be [O, C/groups, kh, kw], got %s" % list(codes.shape))
        return cls(codes, None if bias is None else torch.as_tensor(np.asarray(bias, _f32)), act_scale, w_scale, stride,
                   padding, dilation, groups)

    def forward(self, x, r=None, out=None, off=0):
        return self.run(x, residual=r, out=out, off=off)[0]

    def extra_repr(self):
        return "%d, %d, kernel_size=%s, stride=%s, padding=%s, dilation=%s, groups=%d, act_scale=%g" % (
            self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding, self.dilation, self.groups,
            self.act_scale)


class Int8Linear(_Int8Layer):
    """nn.Linear executed in int8: the 1x1 convolution of [B, I, 1, 1]."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, act_scale, w_scale):
        return cls(lin.weight.reshape(lin.out_features, lin.in_features, 1, 1), lin.bias, act_scale, w_scale)

    forward = _ConvLayer._linear_forward

    def extra_repr(self):
        return "in_features=%d, out_features=%d, act_scale=%g" % (self.in_channels, self.out_channels, self.act_scale)


# ---- the reference's own quantization: asymmetric per-tensor min / max -------------------------------------------------
AFFINE_MAX_K = 1 << 17          # K = kh * kw * C / groups: codes of -128 reach the int32 sums, K * 128 * 128 < 2^31
_GRID_ULPS = 8                  # weight-grid search: fp32 scales within this many ulps of (max - min) / (2^b - 1)


def act_affine_scalars(running_min, running_max, num_bits):
    """(ma, fa) of QuantMeasure's eval-mode fake quantization (utils/quantize.py, dfq_quant_dequant_dev with the range on the
    device): ma = fp32(running_min), fa = fp32(max((running_max - running_min) / (2^b - 1), 1e-8)), the scale in double."""
    mn, mx = float(_f32(running_min)), float(_f32(running_max))
    s = max((mx - mn) / (2. ** int(num_bits) - 1.), 1e-8)
    with np.errstate(over="ignore"):
        return _f32(mn), _f32(s)


def affine_constants(ma, fa, mw, fw):
    """(kP, kA, kW, kN) of the affine epilogue (include/dfq_b200.h, DfqI8Affine) in double, in this order: the shifted offsets
    ma' = ma + 128 fa and mw' = mw + 128 fw, then kP = fa fw, kA = fa mw', kW = ma' fw, kN = ma' mw'."""
    ma, fa, mw, fw = float(ma), float(fa), float(mw), float(fw)
    ma2 = ma + 128. * fa
    mw2 = mw + 128. * fw
    return fa * fw, fa * mw2, ma2 * fw, ma2 * mw2


def weight_grid_candidates(w_min, w_max, num_bits):
    """fp32 scales fw that may have produced fake-quantized weights with this min / max: fp32((max - min) / (2^b - 1)) in
    double (at least fp32(1e-8), quantize_targ_layer's floor) and its neighbours within _GRID_ULPS ulps, those whose
    top code reproduces max (fp32(fp32((2^b - 1) fw) + min) == max) first, then by distance."""
    mn, mx = _f32(w_min), _f32(w_max)
    qmax = _f32(2. ** int(num_bits) - 1.)
    with np.errstate(over="ignore", invalid="ignore"):
        base = _f32(max((float(mx) - float(mn)) / float(qmax), 1e-8))
    if not (np.isfinite(base) and np.isfinite(mn) and np.isfinite(mx)):
        return []
    cands, up, down = [base], base, base
    for _ in range(_GRID_ULPS):
        up, down = np.nextafter(up, _f32(np.inf)), np.nextafter(down, _f32(0))
        cands += [up, down]
    cands = [c for c in cands if c > 0 and np.isfinite(c)]
    with np.errstate(over="ignore"):
        top = [bool(_f32(_f32(qmax * c) + mn) == mx) for c in cands]
    return [c for t, c in sorted(zip(top, cands), key=lambda tc: not tc[0])]


class _AffineInt8Layer(_ConvLayer):
    """One layer of a fake-quantized model executed in integer arithmetic (dfq_i8_affine_*): the input is quantized with the
    range its `quant` observer had at conversion, the weight codes are recovered from the fake-quantized weights, and the
    output is fp32 NCHW.  The ranges are frozen: an observer whose update_stat is truthy would keep widening its range in
    the fake-quantized model (set_layer_bits leaves update_stat = the bit width, quirk Q1), this layer does not.

    Execution modes, set only on the copies chain_affine makes (`chained`): `codes_in` - the input is the pair (codes, S)
    another layer's epilogue wrote at this layer's range (S None for a depthwise layer); `epilogue` - an Epilogue whose
    out_scale is the consumer's (act_min, act_max, act_bits) (dfq_i8_affine_conv_fused), with `sums` - write S too;
    `out_slice` = (coff, cstride) - the codes go to a channel slice of a concatenation's codes and S adds into its sums;
    `pad_code` - the shifted code every out-of-image tap reads (a folded F.pad; dfq_i8_affine_conv_layout)."""

    sums = False
    observers = (None, None)
    tail_observer = None
    rows = False
    pad_code = None
    _copied = _ConvLayer._copied + ("act_bits", "w_bits", "act_min", "act_max", "w_min", "w_scale", "constants", "pad_code")
    # what chained() and observe() set
    _modes = ("codes_in", "layer_name", "epilogue", "sums", "out_slice", "rows", "observers", "tail_observer")

    def __init__(self, weight, bias, act_min, act_max, act_bits=8, w_bits=8, stride=1, padding=0, dilation=1, groups=1,
                 name=None):
        super().__init__(weight, stride, padding, dilation, groups)
        O, _, kh, kw = weight.shape
        self.layer_name = name
        _affine_refusal(self._who(), self.in_channels, self.out_channels, self.groups, self.kernel_size, act_bits, w_bits)
        self.w_bits = int(w_bits)
        self.act_min, self.act_max, self.act_bits = _affine_range(_f32(act_min), act_max, act_bits, "layer %s" % self._who(),
                                                                  "activation range")
        ma, fa = act_affine_scalars(act_min, act_max, act_bits)
        dev = engine._default_device()
        depthwise = self.groups > 1
        taps = kh * kw
        self.register_buffer("weight_codes", torch.zeros((taps * self.cpad,) if depthwise else (O * taps * self.cpad,),
                                                         dtype=torch.int8, device=dev))
        self.register_buffer("tap_table", torch.zeros((0,) if depthwise else (O * (kh + 1) * (kw + 1),), dtype=torch.int32,
                                                      device=dev))
        b = torch.zeros(O) if bias is None else bias.detach().float()
        self.register_buffer("bias", b.to(dev).contiguous())
        w = weight.detach().float().to(dev).contiguous()
        mw, mx = _f32(w.min().item()), _f32(w.max().item())
        fw = self._pack(w, mw, mx)
        self.w_min, self.w_scale = float(mw), float(fw)
        k = affine_constants(ma, fa, mw, fw)
        if not all(np.isfinite(k)):
            raise _lib.DfqError("layer %s: the affine constants %s are not finite" % (self._who(), k))
        self.constants = np.zeros(1, _lib.I8_AFFINE_DT)
        self.constants[0] = k

    def _pack(self, w, mw, mx):
        """Pack the codes at the first candidate scale whose round trip reproduces every weight; returns it."""
        g = self._pack_geometry()
        lib = _lib.load()
        n_bad = torch.zeros(1, dtype=torch.int32, device=w.device)
        fewest = None
        for fw in weight_grid_candidates(mw, mx, self.w_bits):
            with _lib.launch(w, self.weight_codes) as st:
                _lib.check(lib.dfq_i8_affine_pack(_ptr(w), C.c_float(mw), C.c_float(fw), self.w_bits, _ptr(self.weight_codes),
                                                  _ptr(self.tap_table) if self.tap_table.numel() else None, _ptr(n_bad),
                                                  _lib.table_ptr(g), st), "dfq_i8_affine_pack (layer %s)" % self._who())
            bad = int(n_bad.item())
            if bad == 0:
                return fw
            fewest = bad if fewest is None else min(fewest, bad)
        raise _lib.DfqError("layer %s: its weights are not on a %d-bit min / max grid (min %g, max %g; %s of %d weights off "
                            "the best candidate scale): run quantize_targ_layer first"
                            % (self._who(), self.w_bits, mw, mx, "all" if fewest is None else fewest, w.numel()))

    def chained(self, codes_in=False, requant=None, epilogue=None, name=None, sums=False, out_slice=None, rows=False):
        """A new module of the same class on the same buffers (weight_codes, tap_table, bias, constants), in the given
        execution mode: codes_in - take (codes, S) from the previous layer's epilogue instead of quantizing fp32; requant =
        ((act_min, act_max, act_bits), lo, hi) - return the consumer's codes after the clamp (lo, hi), the epilogue
        Epilogue(out, (lo, hi)); epilogue - an Epilogue whose out_scale is the consumer's (act_min, act_max, act_bits) or
        None (the residual epilogue, dfq_i8_affine_conv_fused); sums - the codes come with their per-pixel sums S (a dense
        consumer reads them); out_slice = (coff, cstride), with codes and no fp32 output - write them into channels
        [coff, coff + round_up(C_out, 16)) of a concatenation's codes [N, OH, OW, cstride] and add S into its sums,
        given as forward(x, out=(codes, S | None)) or made (S zeroed) when out is None; rows - the fp32 output
        pixel-major into a detection head's concatenation (dfq_i8_affine_conv_rows), as _Int8Layer.chained(rows=True),
        the clamps from an fp32-only epilogue without residual.  The pad code of a folded F.pad is kept.  name: the layer's
        name in error messages.  self is not modified."""
        new = self._copy(codes_in, name or self.layer_name)
        if requant is not None and epilogue is not None:
            raise _lib.DfqError("layer %s: requant and epilogue are two output modes; give one" % new._who())
        if requant is not None:
            out, lo, hi = requant
            epilogue = Epilogue(out, (lo, hi))
        if epilogue is not None:
            e = Epilogue(*epilogue)
            if e.out_scale is None and not e.fp32:
                raise _lib.DfqError("layer %s: the epilogue returns neither codes nor fp32" % new._who())
            out = None
            if e.out_scale is not None:
                lo, hi, bits = e.out_scale
                who = "%s -> next layer" % new._who()
                _affine_refusal(who, 1, 1, 1, (1, 1), bits, 8)
                out = _affine_range(lo, hi, bits, "layer %s" % who, "output range")
            epilogue = Epilogue(out, _ordered(*e.pre, what="pre-add"), _ordered(*e.post, what="post-add"), bool(e.residual),
                                bool(e.fp32))
        new.epilogue = epilogue
        new.sums = bool(sums) and epilogue is not None and epilogue.out_scale is not None
        if out_slice is not None:
            if epilogue is None or epilogue.out_scale is None or epilogue.fp32 or epilogue.residual:
                raise _lib.DfqError("layer %s: a channel slice takes the codes only, without a residual" % new._who())
            out_slice = _channel_slice(out_slice, self.out_channels, "layer %s" % new._who())
        new.out_slice = out_slice
        if rows:
            if out_slice is not None or self.pad_code is not None or \
                    (epilogue is not None and (epilogue.out_scale is not None or epilogue.residual)):
                raise _lib.DfqError("layer %s: pixel-major fp32 rows exclude codes, a residual and a pad code" % new._who())
            new.epilogue = epilogue or Epilogue(fp32=True)
        new.rows = bool(rows)
        return new

    def fold_pad(self, pad):
        """This layer's copy (chained()) on the input F.pad(x, (l, l, t, t)) of constant zeros, pad = (t, l): padding (t, l)
        and the shifted code of +0.0 at the input range on every out-of-image tap, as the per-layer path quantizes the
        padded zeros.  Needs padding 0: a convolution's own padding is a dequantized 0.0, not a code."""
        if self.padding != (0, 0) or self.pad_code is not None:
            raise _lib.DfqError("layer %s: a pad folds only into a convolution with padding 0" % self._who())
        if self.epilogue is not None or self.out_slice is not None:
            raise _lib.DfqError("layer %s: fold a pad before the chained modes" % self._who())
        new = self.chained(codes_in=self.codes_in, name=self.layer_name)
        new.padding = (int(pad[0]), int(pad[1]))
        new.pad_code = affine_code_of(0.0, self.act_min, self.act_max, self.act_bits)
        return new

    def observe(self, obs=None, res=None, tail=None):
        """Give this chained layer's epilogue the functional-op observers of the reference's evaluation state
        (dfq_i8_affine_conv_observed): obs = (running_min, running_max, num_bits) of the QuantMeasure on v after the first
        clamp (the fused operand of an observed add, the producer's observed fp32 output, or a head's concatenation
        operand), res = that of the one on the residual, tail = (rows mode) that of the one on the head concatenation's
        output, after the second clamp; None: no observer.  Returns self."""
        if self.epilogue is None:
            raise _lib.DfqError("layer %s: observers run in a chained layer's epilogue" % self._who())
        if res is not None and not self.epilogue.residual:
            raise _lib.DfqError("layer %s: an observer on the residual needs a residual input" % self._who())
        if tail is not None and not self.rows:
            raise _lib.DfqError("layer %s: an observer on a head concatenation's output needs rows mode" % self._who())
        self.observers = tuple(None if o is None else _observer_range(o, "layer %s: %s observer" % (self._who(), w))
                               for o, w in ((obs, "operand"), (res, "residual")))
        self.tail_observer = None if tail is None else _observer_range(tail, "layer %s: tail observer" % self._who())
        return self

    def _input(self, x):
        """(codes, S | None, N, H, W) of the input: quantized here from fp32, or the pair a codes_in layer takes."""
        lib = _lib.load()
        if self.codes_in:
            xq, S = x if isinstance(x, tuple) and len(x) == 2 else (x, None)
            if not isinstance(xq, torch.Tensor) or xq.dtype != torch.int8 or xq.dim() != 4 or xq.shape[3] != self.cpad:
                raise _lib.DfqError("chained affine layer %s expects (int8 codes [N, H, W, %d], S), got %s" % (
                    self._who(), self.cpad, "%s %s" % (xq.dtype, tuple(xq.shape)) if isinstance(xq, torch.Tensor)
                    else type(x).__name__))
            N, H, W, _ = xq.shape
            if self.groups == 1 and (S is None or S.dtype != torch.int32 or S.numel() != N * H * W):
                raise _lib.DfqError("chained affine layer %s is dense: it needs the codes' per-pixel sums S, int32 [%d, %d, %d]"
                                    % (self._who(), N, H, W))
            if not xq.is_cuda:
                raise _lib.DfqError("int8 layers run on the GPU only (no CPU fallback): input on %s" % xq.device)
            self._same_device(xq)
            return xq.contiguous(), None if S is None else S.contiguous(), N, H, W
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != self.in_channels:
            raise _lib.DfqError("int8 layer expects fp32 [N, %d, H, W], got %s" % (
                self.in_channels, "%s %s" % (x.dtype, tuple(x.shape)) if isinstance(x, torch.Tensor) else type(x).__name__))
        if not x.is_cuda or not self.bias.is_cuda:
            raise _lib.DfqError("int8 layers run on the GPU only (no CPU fallback): input on %s, layer on %s"
                                % (x.device, self.bias.device))
        self._same_device(x)
        x = x.contiguous()
        N, _, H, W = x.shape
        xq = torch.empty(N * H * W * self.cpad, dtype=torch.int8, device=x.device)
        S = torch.empty(N * H * W, dtype=torch.int32, device=x.device)
        with _lib.launch(x, self.bias) as st:
            _lib.check(lib.dfq_i8_affine_quantize(_ptr(x), _ptr(xq), _ptr(S), N, self.in_channels, H, W, self.cpad,
                                                  C.c_float(self.act_min), C.c_float(self.act_max), self.act_bits, st),
                       "dfq_i8_affine_quantize (layer %s)" % self._who())
        return xq, S, N, H, W

    def _same_device(self, x):
        if x.device != self.bias.device:
            raise _lib.DfqError("layer %s is on %s, its input on %s: an int8 layer runs on its own device"
                                % (self._who(), self.bias.device, x.device))

    def run(self, x, with_acc=False, residual=None, out=None, off=0):
        """(y, P | None) for x fp32 [N, C, H, W] on the GPU; P = the int32 sums of the shifted codes.  In the chained modes
        x is (codes [N, H, W, cpad], S [N, H, W] | None) (codes_in), and with an epilogue y is (codes, S | None), the fp32
        output, or ((codes, S | None), fp32 output) when it returns both; `residual` is the fp32 tensor [N, C_out, OH, OW]
        the epilogue adds (exactly that shape, no broadcasting, on the input's device).  With out_slice, y is `out` (the
        concatenation's (codes, S | None)) or a new such pair, its slice written.  With rows, y is `out` with this layer's
        rows written at `off` of each image, or a new [N, OH * OW, C_out] tensor (see _Int8Layer.chained)."""
        if (self.epilogue is not None or self.pad_code is not None) and with_acc:
            raise _lib.DfqError("a chained affine layer does not return its int32 sums")
        if not self.rows:
            self._check_out(out)
        self._check_residual(residual)
        xq, S, N, H, W = self._input(x)
        g, OH, OW = self._output_geometry(N, H, W)
        if self.rows:
            return self._run_rows(xq, S, out, off, g, N, OH, OW), None
        if self.epilogue is not None or self.pad_code is not None:
            return self._run_fused(xq, S, residual, g, N, OH, OW, out), None
        lib = _lib.load()
        y = torch.empty((N, self.out_channels, OH, OW), dtype=torch.float32, device=xq.device)
        acc = torch.empty(y.shape, dtype=torch.int32, device=xq.device) if with_acc else None
        with _lib.launch(xq, self.weight_codes) as st:
            _lib.check(lib.dfq_i8_affine_conv(_ptr(xq), _ptr(S), _ptr(self.weight_codes),
                                              _ptr(self.tap_table) if self.tap_table.numel() else None,
                                              _lib.table_ptr(self.constants), _ptr(self.bias), _ptr(y), _ptr(acc),
                                              _lib.table_ptr(g), st), "dfq_i8_affine_conv (layer %s)" % self._who())
        return y, acc

    def _run_fused(self, xq, S, r, g, N, OH, OW, out=None):
        e = self.epilogue or Epilogue(fp32=True)                # a folded pad alone: the fp32 output through the layout
        shape = (N, self.out_channels, OH, OW)
        r = self._residual(r, shape, xq.device)
        if self.out_slice is not None:
            yq, S_out = self._slice_buffers(out, N, OH, OW, xq.device)
        else:
            yq = None if e.out_scale is None else \
                torch.empty((N, OH, OW, (self.out_channels + 15) // 16 * 16), dtype=torch.int8, device=xq.device)
            S_out = torch.empty((N, OH, OW), dtype=torch.int32, device=xq.device) if yq is not None and self.sums else None
        y = torch.empty(shape, dtype=torch.float32, device=xq.device) if e.fp32 else None
        d = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
        d[0] = tuple(0 if t is None else t.data_ptr() for t in (r, y, yq, S_out)) + (e.out_scale or (0.0, 0.0, 0)) + \
            e.pre + e.post
        lib, args = _lib.load(), (_ptr(xq), _ptr(S), _ptr(self.weight_codes),
                                  _ptr(self.tap_table) if self.tap_table.numel() else None, _lib.table_ptr(self.constants),
                                  _ptr(self.bias), _lib.table_ptr(d))
        obs, res = self.observers
        if self.out_slice is not None or self.pad_code is not None:
            o = None
            if obs is not None or res is not None:
                o = np.zeros(1, _lib.I8_AFFINE_OBSERVE_DT)
                o[0] = (obs or (0.0, 0.0, 0)) + (res or (0.0, 0.0, 0))
            lay = np.zeros(1, _lib.I8_AFFINE_LAYOUT_DT)
            lay[0] = (self.out_slice or (0, (self.out_channels + 15) // 16 * 16)) + (
                int(self.out_slice is not None), int(self.pad_code is not None), self.pad_code or 0)
            with _lib.launch(xq, self.weight_codes, r, y, yq, S_out) as st:
                _lib.check(lib.dfq_i8_affine_conv_layout(*args, None if o is None else _lib.table_ptr(o), _lib.table_ptr(lay),
                                                         _lib.table_ptr(g), st),
                           "dfq_i8_affine_conv_layout (layer %s)" % self._who())
            if self.out_slice is not None:
                return yq, S_out
        elif obs is None and res is None:
            with _lib.launch(xq, self.weight_codes, r, y, yq, S_out) as st:
                _lib.check(lib.dfq_i8_affine_conv_fused(*args, _lib.table_ptr(g), st),
                           "dfq_i8_affine_conv_fused (layer %s)" % self._who())
        else:
            o = np.zeros(1, _lib.I8_AFFINE_OBSERVE_DT)
            o[0] = (obs or (0.0, 0.0, 0)) + (res or (0.0, 0.0, 0))
            with _lib.launch(xq, self.weight_codes, r, y, yq, S_out) as st:
                _lib.check(lib.dfq_i8_affine_conv_observed(*args, _lib.table_ptr(o), _lib.table_ptr(g), st),
                           "dfq_i8_affine_conv_observed (layer %s)" % self._who())
        codes = None if yq is None else (yq, S_out)
        return (codes, y) if codes is not None and y is not None else (y if codes is None else codes)

    def _run_rows(self, xq, S, out, off, g, N, OH, OW):
        out, off = self._rows_out(out, off, N, OH, OW, xq.device)
        e, (obs, _), tail = self.epilogue, self.observers, self.tail_observer
        r = np.zeros(1, _lib.I8_AFFINE_ROWS_DT)
        r[0] = (out.data_ptr(), int(off), out[0].numel()) + e.pre + e.post + (obs or (0.0, 0.0, 0)) + (tail or (0.0, 0.0, 0))
        with _lib.launch(xq, self.weight_codes, out) as st:
            _lib.check(_lib.load().dfq_i8_affine_conv_rows(_ptr(xq), _ptr(S), _ptr(self.weight_codes),
                                                           _ptr(self.tap_table) if self.tap_table.numel() else None,
                                                           _lib.table_ptr(self.constants), _ptr(self.bias), _lib.table_ptr(r),
                                                           _lib.table_ptr(g), st),
                       "dfq_i8_affine_conv_rows (layer %s)" % self._who())
        return out

    def _slice_buffers(self, out, N, OH, OW, dev):
        """(codes [N, OH, OW, cstride], S [N, OH, OW] | None) of this slice's concatenation: `out`, checked, or new ones
        (S zeroed, when a dense consumer reads it) for the first writer."""
        return _concat_buffers(out, (N, OH, OW, self.out_slice[1]), self.sums, dev, "layer %s" % self._who())

    def extra_repr(self):
        return "%d, %d, kernel_size=%s, stride=%s, padding=%s, dilation=%s, groups=%d, act=[%g, %g] %d-bit, w_min=%g, " \
               "w_scale=%g %d-bit" % (self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding,
                                      self.dilation, self.groups, self.act_min, self.act_max, self.act_bits, self.w_min,
                                      self.w_scale, self.w_bits)


def _observer_range(o, who):
    """(min, max, bits) of an epilogue observer as fp32 / int, or DfqError naming it: 1 to 8 bits and a range whose
    QuantMeasure scale is a finite fp32 number."""
    lo, hi, bits = o
    if not isinstance(bits, (int, np.integer)) or isinstance(bits, bool) or not 1 <= bits <= 8:
        raise _lib.DfqError("%s: %r bits do not fit the int8 epilogue (1 to 8 bits)" % (who, bits))
    return _affine_range(lo, hi, bits, who, "range")


def _affine_range(lo, hi, bits, who, what):
    """(fp32 lo, fp32 hi, bits) of a quantizer's range and bits (1 to 8, checked by the caller), or DfqError
    "<who>: <what> [lo, hi] gives no finite fp32 scale" when its QuantMeasure scale is not a finite fp32 number."""
    ma, fa = act_affine_scalars(lo, hi, bits)
    if not (np.isfinite(ma) and np.isfinite(fa) and np.isfinite(_f32(hi))):
        raise _lib.DfqError("%s: %s [%g, %g] gives no finite fp32 scale" % (who, what, lo, hi))
    return float(_f32(lo)), float(_f32(hi)), int(bits)


def affine_code_of(v, act_min, act_max, num_bits):
    """The shifted code dfq_i8_affine_quantize gives the fp32 value v at this range, with its fp32 ops:
    rint(clamp(fp32(fp32(v + (-min)) * fp32(1 / scale)), 0, 2^b - 1)) - 128, the scale in double (QuantMeasure's)."""
    mn, mx = float(_f32(act_min)), float(_f32(act_max))
    qmax = 2. ** int(num_bits) - 1.
    scale = max((mx - mn) / qmax, 1e-8)
    with np.errstate(over="ignore", invalid="ignore"):
        t = _f32(_f32(_f32(v) + _f32(-mn)) * _f32(1.0 / scale))
    t = 0.0 if np.isnan(t) else min(max(float(t), 0.0), qmax)
    return int(np.rint(t)) - 128


def _concat_buffers(out, shape, sums, dev, who):
    """(codes int8 `shape`, S int32 shape[:3] | None) of a concatenation's codes: `out` checked, or new ones for its first
    writer, S zeroed (the writers add into it) when `sums`."""
    if out is None:
        return (torch.empty(shape, dtype=torch.int8, device=dev),
                torch.zeros(shape[:3], dtype=torch.int32, device=dev) if sums else None)
    codes, S = out if isinstance(out, tuple) and len(out) == 2 else (out, None)
    if not isinstance(codes, torch.Tensor) or codes.dtype != torch.int8 or tuple(codes.shape) != shape or \
            codes.device != dev or not codes.is_contiguous() or (S is None) == bool(sums) or (S is not None and (
                S.dtype != torch.int32 or tuple(S.shape) != shape[:3] or S.device != dev or not S.is_contiguous())):
        raise _lib.DfqError("%s: the concatenation's codes must be contiguous (int8 %s, %s) on %s" % (
            who, list(shape), "int32 %s" % list(shape[:3]) if sums else "None", dev))
    return codes, S


def _affine_refusal(who, C_in, C_out, groups, kernel_size, act_bits, w_bits):
    """Raise DfqError naming the layer if dfq_i8_affine_* cannot run it."""
    if groups != 1 and not (groups == C_in == C_out):
        raise _lib.DfqError("layer %s cannot run in int8: needs groups == 1 or depthwise (groups == C_in == C_out), got "
                            "groups=%d C_in=%d C_out=%d" % (who, groups, C_in, C_out))
    for what, b in (("activation", act_bits), ("weight", w_bits)):
        if not isinstance(b, (int, np.integer)) or isinstance(b, bool) or not 1 <= b <= 8:
            raise _lib.DfqError("layer %s: %s codes of %r bits do not fit the int8 path (1 to 8 bits)" % (who, what, b))
    K = kernel_size[0] * kernel_size[1] * (C_in // groups)
    if K >= AFFINE_MAX_K:
        raise _lib.DfqError("layer %s: K = kh * kw * C / groups = %d reaches %d, where the int32 sums can overflow"
                            % (who, K, AFFINE_MAX_K))


class AffineInt8Conv2d(_AffineInt8Layer):
    """A fake-quantized nn.Conv2d (QuantNConv2d after quantize_targ_layer, or a QConv2d / QuantConv2d) executed in integer
    arithmetic."""

    @classmethod
    def from_conv(cls, conv: nn.Conv2d, act_min, act_max, act_bits=8, w_bits=8, name=None, weight=None, bias=None):
        """weight / bias: the fake-quantized tensors to run in place of conv's own (those a per-forward layer convolves
        with); None: conv.weight, conv.bias."""
        err = _zero_padding_refusal(conv, "layer %s: " % name)
        if err is not None:
            raise err
        return cls(conv.weight if weight is None else weight, conv.bias if bias is None else bias, act_min, act_max,
                   act_bits, w_bits, conv.stride, conv.padding, conv.dilation, conv.groups, name=name)

    def forward(self, x, r=None, out=None, off=0):
        return self.run(x, residual=r, out=out, off=off)[0]


class AffineInt8Linear(_AffineInt8Layer):
    """A fake-quantized nn.Linear executed in integer arithmetic: the 1x1 convolution of [B, I, 1, 1]."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, act_min, act_max, act_bits=8, w_bits=8, name=None, weight=None, bias=None):
        """weight / bias: as AffineInt8Conv2d.from_conv."""
        w = lin.weight if weight is None else weight
        return cls(w.reshape(lin.out_features, lin.in_features, 1, 1), lin.bias if bias is None else bias, act_min, act_max,
                   act_bits, w_bits, name=name)

    forward = _ConvLayer._linear_forward


def _pool_extent(n, k, p, s, d, ceil_mode):
    """torch's pooling output size (floor division; in ceil mode the last window starts inside the input or its left pad)."""
    o = (n + 2 * p - d * (k - 1) - 1 + (s - 1 if ceil_mode else 0)) // s + 1
    return o - 1 if ceil_mode and (o - 1) * s >= n + p else o


class Int8MaxPool2d(nn.Module):
    """F.max_pool2d of a chained model (dfq_i8_maxpool).  codes_in: int8 NHWC codes [N, H, W, round_up(channels, 16)] in,
    the pooled codes out (the max of codes is the code of the max, q being monotone).  Otherwise fp32 NCHW in, bit for bit
    torch's max_pool2d out (`fp32`) and / or its codes at out_scale: (codes, fp32) when both.  sums: ignored (ncnn codes
    have no per-pixel sums), so that AffineInt8MaxPool2d's arguments fit both."""

    def __init__(self, kernel_size, stride, padding, dilation, ceil_mode, channels, codes_in, out_scale=None, fp32=False,
                 name=None, sums=False):
        super().__init__()
        self.kernel_size, self.padding, self.dilation = _pair(kernel_size), _pair(padding), _pair(dilation)
        self.stride = self.kernel_size if stride is None or stride == [] or stride == () else _pair(stride)
        self.ceil_mode, self.channels, self.codes_in = bool(ceil_mode), int(channels), bool(codes_in)
        self.cpad = (self.channels + 15) // 16 * 16
        self.fp32, self.layer_name = bool(fp32), name
        self.out_scale = None if out_scale is None else self._out(out_scale)
        if not codes_in and self.out_scale is None and not self.fp32:
            raise _lib.DfqError("max pool %s returns neither codes nor fp32" % name)

    def _out(self, out_scale):
        """out_scale as the pool keeps it (fp32 mode's codes are at it), checked."""
        s = float(_f32(out_scale))
        check_scale("output", s, "max pool %s" % self.layer_name)
        return s

    def forward(self, x):
        x, g, y, yq = self._launch_args(x)
        with _lib.launch(x) as st:
            _lib.check(_lib.load().dfq_i8_maxpool(_ptr(x) if self.codes_in else None, None if self.codes_in else _ptr(x), _ptr(y),
                                                  _ptr(yq), C.c_float(self.out_scale or 0.0), _lib.table_ptr(g),
                                                  st), "dfq_i8_maxpool (%s)" % self.layer_name)
        return (yq, y) if yq is not None and y is not None else (y if yq is None else yq)

    def _launch_args(self, x):
        """(x contiguous, DfqI8Pool table, y | None, yq | None) of the pool on its input x (codes or fp32, as codes_in
        says), checked: the outputs allocated, fp32 y in fp32 mode when `fp32`, the codes yq when codes_in or out_scale."""
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise _lib.DfqError("int8 max pool %s runs on the GPU only (no CPU fallback)" % self.layer_name)
        if self.codes_in:
            if x.dtype != torch.int8 or x.dim() != 4 or x.shape[3] != self.cpad:
                raise _lib.DfqError("int8 max pool %s expects int8 codes [N, H, W, %d], got %s %s"
                                    % (self.layer_name, self.cpad, x.dtype, tuple(x.shape)))
            N, H, W, _ = x.shape
        else:
            if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != self.channels:
                raise _lib.DfqError("int8 max pool %s expects fp32 [N, %d, H, W], got %s %s"
                                    % (self.layer_name, self.channels, x.dtype, tuple(x.shape)))
            N, _, H, W = x.shape
        x = x.contiguous()
        (kh, kw), (sh, sw), (ph, pw), (dh, dw) = self.kernel_size, self.stride, self.padding, self.dilation
        OH, OW = _pool_extent(H, kh, ph, sh, dh, self.ceil_mode), _pool_extent(W, kw, pw, sw, dw, self.ceil_mode)
        g = np.zeros(1, _lib.I8_POOL_DT)
        g[0] = (N, self.channels, H, W, kh, kw, sh, sw, ph, pw, dh, dw, int(self.ceil_mode), OH, OW, self.cpad)
        yq = torch.empty((N, OH, OW, self.cpad), dtype=torch.int8, device=x.device) \
            if self.codes_in or self.out_scale is not None else None
        y = torch.empty((N, self.channels, OH, OW), dtype=torch.float32, device=x.device) \
            if not self.codes_in and self.fp32 else None
        return x, g, y, yq

    def extra_repr(self):
        return "kernel_size=%s, stride=%s, padding=%s, dilation=%s, ceil_mode=%s, channels=%d, %s" % (
            self.kernel_size, self.stride, self.padding, self.dilation, self.ceil_mode, self.channels,
            "codes" if self.codes_in else "fp32 in, out_scale=%s, fp32=%s" % (self.out_scale, self.fp32))


class AffineInt8MaxPool2d(Int8MaxPool2d):
    """F.max_pool2d of a model chained by chain_affine(pools=True) (dfq_i8_affine_maxpool): Int8MaxPool2d's geometry and
    modes on the affine scheme's shifted codes.  codes_in: (codes [N, H, W, round_up(channels, 16)], S | None) in - S is
    not read - and the pooled codes out.  Otherwise fp32 NCHW in, torch's max_pool2d out (`fp32`) and / or its codes at
    out_scale = the consumers' (act_min, act_max, act_bits).  The codes come as (codes, S | None), S their per-pixel sums
    when `sums` (a dense consumer reads them); ((codes, S | None), fp32) when both."""

    def __init__(self, kernel_size, stride, padding, dilation, ceil_mode, channels, codes_in, out_scale=None, fp32=False,
                 sums=False, name=None):
        super().__init__(kernel_size, stride, padding, dilation, ceil_mode, channels, codes_in, out_scale, fp32, name)
        self.sums = bool(sums)

    def _out(self, out_scale):
        return _observer_range(out_scale, "max pool %s: output" % self.layer_name)

    def forward(self, x):
        if self.codes_in and isinstance(x, tuple) and len(x) == 2:
            x = x[0]                                            # the pool sums its own codes
        x, g, y, yq = self._launch_args(x)
        S = torch.empty(yq.shape[:3], dtype=torch.int32, device=x.device) if yq is not None and self.sums else None
        lo, hi, bits = self.out_scale or (0.0, 0.0, 0)
        with _lib.launch(x) as st:
            _lib.check(_lib.load().dfq_i8_affine_maxpool(
                _ptr(x) if self.codes_in else None, None if self.codes_in else _ptr(x), _ptr(y), _ptr(yq), _ptr(S), C.c_float(lo),
                C.c_float(hi), bits, _lib.table_ptr(g), st), "dfq_i8_affine_maxpool (%s)" % self.layer_name)
        codes = None if yq is None else (yq, S)
        return (codes, y) if codes is not None and y is not None else (y if codes is None else codes)

    def extra_repr(self):
        return super().extra_repr() + ", sums=%s" % self.sums


def _upsample_input(x, size, channels, name):
    """(N, H, W, OH, OW) of an int8 bilinear upsample's input x, fp32 [N, channels, H, W] on the GPU, to its run-time size,
    a pair of positive ints; DfqError otherwise."""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise _lib.DfqError("int8 bilinear upsample %s runs on the GPU only (no CPU fallback)" % name)
    if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != channels:
        raise _lib.DfqError("int8 bilinear upsample %s expects fp32 [N, %d, H, W], got %s %s"
                            % (name, channels, x.dtype, tuple(x.shape)))
    if not isinstance(size, (tuple, list)) or len(size) != 2 or \
            not all(isinstance(v, int) and not isinstance(v, bool) and v > 0 for v in size):
        raise _lib.DfqError("int8 bilinear upsample %s: size must be a pair of positive ints, got %r" % (name, size))
    N, _, H, W = x.shape
    return N, H, W, int(size[0]), int(size[1])


class Int8UpsampleBilinear(nn.Module):
    """F.interpolate(x, size, mode='bilinear', align_corners=...) of a chained model (dfq_i8_upsample_bilinear): fp32 NCHW
    [N, channels, H, W] in, the codes q(clamp(y, *clamp), out_scale) of torch's bilinear output y out - int8 NHWC
    [N, OH, OW, round_up(channels, 16)], or with out_slice = (coff, cstride) channels [coff, coff + round_up(channels, 16))
    of `out` (int8 [N, OH, OW, cstride], made when None).  The size comes at run time (often a traced value such as
    x.shape[-2:]) and must be a pair of positive ints.  pre, obs, post, sums: as AffineInt8UpsampleBilinear's (a given
    pre makes the clamp pre then post; ncnn has no observers or sums)."""

    def __init__(self, channels, align_corners, out_scale, clamp=(-float("inf"), float("inf")), out_slice=None, name=None,
                 pre=None, obs=None, post=(-float("inf"), float("inf")), sums=False):
        super().__init__()
        if obs is not None:
            raise _lib.DfqError("bilinear upsample %s: the ncnn scheme runs no observer" % name)
        clamp = clamp if pre is None else _compose(pre, post)
        self.channels, self.align_corners, self.layer_name = int(channels), bool(align_corners), name
        self.cpad = (self.channels + 15) // 16 * 16
        check_scale("output", out_scale, "bilinear upsample %s" % name)
        self.out_scale = float(_f32(out_scale))
        self.clamp = _ordered(*clamp, what="upsample %s clamp" % name)
        self.out_slice = None if out_slice is None else _channel_slice(out_slice, self.channels, "bilinear upsample %s" % name)

    def forward(self, x, size, out=None):
        N, H, W, OH, OW = _upsample_input(x, size, self.channels, self.layer_name)
        coff, cstride = self.out_slice or (0, self.cpad)
        shape = (N, OH, OW, cstride)
        if out is not None and self.out_slice is None:
            raise _lib.DfqError("bilinear upsample %s: takes no output tensor" % self.layer_name)
        if out is None:
            out = torch.empty(shape, dtype=torch.int8, device=x.device)
        elif not isinstance(out, torch.Tensor) or out.dtype != torch.int8 or tuple(out.shape) != shape or \
                out.device != x.device or not out.is_contiguous():
            raise _lib.DfqError("bilinear upsample %s: the concatenation's codes must be contiguous int8 %s on %s, got %s" % (
                self.layer_name, list(shape), x.device, "%s %s on %s" % (out.dtype, list(out.shape), out.device)
                if isinstance(out, torch.Tensor) else type(out).__name__))
        x = x.contiguous()
        g = np.zeros(1, _lib.I8_RESIZE_DT)
        g[0] = (N, self.channels, H, W, OH, OW, int(self.align_corners), coff, cstride, self.out_scale) + self.clamp
        with _lib.launch(x, out) as st:
            _lib.check(_lib.load().dfq_i8_upsample_bilinear(_ptr(x), None, _ptr(out), _lib.table_ptr(g), st),
                       "dfq_i8_upsample_bilinear (%s)" % self.layer_name)
        return out

    def extra_repr(self):
        return "channels=%d, align_corners=%s, out_scale=%g, clamp=%s, out_slice=%s" % (
            self.channels, self.align_corners, self.out_scale, self.clamp, self.out_slice)


class AffineInt8UpsampleBilinear(nn.Module):
    """A bilinear F.interpolate operand of a concatenation chained by chain_affine (dfq_i8_affine_upsample_bilinear): fp32
    NCHW [N, channels, H, W] in; torch's bilinear output through clamp(pre), the operand's observer `obs` ((min, max, bits)
    or None), clamp(post) and the consumer's quantizer out = (act_min, act_max, act_bits), written into channels
    [coff, coff + round_up(channels, 16)) of the concatenation's (codes [N, OH, OW, cstride], S | None) - `out`, or new
    ones (S zeroed when `sums`) - which it returns.  The size comes at run time and must be a pair of positive ints."""

    def __init__(self, channels, align_corners, out, out_slice, pre=(-float("inf"), float("inf")), obs=None,
                 post=(-float("inf"), float("inf")), sums=False, name=None):
        super().__init__()
        self.channels, self.align_corners, self.layer_name, self.sums = int(channels), bool(align_corners), name, bool(sums)
        who = "bilinear upsample %s" % name
        self.out = _observer_range(out, who + " output")
        self.obs = None if obs is None else _observer_range(obs, who + " observer")
        self.pre, self.post = _ordered(*pre, what=who + " pre"), _ordered(*post, what=who + " post")
        self.out_slice = _channel_slice(out_slice, self.channels, who)

    def forward(self, x, size, out=None):
        N, H, W, OH, OW = _upsample_input(x, size, self.channels, self.layer_name)
        coff, cstride = self.out_slice
        codes, S = _concat_buffers(out, (N, OH, OW, cstride), self.sums, x.device, "bilinear upsample %s" % self.layer_name)
        x = x.contiguous()
        g = np.zeros(1, _lib.I8_AFFINE_RESIZE_DT)
        g[0] = (N, self.channels, H, W, OH, OW, int(self.align_corners), coff, cstride) + self.pre + \
            (self.obs or (0.0, 0.0, 0)) + self.post + self.out
        with _lib.launch(x) as st:
            _lib.check(_lib.load().dfq_i8_affine_upsample_bilinear(_ptr(x), _ptr(codes), _ptr(S), _lib.table_ptr(g),
                                                                   st),
                       "dfq_i8_affine_upsample_bilinear (%s)" % self.layer_name)
        return codes, S

    def extra_repr(self):
        return "channels=%d, align_corners=%s, pre=%s, obs=%s, post=%s, out=%s, out_slice=%s, sums=%s" % (
            self.channels, self.align_corners, self.pre, self.obs, self.post, self.out, self.out_slice, self.sums)


class Int8HeadConcat(nn.Module):
    """torch.cat(..., 1) of detection heads laid out as `conv(x_i).permute(0, 2, 3, 1).contiguous().view(N, -1, k)` in a
    chained model: each head (a rows-mode Int8Conv2d or AffineInt8Conv2d, chained(rows=True)) writes its pixel-major fp32
    output straight into its slice of one [N, R, k] tensor (dfq_i8_conv_nhwc, dfq_i8_affine_conv_rows), in order; an
    affine head's input may be the pair (codes, S).  R and the offsets follow from the inputs'
    sizes when the module runs.  batch: the view's constant N (None: the input's batch), checked."""

    def __init__(self, heads, k, batch=None, name=None):
        super().__init__()
        self.heads = nn.ModuleList(heads)
        self.k, self.batch, self.layer_name = int(k), None if batch is None else int(batch), name

    def forward(self, *xs):
        if len(xs) != len(self.heads):
            raise _lib.DfqError("head concatenation %s takes %d inputs, got %d" % (self.layer_name, len(self.heads), len(xs)))
        ts = [x[0] if isinstance(x, tuple) else x for x in xs]  # an affine head's (codes, S)
        N = int(ts[0].shape[0])
        if any(int(t.shape[0]) != N for t in ts) or (self.batch is not None and self.batch != N):
            raise _lib.DfqError("head concatenation %s: inputs of batch %s do not match the view's batch %s"
                                % (self.layer_name, [int(t.shape[0]) for t in ts], self.batch or N))
        ext = [h.out_extent(x) for h, x in zip(self.heads, xs)]
        if any(e % self.k for e in ext):
            raise _lib.DfqError("head concatenation %s: head outputs of %s floats per image do not view as rows of %d"
                                % (self.layer_name, ext, self.k))
        out = torch.empty((N, sum(ext) // self.k, self.k), dtype=torch.float32, device=ts[0].device)
        off = 0
        for h, x, e in zip(self.heads, xs, ext):
            h(x, out=out, off=off)
            off += e
        return out

    def extra_repr(self):
        return "k=%d, batch=%s" % (self.k, self.batch)


def convert_to_int8(model: nn.Module, graph, targ_type, act_scales=None):
    """Replace every target layer of `graph` (types in targ_type, Conv2d or Linear) inside `model` by its int8 executor, in
    place (by parent attribute); returns the replaced modules' names in graph order.

    Weight scales are export.ncnn_scales' 128 / max|W|, one per layer repeated per output channel.  Activation scales are
    ncnn_scales' 128 / max(|running_min|, |running_max|) of each layer's `quant` observer, or act_scales[i] (a list in graph
    order, one per target layer, e.g. the rows of read_ncnn_table).  A zero range gives scale 0.  Call after equalization /
    bias correction and the activation ranges, before quantize_targ_layer (module docstring).  A layer that cannot run in
    int8, or whose activation or weight scale is not a finite non-negative fp32 number (check_scale), raises DfqError naming
    it, before anything is replaced."""
    rows = export.ncnn_scales(graph, targ_type, zero_range_ok=True)
    layers = [graph[k] for k in graph if type(graph[k]) in targ_type]
    if act_scales is not None and len(act_scales) != len(layers):
        raise _lib.DfqError("act_scales has %d entries for %d target layers" % (len(act_scales), len(layers)))
    names = {id(m): n for n, m in model.named_modules()}
    plan = []
    for i, (layer, (w_scale, _, a_scale)) in enumerate(zip(layers, rows)):
        name = names.get(id(layer))
        if name is None:
            raise _lib.DfqError("target layer %d (%s) is not a submodule of the model" % (i, type(layer).__name__))
        a = act_scales[i] if act_scales is not None else a_scale
        if a is None:
            raise _lib.DfqError("layer %s has no activation range (no `quant` observer and no act_scales entry)" % name)
        check_scale("activation", a, name)
        check_scale("weight", w_scale, name)
        if isinstance(layer, nn.Conv2d):
            ok = (layer.groups == 1 or layer.groups == layer.in_channels == layer.out_channels) and \
                _zero_padding_refusal(layer) is None
        else:
            ok = isinstance(layer, nn.Linear)
        if not ok:
            raise _lib.DfqError("layer %s (%s, groups=%s) cannot run in int8: needs a Linear, or a zero-padded Conv2d with "
                                "groups == 1 or depthwise" % (name, type(layer).__name__, getattr(layer, "groups", "-")))
        plan.append((name, layer, a, w_scale))
    done = []
    for name, layer, a, w_scale in plan:
        _set_module(model, name, (Int8Conv2d.from_conv if isinstance(layer, nn.Conv2d) else Int8Linear.from_linear)(
            layer, a, w_scale))
        done.append(name)
    return done


def convert_affine(model: nn.Module, graph, targ_type, bits_weight=8):
    """Replace every target layer of `graph` (types in targ_type, Conv2d or Linear with a `quant` observer) inside `model`,
    in place, by an AffineInt8Conv2d / AffineInt8Linear that computes it in integer arithmetic under the reference's own
    quantization (asymmetric per-tensor min / max, include/dfq_b200.h dfq_i8_affine_*); returns the names in graph order.

    Call it in one of the reference's inference states, after the activation ranges (set_quant_minmax or
    update_quant_range):
      - QuantNConv2d / QuantNLinear (the default --quantize state), after quantize_targ_layer(graph, bits_weight, ...): the
        weights and biases are the layers' own, fake-quantized offline;
      - QConv2d / QLinear (--distill_range) or QuantConv2d / QuantLinear (--trainable), which quantize their weights and
        bias on every forward: the weights are _quant_param_per_forward(weight, layer.num_bits) and the bias
        quantize(bias, num_bits=layer.num_bits_bias) (the implicit-range path, at 32 bits too), both computed on the GPU
        as the forward computes them there.  The layer states its weight bits: layer.num_bits must equal bits_weight.  A
        layer carrying learned scales (scale / scale_prev of set_scale) is refused; merge_scale_to_weight merges them.
    Activation ranges and bits come from each layer's `quant` observer (running_min, running_max, num_bits) and are frozen
    here: an observer left with a truthy update_stat keeps widening its range in the fake-quantized model (set_layer_bits
    does this through quirk Q1), the converted layer does not.  The weight codes are recovered from the fake-quantized
    weights: mw = min(weight), fw an fp32 scale near (max - min) / (2^bits_weight - 1) whose round trip
    fp32(fp32(q fw) + mw) reproduces every weight bit for bit (checked on the device).  The result agrees with the
    fake-quantized layer to fp32 rounding of its sum, not bit for bit.  The original layers' parameters are not modified.

    Every layer is checked and packed before any is replaced: a layer that cannot run (grouping, padding mode, bits above 8,
    K = kh * kw * C / groups >= 131072, no observer, a non-finite range, a per-forward layer's bits other than bits_weight
    or learned scales) or whose weights are not on such a grid raises DfqError naming it, and the model is left as it
    was."""
    layers = [graph[k] for k in graph if type(graph[k]) in targ_type]
    names = {id(m): n for n, m in model.named_modules()}
    plan = []
    for i, layer in enumerate(layers):
        name = names.get(id(layer))
        if name is None:
            raise _lib.DfqError("target layer %d (%s) is not a submodule of the model" % (i, type(layer).__name__))
        quant = getattr(layer, "quant", None)
        if quant is None or not hasattr(quant, "running_min"):
            raise _lib.DfqError("layer %s has no `quant` observer with an activation range" % name)
        if isinstance(layer, nn.Conv2d):
            err = _zero_padding_refusal(layer, "layer %s: " % name)
            if err is not None:
                raise err
            shape = (layer.in_channels, layer.out_channels, layer.groups, tuple(layer.kernel_size))
        elif isinstance(layer, nn.Linear):
            shape = (layer.in_features, layer.out_features, 1, (1, 1))
        else:
            raise _lib.DfqError("layer %s (%s) cannot run in int8: needs a Conv2d or a Linear" % (name, type(layer).__name__))
        _affine_refusal(name, *shape, quant.num_bits, bits_weight)
        weight, bias = _per_forward_params(layer, name, bits_weight)
        plan.append((name, layer, float(quant.running_min.reshape(-1)[0]), float(quant.running_max.reshape(-1)[0]),
                     quant.num_bits, weight, bias))
    new = []
    for name, layer, lo, hi, bits, weight, bias in plan:
        if isinstance(layer, nn.Conv2d):
            new.append(AffineInt8Conv2d.from_conv(layer, lo, hi, bits, bits_weight, name=name, weight=weight, bias=bias))
        else:
            new.append(AffineInt8Linear.from_linear(layer, lo, hi, bits, bits_weight, name=name, weight=weight, bias=bias))
    for (name, *_), mod in zip(plan, new):
        _set_module(model, name, mod)
    return [name for name, *_ in plan]


def _per_forward_params(layer, name, bits_weight):
    """(weight, bias) a QConv2d / QLinear / QuantConv2d / QuantLinear convolves with, on the GPU: its forward's
    _quant_param_per_forward(weight, num_bits) and quantize(bias, num_bits=num_bits_bias) (None without a bias), computed
    from copies of its parameters; (None, None) for any other layer (a QuantN* layer runs its own weight and bias).
    DfqError naming the layer when its num_bits is not bits_weight or it carries learned scales that its forward merges
    into the weights first (a QConv2d / QLinear after set_scale)."""
    from .utils import quantize as Q
    if not isinstance(layer, (Q.QConv2d, Q.QLinear, Q.QuantConv2d, Q.QuantLinear)):
        return None, None
    if isinstance(layer, (Q.QConv2d, Q.QLinear)) and (getattr(layer, "scale", None) is not None or
                                                      getattr(layer, "scale_prev", None) is not None):
        raise _lib.DfqError("layer %s carries learned scales (scale / scale_prev of set_scale): merge them into its weights "
                            "first (merge_scale_to_weight)" % name)
    if layer.num_bits != bits_weight:
        raise _lib.DfqError("layer %s quantizes its weights to %r bits on every forward, not bits_weight = %r"
                            % (name, layer.num_bits, bits_weight))
    dev = engine._default_device()
    with torch.no_grad():
        weight = Q._quant_param_per_forward(layer.weight.detach().to(dev, copy=True), layer.num_bits)
        bias = None if layer.bias is None else Q.quantize(layer.bias.detach().to(dev, copy=True),
                                                          num_bits=layer.num_bits_bias)
    return weight, bias


def _set_module(root, name, mod):
    """Replace the submodule of root at the dotted `name` by mod."""
    parent, _, attr = name.rpartition(".")
    setattr(root.get_submodule(parent) if parent else root, attr, mod)


# ---- chaining converted convolutions through int8 codes ---------------------------------------------------------------
_INF = float("inf")
_FULL = (-_INF, _INF)                                           # no clamp


_TORCH_DIR = os.path.dirname(torch.__file__) + os.sep


class _Int8Tracer(fx.Tracer):
    """symbolic tracing that keeps the int8 layers (whose forward calls the library) as leaves.  To chain_int8 the affine
    layers of convert_affine are opaque leaves (they are no Int8Conv2d, so nothing is fused into or out of them), and to
    chain_affine the ncnn layers are.  callers=True records in node.meta["caller"] the (function name, line) of the first
    frame outside torch that made each call node: the frame the reference's patched ops inspect."""

    def __init__(self, callers=False):
        super().__init__()
        self.callers = callers

    def is_leaf_module(self, m, qualname):
        from .ncnn import PlaneMean                             # an ncnn model's means (ncnn.load) call the library
        return isinstance(m, (_ConvLayer, PlaneMean)) or super().is_leaf_module(m, qualname)

    def create_proxy(self, kind, target, args, kwargs, *rest, **kw):
        proxy = super().create_proxy(kind, target, args, kwargs, *rest, **kw)
        if self.callers and kind in ("call_function", "call_method"):
            f = sys._getframe(1)
            while f is not None and f.f_code.co_filename.startswith(_TORCH_DIR):
                f = f.f_back
            if f is not None:
                proxy.node.meta["caller"] = (f.f_code.co_name, f.f_lineno)
        return proxy


def _arg(node, i, name, default):
    return node.kwargs[name] if name in node.kwargs else (node.args[i] if len(node.args) > i else default)


def _is_identity_bn(bn):
    """True when the eval-mode BatchNorm2d computes x exactly: weight 1, bias 0, mean 0, var 1 and fp32(1 + eps) == 1 (what
    merge_batchnorm leaves behind, utils/layer_transform.py)."""
    if bn.training or not bn.track_running_stats or bn.running_mean is None:
        return False
    if _f32(1) + _f32(bn.eps) != _f32(1):
        return False
    with torch.no_grad():
        ok = bool((bn.running_mean == 0).all()) and bool((bn.running_var == 1).all())
        if bn.affine:
            ok = ok and bool((bn.weight == 1).all()) and bool((bn.bias == 0).all())
    return ok


def _pass_through(node, mods):
    """(lo, hi) of a node that is the identity or an activation clamp on the edge between two converted convolutions, or
    None when it ends the chain."""
    if node.op == "call_module":
        m = mods[node.target]
        if type(m) is nn.BatchNorm2d:
            return (-_INF, _INF) if _is_identity_bn(m) else None
        if type(m) is nn.ReLU:
            return (0.0, _INF)
        if type(m) in (nn.ReLU6, nn.Hardtanh):                  # ReLU6 is Hardtanh(0, 6)
            return (float(m.min_val), float(m.max_val))
        if type(m) is nn.Identity or (type(m) is nn.Dropout and not m.training):
            return (-_INF, _INF)
        return None
    if node.op == "call_function":
        if node.target in (F.relu, torch.relu):
            return (0.0, _INF)
        if node.target is F.relu6:
            return (0.0, 6.0)
        if node.target is F.hardtanh:
            return (float(_arg(node, 1, "min_val", -1.0)), float(_arg(node, 2, "max_val", 1.0)))
        return None
    if node.op == "call_method" and node.target == "relu":
        return (0.0, _INF)
    return None


def _compose(first, then):
    """The one clamp equal to clamp(clamp(v, *first), *then); both keep NaN."""
    (a, b), (c, d) = first, then
    return (min(max(a, c), d), max(min(b, d), c))


def _data_users(node, queries):
    """node's users, without those that only read its shape when `queries`."""
    return [u for u in node.users if not (queries and _shape_query(u, node))]


def _walk_back(node, mods, stop, queries=False):
    """(source, clamp, path) of the single-user pass-through chain that ends at `node`: from node back through
    pass-throughs of one fx node to the first node for which stop(n) holds, every node on the way, the source included,
    with exactly one user (users that only read its shape not counted when `queries`); clamp composes the pass-throughs'
    (the first in graph order runs first), path lists them from node back.  None when the chain ends elsewhere."""
    clamp, path = (-_INF, _INF), []
    while True:
        if len(_data_users(node, queries)) != 1:
            return None
        if stop(node):
            return node, clamp, path
        c = _pass_through(node, mods)
        if c is None or len(node.all_input_nodes) != 1 or not isinstance(node.args[0], fx.Node):
            return None
        clamp = _compose(c, clamp)                              # walking backwards: this clamp runs first
        path.append(node)
        node = node.args[0]


def _is_identity(node, mods):
    """An exact-identity pass-through: an identity eval BatchNorm2d, nn.Identity or an eval nn.Dropout (no clamp)."""
    return node.op == "call_module" and type(mods[node.target]) in (nn.BatchNorm2d, nn.Identity, nn.Dropout) and \
        _pass_through(node, mods) == (-_INF, _INF)


def _is_add(node):
    """operator.add / torch.add / Tensor.add of two distinct fx nodes, without alpha or out."""
    add = (node.op == "call_function" and node.target in (operator.add, torch.add)) or \
        (node.op == "call_method" and node.target == "add")
    return add and not node.kwargs and len(node.args) == 2 and all(isinstance(a, fx.Node) for a in node.args) and \
        node.args[0] is not node.args[1]


def _is_const(v):
    return isinstance(v, (int, bool)) or (isinstance(v, (tuple, list)) and all(isinstance(e, int) for e in v))


def _max_pool(node, mods):
    """(kernel_size, stride, padding, dilation, ceil_mode) of an nn.MaxPool2d / F.max_pool2d / torch.max_pool2d node without
    return_indices, on one fx node and constant arguments; None otherwise."""
    if len(node.all_input_nodes) != 1 or not node.args or not isinstance(node.args[0], fx.Node):
        return None
    if node.op == "call_module" and type(mods[node.target]) is nn.MaxPool2d:
        m = mods[node.target]
        if m.return_indices or len(node.args) != 1 or node.kwargs:
            return None
        return m.kernel_size, m.stride, m.padding, m.dilation, m.ceil_mode
    if node.op == "call_function" and node.target in (F.max_pool2d, torch.max_pool2d):
        a = (_arg(node, 1, "kernel_size", None), _arg(node, 2, "stride", None), _arg(node, 3, "padding", 0),
             _arg(node, 4, "dilation", 1), _arg(node, 5, "ceil_mode", False))
        if _arg(node, 6, "return_indices", False) or not all(v is None or _is_const(v) for v in a) or a[0] is None:
            return None
        return a
    return None


def _orig(name):
    """The unpatched torch.cat / F.interpolate that utils/layer_transform.py saved when replace_op() patched it (what a
    graph traced in the reference's evaluation state calls), or None."""
    from .utils import layer_transform as LT
    return LT.raw_torch_op.get(name) or LT.raw_func_op.get(name)


def _bilinear_upsample(node, mods, raw=False, wrapped=False):
    """(size, align_corners) of an F.interpolate / nn.Upsample node that resizes one fx node bilinearly to a given size:
    mode 'bilinear', size a pair of ints or a traced value, align_corners True or False, no scale_factor,
    recompute_scale_factor or antialias; None otherwise.  raw: the unpatched F.interpolate counts too (_orig).  wrapped:
    _raw_interpolate counts too (what chain_affine and load leave in a graph; the chaining rules never see it)."""
    if not node.args or not isinstance(node.args[0], fx.Node):
        return None
    if node.op == "call_module" and type(mods[node.target]) is nn.Upsample:
        m = mods[node.target]
        if len(node.args) != 1 or node.kwargs:
            return None
        size, sf, mode, ac, rsf, aa = m.size, m.scale_factor, m.mode, m.align_corners, m.recompute_scale_factor, False
    elif node.op == "call_function" and (node.target is F.interpolate or (raw and node.target is _orig("interpolate")) or
                                         (wrapped and node.target is _raw_interpolate)):
        size, sf, mode, ac, rsf, aa = (_arg(node, i, k, d) for i, k, d in (
            (1, "size", None), (2, "scale_factor", None), (3, "mode", "nearest"), (4, "align_corners", None),
            (5, "recompute_scale_factor", None), (6, "antialias", False)))
    else:
        return None
    if mode != "bilinear" or sf is not None or rsf is not None or aa is not False or (ac is not True and ac is not False):
        return None
    if not isinstance(size, fx.Node) and not (isinstance(size, (tuple, list)) and len(size) == 2 and all(
            isinstance(v, fx.Node) or (isinstance(v, int) and not isinstance(v, bool)) for v in size)):
        return None
    return size, ac


def _observer_key(node, mods):
    """(min, max, bits) of a call of a QuantMeasure whose fake quantization the affine epilogue runs bit for bit: eval
    mode, update_stat falsy (its range is frozen), 1 to 8 bits, a range whose scale is a finite fp32 number; None for
    any other node (such an observer stays in torch)."""
    from .utils.quantize import QuantMeasure
    if node.op != "call_module" or len(node.args) != 1 or node.kwargs or not isinstance(node.args[0], fx.Node):
        return None
    m = mods.get(node.target)
    if type(m) is not QuantMeasure or m.training or m.update_stat:
        return None
    try:
        return _observer_range((float(m.running_min.reshape(-1)[0]), float(m.running_max.reshape(-1)[0]), m.num_bits),
                               node.target)
    except _lib.DfqError:
        return None


def _is_view(node):
    """view / reshape / flatten of one fx node by constant or shape-query arguments: the same elements, another shape."""
    if not node.args or not isinstance(node.args[0], fx.Node) or node.kwargs.get("out") is not None:
        return False
    rest = list(node.args[1:]) + list(node.kwargs.values())
    flat = [v for a in rest for v in (a if isinstance(a, (tuple, list)) else (a,))]
    if not all(not isinstance(v, fx.Node) or _shape_only(v) for v in flat):
        return False
    return (node.op == "call_method" and node.target in ("view", "reshape", "flatten")) or \
        (node.op == "call_function" and node.target in (torch.flatten, torch.reshape))


def _shape_query(u, node):
    """True when u only reads node's shape: node.size(), node.size(d), node.shape or node.dim()."""
    if not u.args or u.args[0] is not node or u.kwargs:
        return False
    if u.op == "call_method" and u.target in ("size", "dim"):
        return all(not isinstance(a, fx.Node) for a in u.args[1:])
    return u.op == "call_function" and u.target is getattr and len(u.args) == 2 and u.args[1] == "shape"


def _nchw_view(codes, channels):
    """A tensor of the shape [N, channels, H, W] of the fp32 tensor whose codes `codes` [N, H, W, *] carry, for the shape
    queries on a fused concatenation's operand (sizes taken as `x4.size()[2:]`): a zero-stride view, nothing allocated."""
    if isinstance(codes, tuple):                                # the affine scheme's (codes, S)
        codes = codes[0]
    N, H, W = codes.shape[:3]
    return codes.as_strided((N, channels, H, W), (0, 0, 0, 0))


def _cat_operands(node, raw=False, dims=(1, -3)):
    """The operands of torch.cat / torch.concat along the channels (a dim in `dims`) of >= 2 distinct fx nodes, without
    out; None otherwise.  raw: the unpatched torch.cat counts too (_orig)."""
    cats = (torch.cat, torch.concat) + ((_orig("cat"),) if raw else ())
    if node.op != "call_function" or node.target not in cats or set(node.kwargs) - {"tensors", "dim"}:
        return None
    ops, dim = _arg(node, 0, "tensors", None), _arg(node, 1, "dim", 0)
    if dim not in dims or not isinstance(ops, (list, tuple)) or len(ops) < 2 or \
            not all(isinstance(o, fx.Node) for o in ops) or len(set(ops)) != len(ops):
        return None
    return list(ops)


def _zero_pad(node):
    """(t, l) of an F.pad node that zero-pads one fx node symmetrically: pad (l, r) or (l, r, t, b) with l == r >= 0 and
    t == b >= 0, mode 'constant', value 0 or None; None otherwise."""
    if node.op != "call_function" or node.target not in (F.pad, torch._C._nn.pad) or len(node.all_input_nodes) != 1 or \
            not node.args or not isinstance(node.args[0], fx.Node) or set(node.kwargs) - {"pad", "mode", "value"}:
        return None
    pad, mode, value = _arg(node, 1, "pad", None), _arg(node, 2, "mode", "constant"), _arg(node, 3, "value", None)
    if not isinstance(pad, (tuple, list)) or len(pad) not in (2, 4) or \
            not all(isinstance(v, int) and not isinstance(v, bool) for v in pad):
        return None
    l, r, t, b = (tuple(pad) + (0, 0))[:4]
    if l != r or t != b or l < 0 or t < 0 or mode != "constant" or not (value is None or (
            isinstance(value, (int, float)) and not isinstance(value, bool) and value == 0)):
        return None
    return t, l


def _fold_pads(gm, mods, conv, scheme):
    """Rule (a) of chain_int8(layout=True) and chain_affine(fold_pads=True): fold each qualifying zero F.pad into its only
    user, a `scheme` convolution that takes it (_Scheme.fold_pad); recorded in gm.folded_pads."""
    folded = []
    for node in list(gm.graph.nodes):
        tl = _zero_pad(node)
        if tl is None or len(node.users) != 1:
            continue
        q = next(iter(node.users))
        if not conv(q) or q.args != (node,) or q.kwargs:
            continue
        new = scheme.fold_pad(mods[q.target], q.target, tl)
        if new is None:
            continue
        _set_module(gm, q.target, new)
        mods[q.target] = new
        q.args = (node.args[0],)
        gm.graph.erase_node(node)
        folded.append((node.name, q.target, tl))
    gm.folded_pads = folded


@dataclasses.dataclass
class _Head:
    """A detection-head operand: producer p, its clamp, the nodes deleted with it, the view's k and constant N or None."""
    p: fx.Node
    clamp: tuple
    path: list
    k: int
    batch: Optional[int]


def _head_operand(view, conv, mods):
    """The _Head of a cat operand `view(N, -1, k)` / `reshape` of [`.contiguous()` of] `.permute(0, 2, 3, 1)` of a `conv`
    producer's single-user pass-through chain; None otherwise.  N is a constant or a dim-0 shape query (.size(0),
    .shape[0], .size()[0]) of a node on that path, used only by the view."""
    if view.op != "call_method" or view.target not in ("view", "reshape") or view.kwargs or len(view.args) < 2 or \
            not isinstance(view.args[0], fx.Node) or len(view.users) != 1:
        return None
    sizes = view.args[1] if len(view.args) == 2 and isinstance(view.args[1], (tuple, list)) else view.args[1:]
    if len(sizes) != 3 or sizes[1] != -1 or not isinstance(sizes[2], int) or isinstance(sizes[2], bool) or sizes[2] <= 0:
        return None
    n, k = sizes[0], sizes[2]
    path, node = [view], view.args[0]
    if node.op == "call_method" and node.target == "contiguous" and len(node.args) == 1 and not node.kwargs:
        path.append(node)
        node = node.args[0]
    if not (node.op == "call_method" and node.target == "permute" and not node.kwargs and isinstance(node.args[0], fx.Node)
            and tuple(node.args[1:] if len(node.args) == 5 else (node.args[1] if len(node.args) == 2 else ())) == (0, 2, 3, 1)):
        return None
    path.append(node)
    back = _walk_back(node.args[0], mods, conv, queries=True)
    if back is None:
        return None
    node, clamp, between = back
    if len(node.args) != 1 or node.kwargs or not isinstance(node.args[0], fx.Node):
        return None
    path += between + [node]

    def query_nodes(u, n):
        """[u, ...] when u reads a shape of n and everything it feeds ends at the view; None otherwise."""
        if not (u.op == "call_method" and u.target == "size" and u.args[0] is n and not u.kwargs and len(u.args) <= 2) \
                and not (u.op == "call_function" and u.target is getattr and u.args == (n, "shape")):
            return None
        if u.users.keys() == {view}:
            return [u]
        if all(g.op == "call_function" and g.target is operator.getitem and g.users.keys() == {view} for g in u.users):
            return [u, *u.users]
        return None

    queries = []
    for a, b in zip(path[1:], path):                            # every node but the view: the next node and shape queries
        for u in a.users:
            qn = [] if u is b else query_nodes(u, a)
            if qn is None:
                return None
            queries += qn
    if isinstance(n, fx.Node):
        base = n.args[0] if n.op == "call_function" and n.target is operator.getitem else None
        dim0 = (n.op == "call_method" and n.target == "size" and n.args[1:] == (0,)) or \
            (base is not None and n.args[1] == 0 and base.op in ("call_method", "call_function") and
             (base.target == "size" and len(base.args) == 1 or base.target is getattr))
        if n not in queries or not dim0:
            return None
        n = None
    elif not isinstance(n, int) or isinstance(n, bool) or n <= 0:
        return None
    if any(q.users.keys() - {view} - set(queries) for q in queries):
        return None
    return _Head(node, clamp, path + queries, k, n)


def _replayed_observer(node, mods, scheme):
    """node, when it calls a replayed observer an epilogue of `scheme` runs (_observer_key) and has one user; else None."""
    return node if scheme.observers and len(node.users) == 1 and _observer_key(node, mods) is not None else None


def _fuse_heads(gm, conv, mods, scheme):
    """Rule (b) of chain_int8(layout=True) and chain_affine(heads=True): detection-head concatenations written in place by
    their producers (no pad code), each applying its operand's replayed observer and one on the cat's single user, if
    any; returns (fused heads, fused observers as (observer module, "head" / "tail", producer name))."""
    g, fused, observed = gm.graph, [], []
    for c in list(g.nodes):                                     # a cat's rewrite touches only its own operands' nodes
        ops = _cat_operands(c, scheme.observers, dims=(1,))
        if ops is None:
            continue
        obs = [_replayed_observer(o, mods, scheme) for o in ops]
        heads = [_head_operand(o if ob is None else o.args[0], conv, mods) for o, ob in zip(ops, obs)]
        if any(h is None for h in heads) or len({h.k for h in heads}) != 1 or len({h.p for h in heads}) != len(heads) \
                or len({h.batch for h in heads} - {None}) > 1 or \
                any(getattr(gm.get_submodule(h.p.target), "pad_code", None) is not None for h in heads):
            continue
        tail = _replayed_observer(next(iter(c.users)), mods, scheme) if len(c.users) == 1 else None
        tkey, layers = None if tail is None else _observer_key(tail, mods), []
        for h, ob in zip(heads, obs):
            p = h.p
            layer = gm.get_submodule(p.target).chained(codes_in=gm.get_submodule(p.target).codes_in, name=p.target,
                                                      epilogue=Epilogue(None, h.clamp, fp32=True), rows=True)
            if ob is not None or tail is not None:
                layer = layer.observe(obs=None if ob is None else _observer_key(ob, mods), tail=tkey)
                observed += [(o.target, what, p.target) for o, what in ((ob, "head"), (tail, "tail")) if o is not None]
            _set_module(gm, p.target, layer)
            layers.append(layer)
        name = "int8_heads_" + c.name
        batch = next((h.batch for h in heads if h.batch is not None), None)
        gm.add_submodule(name, Int8HeadConcat(layers, heads[0].k, batch, name=c.name))
        with g.inserting_before(c):
            node = g.call_module(name, tuple(h.p.args[0] for h in heads))
        for old in [c] + ([tail] if tail is not None else []):
            old.replace_all_uses_with(node)
            g.erase_node(old)
        dead = {n for h in heads for n in h.path} | {o for o in obs if o is not None}
        while dead:                                             # each node goes once nothing uses it
            for n in [n for n in dead if not n.users]:
                g.erase_node(n)
                dead.discard(n)
        fused.append((c.name, [h.p.target for h in heads], heads[0].k))
    g.lint()
    gm.recompile()
    return fused, observed


def chain_int8(model: nn.Module, concrete_args=None, residual=False, pool_cat=False, upsample=False,
               layout=False) -> fx.GraphModule:
    """A torch.fx GraphModule that computes what `model` computes, with activations kept in int8 between converted
    convolutions.

    An edge from an Int8Conv2d P to an Int8Conv2d Q (dense or depthwise) is fused when every node from P to Q has exactly
    one user and every node in between is a pass-through: an exact-identity eval BatchNorm2d (merge_batchnorm's leftover),
    nn.ReLU / F.relu / torch.relu / .relu(), nn.ReLU6 / F.relu6, nn.Hardtanh / F.hardtanh, nn.Identity, or an eval
    nn.Dropout.  P then writes Q's int8 NHWC codes (dfq_i8_conv_requant at Q's act_scale, the activations as one clamp),
    Q reads them, and the nodes in between are deleted (nodes, not modules: a module called elsewhere stays there).  The
    result is bit-identical to the per-layer path.  A skip connection or any other second user, pooling, add / cat, a
    BatchNorm that is not an identity, a Linear, or a layer called at several sites ends the chain.

    residual=True adds residual blocks and tensors with several consumers (dfq_i8_conv_fused, `Epilogue`), still
    bit-identical to the per-layer path:
    - fan-out: from an Int8Conv2d P, forward through single-user pass-throughs to a node with several users.  Its Int8Conv2d
      users (single-site, channels matching) take P's codes when their act_scale equals, bit for bit, the first such user's
      in graph order; every other user, a convolution at another scale included, takes P's fp32 output of the same launch.
    - residual add: operator.add / torch.add / Tensor.add of two distinct nodes, without alpha or out.  The fused operand is
      the first argument whose chain back to an Int8Conv2d P is all single-user pass-throughs (they give the clamp before
      the add); the other is P's residual input, with its exact-identity pass-throughs (identity BatchNorm, Identity, eval
      Dropout, single-user) skipped.  Single-user pass-throughs after the add give the clamp after it, and the fan-out rule
      applies to the result.  P moves to the add's position (its residual may be computed after it in graph order, as in
      ResNet's downsample blocks).
    The deleted pass-throughs' and adds' fp32 value is P's fp32 output.  Adds whose operands differ in shape raise DfqError
    naming the layer when the module runs (no broadcasting).

    The layers of the result are new modules sharing the packed buffers of `model`'s; `model` is not modified.  The fused
    edges are recorded in `requantized_edges`: (producer name, consumer name, (lo, hi)) in graph order, (lo, hi) being the
    clamp the consumer's codes were taken after; with residual=True also the fused adds in `fused_adds`: (producer name,
    add node name, residual node name, (lo, hi) before the add, (lo, hi) after it) in graph order, node names being those
    of the traced model (a residual another fusion deleted is that producer's fp32 output in the result).

    pool_cat=True (with residual=True) also carries codes through max pools and channel concatenations, still bit-identical
    to the per-layer path except where noted:
    - max pool: an nn.MaxPool2d (it may be called at several sites) or F.max_pool2d node without return_indices.  Codes mode
      (dfq_i8_maxpool on codes): its input is a tail that carries codes - a producer's single-user chain or fan-out tail, a
      fused concatenation's or another fused pool's - and every user of the pool, past single-user exact identities (which
      are deleted), takes codes at one scale: an Int8Conv2d at that act_scale, bit for bit, or another such pool.  A clamp
      after a pool ends it.  Two inputs the per-layer path treats otherwise: a window holding a NaN gives the max of the
      other codes (per-layer: -127), and an infinite input at scale 0 gives the code of the max (per-layer: -127).
      Fp32 mode: the pool's input is a producer's single-user pass-through chain and some user needs fp32 (ResNet's stem,
      whose pooled tensor is a residual).  The producer writes its clamped fp32 output (dfq_i8_conv_fused, fp32 only); the
      pool writes torch's fp32 max_pool2d for the fp32 users and the codes of the fan-out rule's Int8Conv2d users.
    - concatenation: torch.cat / torch.concat along dim 1 (or -3) of >= 2 distinct nodes, without out.  Each operand is
      reached from its own Int8Conv2d producer through single-user pass-throughs, every operand but the last has a multiple
      of 16 channels, and every user of the cat's tail (the cat and its single-user pass-throughs) takes codes at one scale
      (Int8Conv2d or codes-mode pool).  Each producer writes its codes, after its operand's clamp composed with the tail's,
      into its channel slice of the consumers' int8 input (dfq_i8_conv_slice), one buffer per forward, in graph order; the
      cat and its pass-throughs are deleted.  Any other cat stays in torch, fp32.
    Edges whose codes come through a fused pool or cat name that node (its traced name) as the producer.  `fused_cats`
    records (cat node name, producer names, channel offsets) and `fused_pools` (pool node name, "codes" or "fp32", the
    outputs it writes), in graph order.  pool_cat=True without residual=True raises DfqError.

    upsample=True (with pool_cat=True) also carries codes out of bilinear upsampling, bit-identical to the per-layer path
    (no exceptions: the codes are those of torch's fp32 output):
    - the node: F.interpolate / nn.Upsample with mode='bilinear', size given (constant or traced, e.g. x.shape[-2:]; checked
      to be a pair of positive ints when the module runs), align_corners True or False, and no scale_factor, antialias or
      recompute_scale_factor, whose input is the end of an Int8Conv2d producer's single-user pass-through chain.  The
      producer writes its clamped fp32 output (dfq_i8_conv_fused, fp32 only; other fp32 users of a fan-out take the same
      tensor), and the upsample (Int8UpsampleBilinear, dfq_i8_upsample_bilinear) writes the codes of torch's output after
      the clamp of its single-user pass-throughs (deleted), when either
      (a) it is, through them, an operand of a concatenation: the concatenation rule accepts it in place of a producer, and
          it writes its slice at the consumers' scale, with the cat tail's clamp composed in.  With upsample=True a user
          that only reads a cat operand's shape (x4.size()[2:], .shape, .size(d), .dim(), on any node of the operand's
          chain - where DeepLab-v3+ reads its upsample sizes) does not count as a second user: it reads the shape of a
          zero-stride view of the slice's writer's output instead (_nchw_view); or
      (b) every user takes codes: Int8Conv2d consumers (single-site, channels matching) at one act_scale, bit for bit.
    Any other upsample stays in torch, fp32, as does anything not listed (nearest or bicubic modes, scale_factor,
    adaptive average pools).  `fused_upsamples` records (node name, producer name, "slice" or "codes", align_corners) in
    graph order; edges whose codes come out of a fused upsample name it as the producer.  upsample=True without
    pool_cat=True raises DfqError.

    layout=True (with upsample=True) also removes the layout copies around converted convolutions, bit-identical to the
    per-layer path (no exceptions):
    (a) zero padding: an F.pad node of one fx node with constant arguments - pad (l, r) or (l, r, t, b), l == r >= 0,
        t == b >= 0, mode 'constant', value 0 or None - whose only user is a single-site Int8Conv2d taking it as its sole
        argument is folded into that convolution: it becomes a copy on the same packed buffers with padding + (t, l), on the
        pad's input, and the pad is deleted.  The per-layer path quantizes the padded zeros to code 0, which is what the
        convolution's out-of-image taps read, so the int32 sums are the same (DeepLab-v3+'s fixed_padding before each
        inverted residual block; in front of a 1x1 convolution too).  This runs before every other rule, which then see a
        direct edge.  Any other pad (asymmetric, negative, reflect / replicate, non-zero, several users, not in front of an
        Int8Conv2d, nn.ZeroPad2d) stays in torch.  `folded_pads` records (pad node name, conv name, (t, l)) in graph order.
    (b) detection heads: a torch.cat / torch.concat along dim 1 of >= 2 distinct nodes, without out, each of them
        `view` / `reshape`(N, -1, k) (N a constant, or a dim-0 shape query - .size(0), .shape[0] - of the path below, used
        only by the view; one k for all) of an optional `.contiguous()` of `.permute(0, 2, 3, 1)` of a single-site Int8Conv2d
        producer's single-user pass-through chain (SSD's compute_header).  The producers write their clamped fp32 output
        pixel-major into their slices of one [N, R, k] tensor per forward (dfq_i8_conv_nhwc), run in operand order at the
        cat's position (Int8HeadConcat), R and the offsets following from the inputs' sizes at run time; the cat becomes
        that tensor for its users, and the views, permutes, shape queries and pass-throughs are deleted.  If one operand
        does not qualify the cat stays in torch.  `fused_heads` records (cat node name, producer names, k).
    layout=True without upsample=True raises DfqError."""
    gm, mods, conv = _trace(model, concrete_args, _NCNN.layer)
    for flag, on, base, has in (("pool_cat", pool_cat, "residual", residual), ("upsample", upsample, "pool_cat", pool_cat),
                                ("layout", layout, "upsample", upsample)):
        if on and not has:
            raise _lib.DfqError("chain_int8: %s=True builds on %s=True" % (flag, base))
    if layout:
        _fold_pads(gm, mods, conv, _NCNN)
    rules = _Rules(cats=pool_cat, pools=pool_cat, up_slices=upsample, up_codes=upsample, heads=layout)
    return _Rewriter(gm, mods, conv, _NCNN, rules).run() if residual else _chain_edges(gm, mods, conv, _NCNN)


def chain_affine(model: nn.Module, concrete_args=None, residual=False, concat=False, fold_pads=False,
                 pools=False, heads=False) -> fx.GraphModule:
    """A torch.fx GraphModule that computes what `model` (after convert_affine) computes, with activations kept as the
    consumers' shifted affine codes between AffineInt8Conv2d layers, bit-identical to the per-layer path.

    The rules are chain_int8's, with AffineInt8Conv2d (dense or depthwise, called at one site) in place of Int8Conv2d and a
    consumer's (act_min, act_max, act_bits), compared bit for bit, in place of its act_scale - two consumers with equal
    ranges and bits read identical codes:
    - single-user edges: every node from P to Q has exactly one user and every node in between is one of chain_int8's
      pass-throughs (exact-identity eval BatchNorm2d, ReLU / ReLU6 / Hardtanh in their module and functional forms,
      nn.Identity, eval Dropout).  P's epilogue (dfq_i8_affine_conv_fused) applies them as one clamp and writes the codes
      dfq_i8_affine_quantize would give Q's input, Q reads them and skips its quantizer, and the nodes in between are
      deleted.
    - residual=True adds chain_int8's fan-out and residual-add rules: from P forward through single-user pass-throughs to
      a node with several users, the AffineInt8Conv2d users whose range key equals the first such user's (graph order)
      take P's codes, every other user - a convolution at another range or bit width included - takes P's fp32 output of
      the same launch; an add of two distinct nodes whose fused operand is P's single-user pass-through chain is computed
      in P's epilogue (clamp before it, fp32 add of the residual, clamp after it), P moving to the add's position (ResNet's
      downsample blocks compute the residual after the block's last convolution).  Adds whose operands differ in shape
      raise DfqError naming the layer when the module runs.
    A producer writes the codes' per-pixel sums S (which a dense consumer's epilogue reads) only when some code consumer is
    dense, and its fp32 output only when a user other than those consumers remains.  Ncnn Int8Conv2d layers and
    AffineInt8Linear stay opaque leaves, so no edge crosses the two schemes; detection heads, max pools, concatenations,
    upsampling and pads stay in torch, fp32, unless heads / pools / concat / fold_pads (below) take them.

    The layers of the result are new modules sharing the packed buffers of `model`'s; `model` is not modified.  The fused
    edges are recorded in `requantized_edges`: (producer name, consumer name, (lo, hi)) in graph order, (lo, hi) the clamp
    the consumer's codes were taken after; with residual=True the fused adds in `fused_adds`: (producer name, add node
    name, residual node name, (lo, hi) before the add, (lo, hi) after it), as chain_int8 records them.

    In the reference's evaluation state - replace_op() active and utils.layer_transform.module_tensor_op a CustomTensorOP, as
    main_*.py --quantize run - the functional ops fake-quantize their inputs with their own QuantMeasure.  chain_affine then
    traces with the raw ops (the patched state is restored even when the trace raises), records each call's caller (the
    first frame outside torch) and replays the cursor protocol of utils/layer_transform.py on the graph in node order: an
    operator.add of two tensors matches add_<L>_2 or iadd_<L>_2, torch.cat of n tensors torch_cat_<L>_<n>, torch.mean /
    F.interpolate / F.softmax ..._<L>_1, only when called from a function named `forward`; a match inserts call_module nodes
    of the next observers on the op's operands (add: input, then the other; cat: in order).  DfqError when the live
    cursors are not at 0 or the graph does not consume the records exactly once.  With residual=True:
    - an add whose fused operand is observer(P's single-user pass-through chain) runs in P's epilogue with that observer
      after the clamp before the add and the residual operand's observer on the fp32 residual (dfq_i8_affine_conv_observed);
    - an observer on a producer's single-user pass-through chain, optionally followed by view / reshape / flatten (shape
      queries do not count as users), is applied in that producer's epilogue to its fp32 output;
    - observers with a truthy update_stat, in training mode, above 8 bits or with a non-finite range stay in torch.
    Folded observers are deleted and recorded in `fused_observers`: (observer module, "operand" / "residual" / "output",
    producer name).  The result's tensor adds are torch.add and its cat / mean / interpolate / softmax the raw ops, so its
    forward can run while replace_op() stays active.  Outside that state nothing here changes.

    fold_pads=True folds zero padding, as chain_int8(layout=True)'s rule (a) but for the affine scheme: an F.pad of one fx
    node with constant arguments - pad (l, r) or (l, r, t, b), l == r >= 0, t == b >= 0, mode 'constant', value 0 or None -
    whose only user is a single-site AffineInt8Conv2d with padding 0 taking it as its sole argument becomes that
    convolution's padding (t, l), and the copy's out-of-image taps read the code of +0.0 at its input range
    (affine_code_of; dfq_i8_affine_conv_layout's pad code), which is what the per-layer path quantizes the padded zeros to:
    bit-identical (DeepLab-v3+'s fixed_padding).  A pad in front of a convolution with padding of its own stays in torch
    (those taps are a dequantized 0.0, not codes), as does any pad chain_int8 leaves.  It runs before every other rule and
    records `folded_pads`: (pad node name, conv name, (t, l)) in graph order.

    concat=True (with residual=True) carries codes into channel concatenations, chain_int8(pool_cat=True, upsample=True)'s
    concatenation rule and its upsample-as-operand rule under the affine scheme, bit-identical to the per-layer path:
    - a torch.cat along dim 1 (or -3) of >= 2 distinct nodes, without out, every operand but the last with a multiple of 16
      channels, each operand an AffineInt8Conv2d producer's single-user pass-through chain, optionally ending in a replayed
      observer, or a bilinear upsample (F.interpolate to a size, no scale_factor; chain_int8's conditions) of such a chain -
      its input observer folded into the producer's fp32 output - followed by single-user pass-throughs and an optional
      observer; every user of the cat's tail (the cat and its single-user pass-throughs) an AffineInt8Conv2d at one range
      key.
    - Each producer (dfq_i8_affine_conv_layout) or upsample (AffineInt8UpsampleBilinear) writes its slice of the consumers'
      codes, one buffer per forward, in graph order: the operand chain's clamp, the operand's observer, the tail's clamp,
      then the consumers' code; the slice's channel sums add into one S zeroed by the first writer, only when a consumer
      is dense.  Shape queries on the operands read a zero-stride view of the writer's codes (_nchw_view).
    - any cat not taken stays in torch (SSD's head concatenations along dim 1 of [N, R, k] included).
    `fused_cats` records (cat node name, writer names, channel offsets), `fused_upsamples` (node name, producer name,
    "slice", align_corners), and the operands' observers enter `fused_observers` as (observer module, "cat", writer
    name).  concat=True without residual=True raises DfqError.

    pools=True (with residual=True) carries the codes through max pools, chain_int8(pool_cat=True)'s pool rule under the
    affine scheme (AffineInt8MaxPool2d, dfq_i8_affine_maxpool), with the consumers' range key in place of their scale:
    codes mode pools the codes of a producer's tail, a fused concatenation's (with concat=True) or another fused pool's,
    every user of the pool past exact identities taking codes at one key; fp32 mode pools a producer's clamped fp32 output
    when some user of the pool needs fp32 (ResNet's stem, whose pooled tensor is a residual) and writes the codes of the
    users at the first key too.  The pool writes S only when one of its code consumers is dense.  replace_op() puts no
    observer on max pools; one on a pool's input or output is an fp32 user.  Bit-identical to the per-layer path except for
    a window holding a NaN, which gives the max of the other codes where the per-layer path gives code -128.  `fused_pools`
    records (pool node name, "codes" or "fp32", the outputs it writes), as chain_int8 records it.  pools=True without
    residual=True raises DfqError.

    heads=True (with residual=True) writes detection-head concatenations in place, chain_int8(layout=True)'s rule (b)
    under the affine scheme: a torch.cat along dim 1 of >= 2 operands, each `view(N, -1, k)` / `reshape` of [`.contiguous()`
    of] `.permute(0, 2, 3, 1)` of a distinct single-site AffineInt8Conv2d's single-user pass-through chain (no folded pad),
    optionally followed by the operand's replayed observer, one k and one N.  Each producer becomes a rows-mode copy
    (_AffineInt8Layer.chained(rows=True), dfq_i8_affine_conv_rows) that writes its slice of one [N, R, k] tensor
    (Int8HeadConcat): the clamp, the operand's observer, and - when the cat's only user is a replayed observer (SSD's
    softmax input, an elementwise op, so per slice) - that observer too, which is deleted.  Any operand that does not
    qualify leaves the cat in torch.  `fused_heads` records (cat node name, producer names, k), and the observers enter
    `fused_observers` as (observer module, "head", producer name) and, once per producer, (observer module, "tail",
    producer name).  heads=True without residual=True raises DfqError."""
    for flag, on in (("concat", concat), ("pools", pools), ("heads", heads)):
        if on and not residual:
            raise _lib.DfqError("chain_affine: %s=True builds on residual=True" % flag)
    LT = _observed_state()
    gm, mods, conv = _trace(model, concrete_args, _AFFINE.layer, LT)
    if fold_pads:
        _fold_pads(gm, mods, conv, _AFFINE)
    rules = _Rules(cats=concat, pools=pools, up_slices=concat, up_codes=False, heads=heads)
    gm = _Rewriter(gm, mods, conv, _AFFINE, rules).run() if residual else _chain_edges(gm, mods, conv, _AFFINE)
    if LT is not None:
        _unpatch_adds(gm, LT)
    return gm


def save(gm: fx.GraphModule, path):
    """Write a chained int8 model - the GraphModule chain_int8 / chain_affine returned, with any flags - to the file `path`,
    for load() in another process: the graph as a node list, each layer's packed codes, tables, ranges and execution modes,
    each shared buffer once, and the chain's records (requantized_edges, fused_*, folded_pads).  One torch.save of plain
    containers and CPU tensors (dfq_b200/int8_io.py has the format).  A per-layer model is not taken: save
    chain_int8(model) / chain_affine(model) with no flags, which computes the same bit for bit.  A graph calling a function,
    tensor method or module type outside the allowlist of what the chains emit (a user function, a module class of the
    model's own) raises DfqError naming it, before anything is written; the file appears whole or not at all, and gm is
    not modified."""
    from . import int8_io
    int8_io.save(gm, path)


def load(path, device=None) -> fx.GraphModule:
    """The chained model save() wrote, rebuilt on the current CUDA device from its stored state, computing what the saved
    model computed, bit for bit, with its records; nothing is repacked.  No code from the file runs: it is read with
    torch.load(weights_only=True), every target and module type is checked against save()'s allowlist, and every name the
    generated forward spells as code (node names, parameters, module paths, keywords, dict keys) must be an identifier (or
    an index in a path).  Each layer's buffers must fit its stored geometry.  It needs dfq_b200 alone: not the model's
    classes, the reference's layers or replace_op().  device: None or the current CUDA device - the layers launch on the
    current device's stream, so load and run a model for another GPU inside `with torch.cuda.device(...)`; any other
    device is refused.  A file of another format or version, with a missing key or failing a check raises DfqError, as
    does a machine without a CUDA device."""
    from . import int8_io
    return int8_io.load(path, device)


class _Scheme(NamedTuple):
    """What the chaining rules need of one integer scheme: `layer`, the convolution class whose edges they fuse; key(m),
    what decides the codes layer m reads, compared bit for bit by same(a, b) (consumers with equal keys read identical
    codes); out(key), the producer's output argument for such a consumer (requant's first element, Epilogue.out_scale).
    observers: replayed observers exist and the evaluation state's raw ops count (_orig).  pool, upsample: the fused
    modules' classes (one argument list).  slice(out, pre, post): a cat writer's chained() mode (clamp pre, observer,
    clamp post).  fold_pad(m, name, (t, l)): m's copy reading through a zero pad, or None."""
    layer: type
    key: object
    same: object
    out: object
    observers: bool
    pool: type
    upsample: type
    slice: object
    fold_pad: object


def _fold_ncnn_pad(m, name, pad):
    new = m.chained(name=name)
    new.padding = (m.padding[0] + pad[0], m.padding[1] + pad[1])
    return new


_NCNN = _Scheme(Int8Conv2d, lambda m: _f32(m.act_scale), lambda a, b: a.view(np.int32) == b.view(np.int32), float,
                observers=False, pool=Int8MaxPool2d, upsample=Int8UpsampleBilinear,
                slice=lambda out, pre, post: dict(requant=(out,) + _compose(pre, post)), fold_pad=_fold_ncnn_pad)
_AFFINE = _Scheme(AffineInt8Conv2d, lambda m: (_f32(m.act_min), _f32(m.act_max), int(m.act_bits)),
                  lambda a, b: a[0].view(np.int32) == b[0].view(np.int32) and a[1].view(np.int32) == b[1].view(np.int32)
                  and a[2] == b[2],
                  lambda k: (float(k[0]), float(k[1]), int(k[2])),
                  observers=True, pool=AffineInt8MaxPool2d, upsample=AffineInt8UpsampleBilinear,
                  slice=lambda out, pre, post: dict(epilogue=Epilogue(out, pre, post)),
                  fold_pad=lambda m, name, pad: m.chained(name=name).fold_pad(pad) if m.padding == (0, 0) else None)


class _Rules(NamedTuple):
    """_Rewriter's rules besides fan-out and adds: cats, pools, upsamples into cats or to codes users, detection heads."""
    cats: bool
    pools: bool
    up_slices: bool
    up_codes: bool
    heads: bool


def _observed_state():
    """utils.layer_transform when the reference's evaluation state is active - replace_op() in place and a CustomTensorOP
    as module_tensor_op (what main_*.py --quantize run, through dropin/) - else None."""
    from .utils import layer_transform as LT
    if LT.raw_torch_op.get("cat") is None or torch.cat is not LT.torch_cat or \
            not isinstance(LT.module_tensor_op, LT.CustomTensorOP):
        return None
    return LT


_OBSERVER_ROOT = "custom_tensor_op"


_INT_ARITH = (operator.add, operator.sub, operator.mul, operator.floordiv, operator.truediv, operator.mod, operator.neg,
              operator.pow)


def _shape_only(n):
    """n is an int or a shape - a size / dim / numel / .shape query, an item of one, or arithmetic on such nodes and
    constants (x.size(2) * 2 + 1) - not a tensor."""
    if n.op == "call_method" and n.target in ("size", "dim", "numel"):
        return True
    if n.op == "call_function" and n.target is getattr:
        return True
    if n.op == "call_function" and n.target is operator.getitem:
        return isinstance(n.args[0], fx.Node) and _shape_only(n.args[0])
    if n.op == "call_function" and n.target in _INT_ARITH and not n.kwargs:
        nodes = [a for a in n.args if isinstance(a, fx.Node)]
        return bool(nodes) and all(_shape_only(a) for a in nodes) and \
            all(isinstance(a, fx.Node) or (isinstance(a, (int, float)) and not isinstance(a, bool)) for a in n.args)
    return False


def _replay_observers(gm, model, LT):
    """Insert the observers of LT.module_tensor_op into the traced gm as call_module nodes, where the patched ops would
    apply them: the cursor protocol of utils/layer_transform.py replayed on the graph in node order, on copies of the
    cursors.  Returns nothing; raises DfqError when the cursors are not at 0 or the records are not consumed exactly once."""
    ct = LT.module_tensor_op
    recs = [r[1] for r in ct.name_tensor_op]
    if ct.idx_name_tensor_op != 0 or ct.idx_tensor_op != 0:
        raise _lib.DfqError("chain_affine: the functional-op observers' cursors are at record %d, observer %d, not 0: a "
                            "forward was interrupted" % (ct.idx_name_tensor_op, ct.idx_tensor_op))
    root = {id(m): n for n, m in model.named_modules()}.get(id(ct)) or _OBSERVER_ROOT
    gm.add_submodule(root, ct)                                  # the observers are leaves: called, not traced
    raw = {LT.raw_torch_op["cat"]: "torch_cat", LT.raw_torch_op["mean"]: "torch_mean",
           LT.raw_func_op["interpolate"]: "F_interpolate", LT.raw_func_op["softmax"]: "F_softmax"}
    i_rec, i_obs, consumed = 0, 0, 0
    for node in list(gm.graph.nodes):
        caller = node.meta.get("caller")
        if node.op != "call_function" or caller is None or caller[0] != "forward" or not recs:
            continue
        line = caller[1]
        if node.target is operator.add:
            ops = node.args[:2]
            if len(node.args) != 2 or node.kwargs or not all(isinstance(a, fx.Node) and not _shape_only(a) for a in ops):
                continue
            names_ok = ("add_%d_2" % line, "iadd_%d_2" % line)
        elif node.target in raw and node.args:
            if raw[node.target] == "torch_cat":
                ts = node.args[0]
                if not isinstance(ts, (list, tuple)) or not all(isinstance(t, fx.Node) for t in ts):
                    continue
                ops, names_ok = tuple(ts), ("torch_cat_%d_%d" % (line, len(ts)),)
            elif not isinstance(node.args[0], fx.Node):
                continue
            else:
                ops, names_ok = (node.args[0],), ("%s_%d_1" % (raw[node.target], line),)
        else:
            continue
        if recs[i_rec] not in names_ok:
            continue
        obs = []
        for t in ops:
            with gm.graph.inserting_before(node):
                obs.append(gm.graph.call_module("%s.%d" % (root, i_obs), (t,)))
            i_obs = (i_obs + 1) % ct.len
        if node.target is operator.add:
            node.args = tuple(obs)
        elif raw[node.target] == "torch_cat":
            node.args = (type(node.args[0])(obs),) + tuple(node.args[1:])
        else:
            node.args = (obs[0],) + tuple(node.args[1:])
        i_rec = (i_rec + 1) % len(recs)
        consumed += 1
    if consumed != len(recs):
        raise _lib.DfqError("chain_affine: the traced graph %s the functional-op records: %s" % (
            "consumes more than once" if consumed > len(recs) else "leaves unmatched",
            "%d calls for %d records" % (consumed, len(recs)) if consumed > len(recs) else
            "first unmatched record %r (record %d of %d)" % (recs[i_rec], i_rec, len(recs))))


def _unpatch_adds(gm, LT):
    """Make gm's generated forward immune to the patched ops: tensor operator.add -> torch.add (bit-identical, not
    patched), and torch.cat / mean, F.interpolate / softmax -> the raw ops called through module-level functions (the
    generated code would otherwise name the patched torch.cat etc.)."""
    raw = {LT.raw_torch_op["cat"]: _raw_cat, LT.raw_torch_op["mean"]: _raw_mean,
           LT.raw_func_op["interpolate"]: _raw_interpolate, LT.raw_func_op["softmax"]: _raw_softmax}
    for node in gm.graph.nodes:
        if node.op != "call_function":
            continue
        if node.target is operator.add and node.args and isinstance(node.args[0], fx.Node) and \
                not _shape_only(node.args[0]):
            node.target = torch.add
        elif node.target in raw:
            node.target = raw[node.target]
    gm.recompile()


def _raw(table, name):
    """The unpatched op: the one replace_op() saved, or the live one when replace_op() never ran in this process (a
    chained model loaded by int8.load)."""
    from .utils import layer_transform as LT
    op = getattr(LT, table).get(name)
    return op if op is not None else getattr(torch if table == "raw_torch_op" else F, name)


def _raw_cat(*a, **k):
    return _raw("raw_torch_op", "cat")(*a, **k)


def _raw_mean(*a, **k):
    return _raw("raw_torch_op", "mean")(*a, **k)


def _raw_interpolate(*a, **k):
    return _raw("raw_func_op", "interpolate")(*a, **k)


def _raw_softmax(*a, **k):
    return _raw("raw_func_op", "softmax")(*a, **k)


def _trace(model, concrete_args, layer, observed=None):
    """(GraphModule of `model` traced with the int8 layers as leaves, its modules by name, conv(node): node calls a
    `layer` module that is called at no other site).  observed: utils.layer_transform in the reference's evaluation state
    (_observed_state): the model is traced with the raw ops in place (restored in every case) and the functional-op
    observers are inserted as call_module nodes (_replay_observers)."""
    tracer = _Int8Tracer(callers=observed is not None)
    if observed is None:
        graph = tracer.trace(model, concrete_args)
    else:
        LT = observed
        patched = [(o, n, getattr(o, n)) for o, names in ((torch.Tensor, LT.tensor_magic_op_supported),
                                                          (torch, LT.torch_op_supported), (F, LT.func_op_sopprted))
                   for n in names]
        try:
            LT.restore_op()
            graph = tracer.trace(model, concrete_args)
        finally:
            for o, n, f in patched:
                setattr(o, n, f)
    gm = fx.GraphModule(tracer.root, graph, type(model).__name__ + "Int8Chained")
    if observed is not None:
        _replay_observers(gm, model, observed)
    mods = dict(gm.named_modules())
    sites = collections.Counter(node.target for node in gm.graph.nodes if node.op == "call_module")

    def conv(node):
        return node.op == "call_module" and isinstance(mods[node.target], layer) and sites[node.target] == 1

    return gm, mods, conv


def _chain_edges(gm, mods, conv, scheme):
    """The single-user edge rule of chain_int8 / chain_affine (residual=False) on the traced `gm`; no observer fused."""
    edges, between = [], []
    for q in list(gm.graph.nodes):
        if not conv(q) or len(q.args) != 1 or q.kwargs or not isinstance(q.args[0], fx.Node):
            continue
        back = _walk_back(q.args[0], mods, conv)
        if back is None or mods[back[0].target].out_channels != mods[q.target].in_channels:
            continue
        node, clamp, path = back
        edges.append((node.target, q.target, clamp))
        between.append((node, q, path))
    producers = {p: c for p, _, c in edges}
    consumers = {q for _, q, _ in edges}
    for target in producers.keys() | consumers:
        requant, sums = None, False
        if target in producers:
            nxt = mods[next(q for p, q, _ in edges if p == target)]
            requant = (scheme.out(scheme.key(nxt)),) + tuple(producers[target])
            sums = nxt.groups == 1
        _set_module(gm, target, mods[target].chained(codes_in=target in consumers, requant=requant, sums=sums))
    for p, q, path in between:
        q.args = (p,)
        for node in path:                                       # from the consumer side back: each has no user left
            gm.graph.erase_node(node)
    gm.graph.lint()
    gm.recompile()
    gm.requantized_edges = edges
    if scheme.observers:
        gm.fused_observers = []
    return gm


@dataclasses.dataclass
class _Plan:
    """A producer's plan: p, its pass-throughs `path` (clamp `pre`) to `tail`, whose users `codes` take codes at `scale`;
    a fused `add`, its residual argument ri and the pass-throughs `post_path` after it (clamp `post`); the observers obs
    (without an add: on the fp32 output) and robs (residual); the residual's skipped identities and its name r_name."""
    p: fx.Node
    path: list
    pre: tuple
    tail: fx.Node
    codes: list = dataclasses.field(default_factory=list)
    scale: object = None
    add: Optional[fx.Node] = None
    ri: Optional[int] = None
    post: tuple = _FULL
    post_path: list = dataclasses.field(default_factory=list)
    obs: Optional[fx.Node] = None
    robs: Optional[fx.Node] = None
    skipped: list = dataclasses.field(default_factory=list)
    r_name: Optional[str] = None

    def nodes(self):
        return (self.p, *self.path, *([self.add] if self.add is not None else []), *self.post_path)


@dataclasses.dataclass
class _Codes:
    """A node whose users `codes` take its codes, `channels` wide, at key `scale` after the clamp `clamp`, past the
    pass-throughs `path` to `tail`: a codes-mode upsample's plan, or a max pool's (exact identities; no tail: fp32 mode)."""
    node: fx.Node
    path: list
    tail: Optional[fx.Node]
    clamp: tuple
    codes: list
    scale: object
    channels: int

    def nodes(self):
        return (self.node, *self.path)


@dataclasses.dataclass
class _Operand:
    """A fused cat's operand: writer p, the nodes `path` back to it (clamp `pre`), observer, slice and shape queries."""
    p: fx.Node
    path: list
    pre: tuple
    obs: Optional[fx.Node]
    coff: int
    channels: int
    queries: list


@dataclasses.dataclass
class _CatPlan(_Codes):
    """A concatenation's plan: its _Operands write one buffer, with sums when a consumer is dense."""
    operands: list
    sums: bool

    def nodes(self):
        return (*super().nodes(), *(n for o in self.operands for n in (o.p, *o.path)))


def _split(g, node):
    """(codes, fp32): getitem nodes inserted after `node`, a call that returns both."""
    with g.inserting_after(node):
        y = g.call_function(operator.getitem, (node, 1))
    with g.inserting_after(node):
        codes = g.call_function(operator.getitem, (node, 0))
    return codes, y


class _Rewriter:
    """chain_int8(residual=True, ...) / chain_affine(residual=True, ...) on the traced gm: fan-out, adds and `rules` under
    `scheme`.  The plan_* steps read the graph as traced, as do the memos; run() then rewrites it."""

    def __init__(self, gm, mods, conv, scheme, rules):
        self.gm, self.mods, self.conv, self.scheme, self.rules = gm, mods, conv, scheme, rules
        self.order = {n: i for i, n in enumerate(gm.graph.nodes)}
        self.convs = {n for n in gm.graph.nodes if self.producer(n)}   # before the rewrites give producers a second input
        # bilinear upsamples: the producer whose single-user pass-through chain ends at the upsample's input
        self.ends = {self.forward(p)[0]: p for p in self.convs} if rules.up_slices or rules.up_codes else {}
        self.sources, self.pool_scales, self.pools = {}, {}, []
        self.edges, self.adds, self.modes, self.watched, self.observed, self.cats, self.ups = [], [], {}, {}, [], [], []

    def producer(self, node):
        return self.conv(node) and len(node.args) == 1 and not node.kwargs and isinstance(node.args[0], fx.Node)

    def forward(self, node, identities=False):
        """(last node, composed clamp, nodes walked) from node through single users of one fx input that are
        pass-throughs (exact identities, as after a pool, with `identities`)."""
        clamp, path = _FULL, []
        while len(node.users) == 1:
            u = next(iter(node.users))
            c = (_FULL if _is_identity(u, self.mods) else None) if identities else _pass_through(u, self.mods)
            if c is None or len(u.all_input_nodes) != 1 or u.args[0] is not node:
                break
            clamp, node = _compose(clamp, c), u
            path.append(u)
        return node, clamp, path

    def observer(self, node):
        return _replayed_observer(node, self.mods, self.scheme) is not None

    def up_source(self, node):
        """The producer of a fusable bilinear upsample node, or None."""
        if node not in self.sources:
            src = node.args[0] if node.args else None
            if isinstance(src, fx.Node) and self.observer(src):    # its input observer goes into the producer
                src = src.args[0]
            self.sources[node] = self.ends.get(src) if self.ends and \
                _bilinear_upsample(node, self.mods, self.scheme.observers) is not None else None
        return self.sources[node]

    def pool_scale(self, pool, channels):
        """The key at which every user of a pool (past exact identities) takes codes, or None."""
        if pool not in self.pool_scales:
            self.pool_scales[pool] = None
            tail = self.forward(pool, True)[0]
            scales = [self.user_scale(u, tail, channels) for u in tail.users]
            self.pool_scales[pool] = scales[0] if scales and all(
                s is not None and self.scheme.same(s, scales[0]) for s in scales) else None
        return self.pool_scales[pool]

    def user_scale(self, u, tail, channels, pools=True):
        """The key at which u takes the codes of `tail` (channels wide), or None when it takes fp32."""
        if self.producer(u) and u.args[0] is tail and self.mods[u.target].in_channels == channels:
            return self.scheme.key(self.mods[u.target])
        if pools and self.rules.pools and _max_pool(u, self.mods) is not None and u.args[0] is tail:
            return self.pool_scale(u, channels)
        return None

    def take_codes(self, tail, channels, pools=True):
        """The fan-out rule: the users of tail that take codes at the first such user's key (graph order), and it."""
        codes, scale = [], None
        for u in sorted(tail.users, key=self.order.get):
            s = self.user_scale(u, tail, channels, pools)
            if s is not None and (scale is None or self.scheme.same(s, scale)):
                scale = s
                codes.append(u)
        return codes, scale

    def plan_pools(self, codes, channels, clamp):
        """The codes-mode pools among `codes` (users that take a tail's codes) and among the users after them."""
        for u in codes:
            if not self.producer(u):
                tail, _, ids = self.forward(u, True)
                self.pools.append(_Codes(u, ids, tail, clamp, sorted(tail.users, key=self.order.get),
                                         self.pool_scale(u, channels), channels))
                self.plan_pools(tail.users, channels, clamp)

    def plan_producers(self):
        """Single-user edges, fan-out and residual adds, and fp32-mode pools: the producers' _Plans."""
        plans, mods = [], self.mods
        for p in list(self.gm.graph.nodes):
            if not self.producer(p):
                continue
            end, pre, path = self.forward(p)
            add, ri, post, post_path, tail = None, None, _FULL, [], end
            fobs = robs = None
            if len(end.users) == 1:
                a = next(iter(end.users))
                if self.observer(a):                            # the observer on the fused operand (replace_op's add)
                    fobs, a = a, next(iter(a.users))
                if _is_add(a):
                    ops = [v.args[0] if self.observer(v) else v for v in a.args]
                    fused = next((i for i, v in enumerate(ops) if _walk_back(v, mods, self.producer) is not None), None)
                    if fused is not None and ops[fused] is end and (fobs is None or a.args[fused] is fobs):
                        add, ri = a, 1 - fused
                        tail, post, post_path = self.forward(a)
                        robs = a.args[ri] if self.observer(a.args[ri]) else None
                if add is None:
                    fobs = None
            out_c = mods[p.target].out_channels
            codes, scale = self.take_codes(tail, out_c)
            clamp = post if add is not None else pre
            if add is None and not codes and self.rules.pools and len(tail.users) == 1:
                u = next(iter(tail.users))                      # fp32-mode pool: a user of the pool needs fp32
                if _max_pool(u, mods) is not None and u.args[0] is tail:
                    pc, ps = self.take_codes(u, out_c, pools=False)
                    if pc:
                        self.pools.append(_Codes(u, [], None, clamp, pc, ps, out_c))
                        plans.append(_Plan(p, path, pre, tail))
                continue
            if add is None and not codes:
                continue
            plans.append(_Plan(p, path, pre, tail, codes, scale, add=add, ri=ri, post=post, post_path=post_path, obs=fobs,
                               robs=robs))
            self.plan_pools(codes, out_c, clamp)
        return plans

    def plan_cats(self):
        """Concatenations whose operands come from their own writers and whose users all take codes at one key."""
        plans, up, mods = [], self.rules.up_slices, self.mods
        for c in (list(self.gm.graph.nodes) if self.rules.cats else []):
            ops = _cat_operands(c, self.scheme.observers)
            if ops is None:
                continue
            oobs = [o if self.observer(o) else None for o in ops]   # the operand's writer applies its observer
            ops = [o.args[0] if ob is not None else o for o, ob in zip(ops, oobs)]
            backs = [_walk_back(o, mods, self.producer, up) or
                     (_walk_back(o, mods, lambda n: self.up_source(n) is not None, True) if up else None) for o in ops]
            if any(b is None for b in backs) or len({b[0] for b in backs}) != len(backs):
                continue
            chans = [mods[(self.up_source(q) or q).target].out_channels for q, _, _ in backs]
            if any(k % 16 for k in chans[:-1]):
                continue
            tail, tclamp, tpath = self.forward(c)
            codes, scale = self.take_codes(tail, sum(chans))
            if not codes or len(codes) != len(tail.users):
                continue
            operands = [_Operand(q, opath, clamp, ob, off, k,
                                 [(u, n) for n in (q, *opath) for u in n.users if up and _shape_query(u, n)])
                        for ob, (q, clamp, opath), k, off in zip(oobs, backs, chans, np.cumsum([0] + chans[:-1]).tolist())]
            plans.append(_CatPlan(c, tpath, tail, tclamp, codes, scale, sum(chans), operands,
                                  any(self.producer(u) and mods[u.target].groups == 1 for u in codes)))
            self.plan_pools(codes, sum(chans), tclamp)
        return plans

    def plan_observers(self, plans, cats):
        """Add to `plans` the observers after a producer's pass-throughs and shape-only views, run in its epilogue."""
        taken = {n for pl in plans for n in (pl.obs, pl.robs)} | {o.obs for cp in cats for o in cp.operands}
        planned = {pl.p for pl in plans}
        for o in (list(self.gm.graph.nodes) if self.scheme.observers else []):
            if o in taken or _observer_key(o, self.mods) is None:
                continue
            node = o.args[0]
            while _is_view(node) and len(_data_users(node, True)) == 1:
                node = node.args[0]
            back = _walk_back(node, self.mods, self.producer, queries=True)
            if back is None or back[0] in planned:
                continue
            q, clamp, path = back
            plans.append(_Plan(q, path[::-1], clamp, node, obs=o))
            planned.add(q)

    def plan_upsamples(self, plans, cats):
        """Codes-mode upsamples; their and the fused cats' upsamples' producers write fp32 (a _Plan added if none)."""
        sliced, ups = [o.p for cp in cats for o in cp.operands if not self.producer(o.p)], []
        for u in (list(self.gm.graph.nodes) if self.rules.up_codes else []):
            if u in sliced or self.up_source(u) is None:
                continue
            tail, clamp, path = self.forward(u)
            channels = self.mods[self.up_source(u).target].out_channels
            codes, scale = self.take_codes(tail, channels, pools=False)
            if codes and len(codes) == len(tail.users):
                ups.append(_Codes(u, path, tail, clamp, codes, scale, channels))
        planned = {pl.p for pl in plans}
        for u in sliced + [up.node for up in ups]:
            p = self.up_source(u)
            if p not in planned:
                plans.append(_Plan(p, *self.forward(p)[::-1]))   # (path, pre, tail)
                planned.add(p)
        return ups

    def skip_identities(self, plans, claimed):
        """Skip the residual's exact identities once every plan's nodes are `claimed`: a node another plan deletes (say an
        identity ending its post-add chain) stays the residual, which that plan replaces by its fp32 output."""
        for pl in plans:
            if pl.add is None:
                continue
            r = pl.robs.args[0] if pl.robs is not None else pl.add.args[pl.ri]
            while r not in claimed and len(r.users) == 1 and _is_identity(r, self.mods) and isinstance(r.args[0], fx.Node):
                pl.skipped.append(r)
                r = r.args[0]
            pl.r_name = r.name

    def hand_over(self, plan, src, name):
        """plan's code users read src instead of its tail, its path goes, and its edges are recorded as from `name`."""
        for v in plan.codes:
            v.replace_input_with(plan.tail, src)
            if v in self.convs:
                self.edges.append((name, v.target, plan.clamp))
        for node in reversed(plan.path):
            self.gm.graph.erase_node(node)

    def rewrite_producer(self, pl):
        g, p, add, tail, fobs, robs = self.gm.graph, pl.p, pl.add, pl.tail, pl.obs, pl.robs
        if add is not None:
            for node in pl.skipped:                             # from the add back: each loses its only user
                node.replace_all_uses_with(node.args[0])
                g.erase_node(node)
            add.prepend(p)
            p.args = (p.args[0], robs.args[0] if robs is not None else add.args[pl.ri])
        fp32 = any(u not in pl.codes for u in tail.users)
        scale = self.scheme.out(pl.scale) if pl.codes else None
        clamp = pl.post if add is not None else pl.pre
        codes_node = y_node = p
        if add is None and not fp32:
            self.modes[p.target] = dict(requant=(scale,) + tuple(clamp))
        else:
            self.modes[p.target] = dict(epilogue=Epilogue(scale, pl.pre, pl.post, add is not None, fp32))
            keys = tuple(None if o is None else _observer_key(o, self.mods) for o in (fobs, robs))
            if keys != (None, None):
                self.watched[p.target] = keys
            if scale is not None and fp32:
                codes_node, y_node = _split(g, p)
        for u in pl.codes:
            u.replace_input_with(tail, codes_node)
            if u in self.convs:
                self.edges.append((p.target, u.target, clamp))
        for node in pl.path:                                    # shape queries inside the chain read p's output
            for u in [u for u in node.users if _shape_query(u, node)]:
                u.replace_input_with(node, y_node)
        if tail is not p:
            tail.replace_all_uses_with(y_node)
            on_add = [o for o in (fobs, robs) if o is not None and add is not None]
            for node in reversed([*pl.path, *on_add, *([add] if add is not None else []), *pl.post_path]):
                g.erase_node(node)
        else:
            p.replace_all_uses_with(y_node, delete_user_cb=lambda u: u not in (y_node, codes_node))
        if add is None and fobs is not None:                    # the views now read the observed output
            fobs.replace_all_uses_with(fobs.args[0])
            g.erase_node(fobs)
            self.observed.append((fobs.target, "output", p.target))
        elif add is not None:
            self.observed += [(o.target, w, p.target) for o, w in ((fobs, "operand"), (robs, "residual")) if o is not None]
            self.adds.append((p.target, add.name, pl.r_name, pl.pre, pl.post))

    def fuse_upsample(self, u, scale, pre, post, out_slice=None, out=None, obs=None, sums=False):
        """Make u call the scheme's upsample module: clamp pre, observer obs, clamp post, codes at `scale` [into `out`]."""
        (size, ac), p = _bilinear_upsample(u, self.mods, self.scheme.observers), self.up_source(u)
        mod = self.scheme.upsample(self.mods[p.target].out_channels, ac, self.scheme.out(scale), out_slice=out_slice,
                                   pre=pre, obs=None if obs is None else _observer_key(obs, self.mods), post=post,
                                   sums=sums, name=u.name)
        name = "int8_up_" + u.name
        self.gm.add_submodule(name, mod)
        self.ups.append((self.order[u], (u.name, p.target, "slice" if out_slice else "codes", ac)))
        u.op, u.target, u.args, u.kwargs = "call_module", name, (u.args[0], size), ({} if out is None else {"out": out})

    def rewrite_cat(self, cp):
        """The writers fill their slices of one buffer in graph order, threaded through `out`."""
        g, prev = self.gm.graph, None
        names = [o.p.target if self.producer(o.p) else o.p.name for o in cp.operands]
        for o in sorted(cp.operands, key=lambda o: self.order[o.p]):
            q, out_slice = o.p, (o.coff, (cp.channels + 15) // 16 * 16)
            if not self.producer(q):
                self.fuse_upsample(q, cp.scale, o.pre, cp.clamp, out_slice, prev, o.obs, cp.sums)
            else:
                self.modes[q.target] = dict(self.scheme.slice(self.scheme.out(cp.scale), o.pre, cp.clamp),
                                            out_slice=out_slice, sums=cp.sums)
                if o.obs is not None:
                    self.watched[q.target] = (_observer_key(o.obs, self.mods), None)
                if prev is not None:
                    q.kwargs = {"out": prev}
            prev = q
        self.hand_over(cp, prev, cp.node.name)
        g.erase_node(cp.node)
        for o, name in zip(cp.operands, names):
            if o.obs is not None:                               # the operand's observer, now in its writer
                g.erase_node(o.obs)
                self.observed.append((o.obs.target, "cat", name))
            for u, n in o.queries:                              # shape queries read the shape off the slice's writer
                with g.inserting_before(u):
                    u.replace_input_with(n, g.call_function(_nchw_view, (o.p, o.channels)))
            for node in o.path:                                 # from the cat back to the producer
                g.erase_node(node)
        self.cats.append((cp.node.name, names, [o.coff for o in cp.operands]))

    def rewrite_pool(self, pp):
        """The pool reads its input as the rewrites before it left it; returns its fused_pools record."""
        g, u = self.gm.graph, pp.node
        codes_mode = pp.tail is not None
        sums = any(v in self.convs and self.mods[v.target].groups == 1 for v in pp.codes)   # S only for a dense consumer
        mod = self.scheme.pool(*_max_pool(u, self.mods), pp.channels, codes_mode,
                               None if codes_mode else self.scheme.out(pp.scale), not codes_mode, sums=sums, name=u.name)
        name = "int8_pool_" + u.name
        self.gm.add_submodule(name, mod)
        u.op, u.target, u.args, u.kwargs = "call_module", name, (u.args[0],), {}
        if codes_mode:
            self.hand_over(pp, u, u.name)
            return u.name, "codes", ("codes",)
        codes_node, y_node = _split(g, u)
        for v in pp.codes:
            v.replace_input_with(u, codes_node)
        u.replace_all_uses_with(y_node, delete_user_cb=lambda x: x not in (y_node, codes_node))
        self.edges += [(u.name, v.target, pp.clamp) for v in pp.codes if v in self.convs]
        return u.name, "fp32", ("fp32", "codes")

    def plan_means(self, planned):
        """The tail rule of an ncnn model (ncnn.load): a producer's single-user pass-through chain, an optional flatten,
        a PlaneMean and, past an optional reshape, a dense 1 x 1 Int8Conv2d of its channels.  Returns [(producer, its
        pass-throughs, clamp, flatten | None, mean node, reshape | None, consumer)]."""
        from .ncnn import PlaneMean
        means = []
        for m in (list(self.gm.graph.nodes) if self.scheme is _NCNN else []):
            if m.op != "call_module" or type(self.mods[m.target]) is not PlaneMean or \
                    self.mods[m.target].out_scale is not None or len(m.users) != 1 or len(m.args) != 1 or m.kwargs:
                continue
            x, view = m.args[0], None
            if isinstance(x, fx.Node) and x.op == "call_method" and x.target == "flatten" and len(x.users) == 1:
                x, view = x.args[0], x
            back = _walk_back(x, self.mods, self.producer) if isinstance(x, fx.Node) else None
            if back is None or back[0] in planned:
                continue
            q, reshape = next(iter(m.users)), None
            if q.op == "call_method" and q.target in ("reshape", "view") and len(q.users) == 1 and len(q.all_input_nodes) == 1:
                q, reshape = next(iter(q.users)), q
            if not self.producer(q) or q.args[0] is not (reshape or m):
                continue
            c, mod = self.mods[back[0].target].out_channels, self.mods[q.target]
            if mod.groups != 1 or mod.kernel_size != (1, 1) or mod.in_channels != c:
                continue
            means.append((back[0], back[2], back[1], view, m, reshape, q))
        return means

    def rewrite_mean(self, p, path, clamp, view, m, reshape, q):
        """p writes its clamped fp32 output, the mean writes q's codes [N, 1, 1, Cpad] and q reads them."""
        g = self.gm.graph
        self.modes[p.target] = dict(epilogue=Epilogue(None, clamp, _FULL, False, True))
        first = path[0] if path else p
        first.replace_all_uses_with(p)
        for node in path:                                       # from the flatten back: each has no user left
            g.erase_node(node)
        mean = self.mods[m.target]
        name = "int8_mean_" + m.name
        self.gm.add_submodule(name, type(mean)(mean.divide, self.scheme.out(self.scheme.key(self.mods[q.target])),
                                               name=mean.layer_name))
        m.target = name
        if reshape is not None:
            q.replace_input_with(reshape, m)
            g.erase_node(reshape)
        self.edges.append((m.name, q.target, clamp))

    def run(self):
        plans, cats = self.plan_producers(), self.plan_cats()
        self.plan_observers(plans, cats)
        ups = self.plan_upsamples(plans, cats)
        means = self.plan_means({pl.p for pl in plans})
        plans.sort(key=lambda pl: self.order[pl.p])
        self.skip_identities(plans, {n for plan in (*plans, *cats, *self.pools, *ups) for n in plan.nodes()})
        # rewrite in producer order (a producer's input may be the codes of an earlier one, and a residual its fp32
        # output), then the concatenations, the codes-mode upsamples and, last, the pools
        gm, g, mods = self.gm, self.gm.graph, self.mods
        for pl in plans:
            self.rewrite_producer(pl)
        for cp in cats:
            self.rewrite_cat(cp)
        for up in ups:
            self.fuse_upsample(up.node, up.scale, up.clamp, _FULL)
            self.hand_over(up, up.node, up.node.name)
        pools = [self.rewrite_pool(pp) for pp in sorted(self.pools, key=lambda pp: self.order[pp.node])]
        for mp in means:
            self.rewrite_mean(*mp)
        consumers = {q for _, q, _ in self.edges}
        dense = {p for p, q, _ in self.edges if mods[q].groups == 1}   # producers whose codes a dense consumer reads
        for target in self.modes.keys() | consumers:
            kw = self.modes.get(target, {})
            mod = mods[target].chained(codes_in=target in consumers, name=target,
                                       **dict(kw, sums=target in dense or kw.get("sums", False)))
            _set_module(gm, target, mod.observe(*self.watched[target]) if target in self.watched else mod)
        g.lint()
        gm.recompile()
        if self.rules.heads:
            gm.fused_heads, observed = _fuse_heads(gm, self.conv, mods, self.scheme)
            self.observed += observed
        gm.requantized_edges, gm.fused_adds = self.edges, self.adds
        if self.scheme.observers:
            gm.fused_observers = self.observed
        if self.rules.cats:
            gm.fused_cats = self.cats
        if self.rules.cats or self.rules.pools:
            gm.fused_pools = pools
        if self.rules.up_slices:
            gm.fused_upsamples = [t for _, t in sorted(self.ups)]
        return gm
