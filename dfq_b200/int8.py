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
"""
import ctypes as C
import operator
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


class _Int8Layer(nn.Module):
    """Packed int8 weights, dq and bias of one layer on the device; forward quantizes the input and convolves.

    Execution modes, set only on the copies chain_int8 makes (`chained`): `codes_in` - the input is already int8 NHWC codes
    [N, H, W, cpad] at this layer's act_scale; `requant` = (out_scale, lo, hi) - the output is the next layer's int8 NHWC
    codes (dfq_i8_conv_requant) instead of fp32 NCHW; `epilogue` - the residual epilogue (dfq_i8_conv_fused, see Epilogue).
    A layer convert_to_int8 made takes and returns fp32 only."""

    codes_in = False
    requant = None
    epilogue = None
    out_slice = None
    layer_name = None

    def __init__(self, weight, bias, act_scale, w_scale, stride=1, padding=0, dilation=1, groups=1):
        super().__init__()
        O, Cg, kh, kw = weight.shape
        self.out_channels, self.in_channels, self.groups = int(O), int(Cg) * int(groups), int(groups)
        self.kernel_size, self.stride, self.padding, self.dilation = (int(kh), int(kw)), _pair(stride), _pair(padding), _pair(dilation)
        self.cpad = (self.in_channels + 15) // 16 * 16
        who = "%s(%d, %d, kernel_size=%s)" % (type(self).__name__, self.in_channels, int(O), self.kernel_size)
        check_scale("activation", act_scale, who)
        check_scale("weight", w_scale, who)
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
        w = weight.detach().float().to(dev).contiguous()
        # geometry of a 1-pixel image: the packer only reads O, C, kh, kw, groups and Cpad
        g = self._geometry(1, (kh - 1) * self.dilation[0] + 1, (kw - 1) * self.dilation[1] + 1, stride=(1, 1), padding=(0, 0))
        lib = _lib.load()
        _lib.check(lib.dfq_i8_pack_weights(_ptr(w), _ptr(self.w_scale), _ptr(self.weight_codes), _lib.table_ptr(g),
                                           _lib.stream_ptr()), "dfq_i8_pack_weights")

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

    def chained(self, codes_in=False, requant=None, epilogue=None, name=None, out_slice=None):
        """A new module of the same class on the same packed buffers (weight_codes, dq, bias, w_scale), in the given execution
        mode: codes_in - take int8 NHWC codes; requant = (out_scale, lo, hi) - return the next layer's codes; epilogue - an
        Epilogue: the residual epilogue (not together with requant); out_slice = (coff, cstride), with requant - write the
        codes into channels [coff, coff + round_up(C_out, 16)) of an int8 NHWC tensor [N, OH, OW, cstride] (a channel
        concatenation, dfq_i8_conv_slice), given as forward(x, out=...) or made when out is None.  name: the layer's name
        in error messages.  self is not modified."""
        new = type(self).__new__(type(self))
        nn.Module.__init__(new)
        for k in ("out_channels", "in_channels", "groups", "kernel_size", "stride", "padding", "dilation", "cpad", "act_scale"):
            setattr(new, k, getattr(self, k))
        for k, b in self._buffers.items():
            new.register_buffer(k, b)
        new.codes_in = bool(codes_in)
        new.layer_name = name
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
            coff, cstride = (int(v) for v in out_slice)
            if requant is None:
                raise _lib.DfqError("layer %s: a channel slice needs requant" % new._who())
            if coff < 0 or coff % 16 or cstride % 16 or coff + (self.out_channels + 15) // 16 * 16 > cstride:
                raise _lib.DfqError("layer %s: channel slice (%d, %d) is not 16-aligned inside its tensor"
                                    % (new._who(), coff, cstride))
            out_slice = (coff, cstride)
        new.out_slice = out_slice
        return new

    def _who(self):
        return self.layer_name or "%s(%d, %d, kernel_size=%s)" % (type(self).__name__, self.in_channels, self.out_channels,
                                                                  self.kernel_size)

    def run(self, x, with_acc=False, residual=None, out=None):
        """(y, acc | None) for x [N, C, H, W] fp32 on the GPU; acc = the int32 sums before the epilogue.  In the chained modes
        x is int8 codes [N, H, W, cpad] (codes_in) and y int8 codes [N, OH, OW, round_up(C_out, 16)] (requant).  With an
        epilogue, y is the codes, the fp32 output, or (codes, fp32 output) when it returns both, and `residual` is the fp32
        tensor [N, C_out, OH, OW] the epilogue adds (exactly that shape, no broadcasting, on x's device).  With out_slice, y
        is `out` (int8 [N, OH, OW, cstride] on x's device) or a new such tensor, its slice written."""
        if not x.is_cuda or not self.dq.is_cuda:
            raise _lib.DfqError("int8 layers run on the GPU only (no CPU fallback): input on %s, layer on %s"
                                % (x.device, self.dq.device))
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
        if (residual is not None) != bool(self.epilogue and self.epilogue.residual):
            raise _lib.DfqError("layer %s: %s" % (self._who(), "takes a residual input" if residual is None else
                                                    "takes no residual input"))
        x = x.contiguous()
        g = self._geometry(N, H, W)
        OH, OW = int(g[0]["OH"]), int(g[0]["OW"])
        if OH <= 0 or OW <= 0:
            raise _lib.DfqError("int8 layer: input %dx%d is smaller than the kernel" % (H, W))
        lib, st = _lib.load(), _lib.stream_ptr()
        if self.codes_in:
            xq = x
        else:
            xq = torch.empty(N * H * W * self.cpad, dtype=torch.int8, device=x.device)
            _lib.check(lib.dfq_i8_quantize_nhwc(_ptr(x), _ptr(xq), N, self.in_channels, H, W, self.cpad,
                                                C.c_float(self.act_scale), st), "dfq_i8_quantize_nhwc")
        if self.epilogue is not None:
            return self._run_fused(xq, residual, g, N, OH, OW), None
        if out is not None and self.out_slice is None:
            raise _lib.DfqError("layer %s: takes no output tensor" % self._who())
        if self.out_slice is not None:
            return self._run_slice(xq, out, g, N, OH, OW), None
        if self.requant is not None:
            s, lo, hi = self.requant
            yq = torch.empty((N, OH, OW, (self.out_channels + 15) // 16 * 16), dtype=torch.int8, device=x.device)
            _lib.check(lib.dfq_i8_conv_requant(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias), _ptr(yq),
                                               C.c_float(s), C.c_float(lo), C.c_float(hi), _lib.table_ptr(g), st),
                       "dfq_i8_conv_requant")
            return yq, None
        y = torch.empty((N, self.out_channels, OH, OW), dtype=torch.float32, device=x.device)
        acc = torch.empty(y.shape, dtype=torch.int32, device=x.device) if with_acc else None
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
        _lib.check(_lib.load().dfq_i8_conv_slice(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias),
                                                 _lib.table_ptr(d), coff, cstride, _lib.table_ptr(g), _lib.stream_ptr()),
                   "dfq_i8_conv_slice (layer %s)" % self._who())
        return out

    def _run_fused(self, xq, r, g, N, OH, OW):
        e = self.epilogue
        shape = (N, self.out_channels, OH, OW)
        if r is not None:
            if not isinstance(r, torch.Tensor) or r.dtype != torch.float32 or not r.is_cuda or tuple(r.shape) != shape or \
                    r.device != xq.device:
                raise _lib.DfqError("layer %s: the residual must be fp32 %s on %s, got %s" % (
                    self._who(), list(shape), xq.device, "%s %s on %s" % (r.dtype, list(r.shape), r.device)
                    if isinstance(r, torch.Tensor) else type(r).__name__))
            r = r.contiguous()
        yq = None if e.out_scale is None else \
            torch.empty((N, OH, OW, (self.out_channels + 15) // 16 * 16), dtype=torch.int8, device=xq.device)
        y = torch.empty(shape, dtype=torch.float32, device=xq.device) if e.fp32 else None
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0 if r is None else r.data_ptr(), 0 if y is None else y.data_ptr(), 0 if yq is None else yq.data_ptr(),
                0.0 if e.out_scale is None else e.out_scale) + e.pre + e.post
        lib = _lib.load()
        _lib.check(lib.dfq_i8_conv_fused(_ptr(xq), _ptr(self.weight_codes), _ptr(self.dq), _ptr(self.bias),
                                         _lib.table_ptr(d), _lib.table_ptr(g), _lib.stream_ptr()),
                   "dfq_i8_conv_fused (layer %s)" % self._who())
        return (yq, y) if yq is not None and y is not None else (y if yq is None else yq)


class Int8Conv2d(_Int8Layer):
    """nn.Conv2d executed in int8 (zero padding; groups == 1 or depthwise)."""

    @classmethod
    def from_conv(cls, conv: nn.Conv2d, act_scale, w_scale):
        if isinstance(conv.padding, str) or conv.padding_mode != "zeros":
            raise _lib.DfqError("int8 execution supports numeric zero padding only (padding=%r, padding_mode=%r)"
                                % (conv.padding, conv.padding_mode))
        return cls(conv.weight, conv.bias, act_scale, w_scale, conv.stride, conv.padding, conv.dilation, conv.groups)

    def forward(self, x, r=None, out=None):
        return self.run(x, residual=r, out=out)[0]

    def extra_repr(self):
        return "%d, %d, kernel_size=%s, stride=%s, padding=%s, dilation=%s, groups=%d, act_scale=%g" % (
            self.in_channels, self.out_channels, self.kernel_size, self.stride, self.padding, self.dilation, self.groups,
            self.act_scale)


class Int8Linear(_Int8Layer):
    """nn.Linear executed in int8: the 1x1 convolution of [B, I, 1, 1]."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, act_scale, w_scale):
        return cls(lin.weight.reshape(lin.out_features, lin.in_features, 1, 1), lin.bias, act_scale, w_scale)

    def forward(self, x):
        lead = x.shape[:-1]
        y, _ = self.run(x.reshape(-1, self.in_channels, 1, 1))
        return y.reshape(*lead, self.out_channels)

    def extra_repr(self):
        return "in_features=%d, out_features=%d, act_scale=%g" % (self.in_channels, self.out_channels, self.act_scale)


def _pool_extent(n, k, p, s, d, ceil_mode):
    """torch's pooling output size (floor division; in ceil mode the last window starts inside the input or its left pad)."""
    o = (n + 2 * p - d * (k - 1) - 1 + (s - 1 if ceil_mode else 0)) // s + 1
    return o - 1 if ceil_mode and (o - 1) * s >= n + p else o


class Int8MaxPool2d(nn.Module):
    """F.max_pool2d of a chained model (dfq_i8_maxpool).  codes_in: int8 NHWC codes [N, H, W, round_up(channels, 16)] in,
    the pooled codes out (the max of codes is the code of the max, q being monotone).  Otherwise fp32 NCHW in, bit for bit
    torch's max_pool2d out (`fp32`) and / or its codes at out_scale: (codes, fp32) when both."""

    def __init__(self, kernel_size, stride, padding, dilation, ceil_mode, channels, codes_in, out_scale=None, fp32=False,
                 name=None):
        super().__init__()
        self.kernel_size, self.padding, self.dilation = _pair(kernel_size), _pair(padding), _pair(dilation)
        self.stride = self.kernel_size if stride is None or stride == [] or stride == () else _pair(stride)
        self.ceil_mode, self.channels, self.codes_in = bool(ceil_mode), int(channels), bool(codes_in)
        self.cpad = (self.channels + 15) // 16 * 16
        self.out_scale = None if out_scale is None else float(_f32(out_scale))
        self.fp32, self.layer_name = bool(fp32), name
        if self.out_scale is not None:
            check_scale("output", self.out_scale, "max pool %s" % name)
        if not codes_in and self.out_scale is None and not self.fp32:
            raise _lib.DfqError("max pool %s returns neither codes nor fp32" % name)

    def forward(self, x):
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
        _lib.check(_lib.load().dfq_i8_maxpool(_ptr(x) if self.codes_in else None, None if self.codes_in else _ptr(x), _ptr(y),
                                              _ptr(yq), C.c_float(self.out_scale or 0.0), _lib.table_ptr(g),
                                              _lib.stream_ptr()), "dfq_i8_maxpool (%s)" % self.layer_name)
        return (yq, y) if yq is not None and y is not None else (y if yq is None else yq)

    def extra_repr(self):
        return "kernel_size=%s, stride=%s, padding=%s, dilation=%s, ceil_mode=%s, channels=%d, %s" % (
            self.kernel_size, self.stride, self.padding, self.dilation, self.ceil_mode, self.channels,
            "codes" if self.codes_in else "fp32 in, out_scale=%s, fp32=%s" % (self.out_scale, self.fp32))


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
                layer.padding_mode == "zeros" and not isinstance(layer.padding, str)
        else:
            ok = isinstance(layer, nn.Linear)
        if not ok:
            raise _lib.DfqError("layer %s (%s, groups=%s) cannot run in int8: needs a Linear, or a zero-padded Conv2d with "
                                "groups == 1 or depthwise" % (name, type(layer).__name__, getattr(layer, "groups", "-")))
        plan.append((name, layer, a, w_scale))
    done = []
    for name, layer, a, w_scale in plan:
        new = (Int8Conv2d.from_conv if isinstance(layer, nn.Conv2d) else Int8Linear.from_linear)(layer, a, w_scale)
        parent_name, _, attr = name.rpartition(".")
        setattr(model.get_submodule(parent_name) if parent_name else model, attr, new)
        done.append(name)
    return done


# ---- chaining converted convolutions through int8 codes ---------------------------------------------------------------
_INF = float("inf")


class _Int8Tracer(fx.Tracer):
    """symbolic tracing that keeps the int8 layers (whose forward calls the library) as leaves"""

    def is_leaf_module(self, m, qualname):
        return isinstance(m, _Int8Layer) or super().is_leaf_module(m, qualname)


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
        if type(m) is nn.Identity:
            return (-_INF, _INF)
        if type(m) is nn.Dropout and not m.training:
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


def _cat_operands(node):
    """The operands of torch.cat / torch.concat along the channels (dim 1 or -3) of >= 2 distinct fx nodes, without out;
    None otherwise."""
    if node.op != "call_function" or node.target not in (torch.cat, torch.concat) or set(node.kwargs) - {"tensors", "dim"}:
        return None
    ops, dim = _arg(node, 0, "tensors", None), _arg(node, 1, "dim", 0)
    if dim not in (1, -3) or not isinstance(ops, (list, tuple)) or len(ops) < 2 or \
            not all(isinstance(o, fx.Node) for o in ops) or len(set(ops)) != len(ops):
        return None
    return list(ops)


def chain_int8(model: nn.Module, concrete_args=None, residual=False, pool_cat=False) -> fx.GraphModule:
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
    outputs it writes), in graph order.  pool_cat=True without residual=True raises DfqError."""
    tracer = _Int8Tracer()
    graph = tracer.trace(model, concrete_args)
    gm = fx.GraphModule(tracer.root, graph, type(model).__name__ + "Int8Chained")
    mods = dict(gm.named_modules())
    sites = {}
    for node in gm.graph.nodes:
        if node.op == "call_module":
            sites[node.target] = sites.get(node.target, 0) + 1

    def conv(node):
        return node.op == "call_module" and isinstance(mods[node.target], Int8Conv2d) and sites[node.target] == 1

    if pool_cat and not residual:
        raise _lib.DfqError("chain_int8: pool_cat=True builds on residual=True")
    if residual:
        return _chain_residual(gm, mods, conv, pool_cat)

    edges, between = [], []
    for q in list(gm.graph.nodes):
        if not conv(q) or len(q.args) != 1 or q.kwargs or not isinstance(q.args[0], fx.Node):
            continue
        node, clamp, path = q.args[0], (-_INF, _INF), []
        while len(node.users) == 1:
            if conv(node):
                break
            c = _pass_through(node, mods)
            if c is None or len(node.all_input_nodes) != 1 or not isinstance(node.args[0], fx.Node):
                break
            clamp = _compose(c, clamp)                          # walking backwards: this clamp runs first
            path.append(node)
            node = node.args[0]
        if len(node.users) != 1 or not conv(node) or mods[node.target].out_channels != mods[q.target].in_channels:
            continue
        edges.append((node.target, q.target, clamp))
        between.append((node, q, path))
    producers = {p: c for p, _, c in edges}
    consumers = {q for _, q, _ in edges}
    for target in producers.keys() | consumers:
        requant = None
        if target in producers:
            nxt = mods[next(q for p, q, _ in edges if p == target)]
            requant = (nxt.act_scale,) + tuple(producers[target])
        parent, _, attr = target.rpartition(".")
        setattr(gm.get_submodule(parent) if parent else gm, attr,
                mods[target].chained(codes_in=target in consumers, requant=requant))
    for p, q, path in between:
        q.args = (p,)
        for node in path:                                       # from the consumer side back: each has no user left
            gm.graph.erase_node(node)
    gm.graph.lint()
    gm.recompile()
    gm.requantized_edges = edges
    return gm


def _chain_residual(gm, mods, conv, pool_cat=False):
    """chain_int8(..., residual=True[, pool_cat=True]) on the traced `gm` (see chain_int8)."""
    full = (-_INF, _INF)
    order = {n: i for i, n in enumerate(gm.graph.nodes)}

    def producer(node):
        return conv(node) and len(node.args) == 1 and not node.kwargs and isinstance(node.args[0], fx.Node)

    def forward(node, clamp):
        """Walk from node through single-user pass-throughs: (last node, composed clamp, the pass-throughs)."""
        path = []
        while len(node.users) == 1:
            u = next(iter(node.users))
            c = _pass_through(u, mods)
            if c is None or len(u.all_input_nodes) != 1 or u.args[0] is not node:
                break
            clamp, node = _compose(clamp, c), u
            path.append(u)
        return node, clamp, path

    def back_to_producer(node):
        """The producer whose single-user pass-through chain ends at `node`, or None."""
        while len(node.users) == 1 and not producer(node):
            if _pass_through(node, mods) is None or len(node.all_input_nodes) != 1 or not isinstance(node.args[0], fx.Node):
                return None
            node = node.args[0]
        return node if len(node.users) == 1 and producer(node) else None

    def same(a, b):
        return a.view(np.int32) == b.view(np.int32)

    def after_pool(node):
        """Walk from a pool through single-user exact identities: (last node, the identities)."""
        path = []
        while len(node.users) == 1:
            u = next(iter(node.users))
            if not _is_identity(u, mods) or len(u.all_input_nodes) != 1 or u.args[0] is not node:
                break
            node = u
            path.append(u)
        return node, path

    pool_memo = {}

    def pool_scale(pool, channels):
        """The scale at which every user of a pool (past exact identities) takes codes, or None."""
        if pool not in pool_memo:
            pool_memo[pool] = None
            tail, _ = after_pool(pool)
            scales = [user_scale(u, tail, channels) for u in tail.users]
            if scales and all(s is not None and same(s, scales[0]) for s in scales):
                pool_memo[pool] = scales[0]
        return pool_memo[pool]

    def user_scale(u, tail, channels, pools=True):
        """The scale at which u takes the codes of `tail` (channels wide), or None when it takes fp32."""
        if producer(u) and u.args[0] is tail and mods[u.target].in_channels == channels:
            return _f32(mods[u.target].act_scale)
        if pools and pool_cat and _max_pool(u, mods) is not None and u.args[0] is tail:
            return pool_scale(u, channels)
        return None

    def take_codes(tail, channels, pools=True):
        """The fan-out rule: the users of tail that take codes at the first such user's scale (graph order), and it."""
        codes, scale = [], None
        for u in sorted(tail.users, key=order.get):
            s = user_scale(u, tail, channels, pools)
            if s is not None and (scale is None or same(s, scale)):
                scale = s
                codes.append(u)
        return codes, scale

    pool_plans = []

    def codes_pool(u, channels, clamp):
        tail, ids = after_pool(u)
        pool_plans.append(dict(node=u, mode="codes", tail=tail, path=ids, codes=sorted(tail.users, key=order.get),
                               scale=pool_scale(u, channels), clamp=clamp, channels=channels))
        for v in tail.users:
            if not producer(v):
                codes_pool(v, channels, clamp)

    plans = []
    for p in list(gm.graph.nodes):
        if not producer(p):
            continue
        end, pre, path = forward(p, full)
        add, ri, post, post_path, tail = None, None, full, [], end
        if len(end.users) == 1:
            a = next(iter(end.users))
            if _is_add(a):
                fused = next((i for i, v in enumerate(a.args) if back_to_producer(v) is not None), None)
                if fused is not None and a.args[fused] is end:
                    add, ri = a, 1 - fused
                    tail, post, post_path = forward(a, full)
        out_c = mods[p.target].out_channels
        codes, scale = take_codes(tail, out_c)
        clamp = post if add is not None else pre
        if add is None and not codes and pool_cat and len(tail.users) == 1:
            u = next(iter(tail.users))                          # fp32-mode pool: a user of the pool needs fp32
            if _max_pool(u, mods) is not None and u.args[0] is tail:
                pc, ps = take_codes(u, out_c, pools=False)
                if pc:
                    pool_plans.append(dict(node=u, mode="fp32", codes=pc, scale=ps, clamp=clamp, channels=out_c))
                    plans.append(dict(p=p, path=path, pre=pre, add=None, ri=None, post=full, post_path=[], tail=tail,
                                      codes=[], scale=None))
            continue
        if add is None and not codes:
            continue
        plans.append(dict(p=p, path=path, pre=pre, add=add, ri=ri, post=post, post_path=post_path, tail=tail, codes=codes,
                          scale=scale))
        for u in codes:
            if not producer(u):
                codes_pool(u, out_c, clamp)

    # concatenations whose operands come from their own producers and whose users all take codes at one scale
    cat_plans = []
    for c in (list(gm.graph.nodes) if pool_cat else []):
        ops = _cat_operands(c)
        if ops is None:
            continue
        prods = [back_to_producer(o) for o in ops]
        if any(q is None for q in prods) or len(set(prods)) != len(prods):
            continue
        chans = [mods[q.target].out_channels for q in prods]
        if any(k % 16 for k in chans[:-1]):
            continue
        tail, tclamp, tpath = forward(c, full)
        codes, scale = take_codes(tail, sum(chans))
        if not codes or len(codes) != len(tail.users):
            continue
        operands = []
        for o, q, off in zip(ops, prods, np.cumsum([0] + chans[:-1]).tolist()):
            node, clamp, opath = o, full, []
            while node is not q:
                clamp = _compose(_pass_through(node, mods), clamp)
                opath.append(node)
                node = node.args[0]
            operands.append(dict(p=q, path=opath, clamp=_compose(clamp, tclamp), coff=off))
        cat_plans.append(dict(cat=c, operands=operands, tail=tail, path=tpath, codes=codes, scale=scale, clamp=tclamp,
                              cstride=(sum(chans) + 15) // 16 * 16))
        for u in codes:
            if not producer(u):
                codes_pool(u, sum(chans), tclamp)

    # the residual's exact identities, skipped once every plan's own nodes are known: a node another plan deletes (an
    # identity at the end of its post-add chain, say) stays the residual, and that plan replaces it by its fp32 output
    claimed = {n for pl in plans for n in (pl["p"], *pl["path"], *([pl["add"]] if pl["add"] is not None else []),
                                            *pl["post_path"])}
    claimed |= {n for cp in cat_plans for n in (cp["cat"], *cp["path"], *(n for o in cp["operands"] for n in (o["p"], *o["path"])))}
    claimed |= {n for pp in pool_plans for n in (pp["node"], *pp.get("path", []))}
    for pl in plans:
        pl["skipped"] = []
        if pl["add"] is None:
            continue
        r = pl["add"].args[pl["ri"]]
        while r not in claimed and len(r.users) == 1 and _is_identity(r, mods) and isinstance(r.args[0], fx.Node):
            pl["skipped"].append(r)
            r = r.args[0]
        pl["r_name"] = r.name

    # rewrite in producer order: a producer's input may be the codes of an earlier one, and a residual its fp32 output
    g = gm.graph
    convs = {n for n in g.nodes if producer(n)}                 # before the rewrites give producers a second input
    edges, adds, modes = [], [], {}
    for pl in plans:
        p, add, tail = pl["p"], pl["add"], pl["tail"]
        if add is not None:
            for node in pl["skipped"]:                          # from the add back: each loses its only user
                node.replace_all_uses_with(node.args[0])
                g.erase_node(node)
            add.prepend(p)
            p.args = (p.args[0], add.args[pl["ri"]])
        fp32 = any(u not in pl["codes"] for u in tail.users)
        scale = float(pl["scale"]) if pl["codes"] else None
        clamp = pl["post"] if add is not None else pl["pre"]
        if add is None and not fp32:
            modes[p.target] = ("requant", (scale,) + tuple(clamp))
            codes_node = y_node = p
        else:
            modes[p.target] = ("epilogue", Epilogue(scale, pl["pre"], pl["post"], add is not None, fp32))
            codes_node = y_node = p
            if scale is not None and fp32:
                with g.inserting_after(p):
                    y_node = g.call_function(operator.getitem, (p, 1))
                with g.inserting_after(p):
                    codes_node = g.call_function(operator.getitem, (p, 0))
        for u in pl["codes"]:
            u.replace_input_with(tail, codes_node)
            if u in convs:
                edges.append((p.target, u.target, clamp))
        if tail is not p:
            tail.replace_all_uses_with(y_node)
            for node in reversed([*pl["path"], *([add] if add is not None else []), *pl["post_path"]]):
                g.erase_node(node)
        else:
            p.replace_all_uses_with(y_node, delete_user_cb=lambda u: u not in (y_node, codes_node))
        if add is not None:
            adds.append((p.target, add.name, pl["r_name"], pl["pre"], pl["post"]))

    # concatenations: the producers write their slices of one buffer in graph order, threaded through `out`
    cats = []
    for cp in cat_plans:
        cstride, prev = cp["cstride"], None
        for o in sorted(cp["operands"], key=lambda o: order[o["p"]]):
            q = o["p"]
            modes[q.target] = ("slice", ((float(cp["scale"]),) + tuple(o["clamp"]), (o["coff"], cstride)))
            if prev is not None:
                q.kwargs = {"out": prev}
            prev = q
        for u in cp["codes"]:
            u.replace_input_with(cp["tail"], prev)
            if u in convs:
                edges.append((cp["cat"].name, u.target, cp["clamp"]))
        for node in reversed(cp["path"]):
            g.erase_node(node)
        g.erase_node(cp["cat"])
        for o in cp["operands"]:
            for node in o["path"]:                              # from the cat back to the producer
                g.erase_node(node)
        cats.append((cp["cat"].name, [o["p"].target for o in cp["operands"]], [o["coff"] for o in cp["operands"]]))

    # pools, last: each reads its input as the rewrites above left it
    pools = []
    for pp in sorted(pool_plans, key=lambda pp: order[pp["node"]]):
        u = pp["node"]
        k, s, pad, dil, ceil = _max_pool(u, mods)
        codes_mode = pp["mode"] == "codes"
        fp32 = not codes_mode
        mod = Int8MaxPool2d(k, s, pad, dil, ceil, pp["channels"], codes_mode, None if codes_mode else float(pp["scale"]),
                            fp32, name=u.name)
        name = "int8_pool_" + u.name
        gm.add_submodule(name, mod)
        inp = u.args[0]
        u.op, u.target, u.args, u.kwargs = "call_module", name, (inp,), {}
        if codes_mode:
            for v in pp["codes"]:
                v.replace_input_with(pp["tail"], u)
            for node in reversed(pp["path"]):
                g.erase_node(node)
        else:
            with g.inserting_after(u):
                y_node = g.call_function(operator.getitem, (u, 1))
            with g.inserting_after(u):
                codes_node = g.call_function(operator.getitem, (u, 0))
            for v in pp["codes"]:
                v.replace_input_with(u, codes_node)
            u.replace_all_uses_with(y_node, delete_user_cb=lambda x: x not in (y_node, codes_node))
        for v in pp["codes"]:
            if v in convs:
                edges.append((u.name, v.target, pp["clamp"]))
        pools.append((u.name, pp["mode"], ("codes",) if codes_mode else ("fp32", "codes")))

    consumers = {q for _, q, _ in edges}
    for target in modes.keys() | consumers:
        kind, arg = modes.get(target, (None, None))
        parent, _, attr = target.rpartition(".")
        setattr(gm.get_submodule(parent) if parent else gm, attr,
                mods[target].chained(codes_in=target in consumers, name=target,
                                     requant=arg if kind == "requant" else (arg[0] if kind == "slice" else None),
                                     epilogue=arg if kind == "epilogue" else None,
                                     out_slice=arg[1] if kind == "slice" else None))
    g.lint()
    gm.recompile()
    gm.requantized_edges = edges
    gm.fused_adds = adds
    if pool_cat:
        gm.fused_cats = cats
        gm.fused_pools = pools
    return gm
