"""Fake-quantization ops and modules: drop-in for the reference's ``utils/quantize.py``.

Same public names, constructor signatures and call semantics (UniformQuantize, quantize, QuantMeasure,
QConv2d, QuantConv2d, QuantNConv2d, QLinear, QuantLinear, QuantNLinear, set_layer_bits); the tensor
arithmetic runs in libdfq_sm90.so:

  utils/quantize.py:23-76    UniformQuantize.forward -> dfq_quant_dequant / dfq_quant_dequant_dev
  utils/quantize.py:102-119  QuantMeasure.forward    -> dfq_observe_quant: statistic + running update + quantization in
                                                       ONE launch, no float() host syncs (eval mode without update_stat:
                                                       dfq_quant_dequant_dev on the device-resident range)
  utils/quantize.py:176-205  per-forward weight / bias quantization of the Q*/Quant* layers -> dfq_observe_quant (own range)

Numerics (SURVEY.md H1).  The reference runs the same Python on CPU tensors (weights during
calibration) and on CUDA tensors (activations, per-forward weights during inference), and PyTorch's two
backends differ in ONE op: ``div_(python_float)`` is a true division on CPU and, on CUDA, a multiply by
``fp32(1.0 / scale)`` - the reciprocal formed in DOUBLE from the Python scalar, then rounded (probed on the GPU).  ``quantize`` follows the device of its input: CPU tensors are staged through the GPU
and computed with true division (bit-identical to the reference's CPU result), CUDA tensors use the
reciprocal form (bit-identical to the reference's CUDA result).  There is no CPU implementation.
"""
import ctypes as C

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import InplaceFunction

from .. import _lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _dev_f32(x):
    """(contiguous fp32 CUDA tensor holding x, came_from_cpu)."""
    _lib.require_cuda()
    if x.dtype != torch.float32:
        raise _lib.DfqError("fake quantization expects float32 tensors, got %s" % x.dtype)
    if x.is_cuda:
        return x.contiguous(), False
    return x.contiguous().cuda(non_blocking=False), True


def _quant_scalars(num_bits, min_value, max_value, symmetric):
    """Python-double prologue of quantize.py:49-66 (explicit float range)."""
    if symmetric:
        qmin = -2. ** (num_bits - 1)
        qmax = 2 ** (num_bits - 1) - 1
        max_value = abs(max_value)
        min_value = abs(min_value)
        if max_value < min_value:
            max_value = min_value
        scale = max_value / qmax
        min_value = 0.
    else:
        qmin = 0.
        qmax = 2. ** num_bits - 1.
        scale = (max_value - min_value) / (qmax - qmin)
    scale = max(scale, 1e-8)
    return float(qmin), float(qmax), float(min_value), float(scale)


def fake_quant_explicit(x, num_bits, min_value, max_value, symmetric=False, out=None, div_mode=None):
    """x -> Q(x) for Python-float min/max.  ``div_mode``: 0 true division, 1 reciprocal multiply,
    None = by the device of ``x`` (CPU: 0, CUDA: 1).  Returns a tensor on x's device."""
    lib = _lib.load()
    xd, from_cpu = _dev_f32(x)
    if div_mode is None:
        div_mode = 0 if from_cpu else 1
    qmin, qmax, mn, scale = _quant_scalars(num_bits, float(min_value), float(max_value), symmetric)
    if out is not None and out.is_cuda and out.is_contiguous():
        yd = out
    else:
        yd = torch.empty_like(xd)
    if xd.numel():
        with _lib.launch(xd) as st:
            _lib.check(lib.dfq_quant_dequant(_ptr(xd), _ptr(yd), xd.numel(), C.c_float(mn), C.c_double(scale),
                                             C.c_float(qmin), C.c_float(qmax), int(div_mode), None, st),
                       "dfq_quant_dequant")
    if out is not None and yd is not out:
        out.copy_(yd.view(out.shape))
        return out
    return yd.view(x.shape).cpu() if from_cpu and out is None else yd.view(x.shape)


def fake_quant_device_range(x, num_bits, min_t, max_t, symmetric=False, prologue=0, out=None, div_mode=None):
    """x -> Q(x) with the range read from device tensors (1 element each); nothing syncs with the host."""
    lib = _lib.load()
    xd, from_cpu = _dev_f32(x)
    if div_mode is None:
        div_mode = 0 if from_cpu else 1
    mn = min_t.detach().reshape(-1)[:1].to(device=xd.device, dtype=torch.float32).contiguous()
    mx = max_t.detach().reshape(-1)[:1].to(device=xd.device, dtype=torch.float32).contiguous()
    yd = out if (out is not None and out.is_cuda and out.is_contiguous()) else torch.empty_like(xd)
    if xd.numel():
        with _lib.launch(xd) as st:
            _lib.check(lib.dfq_quant_dequant_dev(_ptr(xd), _ptr(yd), xd.numel(), _ptr(mn), _ptr(mx), int(num_bits),
                                                 1 if symmetric else 0, int(div_mode), int(prologue), None,
                                                 st), "dfq_quant_dequant_dev")
    if out is not None and yd is not out:
        out.copy_(yd.view(out.shape))
        return out
    return yd.view(x.shape).cpu() if from_cpu and out is None else yd.view(x.shape)


def tensor_minmax(x):
    """Device tensor [2] = (min(x), max(x)); stays on the GPU."""
    lib = _lib.load()
    xd, _ = _dev_f32(x.detach())
    out = xd.new_empty((2,))
    with _lib.launch(xd) as st:
        _lib.check(lib.dfq_minmax(_ptr(xd), xd.numel(), _ptr(out), st), "dfq_minmax")
    return out


def _per_sample(numel, batch):
    """Elements per sample of a tensor viewed as [batch, -1]; refuses a batch that does not divide it, as the reference's
    ``view(B // num_chunks, -1)`` does (quantize.py:26)."""
    if numel % batch:
        raise _lib.DfqError("cannot view a tensor of %d elements as [%d, -1]" % (numel, batch))
    return numel // batch


def _running_buffer(t, device, name):
    """(fp32 contiguous 1-element tensor the kernel may update, the caller's tensor to copy the result back into or None)."""
    if t.device != device:
        raise _lib.DfqError("%s is on %s, the input on %s" % (name, t.device, device))
    if t.numel() != 1:
        raise _lib.DfqError("%s must hold one element, got %d" % (name, t.numel()))
    if t.dtype == torch.float32 and t.is_contiguous():
        return t, None
    return t.detach().reshape(1).to(torch.float32).contiguous(), t


def per_sample_minmax_mean(x, batch=None):
    """Device tensor [2] = (mean_b min(x[b]), mean_b max(x[b])) for x viewed as [batch, -1]
    (quantize.py:106-107,110-111)."""
    lib = _lib.load()
    xd, _ = _dev_f32(x.detach())
    if batch is None:
        batch = xd.shape[0]
    per = _per_sample(xd.numel(), batch)
    out = xd.new_empty((2,))
    scratch = xd.new_empty((2 * batch,))
    with _lib.launch(xd) as st:
        _lib.check(lib.dfq_act_minmax_per_sample(_ptr(xd), batch, per, _ptr(out), _ptr(scratch), st),
                   "dfq_act_minmax_per_sample")
    return out


OBS_UPDATE, OBS_EMA, OBS_OWN = 1, 2, 4      # include/dfq_b200.h DFQ_OBS_*


def observe_and_quant(x, num_bits, flags, running_min=None, running_max=None, momentum=0.1, batch=None, symmetric=False,
                      prologue=0, out=None, div_mode=None):
    """ONE launch: per-sample min/max -> batch mean -> running-statistics update -> fake quantization (dfq_observe_quant).
    Returns Q(x) on x's device; the running buffers (device tensors) are updated in place on the GPU, nothing syncs."""
    lib = _lib.load()
    xd, from_cpu = _dev_f32(x)
    if div_mode is None:
        div_mode = 0 if from_cpu else 1
    if batch is None:
        batch = xd.shape[0] if xd.dim() > 0 else 1
    batch = max(1, int(batch))
    per = _per_sample(xd.numel(), batch)
    rmin, rmin_back = _running_buffer(running_min, xd.device, "running_min") if running_min is not None else (None, None)
    rmax, rmax_back = _running_buffer(running_max, xd.device, "running_max") if running_max is not None else (None, None)
    yd = out if (out is not None and out.is_cuda and out.is_contiguous()) else torch.empty_like(xd)
    if xd.numel():
        with _lib.launch(xd) as st:
            _lib.check(lib.dfq_observe_quant(_ptr(xd), _ptr(yd), batch, per,
                                             _ptr(rmin) if rmin is not None else None,
                                             _ptr(rmax) if rmax is not None else None, None, int(flags),
                                             C.c_double(momentum), int(num_bits), 1 if symmetric else 0, int(div_mode), int(prologue),
                                             st), "dfq_observe_quant")
    for back, buf in ((rmin_back, rmin), (rmax_back, rmax)):
        if back is not None:
            back.copy_(buf.view(back.shape))
    if out is not None and yd is not out:
        out.copy_(yd.view(out.shape))
        return out
    return yd.view(x.shape).cpu() if from_cpu and out is None else yd.view(x.shape)


class UniformQuantize(InplaceFunction):
    """Uniform fake quantization with a straight-through gradient (quantize.py:14-83)."""

    @staticmethod
    def forward(ctx, input, num_bits=8, min_value=None, max_value=None, inplace=False, symmetric=False, num_chunks=None):
        num_chunks = input.shape[0] if num_chunks is None else num_chunks
        ctx.inplace = inplace
        ctx.num_bits = num_bits
        ctx.min_value = min_value
        ctx.max_value = max_value
        if ctx.inplace:
            ctx.mark_dirty(input)
        out = input if inplace else None
        if min_value is None and max_value is None:
            # quantize.py:24-35: y = input.view(B // num_chunks, -1); min = y.min(-1)[0].mean(-1)  (0-d tensors) - statistic
            # and quantization in one launch
            res = observe_and_quant(input, num_bits, OBS_OWN, batch=max(1, input.shape[0] // num_chunks), symmetric=symmetric,
                                    prologue=2 if input.is_cuda else 1, out=out)
        elif min_value is None or max_value is None:
            stat = per_sample_minmax_mean(input, batch=max(1, input.shape[0] // num_chunks))
            mn_t = stat[0:1] if min_value is None else stat.new_full((1,), float(min_value))
            mx_t = stat[1:2] if max_value is None else stat.new_full((1,), float(max_value))
            prologue = 2 if input.is_cuda else 1
            res = fake_quant_device_range(input, num_bits, mn_t, mx_t, symmetric, prologue=prologue, out=out)
        else:
            res = fake_quant_explicit(input, num_bits, float(min_value), float(max_value), symmetric, out=out)
        # in place, autograd wants the very tensor it marked dirty back, not a view of it
        return input if inplace else res

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None, None, None, None, None, None


def quantize(x, num_bits=8, min_value=None, max_value=None, inplace=False, symmetric=False, num_chunks=None):
    return UniformQuantize().apply(x, num_bits, min_value, max_value, inplace, symmetric, num_chunks)


class _QuantByBuffers(InplaceFunction):
    """quantize(x, bits, float(min), float(max)) with min/max left on the device (straight-through)."""

    @staticmethod
    def forward(ctx, input, num_bits, min_t, max_t):
        return fake_quant_device_range(input, num_bits, min_t, max_t, False, prologue=0)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None, None, None


class _ObserveQuant(InplaceFunction):
    """The observer's statistic, running update and fake quantization in one launch (straight-through)."""

    @staticmethod
    def forward(ctx, input, num_bits, flags, rmin, rmax, momentum):
        return observe_and_quant(input, num_bits, flags, rmin, rmax, momentum)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None, None, None, None, None


class _QuantOwnRange(InplaceFunction):
    """quantize(w, bits, float(w.min()), float(w.max())) in one launch (straight-through)."""

    @staticmethod
    def forward(ctx, input, num_bits):
        return observe_and_quant(input, num_bits, OBS_OWN, batch=1, prologue=0)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None


class QuantMeasure(nn.Module):
    """Activation observer + fake quantizer (quantize.py:90-122).

    NOTE the positional order (update_stat first) is part of the reference's behaviour: set_layer_bits
    passes the activation bit width as `update_stat` (quirk Q1, quantize.py:366).
    """

    def __init__(self, update_stat=False, num_bits=8, momentum=0.1):
        super(QuantMeasure, self).__init__()
        self.register_buffer('running_min', torch.zeros(1))
        self.register_buffer('running_max', torch.zeros(1))
        self.momentum = momentum
        self.num_bits = num_bits
        self.update_stat = update_stat

    def _buffers_on(self, device):
        if self.running_min.device != device:
            self.running_min = self.running_min.to(device)
            self.running_max = self.running_max.to(device)
        if not self.running_min.is_contiguous() or self.running_min.dim() == 0:
            self.running_min = self.running_min.reshape(1).contiguous()
            self.running_max = self.running_max.reshape(1).contiguous()

    def forward(self, input):
        lib = _lib.load()
        _lib.require_cuda()
        if not input.is_cuda:
            # the reference's observers run wherever the model is (the tracer's forward inside switch_layers feeds CPU
            # tensors, main_cls.py:77,129); this package computes on the GPU and hands the result back where it came from
            staged, from_cpu = _dev_f32(input)
            if from_cpu and staged.device != input.device:
                return self.forward(staged).to(input.device)
        self._buffers_on(input.device)
        flags = (OBS_UPDATE if self.update_stat else 0) | (OBS_EMA if self.training else 0)
        if flags:
            # statistic -> running update (quantize.py:103-113) -> quantization: one stream-ordered launch, no host sync
            return _ObserveQuant.apply(input, self.num_bits, flags, self.running_min, self.running_max, self.momentum)
        return _QuantByBuffers.apply(input, self.num_bits, self.running_min, self.running_max)

    def set_update_stat(self, update_stat):
        self.update_stat = update_stat


def _quant_param_per_forward(w, num_bits):
    """quantize(w, bits, float(w.min()), float(w.max())) (quantize.py:194-196) without the two syncs."""
    return _QuantOwnRange.apply(w, num_bits)


class QConv2d(nn.Conv2d):
    """Conv2d with input observer, learnable per-channel scales and per-forward weight/bias quantization
    (quantize.py:124-205)."""

    def __init__(self, in_channels, out_channels, kernel_size,
                 stride=1, padding=0, dilation=1, groups=1, bias=True, num_bits=8, num_bits_act=8, num_bits_bias=16, momentum=0.1):
        super(QConv2d, self).__init__(in_channels, out_channels, kernel_size,
                                      stride, padding, dilation, groups, bias)
        self.num_bits = num_bits
        self.num_bits_bias = num_bits_bias
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def set_scale(self, scale=None, scale_prev=None):
        if scale is not None:
            self.register_parameter("scale", nn.Parameter(scale.view(-1, 1, 1, 1)))
        if scale_prev is not None:
            self.scale_prev = scale_prev

    def merge_scale_to_weight(self):
        if getattr(self, 'scale_prev', None) is not None:
            self.weight.data.copy_(self.merge_scale_prev(self.weight.detach(), self.scale_prev))
            self.scale_prev = None
        if getattr(self, 'scale', None) is not None:
            weight, bias = self.merge_scale(self.weight.detach(),
                                            self.bias.detach() if self.bias is not None else self.bias, self.scale)
            self.weight.data.copy_(weight)
            if self.bias is not None:
                self.bias.data.copy_(bias)
            self.scale = None

    def merge_scale_prev(self, weight, scale_prev):
        # quantize.py:158-167: input channels of every group divided by the previous layer's scale
        out = weight.clone()
        rows = weight.shape[0] // self.groups
        cols = weight.shape[1]
        flat = scale_prev[:, 0, 0, 0].view(1, -1, 1, 1)
        for g in range(self.groups):
            out[g * rows:(g + 1) * rows] = weight[g * rows:(g + 1) * rows] / flat[:, g * cols:(g + 1) * cols]
        return out

    def merge_scale(self, weight, bias, scale):
        weight = weight * scale
        if bias is not None:
            bias = bias * scale.view(-1)
        return weight, bias

    def forward(self, input):
        input = self.quant(input)
        sbias = self.bias
        if getattr(self, 'scale_prev', None) is not None:
            sweight = self.merge_scale_prev(self.weight, self.scale_prev)
        else:
            sweight = self.weight
        if getattr(self, 'scale', None) is not None:
            sweight, sbias = self.merge_scale(sweight, sbias, self.scale)
        qweight = _quant_param_per_forward(sweight, self.num_bits)
        qbias = quantize(sbias, num_bits=self.num_bits_bias) if sbias is not None else None
        return F.conv2d(input, qweight, qbias, self.stride, self.padding, self.dilation, self.groups)


class QuantConv2d(nn.Conv2d):
    """Conv2d with input observer and per-forward weight/bias quantization (quantize.py:208-233)."""

    def __init__(self, in_channels, out_channels, kernel_size,
                 stride=1, padding=0, dilation=1, groups=1, bias=True, num_bits=8, num_bits_act=8, num_bits_bias=16, momentum=0.1):
        super(QuantConv2d, self).__init__(in_channels, out_channels, kernel_size,
                                          stride, padding, dilation, groups, bias)
        self.num_bits = num_bits
        self.num_bits_bias = num_bits_bias
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def forward(self, input):
        input = self.quant(input)
        qweight = _quant_param_per_forward(self.weight, self.num_bits)
        qbias = quantize(self.bias, num_bits=self.num_bits_bias) if self.bias is not None else None
        return F.conv2d(input, qweight, qbias, self.stride, self.padding, self.dilation, self.groups)


class QuantNConv2d(nn.Conv2d):
    """Conv2d that only quantizes its input; weights were quantized offline (quantize.py:235-251)."""

    def __init__(self, in_channels, out_channels, kernel_size,
                 stride=1, padding=0, dilation=1, groups=1, bias=True, num_bits=8, num_bits_act=8, momentum=0.1):
        super(QuantNConv2d, self).__init__(in_channels, out_channels, kernel_size,
                                           stride, padding, dilation, groups, bias)
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def forward(self, input):
        input = self.quant(input)
        return F.conv2d(input, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)


class QLinear(nn.Linear):
    """Linear counterpart of QConv2d (quantize.py:253-317)."""

    def __init__(self, in_features, out_features, bias=True, num_bits=8, num_bits_act=8, num_bits_bias=16, momentum=0.1):
        super(QLinear, self).__init__(in_features, out_features, bias)
        self.num_bits = num_bits
        self.num_bits_bias = num_bits_bias
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def set_scale(self, scale=None, scale_prev=None):
        if scale is not None:
            self.register_parameter("scale", nn.Parameter(scale.view(-1, 1)))
        if scale_prev is not None:
            self.scale_prev = scale_prev

    def merge_scale_to_weight(self):
        if getattr(self, 'scale_prev', None) is not None:
            self.weight.data.copy_(self.merge_scale_prev(self.weight.detach(), self.scale_prev))
            self.scale_prev = None
        if getattr(self, 'scale', None) is not None:
            weight, bias = self.merge_scale(self.weight.detach(),
                                            self.bias.detach() if self.bias is not None else self.bias, self.scale)
            self.weight.data.copy_(weight)
            if self.bias is not None:
                self.bias.data.copy_(bias)
            self.scale = None

    def merge_scale_prev(self, weight, scale_prev):
        return weight * scale_prev.view(1, -1)        # quantize.py:283 (a product, unlike the conv)

    def merge_scale(self, weight, bias, scale):
        weight = weight * scale
        if bias is not None:
            bias = bias * scale.view(-1)
        return weight, bias

    def forward(self, input):
        input = self.quant(input)
        sbias = self.bias
        sweight = self.weight
        if getattr(self, 'scale_prev', None) is not None:
            sweight = self.merge_scale_prev(sweight, self.scale_prev)
        if getattr(self, 'scale', None) is not None:
            sweight, sbias = self.merge_scale(sweight, sbias, self.scale)
        qweight = _quant_param_per_forward(sweight, self.num_bits)
        qbias = quantize(sbias, num_bits=self.num_bits_bias) if sbias is not None else None
        return F.linear(input, qweight, qbias)


class QuantLinear(nn.Linear):
    """quantize.py:319-341."""

    def __init__(self, in_features, out_features, bias=True, num_bits=8, num_bits_act=8, num_bits_bias=16, momentum=0.1):
        super(QuantLinear, self).__init__(in_features, out_features, bias)
        self.num_bits = num_bits
        self.num_bits_bias = num_bits_bias
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def forward(self, input):
        input = self.quant(input)
        qweight = _quant_param_per_forward(self.weight, self.num_bits)
        qbias = quantize(self.bias, num_bits=self.num_bits_bias) if self.bias is not None else None
        return F.linear(input, qweight, qbias)


class QuantNLinear(nn.Linear):
    """quantize.py:343-356."""

    def __init__(self, in_features, out_features, bias=True, num_bits=8, num_bits_act=8, momentum=0.1):
        super(QuantNLinear, self).__init__(in_features, out_features, bias)
        self.quant = QuantMeasure(num_bits=num_bits_act, momentum=momentum)

    def forward(self, input):
        input = self.quant(input)
        return F.linear(input, self.weight, self.bias)


def set_layer_bits(graph, bits_weight=8, bits_activation=8, bits_bias=16, targ_type=None):
    print("Setting num_bits for targ layers...")
    assert targ_type != None, "targ_type cannot be None"
    for idx in graph:
        layer = graph[idx]
        if type(layer) not in targ_type:
            continue
        if hasattr(layer, 'quant'):
            # quirk Q1 (quantize.py:366): the bit width lands in `update_stat`; activation bits stay 8
            layer.quant = QuantMeasure(bits_activation)
        if hasattr(layer, 'num_bits'):
            layer.num_bits = bits_weight
        if hasattr(layer, 'num_bits_bias'):
            layer.num_bits_bias = bits_bias
