"""ncnn int8 model files (.param + .bin), read into a GraphModule on this package's int8 kernels and written from a
calibrated model, without ONNX or the ncnn tools.

    load(param_path, bin_path)      -> fx.GraphModule: the per-layer model, fp32 between layers as ncnn's int8 runtime keeps
                                       it (Convolution int8 -> dequantize; ReLU, BinaryOp and Softmax in fp32); it chains
                                       (int8.chain_int8) and saves (int8.save) like a traced model
    write(model, graph, targ, ...)  -> the .param, the int8 .bin and optionally the .table of a model int8.convert_to_int8
                                       returned, as convert_ncnn.py --quantize writes them

The .param text format: the magic 7767517, the layer and blob counts, then one line per layer - type, name, bottom and top
counts, bottom and top names, `key=value` pairs; an array value is `-233xx=count,v0,...` and stands for key xx.  The .bin
record of a weighted layer (Convolution, ConvolutionDepthWise, InnerProduct) is
    tag 0x000D4B38 | int8 codes [O][I/g][kh][kw], padded to 4 bytes | fp32 bias [O] when the bias key is set |
    fp32 weight scales [O] (ConvolutionDepthWise: [groups]) | one fp32 input scale
with the code count in key 6 (InnerProduct: 2) and int8_scale_term (key 8) 1 or 2 (ConvolutionDepthWise: 1).  Nothing else is read: any other layer
type, key or value is refused by name before anything is allocated.
"""
import collections
import ctypes as C
import operator
import re
import struct

import numpy as np
import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, engine, export
from . import int8 as I

MAGIC = 7767517
TAG = 0x000D4B38
WEIGHTED = ("Convolution", "ConvolutionDepthWise", "InnerProduct")

# The keys each layer type takes (ncnn's numbering) and their defaults.  Convolution: 0 num_output, 1 kernel_w, 11 kernel_h,
# 2 dilation_w, 12 dilation_h, 3 stride_w, 13 stride_h, 4 pad_left, 14 pad_top, 5 bias_term, 6 weight_data_size,
# 7 group, 8 int8_scale_term.  Pooling: 0 pooling_type, 1 kernel_w, 11 kernel_h, 2 stride_w, 12 stride_h, 3 pad_left,
# 13 pad_top, 4 global_pooling, 5 pad_mode.  Reduction: 0 operation, 1 reduce_all, 2 coeff, 3 axes, 4 keepdims.
_CONV = {0: None, 1: None, 11: None, 2: 1, 12: None, 3: 1, 13: None, 4: 0, 14: None, 5: 0, 6: None, 8: None}
KEYS = {
    "Input": {0: None, 1: None, 2: None},
    "Convolution": _CONV,
    "ConvolutionDepthWise": {**_CONV, 7: None},
    "InnerProduct": {0: None, 1: 0, 2: None, 8: None},
    "ReLU": {}, "Split": {}, "Flatten": {},
    "BinaryOp": {0: 0},
    "Reshape": {0: None, 1: None},
    "Reduction": {0: None, 1: 1, 2: 1.0, 3: None, 4: 0},
    "Softmax": {0: 0},
    "Pooling": {0: 0, 1: None, 11: None, 2: 1, 12: None, 3: 0, 13: None, 4: 0, 5: 0},
}


class NcnnError(_lib.DfqError):
    """A file or model this module does not read or write, refused by name."""


def _refuse(layer, typ, msg):
    raise NcnnError("ncnn layer %s (%s): %s" % (layer, typ, msg))


# ---- the .param ---------------------------------------------------------------------------------------------------------
def _value(layer, typ, key, v):
    try:
        return float(v) if any(ch in v for ch in ".eE") or v in ("nan", "inf", "-inf") else int(v)
    except ValueError:
        _refuse(layer, typ, "key %d: value %r is not a number" % (key, v))


def parse_param(path):
    """[dict(type, name, bottoms, tops, params {key: int | float | [values]})] of every layer, in file order, each checked
    against KEYS (missing keys take their defaults) and each bottom against the blobs produced before it."""
    with open(path) as f:
        lines = f.read().split("\n")
    if not lines or lines[0].strip() != str(MAGIC):
        _refuse("-", "-", "%s does not start with the magic %d" % (path, MAGIC))
    counts = lines[1].split() if len(lines) > 1 else []
    if len(counts) != 2 or not all(c.isdigit() for c in counts):
        _refuse("-", "-", "%s: line 2 is not the layer and blob counts" % path)
    n_layers, n_blobs = int(counts[0]), int(counts[1])
    body = [ln for ln in lines[2:] if ln.strip()]
    if len(body) != n_layers:
        _refuse("-", "-", "%s holds %d layer lines, its header says %d" % (path, len(body), n_layers))
    layers, blobs = [], set()
    for ln in body:
        f = ln.split()
        if len(f) < 4 or not f[2].isdigit() or not f[3].isdigit():
            _refuse(f[1] if len(f) > 1 else "-", f[0], "the line does not give bottom and top counts")
        typ, name, nb, nt = f[0], f[1], int(f[2]), int(f[3])
        if typ not in KEYS:
            _refuse(name, typ, "layer type %s is not implemented" % typ)
        if len(f) < 4 + nb + nt:
            _refuse(name, typ, "the line lists fewer than %d bottoms and %d tops" % (nb, nt))
        bottoms, tops = f[4:4 + nb], f[4 + nb:4 + nb + nt]
        params = {}
        for item in f[4 + nb + nt:]:
            k, eq, v = item.partition("=")
            if not eq or not k.lstrip("-").isdigit():
                _refuse(name, typ, "%r is not a key=value pair" % item)
            k = int(k)
            if k <= -23300:
                k = -k - 23300
                vals = [_value(name, typ, k, x) for x in v.split(",")]
                if not vals or vals[0] != len(vals) - 1:
                    _refuse(name, typ, "key %d: the array %r does not hold its count" % (k, v))
                v = vals[1:]
            else:
                v = _value(name, typ, k, v)
            if k not in KEYS[typ]:
                _refuse(name, typ, "key %d is not implemented" % k)
            params[k] = v
        for k, d in KEYS[typ].items():
            if k not in params and d is not None:
                params[k] = d
        for b in bottoms:
            if b not in blobs:
                _refuse(name, typ, "bottom blob %s is used before it is produced" % b)
        for t in tops:
            if t in blobs:
                _refuse(name, typ, "top blob %s is produced twice" % t)
            blobs.add(t)
        layers.append(dict(type=typ, name=name, bottoms=bottoms, tops=tops, params=params))
    if len(blobs) != n_blobs:
        _refuse("-", "-", "%s produces %d blobs, its header says %d" % (path, len(blobs), n_blobs))
    for lay in layers:
        _check_layer(lay)
    return layers


def _need(lay, *keys):
    for k in keys:
        if k not in lay["params"]:
            _refuse(lay["name"], lay["type"], "key %d is required" % k)


def _check_layer(lay):
    """Refuse a layer whose counts or values this module does not implement."""
    t, name, p = lay["type"], lay["name"], lay["params"]
    want = {"Input": (0, 1), "Split": (1, None), "BinaryOp": (2, 1)}.get(t, (1, 1))
    if len(lay["bottoms"]) != want[0] or (want[1] is not None and len(lay["tops"]) != want[1]):
        _refuse(name, t, "%d bottoms and %d tops, expected %d and %s" % (len(lay["bottoms"]), len(lay["tops"]), want[0],
                                                                         want[1] if want[1] is not None else "any"))
    if t == "Split" and len(lay["tops"]) < 1:
        _refuse(name, t, "a Split with no top")

    def value(k, ok, what):
        if not ok(p[k]):
            _refuse(name, t, "key %d = %r: %s" % (k, p[k], what))
    if t == "Input":
        _need(lay, 0, 1, 2)
        for k in (0, 1, 2):
            value(k, lambda v: type(v) is int and v > 0, "must be a positive int")
    elif t in WEIGHTED:
        _need(lay, *((0, 2, 8) if t == "InnerProduct" else (0, 1, 6, 8) + ((7,) if t == "ConvolutionDepthWise" else ())))
        bias_key = 1 if t == "InnerProduct" else 5
        for k in p:
            if k == bias_key:
                value(k, lambda v: v in (0, 1), "the bias term must be 0 or 1")
            elif k == 8:
                value(k, lambda v: v in ((1,) if t == "ConvolutionDepthWise" else (1, 2)),
                      "int8_scale_term must be %s: only int8 weight records with per-channel scales are implemented"
                      % ("1" if t == "ConvolutionDepthWise" else "1 or 2"))
            elif k in (4, 14):
                value(k, lambda v: type(v) is int and v >= 0, "only explicit non-negative padding is implemented")
            else:
                value(k, lambda v: type(v) is int and v > 0, "must be a positive int")
    elif t == "BinaryOp":
        value(0, lambda v: v == 0, "only op_type 0 (add) is implemented")
    elif t == "Reshape":
        _need(lay, 0, 1)
        value(0, lambda v: v == -1, "only w = -1 (the plane flattened) is implemented")
        value(1, lambda v: type(v) is int and v > 0, "h must be the channel count")
    elif t == "Reduction":
        _need(lay, 0, 3)
        value(0, lambda v: v == 3, "only operation 3 (mean) is implemented")
        value(1, lambda v: v == 0, "only reduce_all 0 (the listed axes) is implemented")
        value(2, lambda v: v == 1, "only coeff 1 is implemented")
        value(4, lambda v: v == 0, "only keepdims 0 is implemented")
        value(3, lambda v: isinstance(v, list) and v == [-1], "only the mean over the last axis (axes -1) is implemented")
    elif t == "Softmax":
        value(0, lambda v: v == 0, "only axis 0 is implemented")
    elif t == "Pooling":
        value(0, lambda v: v in (0, 1), "pooling_type must be 0 (max) or 1 (average)")
        value(4, lambda v: v in (0, 1), "global_pooling must be 0 or 1")
        if p[4] == 1:
            value(0, lambda v: v == 1, "only global average pooling is implemented")
        else:
            value(0, lambda v: v == 0, "only max pooling is implemented for windows")
            _need(lay, 1)
            value(5, lambda v: v == 1, "only pad_mode 1 (explicit pads, floor: torch's ceil_mode=False) is implemented")
            for k in (1, 11, 2, 12):
                if k in p:
                    value(k, lambda v: type(v) is int and v > 0, "must be a positive int")
            for k in (3, 13):
                if k in p:
                    value(k, lambda v: type(v) is int and v >= 0, "must be a non-negative int")


# ---- the .bin -----------------------------------------------------------------------------------------------------------
def _geometry(lay):
    """(O, k (kh, kw), stride, pad, dilation, groups, code count) of a weighted layer."""
    p = lay["params"]
    if lay["type"] == "InnerProduct":
        return p[0], (1, 1), (1, 1), (0, 0), (1, 1), 1, p[2]
    kw, dw, sw, pw = p[1], p[2], p[3], p[4]
    return (p[0], (p.get(11, kw), kw), (p.get(13, sw), sw), (p.get(14, pw), pw), (p.get(12, dw), dw), p.get(7, 1), p[6])


def parse_bin(path, layers):
    """{layer name: dict(codes int8 [count], bias fp32 [O] | None, w_scales fp32, in_scale fp32)} of the weighted layers,
    every byte of the file accounted for."""
    with open(path, "rb") as f:
        data = f.read()
    pos, recs = 0, {}

    def take(lay, n, dtype, what):
        nonlocal pos
        size = n * np.dtype(dtype).itemsize
        if pos + size > len(data):
            _refuse(lay["name"], lay["type"], "the .bin ends at byte %d inside the %s (%d bytes from %d)"
                    % (len(data), what, size, pos))
        v = np.frombuffer(data, dtype, n, pos).copy()
        pos += size
        return v
    for lay in layers:
        if lay["type"] not in WEIGHTED:
            continue
        O, k, _, _, _, groups, count = _geometry(lay)
        fc, dw = lay["type"] == "InnerProduct", lay["type"] == "ConvolutionDepthWise"
        tag = int(take(lay, 1, "<u4", "record tag")[0])
        if tag != TAG:
            _refuse(lay["name"], lay["type"], "record tag 0x%08X at byte %d is not the int8 tag 0x%08X: only int8 weight "
                    "records are implemented" % (tag, pos - 4, TAG))
        codes = take(lay, count, np.int8, "int8 weights")
        take(lay, (count + 3) // 4 * 4 - count, np.int8, "weight padding")
        bias = take(lay, O, "<f4", "bias").astype(np.float32) if lay["params"][1 if fc else 5] else None
        w_scales = take(lay, groups if dw else O, "<f4", "weight scales").astype(np.float32)
        in_scale = np.float32(take(lay, 1, "<f4", "input scale")[0])
        Cg = count // (O * k[0] * k[1])
        if Cg * O * k[0] * k[1] != count or Cg < 1:
            _refuse(lay["name"], lay["type"], "%d weights are not O %d x I/g x %d x %d" % (count, O, k[0], k[1]))
        if dw and not (groups == O and Cg == 1):
            _refuse(lay["name"], lay["type"], "group %d with num_output %d and %d weights is not depthwise"
                    % (groups, O, count))
        recs[lay["name"]] = dict(codes=codes, bias=bias, w_scales=w_scales, in_scale=in_scale, in_channels=Cg * groups)
    if pos != len(data):
        _refuse("-", "-", "%s holds %d bytes; its weighted layers account for %d" % (path, len(data), pos))
    return recs


# ---- the module ncnn's means become --------------------------------------------------------------------------------------
class PlaneMean(nn.Module):
    """ncnn's mean of each (image, channel) plane of x [N, C, ...] (dfq_i8_plane_mean): a sequential fp32 sum from 0.f in
    plane order, then * fp32(1 / P) (Reduction MEAN, divide=False) or / P (Pooling global average, divide=True); returns
    fp32 [N, C].  It is not torch's mean, which sums in another order.  With out_scale (set by chain_int8 only) it returns
    the consumer's int8 codes [N, 1, 1, round_up(C, 16)] instead, q8 at out_scale."""

    def __init__(self, divide, out_scale=None, name=None):
        super().__init__()
        self.divide, self.out_scale, self.layer_name = bool(divide), out_scale, name
        if out_scale is not None:
            I.check_scale("output", out_scale, name or "PlaneMean")
            self.out_scale = float(np.float32(out_scale))

    def forward(self, x):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or x.dim() < 3 or not x.is_cuda:
            raise _lib.DfqError("PlaneMean %s: expects fp32 [N, C, ...] on the GPU, got %s" % (
                self.layer_name or "", "%s %s on %s" % (x.dtype, list(x.shape), x.device)
                if isinstance(x, torch.Tensor) else type(x).__name__))
        x = x.contiguous()
        N, Cn, P = int(x.shape[0]), int(x.shape[1]), int(x[0, 0].numel())
        y = yq = None
        if self.out_scale is None:
            y = torch.empty((N, Cn), dtype=torch.float32, device=x.device)
        else:
            yq = torch.empty((N, 1, 1, (Cn + 15) // 16 * 16), dtype=torch.int8, device=x.device)
        _lib.check(_lib.load().dfq_i8_plane_mean(I._ptr(x), I._ptr(y), I._ptr(yq), N, Cn, P, int(self.divide),
                                                 C.c_float(0.0 if self.out_scale is None else self.out_scale),
                                                 _lib.stream_ptr()), "dfq_i8_plane_mean (layer %s)" % self.layer_name)
        return y if yq is None else yq

    def extra_repr(self):
        return "divide=%s%s" % (self.divide, "" if self.out_scale is None else ", out_scale=%g" % self.out_scale)


# ---- load ---------------------------------------------------------------------------------------------------------------
def ident(blob):
    """The fx node name of an ncnn blob: characters other than letters, digits and '_' become '_', and a leading digit
    gets a '_' in front (blob 619 is node _619), as torch.fx forms names."""
    s = re.sub(r"[^0-9A-Za-z_]", "_", blob)
    return "_" + s if not s or s[0].isdigit() else s


def load(param_path, bin_path, outputs=None, device=None) -> fx.GraphModule:
    """The int8 ncnn model as an fx.GraphModule: its inputs are the Input blobs (fp32 NCHW, any H x W the layers admit),
    its outputs the `outputs` blobs (default: the last layer's top; a list gives a tuple).  Each node is named after its
    blob (ident()); a Split's tops are its bottom's node, and an InnerProduct is three nodes, <blob>_in, <blob>_fc and
    <blob>.  Convolution / ConvolutionDepthWise are int8.Int8Conv2d built from the file's codes (dfq_i8_pack_codes);
    InnerProduct a 1 x 1 Int8Conv2d of [N, C, 1, 1] between two reshapes; ReLU F.relu; BinaryOp add operator.add;
    Reshape / Flatten Tensor.flatten; Reduction mean and Pooling global average PlaneMean; Pooling max F.max_pool2d;
    Softmax F.softmax (the unpatched op).  Everything is parsed and checked before anything is allocated on `device`
    (default and only choice: the current CUDA device)."""
    layers = parse_param(param_path)
    recs = parse_bin(bin_path, layers)
    last = layers[-1]["tops"] if layers else []
    many = isinstance(outputs, (list, tuple))
    outs = list(outputs) if many else [outputs] if outputs is not None else last[-1:]
    produced = {t for lay in layers for t in lay["tops"]}
    for o in outs:
        if o not in produced:
            _refuse("-", "-", "output blob %s is not produced by any layer" % o)
    channels, dims = {}, {}
    for lay in layers:                                  # channel counts and blob dims: refused before any allocation
        t, p, b = lay["type"], lay["params"], lay["bottoms"]
        c = channels.get(b[0]) if b else p[2]
        d = dims.get(b[0]) if b else 3
        need = {"Convolution": 3, "ConvolutionDepthWise": 3, "Reshape": 3, "Pooling": 3, "Reduction": 2, "Softmax": 1}.get(t)
        if need is not None and d != need:
            _refuse(lay["name"], t, "blob %s is %d-D (per image), this layer takes %d-D: %s" % (b[0], d, need, {
                3: "a [C, H, W] blob", 2: "the [C, H * W] output of a Reshape", 1: "a vector"}[need]))
        if t in WEIGHTED:
            r = recs[lay["name"]]
            if c != r["in_channels"]:
                _refuse(lay["name"], t, "its weights take %d input channels, blob %s has %s" % (r["in_channels"], b[0], c))
            c = p[0]
        elif t == "BinaryOp" and (channels[b[0]] != channels[b[1]] or dims[b[0]] != dims[b[1]]):
            _refuse(lay["name"], t, "adds a %d-D blob of %d channels to a %d-D blob of %d channels"
                    % (dims[b[0]], channels[b[0]], dims[b[1]], channels[b[1]]))
        elif t == "Reshape" and p[1] != c:
            _refuse(lay["name"], t, "h %d is not the %d channels of blob %s" % (p[1], c, b[0]))
        d = {"InnerProduct": 1, "Reshape": 2, "Reduction": 1, "Flatten": 1}.get(t, 1 if t == "Pooling" and p[4] else d)
        for top in lay["tops"]:
            channels[top], dims[top] = c, d
    if device is not None and torch.device(device) not in (engine._default_device(), torch.device("cuda")):
        raise _lib.DfqError("ncnn.load: device %s is not the current CUDA device %s; load inside `with "
                            "torch.cuda.device(...)`" % (device, engine._default_device()))
    root, g, env = nn.Module(), fx.Graph(), {}

    def node(op, target, args, name, kwargs=None):
        return g.create_node(op, target, args, kwargs or {}, name=ident(name))

    def module(name, m):
        root.add_module(ident(name), m)
        return ident(name)
    for lay in layers:
        t, p, name, top = lay["type"], lay["params"], lay["name"], lay["tops"][0]
        ins = [env[b] for b in lay["bottoms"]]
        if t == "Input":
            n = node("placeholder", ident(top), (), top)
        elif t == "Split":
            for tp in lay["tops"]:
                env[tp] = ins[0]
            continue
        elif t in WEIGHTED:
            r = recs[name]
            O, k, stride, pad, dil, groups, _ = _geometry(lay)
            conv = I.Int8Conv2d.from_codes(r["codes"].reshape(O, -1, *k), r["bias"], r["in_scale"], r["w_scales"], stride,
                                           pad, dil, groups)
            conv.layer_name = name
            if t == "InnerProduct":
                x = node("call_method", "reshape", (ins[0], (-1, channels[lay["bottoms"][0]], 1, 1)), top + "_in")
                y = node("call_module", module(top + "_fc", conv), (x,), top + "_fc")
                n = node("call_method", "flatten", (y, 1), top)
            else:
                n = node("call_module", module(top + "_conv", conv), (ins[0],), top)
        elif t == "ReLU":
            n = node("call_function", F.relu, (ins[0],), top)
        elif t == "BinaryOp":
            n = node("call_function", operator.add, (ins[0], ins[1]), top)
        elif t in ("Reshape", "Flatten"):
            n = node("call_method", "flatten", (ins[0], 2 if t == "Reshape" else 1), top)
        elif t == "Reduction" or (t == "Pooling" and p[4] == 1):
            n = node("call_module", module(top + "_mean", PlaneMean(t == "Pooling", name=name)), (ins[0],), top)
        elif t == "Pooling":
            kw = p[1]
            n = node("call_function", F.max_pool2d, (ins[0], (p.get(11, kw), kw), (p.get(12, p[2]), p[2]),
                                                     (p.get(13, p[3]), p[3]), 1, False), top)
        else:                                                   # Softmax
            n = node("call_function", I._raw_softmax, (ins[0],), top, {"dim": 1})
        env[top] = n
    g.output(tuple(env[o] for o in outs) if many else env[outs[0]])
    g.lint()
    return fx.GraphModule(root, g, "NcnnInt8")


# ---- write --------------------------------------------------------------------------------------------------------------
_RELU = (F.relu, torch.relu)
_ADD = (operator.add, torch.add)
_MEAN = (torch.mean, I._raw_mean)


def _refuse_node(n, what):
    raise NcnnError("ncnn.write: node %s (%s %s): %s" % (n.name, n.op, getattr(n.target, "__name__", n.target), what))


class _Writer:
    """The layers of a traced converted model: [(type, name, bottoms, tops, keys)] and the weighted layers' modules."""

    def __init__(self, gm, input_hw):
        self.gm, self.mods, self.input_hw = gm, dict(gm.named_modules()), input_hw
        self.layers, self.weighted, self.blob, self.channels = [], [], {}, {}

    def add(self, typ, n, bottoms, keys):
        self.layers.append([typ, n.name, [self.blob[b] for b in bottoms], [n.name], keys])
        self.blob[n] = n.name

    def alias(self, n, src):
        self.blob[n], self.channels[n] = self.blob[src], self.channels[src]

    def data_input(self, n):
        ins = [a for a in n.all_input_nodes if a in self.blob]
        if len(ins) != 1:
            _refuse_node(n, "reads %d tensors, expected one" % len(ins))
        return ins[0]

    def module(self, n):
        m = self.mods[n.target]
        x = self.data_input(n)
        if isinstance(m, (I.Int8Conv2d, I.Int8Linear)):
            if m.codes_in or m.requant is not None or m.epilogue is not None or m.out_slice is not None or m.rows:
                _refuse_node(n, "a chained int8 layer; write the model int8.convert_to_int8 returned")
            if len(n.args) != 1 or n.kwargs:
                _refuse_node(n, "an int8 layer called with more than its input")
            (kh, kw), (sh, sw), (ph, pw), (dh, dw) = m.kernel_size, m.stride, m.padding, m.dilation
            O, wsize = m.out_channels, m.out_channels * (m.in_channels // m.groups) * kh * kw
            if self.channels[x] is None:                            # the input: the first layer gives its channels
                self.channels[x] = m.in_channels
            if self.channels[x] != m.in_channels:
                _refuse_node(n, "takes %d channels, its input has %s" % (m.in_channels, self.channels[x]))
            if isinstance(m, I.Int8Linear):
                self.add("InnerProduct", n, [x], [(0, O), (1, 1), (2, wsize), (8, 2)])
            else:
                dwise = m.groups > 1
                keys = [(0, O), (1, kw)] + ([(11, kh)] if kh != kw else []) + ([(2, dw)] if dw != 1 else []) + \
                    ([(12, dh)] if dh != dw else []) + ([(3, sw)] if sw != 1 else []) + ([(13, sh)] if sh != sw else []) + \
                    ([(4, pw)] if pw != 0 else []) + ([(14, ph)] if ph != pw else []) + [(5, 1), (6, wsize)] + \
                    ([(7, m.groups), (8, 1)] if dwise else [(8, 2)])
                self.add("ConvolutionDepthWise" if dwise else "Convolution", n, [x], keys)
            self.weighted.append((n.name, m))
            self.channels[n] = O
        elif isinstance(m, (nn.ReLU,)):
            self.add("ReLU", n, [x], [])
            self.channels[n] = self.channels[x]
        elif isinstance(m, (nn.Dropout, nn.Identity)):
            self.alias(n, x)
        elif isinstance(m, nn.MaxPool2d):
            self.max_pool(n, x, m.kernel_size, m.stride, m.padding, m.dilation, m.ceil_mode)
        elif isinstance(m, nn.AdaptiveAvgPool2d):
            self.global_pool(n, x, m.output_size)
        elif isinstance(m, nn.Flatten):
            if (m.start_dim, m.end_dim) != (1, -1):
                _refuse_node(n, "only a flatten from dim 1 has an ncnn Flatten")
            self.add("Flatten", n, [x], [])
            self.channels[n] = self.channels[x]
        elif isinstance(m, nn.Softmax):
            self.softmax(n, x, m.dim)
        else:
            _refuse_node(n, "module %s has no ncnn layer ncnn.load reads back" % type(m).__name__)

    def max_pool(self, n, x, k, s, p, d, ceil):
        k, s, p, d = I._pair(k), I._pair(k if s is None else s), I._pair(p), I._pair(d)
        if d != (1, 1) or ceil:
            _refuse_node(n, "only max pools without dilation or ceil_mode have an ncnn Pooling ncnn.load reads back")
        keys = [(0, 0), (1, k[1])] + ([(11, k[0])] if k[0] != k[1] else []) + [(2, s[1])] + \
            ([(12, s[0])] if s[0] != s[1] else []) + [(3, p[1])] + ([(13, p[0])] if p[0] != p[1] else []) + [(5, 1)]
        self.add("Pooling", n, [x], keys)
        self.channels[n] = self.channels[x]

    def global_pool(self, n, x, size):
        if I._pair(size) != (1, 1):
            _refuse_node(n, "only an average pool to 1 x 1 has an ncnn Pooling ncnn.load reads back")
        self.add("Pooling", n, [x], [(0, 1), (4, 1)])
        self.channels[n] = self.channels[x]

    def softmax(self, n, x, dim):
        if dim not in (1, -1):
            _refuse_node(n, "only a softmax over the classes (dim 1) has an ncnn Softmax ncnn.load reads back")
        self.add("Softmax", n, [x], [])
        self.channels[n] = self.channels[x]

    def mean(self, n, x, dims):
        """mean over the plane: a Reshape to [C, H * W] (skipped when the input is already that view) and a Reduction."""
        src = self.views.get(x)
        if src is None:
            if sorted(d % 4 for d in dims) != [2, 3]:
                _refuse_node(n, "only a mean over the spatial dims has an ncnn Reduction ncnn.load reads back")
            src = x
        elif list(dims) not in ([-1], [2]):
            _refuse_node(n, "only a mean over the last dim of a [N, C, -1] view has an ncnn Reduction")
        view = n.name + "_reshape"
        self.layers.append(["Reshape", view, [self.blob[src]], [view], [(0, -1), (1, self.channels[src])]])
        self.layers.append(["Reduction", n.name, [view], [n.name], [(0, 3), (1, 0), (-23303, "1,-1")]])
        self.blob[n], self.channels[n] = n.name, self.channels[src]

    def run(self):
        self.views = {}                 # [N, C, -1] views of a 4-D tensor: their source, for the mean after them
        for n in self.gm.graph.nodes:
            if n.op == "placeholder":
                if self.layers:
                    _refuse_node(n, "a second input")
                self.layers.append(["Input", n.name, [], [n.name], [(0, self.input_hw[1]), (1, self.input_hw[0]),
                                                                   (2, None)]])
                self.blob[n], self.channels[n] = n.name, None
            elif n.op == "output":
                continue
            elif n.op == "call_module":
                self.module(n)
            elif n.op == "call_method" and n.target in ("size", "dim") or \
                    n.op == "call_function" and n.target is getattr:
                continue                                        # shape queries: no tensor, no layer
            elif n.op == "call_method" and n.target in ("view", "reshape") and len(n.args) == 4 and n.args[3] == -1:
                self.views[n] = self.data_input(n)          # x.view(x.size(0), x.size(1), -1): the Reshape of a mean
            elif n.op == "call_method" and n.target == "flatten" or n.op == "call_function" and n.target is torch.flatten:
                x = self.data_input(n)
                if I._arg(n, 1, "start_dim", 0) != 1 or I._arg(n, 2, "end_dim", -1) != -1:
                    _refuse_node(n, "only a flatten from dim 1 has an ncnn Flatten")
                self.add("Flatten", n, [x], [])
                self.channels[n] = self.channels[x]
            elif n.op == "call_method" and n.target == "mean" or n.op == "call_function" and n.target in _MEAN:
                dims = I._arg(n, 1, "dim", None)
                if I._arg(n, 2, "keepdim", False) or dims is None:
                    _refuse_node(n, "only a mean over listed dims without keepdim has an ncnn Reduction")
                self.mean(n, n.args[0], [dims] if isinstance(dims, int) else list(dims))
            elif n.op == "call_method" and n.target == "relu" or n.op == "call_function" and n.target in _RELU:
                x = self.data_input(n)
                self.add("ReLU", n, [x], [])
                self.channels[n] = self.channels[x]
            elif n.op == "call_function" and n.target in _ADD and len(n.args) == 2 and not n.kwargs and \
                    all(a in self.blob for a in n.args):
                a, b = n.args
                if self.channels[a] != self.channels[b]:
                    _refuse_node(n, "adds %s to %s channels" % (self.channels[a], self.channels[b]))
                self.add("BinaryOp", n, [a, b], [])
                self.channels[n] = self.channels[a]
            elif n.op == "call_function" and n.target in (F.max_pool2d, torch.max_pool2d) and I._max_pool(n, self.mods):
                self.max_pool(n, n.args[0], *I._max_pool(n, self.mods))
            elif n.op == "call_function" and n.target is F.adaptive_avg_pool2d:
                self.global_pool(n, self.data_input(n), I._arg(n, 1, "output_size", None))
            elif n.op == "call_function" and n.target in (F.softmax, torch.softmax, I._raw_softmax):
                self.softmax(n, self.data_input(n), I._arg(n, 1, "dim", None))
            else:
                _refuse_node(n, "has no ncnn layer ncnn.load reads back")
        if not self.weighted:
            raise NcnnError("ncnn.write: the model has no int8 layer (convert it with int8.convert_to_int8 first)")
        self.layers[0][4][2] = (2, self.channels[next(n for n in self.blob if n.op == "placeholder")])
        return self.layers

    def with_splits(self):
        """The layers with a Split after every blob that several layers read, its tops handed out as onnx2ncnn does: the
        first reader in file order takes the last top."""
        readers = collections.Counter(b for lay in self.layers for b in lay[2])
        out, taken, k = [], collections.Counter(), 0
        for typ, name, bottoms, tops, keys in self.layers:
            new = []
            for b in bottoms:
                if readers[b] > 1:
                    new.append("%s_splitncnn_%d" % (b, readers[b] - 1 - taken[b]))   # onnx2ncnn counts down
                    taken[b] += 1
                else:
                    new.append(b)
            out.append([typ, name, new, tops, keys])
            for t in tops:
                if readers[t] > 1:
                    out.append(["Split", "splitncnn_%d" % k, [t], ["%s_splitncnn_%d" % (t, i) for i in range(readers[t])], []])
                    k += 1
        return out


def _format_key(k, v):
    return "%d=%s" % (k, v if isinstance(v, str) else repr(v) if isinstance(v, float) else "%d" % v)


def write(model, graph, targ_type, param_path, bin_path, table_path=None, input_hw=(224, 224)):
    """Write `model` (int8.convert_to_int8's result, its layers unchained) as an ncnn int8 model: the .param (layer types,
    keys and Split layers as onnx2ncnn + ncnn2int8 write them for MobileNetV2 and ResNet-18; blob and layer names are the
    traced graph's node names), the int8 .bin (the packed codes read back by dfq_i8_unpack_codes, the bias, the weight
    scales and the layer's activation scale) and, with table_path, the .table (export.write_ncnn_table of `graph` /
    `targ_type`, named by the same blobs).  The Input layer declares input_hw (H, W).  Any node ncnn.load would not read
    back is refused by name before a file is written.  Returns the layers written: [(type, name, bottoms, tops, keys)]."""
    gm, _, _ = I._trace(model, None, I._Int8Layer)
    w = _Writer(gm, tuple(int(v) for v in input_hw))
    w.run()
    layers = w.with_splits()
    blobs = {t for lay in layers for t in lay[3]}
    lines = ["%d" % MAGIC, "%d %d" % (len(layers), len(blobs))]
    for typ, name, bottoms, tops, keys in layers:
        lines.append(" ".join(["%-24s %-24s %d %d" % (typ, name, len(bottoms), len(tops))] + bottoms + tops +
                              [_format_key(k, v) for k, v in keys]))
    for name, m in w.weighted:
        if m.w_scale.numel() != m.out_channels or m.bias.numel() != m.out_channels:
            raise NcnnError("ncnn.write: layer %s holds %d weight scales and %d biases for %d output channels"
                            % (name, m.w_scale.numel(), m.bias.numel(), m.out_channels))
    chunks = []
    for name, m in w.weighted:                  # ConvolutionDepthWise: groups == O, so [O] scales are its [groups]
        codes = m.unpack_codes().cpu().numpy().reshape(-1)
        chunks += [struct.pack("<I", TAG), codes.tobytes(), b"\0" * ((-codes.size) % 4),
                   m.bias.detach().cpu().numpy().astype("<f4").tobytes(),
                   m.w_scale.detach().cpu().numpy().astype("<f4").tobytes(),
                   np.array([m.act_scale], "<f4").tobytes()]
    if table_path is not None:
        rows = export.ncnn_scales(graph, targ_type)
        if len(rows) != len(w.weighted):
            raise NcnnError("ncnn.write: the graph has %d target layers, the model %d int8 layers"
                            % (len(rows), len(w.weighted)))
    with open(param_path, "w") as f:
        f.write("\n".join(lines) + "\n")
    with open(bin_path, "wb") as f:
        f.write(b"".join(chunks))
    if table_path is not None:
        export.write_ncnn_table(graph, table_path, targ_type, names=[name for name, _ in w.weighted])
    return [tuple(lay) for lay in layers]
