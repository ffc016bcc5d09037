"""The file format of int8.save / int8.load: a model chain_int8 / chain_affine returned, as one torch.save of plain
containers and CPU tensors that torch.load(weights_only=True) reads, rebuilt without running code from the file.

    {"format": FORMAT, "version": VERSION, "class_name": str,
     "tensors": [CPU tensor, ...],                     every buffer and parameter, each storage once
     "modules": [{"type": name, "attrs": {...}, "buffers": {name: tensor index}, "params": {name: [index, grad]},
                  "heads": [module index, ...]}, ...],
     "paths": {dotted path: module index},              the graph's call_module targets and the chained layers
     "nodes": [{"op", "name", "target", "args", "kwargs"}, ...],
     "records": {"requantized_edges": [...], ...}}     the chain's records, those the model has

Node arguments are other nodes {"node": name}, {"tuple": [...]}, {"slice": [start, stop, step]}, lists, constants
(None, bool, int, float, str) and, for a model's dict output, {"dict": [[key, value], ...]}.  Every call_function / call_method target and every module type is checked against the
allowlist below when saving and again when loading; anything else is refused by name.  It holds what the two chains emit
on the reference's networks and torchvision's: the int8 modules, the functional-op observers (QuantMeasure), the
torch.nn leaves the tracer keeps, and the functions and tensor methods of those models' forwards.
"""
import keyword
import operator
import os
import pickle
import re

import numpy as np
import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, engine
from . import int8 as I
from . import ncnn as N
from .utils.quantize import QuantMeasure

FORMAT = "dfq_b200.int8.chained"
VERSION = 1
_KEYS = ("format", "version", "class_name", "tensors", "modules", "paths", "nodes", "records")
RECORDS = ("requantized_edges", "fused_adds", "fused_observers", "fused_cats", "fused_pools", "fused_upsamples",
           "fused_heads", "folded_pads")

# int8 modules rebuilt by their constructors from these attributes (layer_name passed as name=); heads are modules
_CONSTRUCTED = {
    I.Int8MaxPool2d: ("kernel_size", "stride", "padding", "dilation", "ceil_mode", "channels", "codes_in", "out_scale",
                      "fp32", "layer_name"),
    I.AffineInt8MaxPool2d: ("kernel_size", "stride", "padding", "dilation", "ceil_mode", "channels", "codes_in",
                            "out_scale", "fp32", "sums", "layer_name"),
    I.Int8UpsampleBilinear: ("channels", "align_corners", "out_scale", "clamp", "out_slice", "layer_name"),
    I.AffineInt8UpsampleBilinear: ("channels", "align_corners", "out", "out_slice", "pre", "obs", "post", "sums",
                                   "layer_name"),
    I.Int8HeadConcat: ("k", "batch", "layer_name"),
    N.PlaneMean: ("divide", "out_scale", "layer_name"),
}
_LAYERS = (I.Int8Conv2d, I.Int8Linear, I.AffineInt8Conv2d, I.AffineInt8Linear)
# modules rebuilt from their plain attributes, parameters and buffers
_PLAIN = (QuantMeasure, nn.ReLU, nn.ReLU6, nn.Hardtanh, nn.BatchNorm2d, nn.Dropout, nn.Identity, nn.MaxPool2d,
          nn.AvgPool2d, nn.AdaptiveAvgPool2d, nn.Upsample, nn.Flatten)
MODULES = {c.__name__: c for c in (*_LAYERS, *_CONSTRUCTED, *_PLAIN)}

METHODS = frozenset(("view", "reshape", "size", "dim", "permute", "contiguous", "flatten", "mean", "relu", "add"))


def functions():
    """{name: function} of the allowed call_function targets.  torch.cat, torch.mean, F.interpolate and F.softmax are the
    unpatched ops, also while the reference's replace_op() is active."""
    raw = {n: I._raw(t, n) for t, names in (("raw_torch_op", ("cat", "mean")), ("raw_func_op", ("interpolate", "softmax")))
           for n in names}
    fns = {"getattr": getattr, "torch.cat": raw["cat"], "torch.concat": torch.concat, "torch.mean": raw["mean"],
           "torch.add": torch.add, "torch.flatten": torch.flatten, "torch.reshape": torch.reshape, "torch.relu": torch.relu,
           "torch.max_pool2d": torch.max_pool2d, "F.relu": F.relu, "F.relu6": F.relu6, "F.hardtanh": F.hardtanh,
           "F.max_pool2d": F.max_pool2d, "F.adaptive_avg_pool2d": F.adaptive_avg_pool2d,
           "F.interpolate": raw["interpolate"], "F.softmax": raw["softmax"], "F.pad": F.pad}
    fns.update(("operator." + f.__name__, f) for f in (operator.getitem, *I._INT_ARITH))
    fns.update(("int8." + f.__name__, f) for f in (I._raw_cat, I._raw_mean, I._raw_interpolate, I._raw_softmax,
                                                   I._nchw_view))
    return fns


def _refuse(msg):
    raise _lib.DfqError("int8 save / load: " + msg)


def _plain(v, what):
    """v, checked to be None, bool, int, float, str or tuples / lists of them."""
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if type(v) in (tuple, list):
        for e in v:
            _plain(e, what)
        return v
    _refuse("%s holds a %s, not a plain value" % (what, type(v).__name__))


_ELEMENT = re.compile(r"[A-Za-z_][A-Za-z0-9_]*|[0-9]+")


def _identifier(v, what):
    """v, checked to be a str that is a Python identifier and no keyword: the generated forward spells it as code."""
    if not isinstance(v, str) or not v.isidentifier() or keyword.iskeyword(v):
        _refuse("%s %r is not an identifier" % (what, v))
    return v


def _module_path(v, what):
    """v, checked to be a dotted module path of identifiers or indices (features.0.conv)."""
    if not isinstance(v, str) or not all(_ELEMENT.fullmatch(e) and not keyword.iskeyword(e) for e in v.split(".")):
        _refuse("%s %r is not a dotted path of identifiers and indices" % (what, v))
    return v


def _check_node(op, name, target, args, kwargs):
    """The names of a node that the generated forward spells as code: its name, a placeholder's target (a parameter, with
    no default value), an output node's target, a module path, keyword names and dict keys."""
    _identifier(name, "node name")
    if op == "placeholder":
        _identifier(target, "placeholder %s: parameter" % name)
        if args != ():
            _refuse("placeholder %s takes no default value" % name)
    elif op == "output" and target != "output":
        _refuse("output node %s: target %r" % (name, target))
    elif op == "call_module":
        _module_path(target, "node %s: module path" % name)
    for k in kwargs:
        _identifier(k, "node %s: keyword" % name)

    def keys(a):
        if isinstance(a, dict):
            for k, v in a.items():
                _identifier(k, "node %s: dict key" % name)
                keys(v)
        elif isinstance(a, (tuple, list)):
            for v in a:
                keys(v)
    keys(args)
    keys(tuple(kwargs.values()))


# ---- save ---------------------------------------------------------------------------------------------------------------
class _Writer:
    def __init__(self):
        self.tensors, self.by_storage, self.modules, self.by_module = [], {}, [], {}

    def tensor(self, t):
        """The index of t's CPU copy, one per (storage, view) whoever holds it."""
        key = (t.untyped_storage().data_ptr(), t.device, t.storage_offset(), tuple(t.shape), tuple(t.stride()), t.dtype)
        if key not in self.by_storage:
            self.by_storage[key] = len(self.tensors)
            self.tensors.append(t.detach().to("cpu", copy=True).contiguous())
        return self.by_storage[key]

    def module(self, m, path):
        if id(m) in self.by_module:
            return self.by_module[id(m)]
        cls = type(m)
        if MODULES.get(cls.__name__) is not cls:
            _refuse("module %s is a %s.%s, which a chained int8 model does not hold" % (path, cls.__module__,
                                                                                       cls.__qualname__))
        rec = {"type": cls.__name__, "attrs": {}, "buffers": {}, "params": {}}
        if cls in _LAYERS:
            for k in m._copied + m._modes:
                v = getattr(m, k)
                if k == "epilogue" and v is not None:
                    v = tuple(v)
                elif k == "constants":
                    v = [float(c) for c in v[0]]
                rec["attrs"][k] = _plain(v, "%s.%s" % (path, k))
        elif cls in _CONSTRUCTED:
            rec["attrs"] = {k: _plain(getattr(m, k), "%s.%s" % (path, k)) for k in _CONSTRUCTED[cls]}
        else:
            rec["attrs"] = {k: _plain(v, "%s.%s" % (path, k)) for k, v in vars(m).items() if not k.startswith("_")}
            rec["params"] = {k: [self.tensor(p), bool(p.requires_grad)] for k, p in m._parameters.items() if p is not None}
            if m._modules:
                _refuse("module %s (%s) has submodules" % (path, cls.__name__))
        rec["buffers"] = {k: self.tensor(b) for k, b in m._buffers.items() if b is not None}
        self.by_module[id(m)] = i = len(self.modules)
        self.modules.append(rec)
        if cls is I.Int8HeadConcat:
            rec["heads"] = [self.module(h, "%s.heads.%d" % (path, j)) for j, h in enumerate(m.heads)]
        return i


def _encode(a, names, where):
    if isinstance(a, fx.Node):
        return {"node": names[a]}
    if isinstance(a, tuple):
        return {"tuple": [_encode(e, names, where) for e in a]}
    if isinstance(a, list):
        return [_encode(e, names, where) for e in a]
    if isinstance(a, slice):
        return {"slice": [_encode(e, names, where) for e in (a.start, a.stop, a.step)]}
    if isinstance(a, dict) and all(isinstance(k, str) for k in a):     # a model's dict output (torchvision's {"out": y})
        return {"dict": [[k, _encode(v, names, where)] for k, v in a.items()]}
    if a is None or isinstance(a, (bool, int, float, str)):
        return a
    _refuse("node %s: argument %r (%s) is not a node, a constant, a tuple, a list or a slice"
            % (where, a, type(a).__name__))


def _uncalled_layers(gm, called):
    """Paths of the chained layers the graph does not call (a detection head's, which its Int8HeadConcat holds too)."""
    mods = list(gm.named_modules(remove_duplicate=False))
    inside = tuple(p + "." for p, m in mods if isinstance(m, I.Int8HeadConcat))
    return [p for p, m in mods if isinstance(m, _LAYERS) and p not in called and not p.startswith(inside)]


def state(gm):
    """The plain-container state of a chained model, checked against the allowlist; gm is only read."""
    if not isinstance(gm, fx.GraphModule) or not hasattr(gm, "requantized_edges"):
        _refuse("takes the GraphModule chain_int8 / chain_affine returned, not a %s; for a per-layer model, save "
                "chain_int8(model) or chain_affine(model) with no flags, which computes the same bit for bit"
                % type(gm).__name__)
    fns = {id(f): n for n, f in reversed(list(functions().items()))}
    w, names, nodes, paths = _Writer(), {}, [], {}
    for n in gm.graph.nodes:
        names[n] = n.name
        if n.op == "call_function":
            target = fns.get(id(n.target))
            if target is None:
                _refuse("node %s calls %s, which is not on the allowlist of a chained int8 model" % (
                    n.name, "%s.%s" % (getattr(n.target, "__module__", "?"), getattr(n.target, "__qualname__", n.target))))
        elif n.op == "call_method":
            if n.target not in METHODS:
                _refuse("node %s calls the tensor method %r, which is not on the allowlist" % (n.name, n.target))
            target = n.target
        elif n.op == "call_module":
            paths[n.target] = w.module(gm.get_submodule(n.target), n.target)
            target = n.target
        elif n.op in ("placeholder", "output"):
            target = n.target
        else:
            _refuse("node %s is a %s node" % (n.name, n.op))
        _check_node(n.op, n.name, n.target, n.args, n.kwargs)
        nodes.append({"op": n.op, "name": n.name, "target": target, "args": _encode(n.args, names, n.name),
                      "kwargs": {k: _encode(v, names, n.name) for k, v in n.kwargs.items()}})
    for path in _uncalled_layers(gm, paths):
        paths[_module_path(path, "module path")] = w.module(gm.get_submodule(path), path)
    records = {k: _plain(getattr(gm, k), k) for k in RECORDS if hasattr(gm, k)}
    return {"format": FORMAT, "version": VERSION, "class_name": _identifier(type(gm).__name__, "class name"), "tensors": w.tensors,
            "modules": w.modules, "paths": paths, "nodes": nodes, "records": records}


def save(gm, path):
    st = state(gm)
    path = os.fspath(path)
    tmp = "%s.%d.tmp" % (path, os.getpid())
    try:
        torch.save(st, tmp)
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)


# ---- load ---------------------------------------------------------------------------------------------------------------
def _get(d, key, what, typ=None):
    if not isinstance(d, dict) or key not in d:
        _refuse("%s has no %r" % (what, key))
    v = d[key]
    if typ is not None and not isinstance(v, typ):
        _refuse("%s: %r is a %s, not a %s" % (what, key, type(v).__name__, typ.__name__))
    return v


def _public(cls, k, what):
    """k, checked to be a name save() writes for a module of cls: a public identifier that is not a class attribute (a
    method, a hook table)."""
    _identifier(k, what)
    if k.startswith("_") or hasattr(cls, k):
        _refuse("%s %r is not a stored attribute of %s" % (what, k, cls.__name__))
    return k


def _pair_of(v, lo):
    return type(v) in (tuple, list) and len(v) == 2 and all(type(e) is int and e >= lo for e in v)


def _check_layer(cls, a, buffers, what):
    """Refuse a layer whose geometry is not one the layer classes make or whose buffers do not fit it (the kernels would
    read or write past them): what __init__ and chained() establish, checked again."""
    if not all(type(a[k]) is int and a[k] > 0 for k in ("out_channels", "in_channels", "groups", "cpad")) or \
            not all(_pair_of(a[k], 1) for k in ("kernel_size", "stride", "dilation")) or not _pair_of(a["padding"], 0):
        _refuse("%s: the geometry %s is not positive ints" % (what, {k: a[k] for k in cls._copied[:8]}))
    O, Cin, groups, (kh, kw) = a["out_channels"], a["in_channels"], a["groups"], a["kernel_size"]
    depthwise = groups > 1
    if (depthwise and not groups == Cin == O) or a["cpad"] != (Cin + 15) // 16 * 16:
        _refuse("%s: groups %d, C_in %d, C_out %d and Cpad %d do not fit together" % (what, groups, Cin, O, a["cpad"]))
    want = {"weight_codes": (torch.int8, kh * kw * a["cpad"] * (1 if depthwise else O)), "bias": (torch.float32, O)}
    if issubclass(cls, I._Int8Layer):
        want.update(w_scale=(torch.float32, O), dq=(torch.float32, O))
    else:
        I._affine_refusal(what, Cin, O, groups, (kh, kw), a["act_bits"], a["w_bits"])
        want.update(tap_table=(torch.int32, 0 if depthwise else O * (kh + 1) * (kw + 1)))
    if buffers.keys() != want.keys():
        _refuse("%s: buffers %s, expected %s" % (what, sorted(buffers), sorted(want)))
    for k, (dtype, n) in want.items():
        t = buffers[k]
        if t.dtype != dtype or t.dim() != 1 or t.numel() != n or not t.is_contiguous():
            _refuse("%s: buffer %s is %s %s, expected %s [%d]" % (what, k, t.dtype, list(t.shape), dtype, n))
    if a["out_slice"] is not None:
        I._channel_slice(a["out_slice"], O, what)


def _rebuild_module(i, recs, tensors, built, layer=False):
    if built[i] is not None:
        return built[i]
    rec = recs[i]
    what = "module record %d" % i
    cls = MODULES.get(_get(rec, "type", what, str))
    if cls is None:
        _refuse("%s: module type %r is not on the allowlist of a chained int8 model" % (what, rec["type"]))
    if layer and cls not in _LAYERS:
        _refuse("%s: a detection head is a %s, not an int8 convolution" % (what, cls.__name__))
    attrs, bufs = _get(rec, "attrs", what, dict), _get(rec, "buffers", what, dict)
    for k, v in attrs.items():
        _plain(v, "%s.%s" % (what, k))

    def tensor(j):
        if type(j) is not int or not 0 <= j < len(tensors):
            _refuse("%s: tensor index %r out of range" % (what, j))
        return tensors[j]
    buffers = {k: tensor(j) for k, j in bufs.items()}
    if cls in _LAYERS:
        want = set(cls._copied + cls._modes)
        if set(attrs) != want:
            _refuse("%s (%s): attributes %s missing, %s unknown" % (what, cls.__name__, sorted(want - set(attrs)),
                                                                   sorted(set(attrs) - want)))
        _check_layer(cls, attrs, buffers, what)
        a = dict(attrs)
        a["epilogue"] = None if a["epilogue"] is None else I.Epilogue(*a["epilogue"])
        if "constants" in a:
            a["constants"] = np.zeros(1, _lib.I8_AFFINE_DT)
            a["constants"][0] = tuple(attrs["constants"])
        m = cls._build(a, buffers)
    elif cls in _CONSTRUCTED:
        kw = {"name" if k == "layer_name" else k: _get(attrs, k, what) for k in _CONSTRUCTED[cls]}
        if cls is I.Int8HeadConcat:
            kw["heads"] = [_rebuild_module(j, recs, tensors, built, layer=True) if type(j) is int and 0 <= j < len(recs)
                           else _refuse("%s: head index %r out of range" % (what, j)) for j in _get(rec, "heads", what, list)]
        m = cls(**kw)
    else:
        m = cls.__new__(cls)
        nn.Module.__init__(m)
        for k, v in attrs.items():
            setattr(m, _public(cls, k, "%s: attribute" % what), v)
        for k, p in _get(rec, "params", what, dict).items():
            if type(p) is not list or len(p) != 2 or type(p[1]) is not bool:
                _refuse("%s: parameter %r is not [tensor index, requires_grad]" % (what, k))
            m.register_parameter(_public(cls, k, "%s: parameter" % what), nn.Parameter(tensor(p[0]), requires_grad=p[1]))
        for k, b in buffers.items():
            m.register_buffer(_public(cls, k, "%s: buffer" % what), b)
    built[i] = m
    return m


def _decode(a, env, where):
    if isinstance(a, dict):
        if len(a) != 1:
            _refuse("node %s: argument %r is not an encoded value" % (where, a))
        (tag, v), = a.items()
        if tag == "node":
            if v not in env:
                _refuse("node %s reads %r, which no earlier node defines" % (where, v))
            return env[v]
        if tag == "tuple" and isinstance(v, list):
            return tuple(_decode(e, env, where) for e in v)
        if tag == "slice" and isinstance(v, list) and len(v) == 3:
            return slice(*(_decode(e, env, where) for e in v))
        if tag == "dict" and isinstance(v, list) and all(isinstance(e, list) and len(e) == 2 and isinstance(e[0], str)
                                                         for e in v):
            return {k: _decode(e, env, where) for k, e in v}
        _refuse("node %s: argument tag %r is unknown" % (where, tag))
    if isinstance(a, list):
        return [_decode(e, env, where) for e in a]
    if a is None or isinstance(a, (bool, int, float, str)):
        return a
    _refuse("node %s: argument %r is not an encoded value" % (where, a))


def load(path, device=None):
    _lib.require_cuda()
    dev = engine._default_device()
    if device is not None and torch.device(device) not in (dev, torch.device("cuda")):
        _refuse("device %s is not the current CUDA device %s: the layers launch on the current device's stream; load "
                "and run the model inside `with torch.cuda.device(...)`" % (torch.device(device), dev))
    try:
        st = torch.load(path, map_location="cpu", weights_only=True)
    except pickle.UnpicklingError as e:
        _refuse("%s does not load as plain containers and tensors: %s" % (path, e))
    if not isinstance(st, dict) or st.get("format") != FORMAT:
        _refuse("%s is not a chained int8 model file (format %r, expected %r)"
                % (path, st.get("format") if isinstance(st, dict) else type(st).__name__, FORMAT))
    if st.get("version") != VERSION:
        _refuse("%s has format version %r; this dfq_b200 reads version %d" % (path, st.get("version"), VERSION))
    for k in _KEYS:
        _get(st, k, "the file")
    tensors = _get(st, "tensors", "the file", list)
    if not all(isinstance(t, torch.Tensor) for t in tensors):
        _refuse("the file's tensor table holds something else than tensors")
    tensors = [t.to(dev) for t in tensors]
    recs = _get(st, "modules", "the file", list)
    built = [None] * len(recs)
    mods = {}
    for p, i in _get(st, "paths", "the file", dict).items():
        _module_path(p, "module path")
        if type(i) is not int or not 0 <= i < len(recs):
            _refuse("path %r: module index %r out of range" % (p, i))
        mods[p] = _rebuild_module(i, recs, tensors, built)
    fns, g, env = functions(), fx.Graph(), {}
    for rec in _get(st, "nodes", "the file", list):
        name, op = _get(rec, "name", "a node", str), _get(rec, "op", "a node", str)
        target = _get(rec, "target", "node %s" % name, str)
        args = _decode(_get(rec, "args", "node %s" % name, dict), env, name)
        kwargs = {k: _decode(v, env, name) for k, v in _get(rec, "kwargs", "node %s" % name, dict).items()}
        if not isinstance(args, tuple):
            _refuse("node %s: its arguments are not a tuple" % name)
        _check_node(op, name, target, args, kwargs)
        if op == "call_function":
            if target not in fns:
                _refuse("node %s calls %r, which is not on the allowlist of a chained int8 model" % (name, target))
            target = fns[target]
        elif op == "call_method":
            if target not in METHODS:
                _refuse("node %s calls the tensor method %r, which is not on the allowlist" % (name, target))
        elif op == "call_module":
            if target not in mods:
                _refuse("node %s calls module %r, which the file does not hold" % (name, target))
        elif op not in ("placeholder", "output"):
            _refuse("node %s is a %r node" % (name, op))
        env[name] = node = g.create_node(op, target, args, kwargs, name=name)
        if node.name != name:
            _refuse("node name %r is not unique" % name)
    g.lint()
    gm = fx.GraphModule(mods, g, _identifier(_get(st, "class_name", "the file", str), "class name"))
    for p, m in mods.items():                                   # with the layers the graph does not call
        gm.add_submodule(p, m)
    records = _get(st, "records", "the file", dict)
    _get(records, "requantized_edges", "the records")
    for k, v in records.items():
        if k not in RECORDS:
            _refuse("unknown record %r" % k)
        setattr(gm, k, _plain(v, k))
    return gm
