"""The reference's int8 ncnn model, modeling/ncnn/model_quant_relu_equal.{param,bin}: the bundled MobileNetV2 after
`--quantize --relu --equalize` turned into int8 codes by ncnn2int8 from the table tests/ncnn_table_case.py reproduces.
Data of the reference, staged by `__graft_entry__.build()` (oracle/ref_data_int8.py) into the git-ignored oracle/_ref/.

Every Convolution / ConvolutionDepthWise / InnerProduct layer of the .bin is
    tag 0x000D4B38 | int8 weights [O, I/g, kh, kw] padded to 4 bytes | fp32 bias [O] | fp32 weight scales [O] (depthwise:
    [groups]) | fp32 input scale
with the weight size in .param key 6 (InnerProduct: 2), the bias flag in 5 (1), the group in 7.  parse() checks that these
records account for every byte of the file.

Int8Net interprets the whole .param (112 layers) with a pluggable executor for the weighted layers: the integer oracle
(oracle_executor), the GPU kernels, or fp32 F.conv2d with a calibrated model's weights (fp32_executor).
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")
TAG = 0x000D4B38


def paths():
    p = [os.path.join(REF, "model_quant_relu_equal." + e) for e in ("param", "bin")]
    return p if all(os.path.isfile(x) for x in p) else None


WEIGHTED = ("Convolution", "ConvolutionDepthWise", "InnerProduct")


def parse_param():
    """Every layer of the .param: [dict(type, name, bottoms, tops, params {key: int | float | [values]})] in file order.
    An array value is written `-23300-key=count,v0,v1,...` and stored under `key`."""
    layers = []
    for line in open(paths()[0]).read().splitlines()[2:]:
        f = line.split()
        nb, nt = int(f[2]), int(f[3])
        params = {}
        for item in f[4 + nb + nt:]:
            k, v = item.split("=")
            k = int(k)
            if k <= -23300:
                vals = [float(x) if "." in x or "e" in x else int(x) for x in v.split(",")]
                assert vals[0] == len(vals) - 1, "layer %s: array %s" % (f[1], item)
                params[-k - 23300] = vals[1:]
            else:
                params[k] = float(v) if "." in v or "e" in v else int(v)
        layers.append(dict(type=f[0], name=f[1], bottoms=f[4:4 + nb], tops=f[4 + nb:4 + nb + nt], params=params))
    return layers


def parse():
    """[dict(type, name, out, group, codes int8 [wsize], bias fp32 [O] | None, w_scales fp32, in_scale fp32, params)] of the
    weighted layers, in file order."""
    data = open(paths()[1], "rb").read()
    pos, layers = 0, []
    for lay in parse_param():
        if lay["type"] not in WEIGHTED:
            continue
        kv = lay["params"]
        fc = lay["type"] == "InnerProduct"
        out, wsize = kv[0], kv[2 if fc else 6]
        has_bias, group = kv.get(1 if fc else 5, 0), kv.get(7, 1)
        assert kv.get(8) in (1, 2), "layer %s is not int8" % lay["name"]
        assert np.frombuffer(data, "<u4", 1, pos)[0] == TAG, "bad tag at %d" % pos
        pos += 4
        codes = np.frombuffer(data, np.int8, wsize, pos).copy()
        pos += (wsize + 3) // 4 * 4
        bias = None
        if has_bias:
            bias = np.frombuffer(data, "<f4", out, pos).astype(np.float32); pos += 4 * out
        n_s = group if lay["type"] == "ConvolutionDepthWise" else out
        w_scales = np.frombuffer(data, "<f4", n_s, pos).astype(np.float32); pos += 4 * n_s
        in_scale = np.frombuffer(data, "<f4", 1, pos).astype(np.float32)[0]; pos += 4
        layers.append(dict(type=lay["type"], name=lay["name"], out=out, group=group, codes=codes, bias=bias,
                           w_scales=w_scales, in_scale=in_scale, params=kv))
    assert pos == len(data), "parsed %d of %d bytes" % (pos, len(data))
    return layers


# ---- interpreter ----------------------------------------------------------------------------------------------------
# The parameter keys each layer type implements (ncnn's numbering); anything else is refused.  Convolution keys: 0 num_output,
# 1 kernel, 2 dilation, 3 stride, 4 pad (the same on both axes: ncnn's _h keys 11-14 default to these), 5 bias term, 6 weight
# data size, 7 group (ConvolutionDepthWise), 8 int8 scale term.
KEYS = {
    "Input": {0, 1, 2}, "Convolution": {0, 1, 2, 3, 4, 5, 6, 8}, "ConvolutionDepthWise": {0, 1, 2, 3, 4, 5, 6, 7, 8},
    "ReLU": set(), "Split": set(), "BinaryOp": {0}, "Reshape": {0, 1}, "Reduction": {0, 1, 3}, "InnerProduct": {0, 1, 2, 8},
    "Softmax": {0},
}


def layer_spec(rec, index):
    """Geometry and data of one weighted layer: dict(index, name, type, O, C, k, stride, pad, dilation, groups, codes int8
    [O, C/g, k, k], bias fp32 [O] | None, w_scales fp32 [O], in_scale fp32)."""
    kv = rec["params"]
    O = kv[0]
    if rec["type"] == "InnerProduct":
        k, groups, stride, pad, dil = 1, 1, 1, 0, 1
    else:
        k, dil, stride, pad, groups = kv[1], kv.get(2, 1), kv.get(3, 1), kv.get(4, 0), kv.get(7, 1)
        if pad < 0:
            raise NotImplementedError("layer %s: SAME padding (%d) is not implemented" % (rec["name"], pad))
    Cg = rec["codes"].size // (O * k * k)
    assert Cg * O * k * k == rec["codes"].size, rec["name"]
    ws = rec["w_scales"]
    if rec["type"] == "ConvolutionDepthWise":
        assert groups == O == Cg * groups and ws.size == groups, rec["name"]       # one scale per group = per channel
    return dict(index=index, name=rec["name"], type=rec["type"], O=O, C=Cg * groups, k=(k, k), stride=(stride, stride),
                pad=(pad, pad), dilation=(dil, dil), groups=groups, codes=rec["codes"].reshape(O, Cg, k, k),
                bias=rec["bias"], w_scales=np.broadcast_to(ws, (O,)).astype(np.float32), in_scale=np.float32(rec["in_scale"]))


def spec_weight(spec):
    """fp32 weights codes / w_scale[o] from which the packer re-derives the codes (|code| <= 127, so fp32(c / s) * s rounds
    back to c)."""
    return (spec["codes"].astype(np.float32) / spec["w_scales"].reshape(-1, 1, 1, 1)).astype(np.float32)


class Int8Net:
    """Interpreter of model_quant_relu_equal.param.  Convolution, ConvolutionDepthWise and InnerProduct go through a pluggable
    executor(spec, x [N, C, H, W] fp32) -> y [N, O, OH, OW] (layer_spec; InnerProduct as a 1x1 convolution of [N, I, 1, 1]);
    everything else runs as plain torch fp32 ops on x's device.  This is this package's dequantizing scheme - fp32 between
    layers - not ncnn's fused requantize (DESIGN.md section 3.8)."""

    def __init__(self):
        self.layers = parse_param()
        recs = iter(parse())
        self.specs = []
        for lay in self.layers:
            if lay["type"] not in KEYS:
                raise NotImplementedError("layer %s: type %s is not implemented" % (lay["name"], lay["type"]))
            extra = set(lay["params"]) - KEYS[lay["type"]]
            if extra:
                raise NotImplementedError("layer %s (%s): parameter keys %s are not implemented" % (lay["name"], lay["type"],
                                                                                                     sorted(extra)))
            if lay["type"] in WEIGHTED:
                rec = next(recs)
                assert rec["name"] == lay["name"]
                lay["spec"] = layer_spec(rec, len(self.specs))
                self.specs.append(lay["spec"])
            p = lay["params"]
            if lay["type"] in ("BinaryOp", "Softmax") and p.get(0, 0) != 0:
                raise NotImplementedError("layer %s: %s with 0=%r" % (lay["name"], lay["type"], p[0]))
            if lay["type"] == "Reduction" and (p.get(0) != 3 or p.get(1, 1) != 0):
                raise NotImplementedError("layer %s: Reduction other than the mean over listed axes" % lay["name"])

    def forward(self, x, executor, upto=None):
        """OrderedDict blob name -> tensor for the batch x [N, 3, 224, 224] (the Input blob), through layer `upto`
        (a name; default: all)."""
        blobs = {}
        for lay in self.layers:
            t, p, ins = lay["type"], lay["params"], [blobs[b] for b in lay["bottoms"]]
            if t == "Input":
                assert tuple(x.shape[1:]) == (p[2], p[1], p[0]), x.shape
                outs = [x]
            elif t in WEIGHTED:
                s = lay["spec"]
                v = ins[0] if t != "InnerProduct" else ins[0].reshape(ins[0].shape[0], -1, 1, 1)
                assert v.shape[1] == s["C"], (lay["name"], v.shape)
                y = executor(s, v)
                outs = [y if t != "InnerProduct" else y.reshape(y.shape[0], -1)]
            elif t == "ReLU":
                outs = [torch.relu(ins[0])]
            elif t == "Split":
                outs = [ins[0]] * len(lay["tops"])
            elif t == "BinaryOp":
                outs = [ins[0] + ins[1]]
            elif t == "Reshape":                                               # ncnn w = key 0, h = key 1: a 2-D [h, w] blob
                outs = [ins[0].reshape(ins[0].shape[0], p[1], p[0])]
            elif t == "Reduction":                                             # mean over the listed axes (w = -1)
                v = ins[0]
                outs = [v.mean(dim=[a % (v.dim() - 1) + 1 for a in p[3]])]
            elif t == "Softmax":
                outs = [torch.softmax(ins[0], dim=1)]
            for name, o in zip(lay["tops"], outs):
                blobs[name] = o
            if upto is not None and lay["name"] == upto:
                break
        return blobs


def oracle_executor(spec, x):
    """The integer oracle (tests/int8_oracle.py) on the CPU: codes of x at in_scale, exact sums, the two-op epilogue."""
    import int8_oracle as I8
    xq = I8.i8_quantize(x.detach().cpu().numpy(), spec["in_scale"])
    acc = I8.i8_conv(xq, spec["codes"], spec["stride"], spec["pad"], spec["dilation"], spec["groups"])
    return torch.from_numpy(I8.i8_dequant(acc, spec["in_scale"], spec["w_scales"], spec["bias"]))


def fp32_executor(layers):
    """F.conv2d with the fp32 weights of `layers` (the 53 target modules, in graph order), on x's device."""
    import torch.nn.functional as F

    def run(spec, x):
        m = layers[spec["index"]]
        w = m.weight.reshape(spec["O"], -1, *spec["k"])
        return F.conv2d(x, w, m.bias, spec["stride"], spec["pad"], spec["dilation"], spec["groups"])
    return run


def calibrated_graph(monkeypatch):
    """(graph, targ) of tests/ncnn_table_case.run: the bundled checkpoint after BN fold, signed equalization and the
    activation ranges, through whichever library is installed."""
    import ncnn_table_case
    from dfq_b200 import export
    seen = {}
    orig = export.ncnn_scales

    def capture(graph, targ_type, **kw):
        seen["graph"], seen["targ"] = graph, targ_type
        return orig(graph, targ_type, **kw)

    monkeypatch.setattr(export, "ncnn_scales", capture)
    ncnn_table_case.run(monkeypatch)
    monkeypatch.setattr(export, "ncnn_scales", orig)
    return seen["graph"], seen["targ"]
