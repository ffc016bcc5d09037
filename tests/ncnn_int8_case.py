"""The reference's int8 ncnn model, modeling/ncnn/model_quant_relu_equal.{param,bin}: the bundled MobileNetV2 after
`--quantize --relu --equalize` turned into int8 codes by ncnn2int8 from the table tests/ncnn_table_case.py reproduces.
Data of the reference, staged by `__graft_entry__.build()` (oracle/ref_data_int8.py) into the git-ignored oracle/_ref/.

Every Convolution / ConvolutionDepthWise / InnerProduct layer of the .bin is
    tag 0x000D4B38 | int8 weights [O, I/g, kh, kw] padded to 4 bytes | fp32 bias [O] | fp32 weight scales [O] (depthwise:
    [groups]) | fp32 input scale
with the weight size in .param key 6 (InnerProduct: 2), the bias flag in 5 (1), the group in 7.  parse() checks that these
records account for every byte of the file.
"""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")
TAG = 0x000D4B38


def paths():
    p = [os.path.join(REF, "model_quant_relu_equal." + e) for e in ("param", "bin")]
    return p if all(os.path.isfile(x) for x in p) else None


def parse():
    """[dict(type, name, out, group, codes int8 [wsize], bias fp32 [O] | None, w_scales fp32, in_scale fp32)] in file order."""
    param, binf = paths()
    data = open(binf, "rb").read()
    pos, layers = 0, []
    for line in open(param).read().splitlines()[2:]:
        f = line.split()
        if f[0] not in ("Convolution", "ConvolutionDepthWise", "InnerProduct"):
            continue
        kv = dict(x.split("=") for x in f[4 + int(f[2]) + int(f[3]):])
        fc = f[0] == "InnerProduct"
        out, wsize = int(kv["0"]), int(kv["2" if fc else "6"])
        has_bias, group = int(kv.get("1" if fc else "5", 0)), int(kv.get("7", 1))
        assert kv.get("8") in ("1", "2"), "layer %s is not int8" % f[1]
        assert np.frombuffer(data, "<u4", 1, pos)[0] == TAG, "bad tag at %d" % pos
        pos += 4
        codes = np.frombuffer(data, np.int8, wsize, pos).copy()
        pos += (wsize + 3) // 4 * 4
        bias = None
        if has_bias:
            bias = np.frombuffer(data, "<f4", out, pos).astype(np.float32); pos += 4 * out
        n_s = group if f[0] == "ConvolutionDepthWise" else out
        w_scales = np.frombuffer(data, "<f4", n_s, pos).astype(np.float32); pos += 4 * n_s
        in_scale = np.frombuffer(data, "<f4", 1, pos).astype(np.float32)[0]; pos += 4
        layers.append(dict(type=f[0], name=f[1], out=out, group=group, codes=codes, bias=bias, w_scales=w_scales,
                           in_scale=in_scale))
    assert pos == len(data), "parsed %d of %d bytes" % (pos, len(data))
    return layers


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
