"""Int8 execution without a GPU: the integer oracle (tests/int8_oracle.py), the reference's int8 ncnn model against the
calibration this package computes, and the host path of dfq_b200.int8 (packing plan, scale choice, module swap,
read_ncnn_table) through the oracle-backed fake library."""
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import fakelib
import fakelib_int8
import int8_oracle as O

f32 = np.float32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_quantizer_rounds_ties_away_from_zero_and_clamps():
    s = f32(0.5)
    v = np.array([1, 3, 5, -1, -3, -5, 253, -253, 255, -255, 1e30, -1e30, 0.0, -0.0], f32)   # v * 0.5 = k + 0.5 exactly
    assert np.all((v[:10] * s) % 1 == 0.5)
    got = O.i8_quantize(v, s)
    assert got.dtype == np.int8
    assert got.tolist() == [1, 2, 3, -1, -2, -3, 127, -127, 127, -127, 127, -127, 0, 0]
    # the product is rounded to fp32 first: 0.49999997 * 1 stays below the tie, 2.5 - ulp rounds down
    assert O.i8_quantize(np.array([np.nextafter(f32(0.5), f32(0)), np.nextafter(f32(2.5), f32(0))], f32), 1.0).tolist() == [0, 2]
    assert O.i8_quantize(np.array([-128.0, 126.5], f32), 1.0).tolist() == [-127, 127]


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


GRID = [  # (N, C, H, W, O, k, stride, pad, dil, groups); k / stride / pad / dil: an int, or (h, w)
    (1, 3, 9, 9, 8, 3, 1, 1, 1, 1), (3, 16, 8, 7, 24, 1, 2, 0, 1, 1), (1, 24, 11, 10, 100, 7, 2, 3, 1, 1),
    (2, 5, 13, 13, 6, 3, 1, 3, 6, 1), (1, 12, 7, 7, 12, 3, 2, 1, 1, 12), (2, 8, 10, 9, 8, 5, 1, 4, 2, 8),
    (1, 6, 3, 3, 4, 3, 1, 0, 1, 1), (1, 8, 6, 6, 8, 3, 1, 1, 1, 2),
    # off the square: every pair below has different h and w values, so a swapped axis changes the sums
    (2, 5, 9, 11, 7, (1, 7), 1, (0, 3), 1, 1), (1, 6, 11, 8, 6, (7, 1), 1, (3, 0), 1, 6),             # 1x7 dense, 7x1 dw
    (2, 4, 10, 13, 5, (3, 5), (2, 1), (1, 2), (1, 2), 1), (1, 9, 12, 10, 9, (3, 5), (2, 1), (1, 2), (1, 2), 9),
    (1, 3, 13, 14, 4, (5, 3), (1, 3), 0, (2, 1), 1), (2, 7, 13, 14, 7, (5, 3), (1, 3), 0, (2, 1), 7),
    (2, 10, 5, 6, 10, 1, (1, 2), 0, 1, 10),                                                           # 1x1 dw
    (2, 6, 7, 5, 8, (2, 3), (3, 2), (2, 1), (2, 1), 2),                                               # grouped
]


@pytest.mark.parametrize("case", GRID)
def test_integer_conv_oracle_equals_float64_conv(case):
    N, Cn, H, W, Oc, k, s, p, d, g = case
    k, s, p, d = map(_pair, (k, s, p, d))
    rng = np.random.default_rng(hash(case) % 2 ** 32)
    x = rng.integers(-127, 128, (N, Cn, H, W))
    w = rng.integers(-127, 128, (Oc, Cn // g) + k)
    acc = O.i8_conv(x, w, s, p, d, g)
    ref = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, s, p, d, g).numpy()
    assert acc.dtype == np.int64 and acc.shape == ref.shape and np.array_equal(acc, ref.astype(np.int64))


def test_quantizer_maps_nan_products_to_minus_127():
    """NaN (a NaN input, inf * 0, 0 * inf) -> -127 like the kernel's fminf(fmaxf(NaN, -127), 127); +-inf and products that
    overflow fp32 clamp to +-127; subnormal inputs are not flushed: 1e-38 * 3e38 = 3."""
    v = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, 1e30, -1e30, 1.1e-38, -1.1e-38], f32)
    s = np.array([1.0, 1.0, 0.0, 0.0, np.inf, 1e10, 1e10, 3e38, 3e38], f32)
    assert O.i8_quantize(v, s).tolist() == [-127, -127, -127, -127, -127, 127, -127, 3, -3]
    assert O.i8_quantize(np.array([np.nan, 2.0], f32), f32(np.nan)).tolist() == [-127, -127]


def test_dequant_epilogue_is_two_rounded_fp32_ops():
    acc = np.array([[[[2 ** 24 + 1]], [[-7]], [[5]]]], np.int64)           # 2^24 + 1 is not an fp32: rounds to even
    a, ws, b = f32(48.484846), np.array([163.08817, 0.0, 3.0], f32), np.array([0.25, 1.0, -0.0], f32)
    y = O.i8_dequant(acc, a, ws, b)
    dq0 = f32(1) / (a * ws[0])
    assert y[0, 0, 0, 0] == f32(f32(2 ** 24) * dq0) + f32(0.25)
    assert y[0, 1, 0, 0] == f32(1.0)                                        # zero scale: dq 0, the bias remains
    assert y[0, 2, 0, 0] == f32(5) * (f32(1) / (a * ws[2]))


# ---- the reference's int8 ncnn model -------------------------------------------------------------------------------
def _staged():
    import ncnn_int8_case as case
    import ncnn_table_case
    if case.paths() is None or ncnn_table_case.checkpoint_path() is None:
        pytest.skip("reference int8 model / checkpoint not staged in oracle/_ref")
    return case


def test_reference_int8_model_parses_completely():
    case = _staged()
    layers = case.parse()
    assert len(layers) == 53 and sum(l["codes"].size for l in layers) == 3_469_760
    assert min(int(l["codes"].min()) for l in layers) == -127                  # never -128: the clamp is +-127
    rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
    assert np.array_equal(np.array([l["w_scales"][0] for l in layers]), rows["weight_scales"].astype(f32))
    assert np.abs(np.array([l["in_scale"] for l in layers]) / rows["activation_scales"] - 1).max() < 1e-6


def test_reference_codes_and_biases_from_this_calibration(monkeypatch):
    """Oracle-calibrated weights (BN fold + signed CLE on the bundled checkpoint) quantized with the table's weight scales
    reproduce the reference's int8 codes but for last-bit weight differences (DESIGN.md section 4); its biases agree."""
    case = _staged()
    fakelib.install(monkeypatch, fakelib.torch_sqrt)
    graph, targ = case.calibrated_graph(monkeypatch)
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    ref = case.parse()
    rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
    same = total = 0
    worst_bias = 0.0
    for m, r, ws in zip(layers, ref, rows["weight_scales"]):
        codes = O.i8_quantize(m.weight.detach().numpy().reshape(-1), f32(ws)).astype(np.int16)
        d = np.abs(codes - r["codes"].astype(np.int16))
        assert d.max() <= 1, r["name"]
        same += int((d == 0).sum()); total += d.size
        b = m.bias.detach().numpy()
        worst_bias = max(worst_bias, float(np.abs(b - r["bias"]).max() / np.abs(b).max()))
    print("reference int8 codes reproduced: %d of %d; worst bias error %.3g of the layer's max|bias|" % (same, total, worst_bias))
    assert total == 3_469_760 and same >= 3_469_750
    assert worst_bias < 2e-6


def test_interpreter_walks_all_112_layers_in_the_order_of_the_topology():
    """Int8Net consumes every layer of the .param; its Convolution / ConvolutionDepthWise / InnerProduct sequence is the 53
    target layers of topology_mobilenetv2.json, in order and geometry."""
    import json
    case = _staged()
    net = case.Int8Net()
    assert len(net.layers) == 112 and len(net.specs) == 53
    topo = json.load(open(os.path.join(GOLD, "topology_mobilenetv2.json")))
    targets = [n for n in topo["nodes"] if n["type"] in ("Conv2d", "Linear")]
    assert len(targets) == 53
    for s, n in zip(net.specs, targets):
        a = n["args"]
        if n["type"] == "Linear":
            got = (s["type"], s["C"], s["O"], s["k"], s["groups"])
            assert got == ("InnerProduct", a["in_features"], a["out_features"], (1, 1), 1), s["name"]
        else:
            assert s["type"] == ("ConvolutionDepthWise" if a["groups"] > 1 else "Convolution"), s["name"]
            assert (s["C"], s["O"], s["groups"]) == (a["in_channels"], a["out_channels"], a["groups"]), s["name"]
            assert (s["k"], s["stride"], s["pad"], s["dilation"]) == tuple(tuple(a[k]) for k in (
                "kernel_size", "stride", "padding", "dilation")), s["name"]


def test_interpreter_refuses_what_it_does_not_implement(monkeypatch):
    case = _staged()
    layers = case.parse_param()
    for edit, msg in ((lambda l: l[4]["params"].__setitem__(11, 5), r"keys \[11\]"),
                      (lambda l: l[4].__setitem__("type", "Pooling"), "type Pooling"),
                      (lambda l: [x for x in l if x["type"] == "BinaryOp"][0]["params"].__setitem__(0, 2), "BinaryOp")):
        changed = [dict(x, params=dict(x["params"])) for x in layers]
        edit(changed)
        monkeypatch.setattr(case, "parse_param", lambda changed=changed: changed)
        with pytest.raises(NotImplementedError, match=msg):
            case.Int8Net()


def test_reference_int8_mobilenetv2_rehearsal_on_the_cpu(monkeypatch):
    """The comparisons of the -m gpu end-to-end tests with the oracle executor and the oracle-backed library: the
    reference's int8 model and this package's calibration converted to int8 against the calibrated fp32 model.  The
    thresholds are test_gpu_int8.py's (measured here: 0.26-0.27, 0.10, top-1 4 of 4)."""
    import test_gpu_int8 as G
    from dfq_b200 import int8
    case = _staged()
    net = case.Int8Net()
    fakelib_int8.install(monkeypatch, fakelib.torch_sqrt)
    graph, targ = case.calibrated_graph(monkeypatch)
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    x = G._ref_images()
    with torch.no_grad():
        fp32 = net.forward(x, case.fp32_executor(layers))["781"]
        theirs = net.forward(x, case.oracle_executor)["781"]
        holder = nn.ModuleList(layers)
        rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
        int8.convert_to_int8(holder, graph, targ, act_scales=list(rows["activation_scales"]))
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        ours = net.forward(x, lambda s, v: holder[s["index"]].run(v)[0])["781"]
    top1 = lambda a, b: float((a.argmax(1) == b.argmax(1)).float().mean())
    print("int8 vs fp32: reference codes %.4g, this calibration %.4g; this calibration vs reference codes %.4g" % (
        G._rel(theirs, fp32), G._rel(ours, fp32), G._rel(ours, theirs)))
    assert G._rel(theirs, fp32) < G.INT8_VS_FP32_REL and G._rel(ours, fp32) < G.INT8_VS_FP32_REL
    assert G._rel(ours, theirs) < G.PKG_VS_REF_REL
    assert top1(theirs, fp32) >= G.TOP1_AGREE and top1(ours, fp32) >= G.TOP1_AGREE


# ---- host path of dfq_b200.int8 ------------------------------------------------------------------------------------
class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.features = nn.Sequential(nn.Conv2d(3, 16, 3, 2, 1), nn.ReLU(), nn.Conv2d(16, 16, 3, 1, 2, 2, groups=16), nn.ReLU())
        self.head = nn.Linear(16, 10)

    def forward(self, x):
        return self.head(self.features(x).mean((2, 3)))


def _graph(model):
    """The target-layer nodes of the tracer's graph (keys id(module), graph order) - all that the converter reads."""
    return OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))


def test_convert_to_int8_packs_scales_and_swaps_through_the_fake_library(monkeypatch):
    from dfq_b200 import _lib, int8
    fake = fakelib_int8.install(monkeypatch)
    torch.manual_seed(0)
    model = _Net().eval()
    w = [model.features[0].weight, model.features[2].weight, model.head.weight]
    with torch.no_grad():
        model.features[2].weight[3].zero_()                                    # a zero channel packs to zeros
    graph = _graph(model)
    targ = [nn.Conv2d, nn.Linear]
    acts = [40.0, 12.5, 3.0]
    ws_ref = [f32(128. / float(t.detach().abs().max())) for t in w]
    names = int8.convert_to_int8(model, graph, targ, act_scales=acts)
    assert names == ["features.0", "features.2", "head"]
    assert isinstance(model.features[0], int8.Int8Conv2d) and isinstance(model.features[2], int8.Int8Conv2d)
    assert isinstance(model.head, int8.Int8Linear) and fake.calls.count("dfq_i8_pack_weights") == 3
    dense, dw, fc = model.features[0], model.features[2], model.head
    assert dense.cpad == 16 and dw.cpad == 16 and fc.cpad == 16
    codes = dense.weight_codes.numpy().reshape(16, 3, 3, 16)                   # [O][kh][kw][Cpad]
    assert np.array_equal(codes[..., :3], O.i8_quantize(w[0].detach().numpy(), ws_ref[0]).transpose(0, 2, 3, 1))
    assert not codes[..., 3:].any()
    dcodes = dw.weight_codes.numpy().reshape(9, 16)                            # [kh*kw][Cpad]
    assert np.array_equal(dcodes, O.i8_quantize(w[1].detach().numpy(), ws_ref[1]).reshape(16, 9).T)
    assert not dcodes[:, 3].any()
    for mod, a, ws in zip((dense, dw, fc), acts, ws_ref):
        assert mod.act_scale == float(f32(a)) and np.all(mod.w_scale.numpy() == ws)
        assert np.array_equal(mod.dq.numpy(), (f32(1) / (f32(a) * np.full(mod.out_channels, ws, f32))).astype(f32))
    with pytest.raises(_lib.DfqError, match="GPU"):
        model(torch.randn(1, 3, 8, 8))


def test_convert_to_int8_uses_the_observers_and_refuses_what_it_cannot_run(monkeypatch):
    from dfq_b200 import _lib, export, int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8.install(monkeypatch)
    model = nn.Sequential(Q.QuantNConv2d(8, 16, 3, padding=1), nn.ReLU(), Q.QuantNConv2d(16, 16, 1, groups=2))
    graph = _graph(model)
    targ = [Q.QuantNConv2d]
    for m, (lo, hi) in zip((model[0], model[2]), ((-2.0, 3.2), (0.0, 0.0))):
        m.quant.running_min.fill_(lo); m.quant.running_max.fill_(hi)
    with pytest.raises(_lib.DfqError, match=r"layer 2 .*cannot run in int8"):
        int8.convert_to_int8(model, graph, targ)
    assert isinstance(model[0], Q.QuantNConv2d)                                # nothing replaced
    with pytest.raises(_lib.DfqError, match="act_scales has 1 entries"):
        int8.convert_to_int8(model, graph, targ, act_scales=[1.0])
    model2 = nn.Sequential(Q.QuantNConv2d(8, 16, 3, padding=1), nn.ReLU(), Q.QuantNConv2d(16, 16, 1))
    model2[0].quant.running_min.fill_(-2.0); model2[0].quant.running_max.fill_(3.2)      # model2[2]: zero range
    g2 = _graph(model2)
    assert int8.convert_to_int8(model2, g2, targ) == ["0", "2"]
    assert model2[0].act_scale == float(f32(128. / 3.2)) and model2[2].act_scale == 0.0
    with pytest.raises(ZeroDivisionError):                                     # export's default is unchanged
        export.ncnn_scales(g2, targ)
    assert not model2[2].dq.numpy().any()
    with pytest.raises(_lib.DfqError, match="no activation range"):
        m3 = nn.Sequential(nn.Conv2d(4, 4, 1))
        int8.convert_to_int8(m3, _graph(m3), [nn.Conv2d])


def test_fake_library_runs_the_abi_end_to_end(monkeypatch):
    """The three entries' host twins compose: quantize -> pack -> conv equals the oracle chain (a CPU rehearsal of the -m gpu
    tests' comparison)."""
    from dfq_b200 import int8
    fakelib_int8.install(monkeypatch)
    torch.manual_seed(1)
    conv = nn.Conv2d(5, 7, 3, 2, 1)
    layer = int8.Int8Conv2d.from_conv(conv, 30.0, f32(128. / float(conv.weight.abs().max())))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    x = torch.randn(2, 5, 9, 8)
    y, acc = layer.run(x, with_acc=True)
    xq = O.i8_quantize(x.numpy(), f32(30.0))
    wq = O.i8_quantize(conv.weight.detach().numpy(), layer.w_scale.numpy()[0])
    ref_acc = O.i8_conv(xq, wq, (2, 2), (1, 1), (1, 1), 1)
    assert np.array_equal(acc.numpy(), ref_acc)
    assert np.array_equal(y.numpy(), O.i8_dequant(ref_acc, 30.0, layer.w_scale.numpy(), conv.bias.detach().numpy()))


def test_read_ncnn_table_inverts_write_ncnn_table(monkeypatch, tmp_path):
    from dfq_b200 import export
    from dfq_b200.utils import quantize as Q
    fakelib_int8.install(monkeypatch)
    torch.manual_seed(2)
    model = nn.Sequential(Q.QuantNConv2d(3, 8, 3), nn.ReLU(), Q.QuantNConv2d(8, 4, 1), nn.Flatten(), Q.QuantNLinear(4 * 4, 3))
    for i, m in enumerate((model[0], model[2], model[4])):
        m.quant.running_min.fill_(-1.0 - i); m.quant.running_max.fill_(0.5 + 3 * i)
    graph = _graph(model)
    path = str(tmp_path / "t.table")
    rows = export.write_ncnn_table(graph, path, [Q.QuantNConv2d, Q.QuantNLinear], ["a", "b", "c"])
    names, back = export.read_ncnn_table(path)
    assert names == ["a", "b", "c"] and back == rows
    with open(path, "a") as f:
        f.write("d_param_0 1.0 2.0\n")
    with pytest.raises(ValueError, match="differ"):
        export.read_ncnn_table(path)



@pytest.mark.parametrize("bad", [float("inf"), float("nan"), -2.0, 1.28e40])
def test_non_finite_or_negative_scales_are_refused(monkeypatch, bad):
    """128 / range of a range below about 3.8e-37 is inf in fp32: refused, by the layer and by the converter, naming the
    layer and the range, before anything is replaced."""
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8.install(monkeypatch)
    conv = nn.Conv2d(4, 6, 3)
    with pytest.raises(_lib.DfqError, match=r"activation scale .*\(range 128 / scale"):
        int8.Int8Conv2d.from_conv(conv, bad, 1.0)
    ws = np.ones(6, f32)
    ws[4] = bad
    with pytest.raises(_lib.DfqError, match="weight scale .* of channel 4"):
        int8.Int8Conv2d.from_conv(conv, 1.0, ws)
    model = nn.Sequential(Q.QuantNConv2d(4, 8, 3, padding=1), nn.ReLU(), Q.QuantNConv2d(8, 8, 1))
    model[0].quant.running_min.fill_(-1.0); model[0].quant.running_max.fill_(1.0)
    model[2].quant.running_min.fill_(0.0); model[2].quant.running_max.fill_(1e-38)        # 128 / 1e-38: inf in fp32
    with pytest.raises(_lib.DfqError, match=r"layer 2: activation scale 1.28e\+40 \(range 128 / scale = 1e-38\)"):
        int8.convert_to_int8(model, _graph(model), [Q.QuantNConv2d])
    with pytest.raises(_lib.DfqError, match="layer 0: activation scale"):
        int8.convert_to_int8(model, _graph(model), [Q.QuantNConv2d], act_scales=[bad, 1.0])
    assert isinstance(model[0], Q.QuantNConv2d) and isinstance(model[2], Q.QuantNConv2d)   # nothing replaced
