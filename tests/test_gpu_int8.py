"""Int8 execution on the H100 (dfq_i8_* in libdfq_sm90.so, dfq_b200.int8) against the integer oracle, bit for bit."""
import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_oracle as O

pytestmark = pytest.mark.gpu
f32 = np.float32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _wscale(w):
    return f32(128. / float(w.detach().abs().max()))


def _ascale(x):
    return f32(128. / float(x.abs().max()))


def _oracle(x, conv, a, ws):
    """(acc, y) of the int8 layer by the oracle, from the fp32 input and the module's fp32 weights."""
    xq = O.i8_quantize(x.detach().cpu().numpy(), a)
    w = conv.weight.detach().cpu().numpy()
    wq = O.i8_quantize(w, np.full(w.shape[0], ws, f32).reshape(-1, 1, 1, 1))
    acc = O.i8_conv(xq, wq, conv.stride, conv.padding, conv.dilation, conv.groups)
    b = None if conv.bias is None else conv.bias.detach().cpu().numpy()
    return acc, O.i8_dequant(acc, a, np.full(w.shape[0], ws, f32), b)


def _run_conv(N, Cin, H, W, Cout, k, s, p, d, g=1, seed=0, x=None, conv=None):
    from dfq_b200 import int8
    torch.manual_seed(seed)
    conv = conv or nn.Conv2d(Cin, Cout, k, s, p, d, g).cuda()
    x = torch.randn(N, Cin, H, W, device="cuda") * 2 if x is None else x
    a, ws = _ascale(x), _wscale(conv.weight)
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    y, acc = layer.run(x, with_acc=True)
    acc_ref, y_ref = _oracle(x, conv, a, ws)
    assert np.array_equal(acc.cpu().numpy(), acc_ref), "acc"
    assert np.array_equal(y.cpu().numpy().view(np.int32), y_ref.view(np.int32)), "y"
    return layer, x, y


def test_quantizer_and_packer_are_bit_exact_with_ties_saturation_and_negative_zero():
    from dfq_b200 import _lib, int8
    lib = _lib.load()
    ties = np.array([1, 3, -1, -3, 253, -253, 255, -255, 0.0, -0.0, 1e30, -1e30], f32)       # * 0.5: k + 0.5
    N, Cn, H, W = 2, 19, 5, 3
    x = np.random.default_rng(0).standard_normal((N, Cn, H, W)).astype(f32) * 100
    x.reshape(-1)[:ties.size] = ties
    xt = torch.from_numpy(x).cuda()
    q = torch.full((N * H * W * 32,), 99, dtype=torch.int8, device="cuda")
    _lib.check(lib.dfq_i8_quantize_nhwc(C.c_void_p(xt.data_ptr()), C.c_void_p(q.data_ptr()), N, Cn, H, W, 32, C.c_float(0.5),
                                        _lib.stream_ptr()), "quantize")
    got = q.cpu().numpy().reshape(N, H, W, 32)
    assert np.array_equal(got[..., :Cn], O.i8_quantize(x, f32(0.5)).transpose(0, 2, 3, 1))
    assert not got[..., Cn:].any()
    # packer: dense [O][kh][kw][Cpad] and depthwise [kh*kw][Cpad], per-channel scales with ties and saturation
    for groups, (O_, Cin) in ((1, (5, 21)), (21, (21, 21))):
        w = np.random.default_rng(1).standard_normal((O_, Cin // groups, 3, 2)).astype(f32)
        w.reshape(-1)[:ties.size] = ties
        conv = nn.Conv2d(Cin, O_, (3, 2), groups=groups, bias=False).cuda()
        with torch.no_grad():
            conv.weight.copy_(torch.from_numpy(w))
        ws = np.full(O_, f32(0.5), f32)
        layer = int8.Int8Conv2d(conv.weight, None, 1.0, ws, groups=groups)
        codes = layer.weight_codes.cpu().numpy()
        ref = O.i8_quantize(w, f32(0.5))
        if groups == 1:
            codes = codes.reshape(O_, 3, 2, 32)
            assert np.array_equal(codes[..., :Cin], ref.transpose(0, 2, 3, 1)) and not codes[..., Cin:].any()
        else:
            codes = codes.reshape(6, 32)
            assert np.array_equal(codes[:, :Cin], ref.reshape(Cin, 6).T) and not codes[:, Cin:].any()


DENSE = [  # (N, Cin, H, W, Cout, k, stride, pad, dil)
    (1, 3, 15, 15, 8, 3, 1, 1, 1), (3, 16, 8, 9, 24, 1, 2, 0, 1), (1, 24, 17, 16, 100, 7, 2, 3, 1),
    (3, 96, 10, 10, 1000, 1, 1, 0, 1), (1, 160, 9, 7, 24, 3, 1, 3, 2), (1, 512, 7, 7, 100, 3, 2, 1, 1),
    (3, 3, 30, 31, 24, 7, 2, 3, 1), (1, 16, 20, 20, 8, 3, 1, 3, 6), (1, 24, 5, 5, 8, 3, 1, 0, 1),
    (3, 512, 1, 1, 1000, 1, 1, 0, 1), (1, 96, 7, 7, 24, 7, 1, 0, 1), (1, 160, 11, 12, 8, 3, 2, 1, 2),
    (3, 24, 14, 13, 1000, 3, 1, 1, 1), (1, 3, 224, 224, 24, 3, 2, 1, 1), (3, 512, 6, 5, 8, 1, 2, 0, 1),
    (1, 16, 13, 13, 100, 3, 2, 0, 6), (3, 160, 4, 4, 100, 7, 1, 3, 1),
]


@pytest.mark.parametrize("case", DENSE, ids=lambda c: "x".join(map(str, c)))
def test_dense_conv_acc_and_output_bit_exact(case):
    _run_conv(*case, seed=sum(case))


def test_dense_conv_accumulates_beyond_2_pow_24_exactly():
    """All codes +-127 with K = 3*3*512 = 4608: |acc| reaches 127^2 * 4608 = 74,322,432 > 2^24, where fp32_rn(acc) rounds."""
    conv = nn.Conv2d(512, 24, 3, 1, 1, bias=True).cuda()
    with torch.no_grad():
        sign = torch.ones(24, 512, 3, 3)
        sign[1::2, ::3] = -1
        conv.weight.copy_(sign)
    x = torch.ones(1, 512, 6, 6, device="cuda")
    layer = _run_conv(1, 512, 6, 6, 24, 3, 1, 1, 1, x=x, conv=conv)[0]
    acc = layer.run(x, with_acc=True)[1]
    assert int(acc.max()) == 127 * 127 * 4608 and int(acc.abs().max()) > 2 ** 24


DW = [  # (N, C, H, W, k, stride, pad, dil)
    (1, 32, 15, 15, 3, 1, 1, 1), (3, 96, 14, 13, 3, 2, 1, 1), (1, 144, 9, 9, 3, 1, 2, 2), (1, 24, 17, 16, 3, 2, 4, 4),
    (3, 19, 8, 8, 5, 1, 2, 1), (1, 960, 7, 7, 3, 1, 1, 1), (1, 40, 3, 3, 3, 1, 0, 1), (1, 16, 11, 10, 7, 2, 3, 2),
]


@pytest.mark.parametrize("case", DW, ids=lambda c: "x".join(map(str, c)))
def test_depthwise_conv_acc_and_output_bit_exact(case):
    N, Cn, H, W, k, s, p, d = case
    _run_conv(N, Cn, H, W, Cn, k, s, p, d, g=Cn, seed=sum(case))


@pytest.mark.parametrize("B", [1, 7, 256])
def test_linear_bit_exact(B):
    from dfq_b200 import int8
    torch.manual_seed(B)
    lin = nn.Linear(1280, 1000).cuda()
    x = torch.randn(B, 1280, device="cuda")
    a, ws = _ascale(x), _wscale(lin.weight)
    layer = int8.Int8Linear.from_linear(lin, a, ws)
    y = layer(x)
    conv = nn.Conv2d(1280, 1000, 1).cuda()
    with torch.no_grad():
        conv.weight.copy_(lin.weight.reshape(1000, 1280, 1, 1)); conv.bias.copy_(lin.bias)
    _, y_ref = _oracle(x.reshape(B, 1280, 1, 1), conv, a, ws)
    assert y.shape == (B, 1000) and np.array_equal(y.cpu().numpy(), y_ref.reshape(B, 1000))


def test_refusals():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="groups"):
        int8.Int8Conv2d.from_conv(nn.Conv2d(8, 8, 3, groups=2).cuda(), 1.0, 1.0)
    # the C ABI itself refuses the grouping and names the condition
    lib = _lib.load()
    g = np.zeros(1, _lib.I8_CONV_DT)
    for k, v in dict(N=1, C=8, H=4, W=4, O=8, kh=1, kw=1, stride_h=1, stride_w=1, dil_h=1, dil_w=1, groups=2, OH=4, OW=4,
                     Cpad=16).items():
        g[0][k] = v
    buf = torch.zeros(1024, dtype=torch.int8, device="cuda")
    f = torch.zeros(1024, device="cuda")
    rc = lib.dfq_i8_conv(C.c_void_p(buf.data_ptr()), C.c_void_p(buf.data_ptr()), C.c_void_p(f.data_ptr()), None,
                         C.c_void_p(f.data_ptr()), None, _lib.table_ptr(g), _lib.stream_ptr())
    assert rc == -2 and b"groups=2" in lib.dfq_last_error()
    layer = int8.Int8Conv2d.from_conv(nn.Conv2d(8, 8, 3).cuda(), 1.0, 1.0)
    with pytest.raises(_lib.DfqError, match="GPU"):
        layer(torch.randn(1, 8, 5, 5))


def test_single_layer_twin_of_dequantized_codes():
    """F.conv2d (TF32 off) on the dequantized codes is the float model of the int8 layer: they agree to 1e-5 normwise."""
    from dfq_b200 import int8
    torch.manual_seed(3)
    conv = nn.Conv2d(96, 100, 3, 1, 1).cuda()
    x = torch.randn(2, 96, 14, 14, device="cuda")
    a, ws = _ascale(x), _wscale(conv.weight)
    y = int8.Int8Conv2d.from_conv(conv, a, ws)(x)
    xd = torch.from_numpy(O.i8_quantize(x.cpu().numpy(), a).astype(f32) / a).cuda()
    wd = torch.from_numpy(O.i8_quantize(conv.weight.detach().cpu().numpy(), ws).astype(f32) / ws).cuda()
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        twin = F.conv2d(xd, wd, conv.bias, 1, 1)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    err = float((y - twin).norm() / twin.norm())
    assert err < 1e-5, err


def _convert_and_check_every_layer(model, x):
    """Convert every Conv2d / Linear of `model` (activation scales from a float forward's max|input|) and check each int8
    layer's output against the oracle on the input it saw in the int8 forward."""
    from dfq_b200 import int8
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    layers = list(graph.values())
    amax = {}
    hooks = [m.register_forward_pre_hook(lambda m, inp: amax.__setitem__(id(m), max(amax.get(id(m), 0.0),
                                                                                    float(inp[0].abs().max())))) for m in layers]
    with torch.no_grad():
        model(x)
    for h in hooks:
        h.remove()
    acts = [128. / amax[id(m)] for m in layers]
    names = int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=acts)
    assert len(names) == len(layers)
    seen = {}
    mods = dict(model.named_modules())
    for n in names:
        mods[n].register_forward_hook(lambda m, inp, out, n=n: seen.__setitem__(n, (inp[0], out)))
    with torch.no_grad():
        model(x)
    for n, src, a in zip(names, layers, acts):
        inp, out = seen[n]
        conv = src
        if isinstance(src, nn.Linear):
            conv = nn.Conv2d(src.in_features, src.out_features, 1).cuda()
            with torch.no_grad():
                conv.weight.copy_(src.weight.reshape(conv.weight.shape)); conv.bias.copy_(src.bias)
            inp, out = inp.reshape(inp.shape[0], -1, 1, 1), out.reshape(out.shape[0], -1, 1, 1)
        _, y_ref = _oracle(inp, conv, f32(a), _wscale(src.weight))
        assert np.array_equal(out.cpu().numpy(), y_ref), n
    return names


def test_resnet18_every_layer_bit_exact():
    """torchvision ResNet-18 (seeded): the 7x7/s2 stem, 3x3 convs, 1x1/s2 downsamples and the classifier."""
    import torchvision
    torch.manual_seed(0)
    model = torchvision.models.resnet18(num_classes=1000).cuda().eval()
    names = _convert_and_check_every_layer(model, torch.randn(2, 3, 224, 224, device="cuda"))
    assert "conv1" in names and "layer2.0.downsample.0" in names and "fc" in names


def test_mobilenetv2_every_layer_bit_exact():
    """torchvision MobileNetV2 (seeded, ReLU6 -> ReLU): dense, depthwise and pointwise layers and the classifier."""
    import torchvision
    torch.manual_seed(1)
    model = torchvision.models.mobilenet_v2(num_classes=1000).cuda().eval()
    for m in model.modules():
        for k, c in m.named_children():
            if isinstance(c, nn.ReLU6):
                setattr(m, k, nn.ReLU())
    names = _convert_and_check_every_layer(model, torch.randn(1, 3, 224, 224, device="cuda"))
    assert len(names) == 53


def test_reference_int8_model_codes_from_the_cuda_calibration(monkeypatch):
    """The bundled checkpoint calibrated by libdfq_sm90.so (BN fold, signed equalization) and converted with the table's
    activation scales: the packed codes reproduce the reference's int8 model (ncnn2int8 output) to the CPU bound, and the
    converted layers carry its biases."""
    import ncnn_int8_case as case
    import ncnn_table_case
    from dfq_b200 import int8
    if case.paths() is None or ncnn_table_case.checkpoint_path() is None:
        pytest.skip("reference int8 model / checkpoint not staged in oracle/_ref")
    graph, targ = case.calibrated_graph(monkeypatch)
    rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    holder = nn.ModuleList(layers).cuda()
    names = int8.convert_to_int8(holder, graph, targ, act_scales=list(rows["activation_scales"]))
    ref = case.parse()
    same = total = 0
    for n, r in zip(names, ref):
        m = holder[int(n)]
        codes = m.weight_codes.cpu().numpy()
        if m.groups == 1:
            kh, kw = m.kernel_size
            codes = codes.reshape(m.out_channels, kh, kw, m.cpad)[..., :m.in_channels].transpose(0, 3, 1, 2).reshape(-1)
        else:
            codes = codes.reshape(-1, m.cpad)[:, :m.in_channels].T.reshape(-1)
        d = np.abs(codes.astype(np.int16) - r["codes"].astype(np.int16))
        assert d.max() <= 1, n
        same += int((d == 0).sum()); total += d.size
        assert np.abs(m.bias.cpu().numpy() - r["bias"]).max() <= 1e-5 * np.abs(r["bias"]).max(), n
    print("reference int8 codes from the CUDA calibration: %d of %d" % (same, total))
    assert total == 3_469_760 and same >= 3_469_750
