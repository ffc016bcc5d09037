"""Int8 chaining on the H100: dfq_i8_conv_requant against the integer oracle byte for byte, and dfq_b200.int8.chain_int8
on whole models bit for bit against the per-layer path."""
import ctypes as C
import math
from collections import Counter, OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_chain_oracle as CO
import int8_oracle as O
import test_gpu_int8 as G

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
SENTINEL, TAIL = -128, 64                        # never a code (the clamp is +-127); bytes checked past the end of yq
ACTS = {"none": (-INF, INF), "relu": (0.0, INF), "relu6": (0.0, 6.0), "hardtanh": (-1.0, 2.5)}


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _requant_abi(layer, xq_nhwc, out_scale, lo, hi, offset=0):
    """dfq_i8_conv_requant of `layer` on codes xq [N, H, W, cpad] into a sentinel-filled buffer with a sentinel tail; returns
    (rc, the whole buffer as numpy).  offset shifts yq off its 16-byte alignment."""
    from dfq_b200 import _lib
    N, H, W, _ = xq_nhwc.shape
    g = layer._geometry(N, H, W)
    n = N * int(g[0]["OH"]) * int(g[0]["OW"]) * ((layer.out_channels + 15) // 16 * 16)
    buf = torch.full((n + TAIL + 16,), SENTINEL, dtype=torch.int8, device="cuda")
    xq = torch.from_numpy(np.ascontiguousarray(xq_nhwc)).cuda()
    rc = _lib.load().dfq_i8_conv_requant(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias),
                                         C.c_void_p(buf.data_ptr() + offset), C.c_float(out_scale), C.c_float(lo),
                                         C.c_float(hi), _lib.table_ptr(g), _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc, buf.cpu().numpy()[offset:offset + n + TAIL], n


def _check_requant(conv, x, a, ws, lo, hi, out_scale=None):
    """Run dfq_i8_conv_requant on the oracle's codes of x and compare every byte of yq (pad channels included) and of the
    tail with the oracle; returns (codes [N, O, OH, OW], out_scale)."""
    from dfq_b200 import _lib, int8
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    xn = x.detach().cpu().numpy()
    xq = O.i8_quantize(xn, a)
    acc, y = G._oracle(x, conv, a, ws)
    if out_scale is None:
        v = CO.i8_clamp(y, lo, hi)
        m = float(np.abs(v[np.isfinite(v)]).max()) if np.isfinite(v).any() else 0.0
        out_scale = f32(160.0 / m) if m > 0 else f32(1.0)               # some codes saturate at +-127
    b = None if conv.bias is None else conv.bias.detach().cpu().numpy()
    ref = CO.i8_requantize(acc, a, np.broadcast_to(np.asarray(ws, f32), (conv.out_channels,)), b, out_scale, lo, hi)
    pad = np.zeros((xq.shape[0], xq.shape[2], xq.shape[3], layer.cpad), np.int8)
    pad[..., :xq.shape[1]] = xq.transpose(0, 2, 3, 1)
    rc, got, n = _requant_abi(layer, pad, out_scale, lo, hi)
    _lib.check(rc, "dfq_i8_conv_requant")
    assert np.array_equal(got[:n], CO.to_nhwc_codes(ref).reshape(-1)), "codes"
    assert np.all(got[n:] == SENTINEL), "written past the end of yq"
    return ref, out_scale


def _dense(case, act):
    N, Cn, H, W, Oc, k, s, p, d = case
    torch.manual_seed(G._seed(case))
    conv = nn.Conv2d(Cn, Oc, k, s, p, d).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda") * 2
    _check_requant(conv, x, G._ascale(x), G._channel_scales(conv.weight, G._seed(case)), *ACTS[act])


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("case", G.DENSE, ids=G._case_id)
def test_dense_requant_bit_exact(case, act):
    _dense(case, act)


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("case", G.TILES, ids=G._case_id)
def test_dense_requant_tile_edges_bit_exact(case, act):
    _dense(case, act)


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("case", G.DW, ids=G._case_id)
def test_depthwise_requant_bit_exact(case, act):
    N, Cn, H, W, k, s, p, d = case
    torch.manual_seed(G._seed(case))
    conv = nn.Conv2d(Cn, Cn, k, s, p, d, Cn).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda") * 2
    _check_requant(conv, x, G._ascale(x), G._channel_scales(conv.weight, G._seed(case)), *ACTS[act])


@pytest.mark.parametrize("groups", [1, 40])
def test_requant_single_weight_scale_and_out_channels_below_16(groups):
    """One weight scale for the layer; O = 5 (cpad 16, 11 pad channels) dense, and O = 40 depthwise."""
    torch.manual_seed(groups)
    conv = nn.Conv2d(40, 5 if groups == 1 else 40, 3, 1, 1, groups=groups).cuda()
    x = torch.randn(2, 40, 7, 9, device="cuda")
    _check_requant(conv, x, G._ascale(x), G._wscale(conv.weight), 0.0, INF)


@pytest.mark.parametrize("groups", [1, 24])
def test_requant_zero_out_scale(groups):
    torch.manual_seed(20 + groups)
    conv = nn.Conv2d(24, 24, 3, 1, 1, groups=groups).cuda()
    x = torch.randn(2, 24, 6, 6, device="cuda")
    ref, _ = _check_requant(conv, x, G._ascale(x), G._wscale(conv.weight), -INF, INF, out_scale=f32(0.0))
    assert not ref.any()


@pytest.mark.parametrize("act", ["none", "relu", "relu6"])
@pytest.mark.parametrize("groups", [1, 24])
def test_requant_non_finite_and_overflowing_bias(groups, act):
    """NaN bias -> NaN through the clamp -> -127; +-inf and 3e38 -> +-127 (or the clamp bound's code)."""
    torch.manual_seed(30 + groups)
    conv = nn.Conv2d(24, 24, 3, 1, 1, groups=groups).cuda()
    with torch.no_grad():
        conv.bias[:6] = torch.tensor([float("nan"), float("inf"), float("-inf"), 3e38, -3e38, float("nan")])
    x = torch.randn(2, 24, 6, 6, device="cuda")
    lo, hi = ACTS[act]
    ref, s = _check_requant(conv, x, G._ascale(x), G._wscale(conv.weight), lo, hi, out_scale=f32(20.0))
    assert np.all(ref[:, 0] == -127) and np.all(ref[:, 5] == -127)
    top = 127 if hi == INF else int(O.i8_quantize(f32(hi), s))
    bottom = -127 if lo == -INF else int(O.i8_quantize(f32(lo), s))
    assert np.all(ref[:, 1] == top) and np.all(ref[:, 3] == top)
    assert np.all(ref[:, 2] == bottom) and np.all(ref[:, 4] == bottom)


@pytest.mark.parametrize("groups, C_, cpad_in", [(16, 16, 32), (24, 24, 64), (1, 16, 32), (1, 5, 48)])
def test_requant_input_cpad_wider_than_the_output(groups, C_, cpad_in):
    """The ABI accepts any input Cpad that is a multiple of 16 holding C.  yq keeps round_up(O, 16) channels: a depthwise
    launch covers cpad_in / 16 chunks per pixel, and those past yq's width must write nothing (sentinel-filled buffer and
    tail).  Dense layers read the wider rows through their K loop."""
    from dfq_b200 import _lib, int8
    lib = _lib.load()
    torch.manual_seed(50 + cpad_in + groups)
    N, H, W = 2, 7, 9
    conv = nn.Conv2d(C_, C_ if groups > 1 else 24, 3, 1, 1, groups=groups).cuda()
    x = torch.randn(N, C_, H, W, device="cuda") * 2
    a, ws = G._ascale(x), G._channel_scales(conv.weight, 50)
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    g = layer._geometry(N, H, W)
    g[0]["Cpad"] = cpad_in
    taps = 9
    wq = torch.full(((conv.out_channels if groups == 1 else 1) * taps * cpad_in,), SENTINEL, dtype=torch.int8, device="cuda")
    w = conv.weight.detach().contiguous()
    _lib.check(lib.dfq_i8_pack_weights(_vp(w), _vp(layer.w_scale), _vp(wq), _lib.table_ptr(g), _lib.stream_ptr()), "pack")
    xq = np.zeros((N, H, W, cpad_in), np.int8)
    xq[..., :C_] = O.i8_quantize(x.cpu().numpy(), a).transpose(0, 2, 3, 1)
    xq_d = torch.from_numpy(xq).cuda()
    n = N * H * W * ((conv.out_channels + 15) // 16 * 16)
    buf = torch.full((n + TAIL,), SENTINEL, dtype=torch.int8, device="cuda")
    s = f32(20.0)
    _lib.check(lib.dfq_i8_conv_requant(_vp(xq_d), _vp(wq), _vp(layer.dq), _vp(layer.bias), _vp(buf), C.c_float(s),
                                       C.c_float(0.0), C.c_float(6.0), _lib.table_ptr(g), _lib.stream_ptr()),
               "dfq_i8_conv_requant")
    got = buf.cpu().numpy()
    acc, _ = G._oracle(x, conv, a, ws)
    ref = CO.i8_requantize(acc, a, ws, conv.bias.detach().cpu().numpy(), s, 0.0, 6.0)
    assert np.array_equal(got[:n], CO.to_nhwc_codes(ref).reshape(-1)), "codes"
    assert np.all(got[n:] == SENTINEL), "written past the end of yq"


def test_depthwise_requant_grid_stride_loop_covers_every_item():
    N, Cn, H, W = 48, 144, 56, 56
    assert N * (Cn // 16) * H * W > G._launch_cap(), "the case no longer takes a second trip through the loop"
    torch.manual_seed(7)
    conv = nn.Conv2d(Cn, Cn, 3, 1, 1, groups=Cn).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda")
    _check_requant(conv, x, G._ascale(x), G._channel_scales(conv.weight, 7), 0.0, 6.0)


def test_requant_refusals_leave_the_buffer_untouched():
    from dfq_b200 import _lib, int8
    lib = _lib.load()
    torch.manual_seed(40)
    layer = int8.Int8Conv2d.from_conv(nn.Conv2d(16, 16, 3, 1, 1).cuda(), 1.0, 1.0)
    xq = np.zeros((1, 5, 5, 16), np.int8)
    for args, what in (((1.0, 0.0, INF, 1), "yq"), ((1.0, float("nan"), 6.0, 0), "bounds"), ((1.0, 0.0, float("nan"), 0), "bounds"),
                       ((1.0, 6.0, 0.0, 0), "bounds"), ((float("inf"), 0.0, 6.0, 0), "out_scale"),
                       ((float("nan"), 0.0, 6.0, 0), "out_scale"), ((-1.0, 0.0, 6.0, 0), "out_scale")):
        s, lo, hi, off = args
        rc, got, _ = _requant_abi(layer, xq, s, lo, hi, offset=off)
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (args, lib.dfq_last_error())
        assert np.all(got == SENTINEL)
    g = np.zeros(1, _lib.I8_CONV_DT)
    for k, v in dict(N=1, C=8, H=4, W=4, O=8, kh=1, kw=1, stride_h=1, stride_w=1, dil_h=1, dil_w=1, groups=2, OH=4, OW=4,
                     Cpad=16).items():
        g[0][k] = v
    buf = torch.zeros(1024, dtype=torch.int8, device="cuda")
    f = torch.zeros(1024, device="cuda")
    rc = lib.dfq_i8_conv_requant(_vp(buf), _vp(buf), _vp(f), None, _vp(buf), C.c_float(1.0), C.c_float(0.0), C.c_float(6.0),
                                 _lib.table_ptr(g), _lib.stream_ptr())
    assert rc == -2 and b"groups=2" in lib.dfq_last_error()


# ---- whole models -----------------------------------------------------------------------------------------------------
def _folded_and_converted(net, relu6=True, batch=2):
    """torchvision `net` (seeded) with its BN folded by trace_graph + merge_batchnorm, every Conv2d / Linear converted with
    activation scales 128 / max|input| of a forward pass; returns (model, x)."""
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm
    torch.manual_seed(0)
    model = getattr(torchvision.models, net)(num_classes=1000).cuda().eval()
    if not relu6:
        for m in model.modules():
            for k, c in m.named_children():
                if isinstance(c, nn.ReLU6):
                    setattr(m, k, nn.ReLU())
    graph, bottoms = trace_graph(model)
    merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
    x = torch.randn(batch, 3, 224, 224, device="cuda")
    layers = OrderedDict((n, m) for n, m in model.named_modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    amax = {}
    hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, float(i[0].abs().max())))
             for n, m in layers.items()]
    with torch.no_grad():
        model(x)
    for h in hooks:
        h.remove()
    int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                         act_scales=[128. / amax[n] for n in layers])
    return model, x


@pytest.mark.parametrize("net, relu6, fused", [("mobilenet_v2", True, 36), ("mobilenet_v2", False, 36), ("resnet18", True, 8)],
                         ids=["mobilenet_v2", "mobilenet_v2_relu", "resnet18"])
def test_chained_model_is_bit_identical_to_the_per_layer_path(net, relu6, fused):
    from dfq_b200 import int8
    model, x = _folded_and_converted(net, relu6)
    with torch.no_grad():
        before = model(x)
        gm = int8.chain_int8(model)
        assert len(gm.requantized_edges) == fused
        seen_fp32, seen_codes = {}, {}
        mods = dict(model.named_modules())
        hooks = [mods[q].register_forward_pre_hook(lambda m, i, q=q: seen_fp32.__setitem__(q, i[0].clone()))
                 for _, q, _ in gm.requantized_edges]
        hooks += [gm.get_submodule(q).register_forward_pre_hook(lambda m, i, q=q: seen_codes.__setitem__(q, i[0].clone()))
                  for _, q, _ in gm.requantized_edges]
        ref = model(x)
        got = gm(x)
        for h in hooks:
            h.remove()
        after = model(x)
    assert G._same_bits(got.cpu().numpy(), ref.cpu().numpy()), "chained logits"
    assert torch.equal(before, ref) and torch.equal(after, ref), "the converted model changed"
    for p, q, _ in gm.requantized_edges:
        want = CO.to_nhwc_codes(O.i8_quantize(seen_fp32[q].cpu().numpy(), f32(mods[q].act_scale)))
        assert np.array_equal(seen_codes[q].cpu().numpy(), want), (p, q)


# ---- the reference's int8 MobileNetV2, blob by blob --------------------------------------------------------------------
CONVS = ("Convolution", "ConvolutionDepthWise")


def _chain_plan(net):
    """producer layer name -> (consumer layer name, clamp, carried blob, skipped ReLU name | None) for every Conv -> [ReLU] ->
    Conv edge of the .param whose blobs each have one consumer."""
    users = Counter(b for l in net.layers for b in l["bottoms"])
    consumer = {b: l for l in net.layers for b in l["bottoms"]}
    plan = {}
    for l in net.layers:
        if l["type"] not in CONVS:
            continue
        top, clamp, relu = l["tops"][0], (-INF, INF), None
        if users[top] != 1:
            continue
        nxt = consumer[top]
        if nxt["type"] == "ReLU":
            relu, clamp, top = nxt["name"], (0.0, INF), nxt["tops"][0]
            if users[top] != 1:
                continue
            nxt = consumer[top]
        if nxt["type"] in CONVS:
            plan[l["name"]] = (nxt["name"], clamp, top, relu)
    return plan


def test_reference_int8_mobilenetv2_chained_blob_by_blob():
    """The reference's deployed int8 model (tests/ncnn_int8_case.py) walked with its single-consumer Conv -> [ReLU] -> Conv
    edges fused: every fp32 blob up to the last ReLU and the logits equal the per-layer GPU run's bit for bit, and every
    carried code blob equals i8_quantize of the per-layer blob at the consumer's input scale."""
    case, net = G._ref_net()
    from dfq_b200 import int8
    mods = []
    for s in net.specs:
        w = torch.from_numpy(case.spec_weight(s)).cuda()
        b = None if s["bias"] is None else torch.from_numpy(s["bias"]).cuda()
        mods.append(int8.Int8Linear(w, b, s["in_scale"], s["w_scales"]) if s["type"] == "InnerProduct" else
                    int8.Int8Conv2d(w, b, s["in_scale"], s["w_scales"], s["stride"], s["pad"], s["dilation"], s["groups"]))
    plan = _chain_plan(net)
    consumers = {q for q, _, _, _ in plan.values()}
    skipped = {r for _, _, _, r in plan.values() if r}
    by_name = {l["name"]: l for l in net.layers}
    assert len(plan) == 36, len(plan)
    x = G._ref_images().cuda()
    blobs, codes = {}, {}
    with torch.no_grad():
        ref = net.forward(x, lambda s, v: mods[s["index"]].run(v)[0])
        for l in net.layers:
            t, p, name = l["type"], l["params"], l["name"]
            if name in skipped:
                continue
            if t in CONVS:
                m, codes_in = mods[l["spec"]["index"]], name in consumers
                v = codes[l["bottoms"][0]] if codes_in else blobs[l["bottoms"][0]]
                if name in plan:
                    q, clamp, top, _ = plan[name]
                    nxt = mods[by_name[q]["spec"]["index"]]
                    codes[top] = m.chained(codes_in=codes_in, requant=(nxt.act_scale,) + clamp).run(v)[0]
                else:
                    blobs[l["tops"][0]] = (m.chained(codes_in=True) if codes_in else m).run(v)[0]
                continue
            ins = [blobs[b] for b in l["bottoms"]]
            if t == "Input":
                outs = [x]
            elif t == "InnerProduct":
                outs = [mods[l["spec"]["index"]].run(ins[0].reshape(ins[0].shape[0], -1, 1, 1))[0].reshape(ins[0].shape[0], -1)]
            elif t == "ReLU":
                outs = [torch.relu(ins[0])]
            elif t == "Split":
                outs = [ins[0]] * len(l["tops"])
            elif t == "BinaryOp":
                outs = [ins[0] + ins[1]]
            elif t == "Reshape":
                outs = [ins[0].reshape(ins[0].shape[0], p[1], p[0])]
            elif t == "Reduction":
                outs = [ins[0].mean(dim=[a % (ins[0].dim() - 1) + 1 for a in p[3]])]
            elif t == "Softmax":
                outs = [torch.softmax(ins[0], dim=1)]
            for b, o in zip(l["tops"], outs):
                blobs[b] = o
    names = list(ref)
    last_relu = [l for l in net.layers if l["type"] == "ReLU"][-1]["tops"][0]
    for n in names[:names.index(last_relu) + 1]:
        if n in blobs:
            assert G._same_bits(blobs[n].cpu().numpy(), ref[n].cpu().numpy()), n
    logits = [l for l in net.layers if l["type"] == "InnerProduct"][0]["tops"][0]
    assert G._same_bits(blobs[logits].cpu().numpy(), ref[logits].cpu().numpy())
    for prod, (q, _, top, _) in plan.items():
        want = CO.to_nhwc_codes(O.i8_quantize(ref[top].cpu().numpy(), f32(mods[by_name[q]["spec"]["index"]].act_scale)))
        assert np.array_equal(codes[top].cpu().numpy(), want), (prod, q)
    print("reference int8 MobileNetV2: %d of %d convolution inputs carried as int8 codes" % (len(plan), len(mods) - 1))
