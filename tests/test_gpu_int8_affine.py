"""The affine int8 scheme on the H100 (dfq_i8_affine_* in libdfq_sm90.so, dfq_b200.int8.convert_affine): codes, sums and
outputs against tests/int8_affine_oracle.py bit for bit, and calibrated torchvision networks against their fake-quantized
twins."""
import ctypes as C
import copy
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_calibrated
import int8_affine_oracle as A
import test_gpu_int8 as G

pytestmark = pytest.mark.gpu
f32 = np.float32


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))


def _quantize(x, lo, hi, bits, cpad):
    """dfq_i8_affine_quantize into sentinel-filled buffers: ([N, H, W, cpad] codes, [N, H, W] S)."""
    from dfq_b200 import _lib
    N, Cn, H, W = x.shape
    q = torch.full((N * H * W * cpad,), 99, dtype=torch.int8, device="cuda")
    S = torch.full((N * H * W,), -2 ** 31, dtype=torch.int32, device="cuda")
    _lib.check(_lib.load().dfq_i8_affine_quantize(C.c_void_p(x.data_ptr()), C.c_void_p(q.data_ptr()), C.c_void_p(S.data_ptr()),
                                                  N, Cn, H, W, cpad, C.c_float(lo), C.c_float(hi), bits, _lib.stream_ptr()),
               "dfq_i8_affine_quantize")
    return q.reshape(N, H, W, cpad).cpu().numpy(), S.reshape(N, H, W).cpu().numpy()


@pytest.mark.parametrize("shape,bits", [((2, 19, 5, 3), 8), ((1, 33, 7, 9), 5), ((3, 16, 1, 1), 2), ((24, 3, 224, 224), 8)],
                         ids=["19ch", "33ch-5bit", "16ch-2bit", "grid-stride"])
def test_quantizer_codes_and_sums_match_the_oracle_and_dequantize_to_quant_measure(shape, bits):
    """Unaligned channel counts, 2-8 bits, values at each code's half point, +-inf, and (last case: 24 * 224 * 224 pixels)
    more pixels than one launch has threads."""
    from dfq_b200.utils.quantize import QuantMeasure
    N, Cn, H, W = shape
    rng = np.random.default_rng(N * Cn)
    lo, hi = f32(-1.7), f32(2.3)
    x = (rng.standard_normal(shape) * 2).astype(f32)
    _, ma, fa, _, qmax = A.act_scalars(lo, hi, bits)
    special = np.concatenate([((np.arange(int(qmax) + 1) + 0.5) * float(fa) + float(ma)).astype(f32),
                              np.array([np.inf, -np.inf, lo, hi, -0.0], f32)])
    x.reshape(-1)[:special.size] = special[:x.size]
    cpad = (Cn + 15) // 16 * 16
    q, S = _quantize(torch.from_numpy(x).cuda(), lo, hi, bits, cpad)
    q_ref, S_ref = A.act_codes(x, lo, hi, bits)
    assert np.array_equal(q[..., :Cn], q_ref.transpose(0, 2, 3, 1)) and not q[..., Cn:].any()
    assert np.array_equal(S, S_ref)
    qm = QuantMeasure(num_bits=bits).cuda().eval()
    qm.running_min.fill_(float(lo)); qm.running_max.fill_(float(hi))
    with torch.no_grad():
        ref = qm(torch.from_numpy(x).cuda()).cpu().numpy()
    assert _same_bits(A.act_dequant(q[..., :Cn].transpose(0, 3, 1, 2), lo, hi, bits), ref)


def _fake_quantized_conv(conv, bits=8):
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(A.fake_quant_weights(conv.weight.detach().cpu().numpy(), bits)))
    return conv


def _run_affine(N, Cin, H, W, Cout, k, s, p, d, g=1, seed=0, x=None, conv=None, lo=None, hi=None):
    """Convert, run with P, and check the codes, the prefix table, P and y against the oracle."""
    from dfq_b200 import int8
    torch.manual_seed(seed)
    conv = conv or _fake_quantized_conv(nn.Conv2d(Cin, Cout, k, s, p, d, g).cuda())
    x = torch.randn(N, Cin, H, W, device="cuda") * 2 if x is None else x
    lo = f32(float(x.min()) * 0.8) if lo is None else lo
    hi = f32(float(x.max()) * 0.8) if hi is None else hi
    layer = int8.AffineInt8Conv2d.from_conv(conv, lo, hi)
    y, P = layer.run(x, with_acc=True)
    w_hat = conv.weight.detach().cpu().numpy()
    P_ref, y_ref = A.conv(x.cpu().numpy(), lo, hi, 8, w_hat, layer.w_min, layer.w_scale, 8,
                          None if conv.bias is None else conv.bias.detach().cpu().numpy(), conv.stride, conv.padding,
                          conv.dilation, conv.groups)
    wq, _ = A.weight_codes(w_hat, layer.w_min, layer.w_scale, 8)
    kh, kw = layer.kernel_size
    codes = layer.weight_codes.cpu().numpy()
    if layer.groups == 1:
        codes = codes.reshape(Cout, kh, kw, layer.cpad)
        assert np.array_equal(codes[..., :Cin], wq.transpose(0, 2, 3, 1)) and not codes[..., Cin:].any()
        assert np.array_equal(layer.tap_table.cpu().numpy().reshape(-1, kh + 1, kw + 1), A.tap_table(wq))
    else:
        codes = codes.reshape(kh * kw, layer.cpad)
        assert np.array_equal(codes[:, :Cin], wq.reshape(Cin, kh * kw).T) and not codes[:, Cin:].any()
    assert np.array_equal(P.cpu().numpy(), P_ref), "P"
    assert _same_bits(y.cpu().numpy(), y_ref), "y"
    return layer, x, y, P


@pytest.mark.parametrize("case", G.DENSE, ids=G._case_id)
def test_dense_affine_conv_bit_exact(case):
    _run_affine(*case, seed=G._seed(case))


@pytest.mark.parametrize("case", G.TILES, ids=G._case_id)
def test_dense_affine_conv_tile_edges_bit_exact(case):
    _run_affine(*case, seed=sum(G.tile_geometry(case)))


@pytest.mark.parametrize("case", G.DW, ids=G._case_id)
def test_depthwise_affine_conv_bit_exact(case):
    N, Cn, H, W, k, s, p, d = case
    _run_affine(N, Cn, H, W, Cn, k, s, p, d, g=Cn, seed=G._seed(case))


def test_affine_sums_reach_past_2_pow_24_exactly():
    """Every input at the range's minimum (code -128) and every weight but one per channel at its minimum (code -128), K =
    3 * 3 * 512: P reaches 128^2 * 4608 = 75,497,472 > 2^24 at the interior pixels."""
    conv = nn.Conv2d(512, 24, 3, 1, 1).cuda()
    with torch.no_grad():
        w = torch.full((24, 512, 3, 3), -0.5)
        w[:, 0, 0, 0] = 0.5
        conv.weight.copy_(w)
    _fake_quantized_conv(conv)
    x = torch.full((1, 512, 6, 6), -1.0, device="cuda")
    _, _, _, P = _run_affine(1, 512, 6, 6, 24, 3, 1, 1, 1, x=x, conv=conv, lo=f32(-1), hi=f32(1))
    assert int(P.max()) > 2 ** 24 and int(P.max()) == 128 * 128 * (4608 - 1) - 128 * 127


@pytest.mark.parametrize("B", [1, 7, 256])
def test_affine_linear_bit_exact(B):
    from dfq_b200 import int8
    torch.manual_seed(B)
    lin = nn.Linear(1000, 37).cuda()
    with torch.no_grad():
        lin.weight.copy_(torch.from_numpy(A.fake_quant_weights(lin.weight.detach().cpu().numpy(), 8)))
    x = torch.randn(B, 1000, device="cuda")
    layer = int8.AffineInt8Linear.from_linear(lin, f32(-2.5), f32(3.0))
    y = layer(x)
    _, y_ref = A.conv(x.cpu().numpy().reshape(B, 1000, 1, 1), f32(-2.5), f32(3.0), 8,
                      lin.weight.detach().cpu().numpy().reshape(37, 1000, 1, 1), layer.w_min, layer.w_scale, 8,
                      lin.bias.detach().cpu().numpy())
    assert y.shape == (B, 37) and _same_bits(y.cpu().numpy(), y_ref.reshape(B, 37))


# ---- calibrated torchvision networks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["resnet18", "mobilenet_v2"])
def test_calibrated_network_layer_by_layer_and_logits(net):
    """Every layer: the weight round trip is exact (convert_affine packs only then), and its output on the input its
    fake-quantized twin saw stays within 16 ulp of sum |x^| |w^| + |b| of the twin's fp32 output (measured on an H100:
    6 ulp on ResNet-18, 8 on MobileNetV2) and within 4 ulp of sum (|x^| + |ma|)(|w^| + |mw|) + |b| of the same sum
    computed in double from x^ and w^: x^ and w^ are rounded at the magnitude of their offsets ma, mw, not at their own.
    Whole network: the relative logit error against the fake-quantized model over 8 synthetic images was 5.4e-3
    (ResNet-18) and 2.9e-3 (MobileNetV2) on an H100 and is asserted below 1e-2: the per-layer differences of fp32 rounding
    move activations that sit on a rounding boundary of the next layer's quantizer by one code."""
    from dfq_b200 import int8
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        fq, qgraph, qtarg = affine_calibrated.calibrated(net)
        aff = copy.deepcopy(fq)
        names = int8.convert_affine(aff, OrderedDict((id(m), m) for m in aff.modules() if type(m) in qtarg), qtarg)
        assert len(names) == len(qgraph) and all(isinstance(m, int8._AffineInt8Layer) for n, m in aff.named_modules()
                                                   if n in names)
        x = torch.randn(8, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
        seen = {}
        mods = dict(fq.named_modules())
        hooks = [mods[n].register_forward_hook(lambda m, i, o, n=n: seen.__setitem__(n, (i[0].detach(), o.detach())))
                 for n in names]
        with torch.no_grad():
            ref = fq(x)
            for h in hooks:
                h.remove()
            worst, worst64 = 0.0, 0.0
            amods = dict(aff.named_modules())
            for n in names:
                xin, yfq = seen[n]
                lay, twin = amods[n], mods[n]
                xh = twin.quant(xin)
                w = twin.weight
                y = lay(xin)
                if isinstance(twin, nn.Conv2d):
                    conv = lambda a, b: F.conv2d(a, b, None, twin.stride, twin.padding, twin.dilation, twin.groups)
                else:
                    conv = lambda a, b: F.linear(a, b)
                bound = conv(xh.abs().double(), w.abs().double()) + twin.bias.abs().double().reshape((-1,) + (1,) * (y.dim() - 2))
                y64 = conv(xh.double(), w.double()) + twin.bias.double().reshape((-1,) + (1,) * (y.dim() - 2))
                ma, mw = abs(float(twin.quant.running_min)), abs(float(w.min()))
                bound64 = conv(xh.abs().double() + ma, w.abs().double() + mw) + \
                    twin.bias.abs().double().reshape((-1,) + (1,) * (y.dim() - 2))
                ulp = torch.from_numpy(np.spacing(bound.float().cpu().numpy())).cuda().double()
                ulp64 = torch.from_numpy(np.spacing(bound64.float().cpu().numpy())).cuda().double()
                worst = max(worst, float(((y.double() - yfq.double()).abs() / ulp).max()))
                worst64 = max(worst64, float(((y.double() - y64).abs() / ulp64).max()))
            got = aff(x)
        err = float((got - ref).norm() / ref.norm())
        print("%s: %d layers, worst |int - fake quant| %.2f ulp, |int - double| %.2f ulp, relative logit error %.3g"
              % (net, len(names), worst, worst64, err))
        assert worst <= 16 and worst64 <= 4, (worst, worst64)
        assert err < 1e-2, err
        gm = int8.chain_int8(aff, residual=True, pool_cat=True)
        with torch.no_grad():
            chained = gm(x)
        assert gm.requantized_edges == [] and gm.fused_adds == [] and gm.fused_pools == [] and gm.fused_cats == []
        assert torch.equal(chained.view(torch.int32), got.view(torch.int32))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_abi_refusals():
    from dfq_b200 import _lib, int8
    lib, st = _lib.load(), _lib.stream_ptr()
    conv = _fake_quantized_conv(nn.Conv2d(16, 8, 3, padding=1).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.0, 1.0)
    g = layer._geometry(1, 4, 4)
    x = torch.zeros(1, 16, 4, 4, device="cuda")
    q = torch.zeros(16 * 16, dtype=torch.int8, device="cuda")
    S = torch.zeros(16, dtype=torch.int32, device="cuda")
    y = torch.zeros(1, 8, 4, 4, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())

    def quantize(lo, hi, bits):
        return lib.dfq_i8_affine_quantize(p(x), p(q), p(S), 1, 16, 4, 4, 16, C.c_float(lo), C.c_float(hi), bits, st)

    assert quantize(-1, 1, 9) == -2 and quantize(-1, 1, 0) == -1
    assert quantize(float("nan"), 1, 8) == -1 and quantize(-1, float("inf"), 8) == -1 and quantize(-3e38, 3e38, 1) == -1
    assert quantize(-1, 1, 8) == 0

    def conv_call(k, g_=g, table=layer.tap_table):
        d = np.zeros(1, _lib.I8_AFFINE_DT)
        d[0] = k
        return lib.dfq_i8_affine_conv(p(q), p(S), p(layer.weight_codes), p(table) if table is not None else None,
                                      _lib.table_ptr(d), p(layer.bias), p(y), None, _lib.table_ptr(g_), st)

    assert conv_call(tuple(layer.constants[0])) == 0
    assert conv_call((float("inf"), 0, 0, 0)) == -1 and conv_call((0, 0, float("nan"), 0)) == -1
    assert conv_call(tuple(layer.constants[0]), table=None) == -1
    assert "prefix table" in lib.dfq_last_error().decode()
    g2 = g.copy()
    g2[0]["groups"] = 2
    assert conv_call(tuple(layer.constants[0]), g_=g2) == -2
    wide = g.copy()
    wide[0]["C"], wide[0]["Cpad"] = 16384, 16384                               # K = 9 * 16384 = 147456
    assert conv_call(tuple(layer.constants[0]), g_=wide) == -2 and "131072" in lib.dfq_last_error().decode()
    n_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    w = conv.weight.detach().contiguous()
    pack = lambda mn, s, bits: lib.dfq_i8_affine_pack(p(w), C.c_float(mn), C.c_float(s), bits, p(layer.weight_codes),
                                                      p(layer.tap_table), p(n_bad), _lib.table_ptr(g), st)
    assert pack(layer.w_min, layer.w_scale, 9) == -2 and pack(layer.w_min, 0.0, 8) == -1
    assert pack(float("inf"), layer.w_scale, 8) == -1
    assert pack(layer.w_min, layer.w_scale, 8) == 0 and int(n_bad.item()) == 0
    assert pack(layer.w_min, float(np.nextafter(f32(layer.w_scale), f32(1))) * 1.01, 8) == 0 and int(n_bad.item()) > 0
