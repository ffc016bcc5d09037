"""The affine residual epilogue on the H100 (dfq_i8_affine_conv_fused, dfq_b200.int8.chain_affine): y, codes and S against
tests/int8_affine_chain_oracle.py bit for bit, the codes and S against dfq_i8_affine_quantize of the per-layer value, the
entry's refusals, and calibrated torchvision networks chained against their per-layer affine model."""
import ctypes as C
import copy
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

import affine_calibrated
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A
from test_gpu_int8_affine import _fake_quantized_conv, _quantize, _same_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-41], f32)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _launch(layer, xq, S, g, r=None, y=None, yq=None, S_out=None, out=(0.0, 0.0, 0), pre=NONE, post=NONE):
    from dfq_b200 import _lib
    d = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
    d[0] = tuple(0 if t is None else t.data_ptr() for t in (r, y, yq, S_out)) + tuple(out) + tuple(pre) + tuple(post)
    return _lib.load().dfq_i8_affine_conv_fused(_p(xq), _p(S), _p(layer.weight_codes),
                                                _p(layer.tap_table) if layer.tap_table.numel() else None,
                                                _lib.table_ptr(layer.constants), _p(layer.bias), _lib.table_ptr(d),
                                                _lib.table_ptr(g), _lib.stream_ptr())


def _case(N, Cin, H, W, O, k, s, p, d, g=1, bits=8, lo=-1.3, outputs="both", residual=True, special=True, seed=0,
          pre=(0.0, 6.0), post=(0.0, INF), oracle=True):
    """Run the epilogue into sentinel-filled buffers and check y, the codes (pad channels 0, nothing past them) and S against
    the oracle and against dfq_i8_affine_quantize of the per-layer value clamp(clamp(y) + r)."""
    from dfq_b200 import _lib, int8
    torch.manual_seed(seed)
    conv = _fake_quantized_conv(nn.Conv2d(Cin, O, k, s, p, d, g).cuda())
    bias = conv.bias.detach().cpu().numpy().copy()
    if special:
        bias[:min(O, SPECIAL.size)] = SPECIAL[:min(O, SPECIAL.size)]
        with torch.no_grad():
            conv.bias.copy_(torch.from_numpy(bias))
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    layer = int8.AffineInt8Conv2d.from_conv(conv, f32(float(x.min()) * 0.8), f32(float(x.max()) * 0.8))
    xq, S, *_ = layer._input(x)
    geo = layer._geometry(N, H, W)
    OH, OW = int(geo[0]["OH"]), int(geo[0]["OW"])
    cpad = (O + 15) // 16 * 16
    y_pl, _ = layer.run(x)                                      # the per-layer value
    r = None
    if residual:
        rng = np.random.default_rng(seed + 1)
        rn = (rng.standard_normal((N, O, OH, OW)) * 3).astype(f32)
        rn.reshape(-1)[::97][:SPECIAL.size] = SPECIAL[:rn.reshape(-1)[::97].size]
        r = torch.from_numpy(rn).cuda()
    out = (f32(lo), f32(lo + 4.5), bits)
    want_y, want_q = outputs in ("both", "y"), outputs in ("both", "codes", "codes_noS")
    y = torch.full((N, O, OH, OW), 7.25, device="cuda") if want_y else None
    yq = torch.full((N * OH * OW * cpad + 64,), 99, dtype=torch.int8, device="cuda") if want_q else None
    S_out = torch.full((N * OH * OW + 16,), -2 ** 31, dtype=torch.int32, device="cuda") if outputs in ("both", "codes") \
        else None
    _lib.check(_launch(layer, xq, S, geo, r, y, yq, S_out, out, pre, post), "dfq_i8_affine_conv_fused")
    torch.cuda.synchronize()
    # the per-layer path: the fp32 clamps and add of torch's ops (numpy here: the same IEEE ops), then the quantizer
    v_pl = AC.epilogue_value(y_pl.cpu().numpy(), None if r is None else r.cpu().numpy(), pre, post)
    q_pl, S_pl = _quantize(torch.from_numpy(v_pl).cuda(), *out[:2], bits, cpad)
    if oracle:
        xo, _ = A.act_codes(x.cpu().numpy(), layer.act_min, layer.act_max, 8)
        wo, bad = A.weight_codes(conv.weight.detach().cpu().numpy(), layer.w_min, layer.w_scale, 8)
        assert bad == 0
        terms = A.terms(xo, wo, conv.stride, conv.padding, conv.dilation, conv.groups)
        v_o, q_o, S_o = AC.fused(*terms, tuple(layer.constants[0]), bias, None if r is None else r.cpu().numpy(), pre,
                                 post, out)
    if want_y:
        got = y.cpu().numpy()
        nan = np.isnan(v_pl)                                    # numpy keeps a NaN's payload, the GPU's add does not
        assert np.array_equal(np.isnan(got), nan) and _same_bits(np.where(nan, 0, got), np.where(nan, 0, v_pl)), \
            "y vs per-layer"
        if oracle:
            assert _same_bits(got, v_o), "y vs oracle"
    if want_q:
        codes = yq.cpu().numpy()
        assert (codes[N * OH * OW * cpad:] == 99).all(), "past the codes"
        codes = codes[:N * OH * OW * cpad].reshape(N, OH, OW, cpad)
        assert np.array_equal(codes, q_pl), "codes vs the quantizer of the per-layer value"
        assert not codes[..., O:].any()
        if oracle:
            assert np.array_equal(codes, AC.to_nhwc(q_o)), "codes vs oracle"
    if S_out is not None:
        s = S_out.cpu().numpy()
        assert (s[N * OH * OW:] == -2 ** 31).all()
        assert np.array_equal(s[:N * OH * OW].reshape(N, OH, OW), S_pl), "S vs the quantizer of the per-layer value"
        if oracle:
            assert np.array_equal(s[:N * OH * OW].reshape(N, OH, OW), S_o)
    return layer


# O across the 64-channel tile (1 tile: S stored; several: S added atomically), M tails (M = N OH OW not a multiple of
# 128), 1-8 output bits, negative and positive act_min, with and without a residual
DENSE = [  # (N, Cin, H, W, O, k, s, p, d), bits, lo, residual
    ((2, 19, 9, 7, 1, 3, 1, 1, 1), 8, -1.3, True),
    ((2, 19, 9, 7, 15, 3, 1, 1, 1), 7, 0.4, False),
    ((1, 32, 15, 15, 16, 3, 2, 1, 1), 6, -1.3, True),
    ((3, 16, 7, 7, 17, 1, 1, 0, 1), 5, 0.4, True),
    ((2, 24, 10, 11, 63, 3, 1, 2, 2), 4, -1.3, False),
    ((2, 40, 8, 8, 64, 3, 1, 1, 1), 3, 0.4, True),
    ((1, 16, 12, 13, 65, 3, 2, 1, 1), 2, -1.3, True),
    ((2, 33, 9, 9, 130, 3, 1, 1, 1), 1, 0.4, True),
    ((4, 64, 14, 14, 130, 1, 1, 0, 1), 8, -0.2, False),
]


@pytest.mark.parametrize("case,bits,lo,residual", DENSE, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_dense_epilogue_bit_exact(case, bits, lo, residual):
    _case(*case, bits=bits, lo=lo, residual=residual, seed=sum(case))


DW = [  # (N, C, H, W, k, s, p, d), bits, lo, residual
    ((2, 15, 9, 7, 3, 1, 1, 1), 8, -1.3, True),
    ((2, 16, 8, 8, 3, 2, 1, 1), 5, 0.4, False),
    ((1, 17, 11, 9, 5, 1, 2, 1), 3, -1.3, True),
    ((2, 65, 7, 7, 3, 1, 2, 2), 1, 0.4, True),
    ((1, 130, 10, 10, 3, 2, 1, 1), 8, -0.2, True),
]


@pytest.mark.parametrize("case,bits,lo,residual", DW, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_depthwise_epilogue_bit_exact(case, bits, lo, residual):
    N, Cn, H, W, k, s, p, d = case
    _case(N, Cn, H, W, Cn, k, s, p, d, g=Cn, bits=bits, lo=lo, residual=residual, seed=sum(case))


@pytest.mark.parametrize("outputs", ["y", "codes", "codes_noS", "both"])
@pytest.mark.parametrize("depthwise", [False, True])
def test_output_selection(outputs, depthwise):
    """y only, codes only, codes without S, both; every unrequested buffer stays NULL and what is requested is exact."""
    if depthwise:
        _case(2, 40, 9, 9, 40, 3, 1, 1, 1, g=40, outputs=outputs, seed=11)
    else:
        _case(2, 24, 9, 9, 80, 3, 1, 1, 1, outputs=outputs, seed=12)


@pytest.mark.parametrize("bits", range(1, 9))
def test_every_output_bit_width(bits):
    _case(1, 16, 6, 6, 20, 3, 1, 1, 1, bits=bits, lo=-0.7 if bits % 2 else 0.3, seed=bits, pre=NONE, post=(-1.0, 2.0))


def test_depthwise_grid_stride_loop():
    """16 x 96 x 112 x 112: 1.2M (pixel, 16-channel) threads, more than one launch covers; S added atomically.  Checked
    against the quantizer of the per-layer value (the numpy oracle is too slow at this size)."""
    _case(16, 96, 112, 112, 96, 3, 1, 1, 1, g=96, special=False, seed=13, oracle=False)


def test_abi_refusals_leave_the_buffers_untouched():
    from dfq_b200 import int8
    conv = _fake_quantized_conv(nn.Conv2d(16, 8, 3, padding=1).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.0, 1.0)
    g = layer._geometry(1, 4, 4)
    xq, S, *_ = layer._input(torch.randn(1, 16, 4, 4, device="cuda"))
    y, r = torch.full((128,), 3.5, device="cuda"), torch.zeros(128, device="cuda")
    yq, S_out = torch.full((256 + 16,), 99, dtype=torch.int8, device="cuda"), torch.full((16,), -7, dtype=torch.int32,
                                                                                            device="cuda")
    base = dict(r=None, y=y, yq=yq[:256], S_out=S_out, out=(-1.0, 1.0, 8), pre=NONE, post=NONE)

    def call(**kw):
        a = dict(base)
        a.update(kw)
        return _launch(layer, xq, S, g, **a)

    refused = [
        (dict(y=None, yq=None, S_out=None), -1), (dict(yq=None), -1), (dict(yq=yq[1:257]), -1),
        (dict(y=y.view(torch.int8)[1:]), -1), (dict(S_out=S_out.view(torch.int8)[1:]), -1), (dict(r=y), -1),
        (dict(S_out=y.view(torch.int32)), -1), (dict(pre=(1.0, 0.0)), -1), (dict(post=(math.nan, 1.0)), -1),
        (dict(out=(-1.0, math.inf, 8)), -1), (dict(out=(-3e38, 3e38, 1)), -1), (dict(out=(-1.0, 1.0, 0)), -1),
        (dict(out=(-1.0, 1.0, 9)), -2),
    ]
    for kw, rc in refused:
        assert call(**kw) == rc, kw
        torch.cuda.synchronize()
        assert (y == 3.5).all() and (yq == 99).all() and (S_out == -7).all(), kw
    assert call(r=r) == 0
    torch.cuda.synchronize()
    assert (yq[256:] == 99).all() and not (S_out == -7).any()


# ---- calibrated torchvision networks ----------------------------------------------------------------------------------
# (net, chain_affine edges, chain_affine(residual=True) edges, fused adds), as measured on an H100.  The ncnn residual chain
# carries 51 convolution inputs with 10 adds on MobileNetV2 and 18 with 8 on ResNet-18: the affine one carries the same -
# the consumers of a fan-out (ResNet's conv1 and downsample) observe the same tensor, so their observers end with the same
# range and take the same codes.
NETS = [("mobilenet_v2", 36, 51, 10), ("resnet18", 8, 18, 8)]


@pytest.mark.parametrize("net,edges,res_edges,adds", NETS, ids=[n[0] for n in NETS])
def test_calibrated_network_chained_logits_equal_the_per_layer_model(net, edges, res_edges, adds):
    from dfq_b200 import int8
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        fq, _, qtarg = affine_calibrated.calibrated(net)
        aff = copy.deepcopy(fq)
        int8.convert_affine(aff, OrderedDict((id(m), m) for m in aff.modules() if type(m) in qtarg), qtarg)
        x = torch.randn(8, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
        chained, gm = int8.chain_affine(aff), int8.chain_affine(aff, residual=True)
        with torch.no_grad():
            ref = aff(x)
            got = {"chained": chained(x), "residual": gm(x)}
        print("%s: edges %d / %d, adds %d" % (net, len(chained.requantized_edges), len(gm.requantized_edges),
                                              len(gm.fused_adds)))
        for k, v in got.items():
            assert torch.equal(ref.view(torch.int32), v.view(torch.int32)), k
        assert (len(chained.requantized_edges), len(gm.requantized_edges), len(gm.fused_adds)) == (edges, res_edges, adds)
        assert isinstance(gm.get_submodule("classifier.1" if net == "mobilenet_v2" else "fc"), int8.AffineInt8Linear)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
