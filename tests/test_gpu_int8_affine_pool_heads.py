"""The affine max pool and detection-head rows on the H100 (dfq_i8_affine_maxpool, dfq_i8_affine_conv_rows,
dfq_b200.int8.chain_affine(pools=True / heads=True)): codes mode against the oracle and against dfq_i8_affine_quantize of
torch's max_pool2d, fp32 mode against torch and the quantizer of its output, the NaN-window exception, the rows against
the per-layer layer's output permuted and passed through QuantMeasure, the refusals of both entries, and ResNet-18,
GoogLeNet and SSD-Lite in the reference's evaluation state (SqueezeNet 1.1 with fixed ranges) against their per-layer
affine models."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import affine_observed_state
import int8_affine_pool_heads_oracle as AP

pytestmark = pytest.mark.gpu
f32 = np.float32
SPECIAL = [np.inf, -np.inf, -0.0, 1e-40, -1e-41, 0.0]


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _geometry(N, Cn, H, W, k, s, p, d, ceil):
    from dfq_b200 import _lib
    g = np.zeros(1, _lib.I8_POOL_DT)
    OH, OW = AP.PO.pool_extent(H, k[0], p[0], s[0], d[0], ceil), AP.PO.pool_extent(W, k[1], p[1], s[1], d[1], ceil)
    g[0] = (N, Cn, H, W, *k, *s, *p, *d, int(ceil), OH, OW, (Cn + 15) // 16 * 16)
    return g, OH, OW


def _quantize(x, out):
    """(codes [N, H, W, cpad], S [N, H, W]) of fp32 NCHW x from dfq_i8_affine_quantize at out = (min, max, bits)."""
    from dfq_b200 import _lib
    N, Cn, H, W = x.shape
    cpad = (Cn + 15) // 16 * 16
    q = torch.empty((N, H, W, cpad), dtype=torch.int8, device="cuda")
    S = torch.empty((N, H, W), dtype=torch.int32, device="cuda")
    _lib.check(_lib.load().dfq_i8_affine_quantize(_p(x.contiguous()), _p(q), _p(S), N, Cn, H, W, cpad, C.c_float(out[0]),
                                                  C.c_float(out[1]), out[2], _lib.stream_ptr()), "quantize")
    return q, S


def _pool(g, xq=None, x=None, y=None, yq=None, S=None, out=(0.0, 0.0, 0)):
    from dfq_b200 import _lib
    return _lib.load().dfq_i8_affine_maxpool(_p(xq), _p(x), _p(y), _p(yq), _p(S), C.c_float(out[0]), C.c_float(out[1]),
                                             out[2], _lib.table_ptr(g), _lib.stream_ptr())


def _input(N, Cn, H, W, seed, special=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Cn, H, W, device="cuda", generator=g) * 1.5 + 0.7
    if special and x.numel() >= 2 * len(SPECIAL):
        x.view(-1)[:len(SPECIAL)] = torch.tensor(SPECIAL, device="cuda")
        x.view(-1)[-len(SPECIAL):] = torch.tensor(SPECIAL[::-1], device="cuda")
    return x


GEOMETRY = [  # (k, s, p, d, ceil_mode, H, W)
    ((2, 2), (2, 2), (0, 0), (1, 1), False, 9, 8),
    ((3, 3), (2, 2), (1, 1), (1, 1), True, 11, 10),
    ((3, 3), (1, 1), (1, 1), (1, 1), False, 7, 9),
    ((3, 2), (2, 1), (1, 1), (2, 1), True, 10, 7),
    ((2, 2), (1, 1), (1, 1), (2, 2), False, 1, 1),            # every window empty: taps at -1 and 1
    ((3, 3), (3, 2), (1, 0), (2, 2), True, 8, 9),
]
CHANNELS = [1, 15, 16, 17, 64, 65, 130]
OUTS = [(-1.3, 2.2, 8), (0.0, 3.0, 8), (0.4, 3.3, 7), (-0.9, 1.1, 4), (0.0, 1.0, 1), (-2.0, 0.5, 2), (0.3, 6.0, 5),
        (-1.0, 4.0, 3), (-0.5, 2.5, 6)]


@pytest.mark.parametrize("gi", range(len(GEOMETRY)))
@pytest.mark.parametrize("Cn", CHANNELS)
def test_codes_mode_equals_the_quantizer_of_max_pool(gi, Cn):
    k, s, p, d, ceil, H, W = GEOMETRY[gi]
    out = OUTS[(gi * len(CHANNELS) + CHANNELS.index(Cn)) % len(OUTS)]
    x = _input(2, Cn, H, W, gi * 1000 + Cn)
    xq, _ = _quantize(x, out)
    g, OH, OW = _geometry(2, Cn, H, W, k, s, p, d, ceil)
    yq = torch.full((2, OH, OW, xq.shape[3]), 99, dtype=torch.int8, device="cuda")
    S = torch.full((2, OH, OW), -7, dtype=torch.int32, device="cuda")
    assert _pool(g, xq=xq, yq=yq, S=S) == 0
    want_q, want_S = _quantize(F.max_pool2d(x, k, s, p, d, ceil), out)
    assert torch.equal(yq, want_q) and torch.equal(S, want_S)
    oq, oS = AP.maxpool_codes(xq.cpu().numpy(), Cn, k, s, p, d, ceil)
    assert np.array_equal(yq.cpu().numpy(), oq) and np.array_equal(S.cpu().numpy(), oS)
    yq2 = torch.full_like(yq, 99)
    assert _pool(g, xq=xq, yq=yq2) == 0 and torch.equal(yq2, yq)       # S is optional
    if H == 1:
        assert (yq[..., :Cn] == -128).all() and (yq[..., Cn:] == 0).all()


@pytest.mark.parametrize("bits", range(1, 9))
def test_codes_mode_every_bit_width(bits):
    for lo in (-1.1, 0.0, 0.6):
        out = (lo, 2.4, bits)
        x = _input(3, 33, 13, 12, bits)
        xq, _ = _quantize(x, out)
        g, OH, OW = _geometry(3, 33, 13, 12, (3, 3), (2, 2), (1, 1), (1, 1), True)
        yq = torch.empty((3, OH, OW, 48), dtype=torch.int8, device="cuda")
        S = torch.empty((3, OH, OW), dtype=torch.int32, device="cuda")
        assert _pool(g, xq=xq, yq=yq, S=S) == 0
        want_q, want_S = _quantize(F.max_pool2d(x, 3, 2, 1, ceil_mode=True), out)
        assert torch.equal(yq, want_q) and torch.equal(S, want_S), out


def test_grid_stride_loop():
    """More (pixel, chunk) threads than the grid's 32 blocks of 256 per SM: ResNet-18's stem pool at batch 32."""
    x = _input(32, 64, 224, 224, 5)
    out = (0.0, 4.0, 8)
    xq, _ = _quantize(x, out)
    g, OH, OW = _geometry(32, 64, 224, 224, (3, 3), (2, 2), (1, 1), (1, 1), False)
    assert 32 * OH * OW * 4 > torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256
    want_q, want_S = _quantize(F.max_pool2d(x, 3, 2, 1), out)
    yq, S = torch.empty_like(want_q), torch.empty_like(want_S)
    assert _pool(g, xq=xq, yq=yq, S=S) == 0
    assert torch.equal(yq, want_q) and torch.equal(S, want_S)
    y = torch.empty((32, 64, OH, OW), device="cuda")
    yq.fill_(99)
    assert _pool(g, x=x, y=y, yq=yq, S=S, out=out) == 0
    assert torch.equal(y.view(torch.int32), F.max_pool2d(x, 3, 2, 1).view(torch.int32))
    assert torch.equal(yq, want_q) and torch.equal(S, want_S)


@pytest.mark.parametrize("gi", range(len(GEOMETRY)))
@pytest.mark.parametrize("Cn", [1, 17, 65])
def test_fp32_mode_every_output_selection(gi, Cn):
    k, s, p, d, ceil, H, W = GEOMETRY[gi]
    out = OUTS[gi % len(OUTS)]
    x = _input(2, Cn, H, W, gi + Cn)
    x.view(-1)[7 % x.numel()] = math.nan                                    # torch's NaN rule: NaN wins and stays
    g, OH, OW = _geometry(2, Cn, H, W, k, s, p, d, ceil)
    ref = F.max_pool2d(x, k, s, p, d, ceil)
    want_q, want_S = _quantize(ref, out)
    cpad = (Cn + 15) // 16 * 16
    for sel in ("y", "yq", "yq S", "y yq", "y yq S"):
        y = torch.full((2, Cn, OH, OW), 5.0, device="cuda") if "y" in sel.split() else None
        yq = torch.full((2, OH, OW, cpad), 99, dtype=torch.int8, device="cuda") if "yq" in sel else None
        S = torch.full((2, OH, OW), -7, dtype=torch.int32, device="cuda") if "S" in sel else None
        assert _pool(g, x=x, y=y, yq=yq, S=S, out=out) == 0, sel
        if y is not None:
            assert torch.equal(y.view(torch.int32), ref.view(torch.int32)), sel
        if yq is not None:
            assert torch.equal(yq, want_q), sel
        if S is not None:
            assert torch.equal(S, want_S), sel


def test_nan_window_gives_the_max_of_the_other_codes():
    """The documented exception of codes mode: the per-layer path quantizes max_pool2d's NaN to code -128, the pool of the
    codes (NaN -> -128 at quantization) gives the max of the window's other codes."""
    out = (-1.0, 1.0, 8)
    x = torch.full((1, 1, 2, 2), 0.5, device="cuda")
    x[0, 0, 0, 0] = math.nan
    xq, _ = _quantize(x, out)
    g, _, _ = _geometry(1, 1, 2, 2, (2, 2), (2, 2), (0, 0), (1, 1), False)
    yq = torch.empty((1, 1, 1, 16), dtype=torch.int8, device="cuda")
    assert _pool(g, xq=xq, yq=yq) == 0
    per_layer, _ = _quantize(F.max_pool2d(x, 2), out)
    half, _ = _quantize(torch.full((1, 1, 1, 1), 0.5, device="cuda"), out)
    assert per_layer[0, 0, 0, 0] == -128 and yq[0, 0, 0, 0] == half[0, 0, 0, 0] != -128


def test_refusals_leave_the_buffers_untouched():
    x = torch.randn(1, 20, 8, 8, device="cuda")
    xq, _ = _quantize(x, (-1.0, 1.0, 8))
    g, OH, OW = _geometry(1, 20, 8, 8, (3, 3), (2, 2), (1, 1), (1, 1), False)
    n = OH * OW
    y = torch.full((20 * n + 4,), 5.0, device="cuda")
    yq = torch.full((32 * n + 16,), 99, dtype=torch.int8, device="cuda")
    S = torch.full((n + 4,), -7, dtype=torch.int32, device="cuda")

    def untouched():
        torch.cuda.synchronize()
        return (y == 5.0).all() and (yq == 99).all() and (S == -7).all()

    def bad(**kw):
        b = g.copy()
        for k, v in kw.items():
            b[0][k] = v
        return b
    Y, YQ, SS = y[:20 * n], yq[:32 * n], S[:n]
    refused = [
        (dict(g=bad(N=0), xq=xq, yq=YQ), -1), (dict(g=bad(pad_h=2), xq=xq, yq=YQ), -1),
        (dict(g=bad(ceil_mode=2), xq=xq, yq=YQ), -1), (dict(g=bad(Cpad=24), xq=xq, yq=YQ), -1),
        (dict(g=bad(OH=OH + 1), xq=xq, yq=YQ), -1), (dict(g=g, xq=xq, x=x, yq=YQ), -1), (dict(g=g, yq=YQ), -1),
        (dict(g=g, xq=xq, yq=YQ, y=Y), -1), (dict(g=g, xq=xq), -1), (dict(g=g, xq=xq, yq=yq[1:32 * n + 1]), -1),
        (dict(g=g, xq=xq, S=SS), -1),
        (dict(g=g, xq=xq, yq=xq.view(-1)[:32 * n]), -1), (dict(g=g, x=x), -1), (dict(g=g, x=x, S=SS), -1),
        (dict(g=g, x=x, yq=YQ, out=(-1.0, 1.0, 9)), -2), (dict(g=g, x=x, yq=YQ, out=(-1.0, 1.0, 0)), -1),
        (dict(g=g, x=x, yq=YQ, out=(-1.0, math.inf, 8)), -1), (dict(g=g, x=x, yq=YQ, out=(math.nan, 1.0, 8)), -1),
        (dict(g=g, x=x, yq=YQ, out=(-3e38, 3e38, 1)), -1), (dict(g=g, x=x, y=x.view(-1)[:20 * n]), -1),
        (dict(g=g, x=x, y=Y, yq=Y.view(torch.int8)[:32 * n], out=(-1.0, 1.0, 8)), -1),
    ]
    for kw, rc in refused:
        assert _pool(**kw) == rc, kw
        assert untouched(), kw
    assert _pool(g, x=x, y=Y, yq=YQ, out=(-1.0, 1.0, 8)) == 0          # codes mode's out is not read
    assert _pool(g, xq=xq, yq=YQ, S=SS, out=(math.nan, 1.0, 99)) == 0
    torch.cuda.synchronize()
    assert (y[20 * n:] == 5.0).all() and (yq[32 * n:] == 99).all() and (S[n:] == -7).all()


# ---- models in the reference's evaluation state -------------------------------------------------------------------------
def _equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_equal(u, v) for u, v in zip(a, b))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# (network, chain_affine flags, convolution inputs carried as codes, convolutions, fused concatenations, pool modes),
# measured on an H100: every pool is fused, ResNet-18's stem in fp32 mode (its output is also layer1.0's residual).
# SqueezeNet 1.1 has no BatchNorm, which the equalization of the evaluation state needs: it is tested below with fixed
# ranges instead.
NETWORKS = [("resnet18", dict(), (19, 20), 0, ["fp32"]),
            ("googlenet", dict(concat=True), (56, 57), 8, ["codes"] * 13)]


@pytest.mark.parametrize("net,kw,carried,cats,pools", NETWORKS, ids=[n[0] for n in NETWORKS])
def test_evaluation_state_chained_through_max_pools(net, kw, carried, cats, pools):
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state(net, batch=4) as (model, qgraph, qtarg):
            ct = LT.module_tensor_op
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True, pools=True, **kw)
            base = int8.chain_affine(model, residual=True, **kw)
            x = torch.randn(2, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
            x.clamp_(-2.5, 2.5)
            with torch.no_grad():
                ref = model(x)
                assert _equal(ref, gm(x)) and _equal(ref, base(x))
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
            convs = [n for n, m in gm.named_modules() if isinstance(m, int8.AffineInt8Conv2d)]
            got = (len({q for _, q, _ in gm.requantized_edges}), len(convs))
            print("%s: carried %d of %d (without pools %d), cats %d, pools %s, observers %d of %d" % (
                net, got[0], got[1], len({q for _, q, _ in base.requantized_edges}), len(getattr(gm, "fused_cats", [])),
                [p[:2] for p in gm.fused_pools], len(gm.fused_observers), ct.len))
            assert got == carried and len(getattr(gm, "fused_cats", [])) == cats
            assert [m for _, m, _ in gm.fused_pools] == pools
            assert len(gm.fused_observers) == len(base.fused_observers) == ct.len
            assert any(isinstance(m, int8.AffineInt8MaxPool2d) for m in gm.modules())
            # the same model without functional-op observers
            LT.restore_op()
            LT.module_tensor_op = None
            try:
                gm2 = int8.chain_affine(model, residual=True, pools=True, **kw)
                with torch.no_grad():
                    assert _equal(model(x), gm2(x))
                assert [m for _, m, _ in gm2.fused_pools] == pools and gm2.fused_observers == []
            finally:
                LT.module_tensor_op = ct
                LT.replace_op()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_squeezenet_with_fixed_ranges_chained_through_max_pools():
    """SqueezeNet 1.1 with BN folded, 8-bit weights, input ranges [-2, 6] and the functional-op observers of an eager run
    (tests/test_int8_affine_pool_heads_host.py fixed_range_model): 8 concatenations and 3 pools fused, 25 of 26 convolution
    inputs carried, every observer fused, equal to the per-layer model."""
    from collections import OrderedDict
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    from test_int8_affine_observe_host import _state
    from test_int8_affine_pool_heads_host import fixed_range_model
    model = fixed_range_model("squeezenet1_1").cuda().eval()
    x = torch.randn(2, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
    records = affine_observed_state.record_ops(model, x)
    with _state(model, records) as ct:
        ct.cuda()
        int8.convert_affine(model, OrderedDict((id(m), m) for m in model.modules() if isinstance(m, Q.QuantNConv2d)),
                            [Q.QuantNConv2d])
        gm = int8.chain_affine(model, residual=True, concat=True, pools=True)
        with torch.no_grad():
            assert _equal(model(x), gm(x))
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
        convs = [n for n, m in gm.named_modules() if isinstance(m, int8.AffineInt8Conv2d)]
        assert (len({q for _, q, _ in gm.requantized_edges}), len(convs)) == (25, 26)
        assert len(gm.fused_cats) == 8 and [m for _, m, _ in gm.fused_pools] == ["codes"] * 3
        assert len(gm.fused_observers) == ct.len == 16


# ---- detection-head rows ----------------------------------------------------------------------------------------------------
ROWS = [  # (N, Cin, H, W, O, k, stride, groups)
    (2, 19, 9, 7, 12, 1, 1, 1),
    (3, 33, 10, 10, 126, 3, 1, 1),
    (1, 24, 19, 19, 130, 3, 2, 1),
    (2, 65, 7, 9, 65, 3, 1, 65),
    (3, 16, 10, 10, 16, 3, 2, 16),
]


def _measure(lo, hi, bits=8):
    from dfq_b200.utils.quantize import QuantMeasure
    q = QuantMeasure(num_bits=bits).cuda().eval()
    q.running_min.fill_(float(f32(lo)))
    q.running_max.fill_(float(f32(hi)))
    return q


@pytest.mark.parametrize("case", range(len(ROWS)))
@pytest.mark.parametrize("codes_in", [False, True])
@pytest.mark.parametrize("observers", ["off", "operand", "operand_tail"])
def test_rows_equal_the_permuted_observed_layer(case, codes_in, observers):
    import torch.nn as nn
    from dfq_b200 import int8
    from test_gpu_int8_affine import _fake_quantized_conv
    N, Cin, H, W, O, k, stride, groups = ROWS[case]
    torch.manual_seed(case)
    conv = _fake_quantized_conv(nn.Conv2d(Cin, O, k, stride, k // 2, groups=groups).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.3, 2.9, name="h")
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    clamp = (0.0, 6.0) if case % 2 else (-math.inf, math.inf)
    obs = (-2.1, 3.3, 8) if observers != "off" else None
    tail = (-0.7, 1.9, 6) if observers == "operand_tail" else None
    rows = layer.chained(codes_in=codes_in, name="h", epilogue=int8.Epilogue(None, clamp, fp32=True), rows=True)
    if obs is not None:
        rows = rows.observe(obs=obs, tail=tail)
    with torch.no_grad():
        v = layer(x).clamp(*clamp) if clamp[0] > -math.inf else layer(x)
        if obs is not None:
            v = _measure(*obs)(v)
        if tail is not None:
            v = _measure(*tail)(v)
    OH, OW = v.shape[2:]
    n, off, stride_ = OH * OW * O, 37, OH * OW * O + 53
    out = torch.full((N, stride_), 7.5, device="cuda")
    if codes_in:
        xq, S, *_ = layer._input(x)
        arg = (xq.view(N, H, W, -1), S)
    else:
        arg = x
    assert rows(arg, out=out, off=off) is out
    want = torch.full_like(out, 7.5)
    want[:, off:off + n] = v.permute(0, 2, 3, 1).reshape(N, n)
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))
    alone = rows(arg)                                           # a tensor of its own
    assert torch.equal(alone.reshape(N, n).view(torch.int32), want[:, off:off + n].contiguous().view(torch.int32))


def test_rows_refusals_leave_the_buffers_untouched():
    import torch.nn as nn
    from dfq_b200 import _lib, int8
    from test_gpu_int8_affine import _fake_quantized_conv
    conv = _fake_quantized_conv(nn.Conv2d(16, 20, 3).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.0, 1.0)
    g = layer._geometry(1, 6, 6)                                            # 4 x 4 output: 320 floats
    xq, S, *_ = layer._input(torch.randn(1, 16, 6, 6, device="cuda"))
    y = torch.full((400,), 5.0, device="cuda")

    def call(**kw):
        d = dict(y=y.data_ptr(), off=8, img_stride=400, pre_lo=-math.inf, pre_hi=math.inf, post_lo=-math.inf,
                 post_hi=math.inf, obs_min=-1.0, obs_max=1.0, obs_bits=8, tail_min=-1.0, tail_max=1.0, tail_bits=0)
        d.update(kw)
        r = np.zeros(1, _lib.I8_AFFINE_ROWS_DT)
        for k, v in d.items():
            r[0][k] = v
        return _lib.load().dfq_i8_affine_conv_rows(_p(xq), _p(S), _p(layer.weight_codes), _p(layer.tap_table),
                                                   _lib.table_ptr(layer.constants), _p(layer.bias), _lib.table_ptr(r),
                                                   _lib.table_ptr(g), _lib.stream_ptr())
    refused = [
        (dict(y=0), -1), (dict(y=y.data_ptr() + 2), -1), (dict(off=-1), -1), (dict(img_stride=327), -1),
        (dict(pre_lo=math.nan), -1), (dict(post_lo=2.0, post_hi=1.0), -1), (dict(obs_bits=-1), -1),
        (dict(obs_bits=9), -2), (dict(obs_max=math.inf), -1), (dict(tail_bits=9), -2),
        (dict(tail_bits=4, tail_min=math.nan), -1), (dict(y=xq.data_ptr()), -1), (dict(y=S.data_ptr()), -1),
    ]
    for kw, rc in refused:
        assert call(**kw) == rc, kw
        torch.cuda.synchronize()
        assert (y == 5.0).all(), kw
    assert call() == 0 and call(off=80, tail_bits=8) == 0
    torch.cuda.synchronize()
    assert (y[:8] == 5.0).all() and (y[8:] != 5.0).any()


def test_ssd_evaluation_state_heads_written_in_place():
    """SSD-Lite (is_test) in the evaluation state under residual=True, concat=True, fold_pads=True, heads=True: both
    outputs torch.equal to the per-layer model at batch 2 and 3 through the same GraphModule, 2 head concatenations of
    6 producers (k = 21 and 4), and every observer the replay inserts fused: 10 adds x 2 operands, 12 head operands and
    the softmax input, 33; the same model without functional-op observers too."""
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
            ct = LT.module_tensor_op
            int8.convert_affine(model, qgraph, qtarg)
            kw = dict(residual=True, concat=True, fold_pads=True)
            gm = int8.chain_affine(model, heads=True, **kw)
            base = int8.chain_affine(model, **kw)
            g = torch.Generator(device="cuda").manual_seed(2)
            for n in (2, 3):
                x = torch.randn(n, 3, 300, 300, device="cuda", generator=g).clamp_(-2.5, 2.5)
                with torch.no_grad():
                    ref = model(x)
                    assert _equal(ref, gm(x)) and _equal(ref, base(x)), n
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
            kinds = [w for _, w, _ in gm.fused_observers]
            print("ssd: heads %s, observers %d distinct of %d (%s), edges %d" % (
                [(c, len(p), k) for c, p, k in gm.fused_heads], len({o for o, _, _ in gm.fused_observers}), ct.len,
                {w: kinds.count(w) for w in set(kinds)}, len(gm.requantized_edges)))
            assert [(len(p), k) for _, p, k in gm.fused_heads] == [(6, 21), (6, 4)]
            assert ct.len == 33 and len({o for o, _, _ in gm.fused_observers}) == 33
            assert (kinds.count("head"), kinds.count("tail")) == (12, 6)
            assert not any(n.op == "call_function" and "cat" in getattr(n.target, "__name__", "") for n in gm.graph.nodes)
            LT.restore_op()
            LT.module_tensor_op = None
            try:
                gm2 = int8.chain_affine(model, heads=True, **kw)
                x = torch.randn(2, 3, 300, 300, device="cuda", generator=g).clamp_(-2.5, 2.5)
                with torch.no_grad():
                    assert _equal(model(x), gm2(x))
                assert [(len(p), k) for _, p, k in gm2.fused_heads] == [(6, 21), (6, 4)] and gm2.fused_observers == []
            finally:
                LT.module_tensor_op = ct
                LT.replace_op()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
