"""The affine layout epilogue and upsample on the H100 (dfq_i8_affine_conv_layout, dfq_i8_affine_upsample_bilinear,
dfq_b200.int8.chain_affine(concat=True, fold_pads=True)): a folded pad against the layer on F.pad(x) and the oracle, slices
of a concatenation against the quantizer of the concatenated per-layer values, the upsample against QuantMeasure and the
quantizer applied to F.interpolate, the refusals, and DeepLab-v3+ / SSD-Lite in the evaluation state against their
per-layer affine models."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_observed_state
import int8_affine_chain_oracle as AC
import int8_affine_layout_oracle as AL
import int8_affine_oracle as A
from test_gpu_int8_affine import _fake_quantized_conv, _same_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-41], f32)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _quantized(v, out):
    """(codes [N, H, W, cpad], S [N, H, W]) of the fp32 NCHW v at out = (min, max, bits): the host oracle of
    dfq_i8_affine_quantize, itself checked against the device by tests/test_gpu_int8_affine.py."""
    q, S = A.act_codes(v.cpu().numpy(), *out)
    return AC.to_nhwc(q), S


# ---- the pad code -------------------------------------------------------------------------------------------------------
PAD = [  # (N, Cin, H, W, O, k, stride, dilation, (t, l), groups)
    (2, 19, 9, 7, 1, 1, 1, 1, (1, 1), 1),
    (2, 19, 9, 7, 16, 3, 1, 1, (1, 1), 1),
    (1, 24, 10, 11, 17, 3, 2, 1, (2, 1), 1),
    (3, 16, 7, 7, 64, 3, 1, 2, (2, 2), 1),
    (2, 33, 9, 9, 65, 3, 1, 1, (1, 2), 1),
    (1, 40, 13, 5, 130, 3, 2, 2, (2, 2), 1),
    (2, 17, 9, 7, 17, 3, 1, 1, (1, 1), 17),
    (1, 32, 12, 13, 32, 3, 2, 1, (1, 1), 32),
    (2, 65, 7, 7, 65, 3, 1, 2, (2, 2), 65),
    (3, 24, 11, 9, 24, 3, 1, 1, (2, 1), 24),
]
RANGES = {"neg": (-1.7, 2.9), "zero": (0.0, 3.1), "pos": (0.4, 3.3)}


def _pad_case(N, Cin, H, W, O, k, stride, dil, pad, groups, bits=8, rng="neg", seed=0):
    from dfq_b200 import int8
    torch.manual_seed(seed)
    conv = _fake_quantized_conv(nn.Conv2d(Cin, O, k, stride, 0, dil, groups).cuda())
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    lo, hi = RANGES[rng]
    layer = int8.AffineInt8Conv2d.from_conv(conv, f32(lo), f32(hi), act_bits=bits)
    t, l = pad
    xp = F.pad(x, (l, l, t, t))
    folded = layer.fold_pad(pad)
    assert folded.pad_code == AL.zero_code(lo, hi, bits)
    if rng == "pos":
        assert folded.pad_code == -128                          # +0.0 clamps to the bottom code
    want, _ = layer.run(xp)
    got, _ = folded.run(x)
    assert _same_bits(got.cpu().numpy(), want.cpu().numpy()), "y vs the layer on F.pad(x)"
    wo = conv.weight.detach().cpu().numpy()
    y_o = AL.folded_conv(x.cpu().numpy(), (lo, hi, bits), wo, layer.w_min, layer.w_scale, 8, conv.bias.detach().cpu().numpy(),
                         pad, conv.stride, conv.dilation, groups)
    assert _same_bits(got.cpu().numpy(), y_o), "y vs oracle"
    # codes and S for a consumer, from fp32 input and from the codes / S of the input
    out = (f32(-1.1), f32(5.5), 8)
    ref = layer.chained(requant=(out, 0.0, 6.0), sums=True)(xp)
    codes_in = folded.chained(codes_in=True, requant=(out, 0.0, 6.0), sums=True)
    xq, S, *_ = layer._input(x)
    for got in (folded.chained(requant=(out, 0.0, 6.0), sums=True)(x),
                codes_in((xq.view(N, H, W, -1), S.view(N, H, W) if groups == 1 else None))):
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


@pytest.mark.parametrize("case", PAD, ids=lambda c: "x".join(map(str, c[:8])) + "_p%d%d_g%d" % (*c[8], c[9]))
@pytest.mark.parametrize("rng", sorted(RANGES))
def test_folded_pad_equals_the_layer_on_the_padded_input(case, rng):
    _pad_case(*case, rng=rng, seed=sum(case[:8]))


@pytest.mark.parametrize("bits", range(1, 9))
@pytest.mark.parametrize("dw", [False, True])
def test_folded_pad_every_activation_bit_width(bits, dw):
    case = (2, 20, 8, 9, 20, 3, 1, 1, (1, 2), 20) if dw else (2, 20, 8, 9, 33, 3, 1, 1, (1, 2), 1)
    _pad_case(*case, bits=bits, rng="neg", seed=bits)


def test_folded_pad_m_tail_and_grid_stride():
    _pad_case(3, 16, 31, 29, 70, 3, 1, 1, (1, 1), 1, seed=3)                 # M = 2697: a partial last tile
    _pad_case(8, 96, 57, 57, 96, 3, 1, 1, (1, 1), 96, seed=4)                # the depthwise grid-stride loop


# ---- channel slices -----------------------------------------------------------------------------------------------------
def _slices(widths, dw, observers, seed=0):
    from dfq_b200 import int8
    torch.manual_seed(seed)
    N, H, W = 2, 9, 7
    out = (f32(-0.9), f32(4.7), 8)
    layers, xs, vs = [], [], []
    for i, O in enumerate(widths):
        Cin = O if dw else 13 + 7 * i
        conv = _fake_quantized_conv(nn.Conv2d(Cin, O, 3, 1, 1, 1, O if dw else 1).cuda())
        b = conv.bias.detach().cpu().numpy().copy()
        b[:min(O, SPECIAL.size)] = SPECIAL[:min(O, SPECIAL.size)]
        with torch.no_grad():
            conv.bias.copy_(torch.from_numpy(b))
        x = torch.randn(N, Cin, H, W, device="cuda") * 2
        layers.append(int8.AffineInt8Conv2d.from_conv(conv, f32(float(x.min()) * 0.8), f32(float(x.max()) * 0.8)))
        xs.append(x)
    offs = np.cumsum([0] + [(w + 15) // 16 * 16 for w in widths[:-1]]).tolist()
    cstride = offs[-1] + (widths[-1] + 15) // 16 * 16 + 32        # 32 sentinel channels past the last slice
    codes = torch.full((N, H, W, cstride), 99, dtype=torch.int8, device="cuda")
    S = torch.zeros((N, H, W), dtype=torch.int32, device="cuda")
    from dfq_b200.utils.quantize import QuantMeasure
    for i, (layer, x, off) in enumerate(zip(layers, xs, offs)):
        obs = (f32(-0.4 - 0.1 * i), f32(3.9 + 0.3 * i), 8 - i) if observers else None
        w = layer.chained(epilogue=int8.Epilogue(out, (0.0, 6.0), (-1.0, 4.0)), sums=True, out_slice=(off, cstride))
        if obs is not None:
            w.observe(obs)
        assert w(x, out=(codes, S))[0] is codes
        v = layer.run(x)[0].clamp(0.0, 6.0)                       # the per-layer value: clamp, observer, clamp
        if obs is not None:
            q = QuantMeasure(num_bits=obs[2]).cuda().eval()
            q.running_min.fill_(float(obs[0])); q.running_max.fill_(float(obs[1]))
            with torch.no_grad():
                v = q(v)
        vs.append(v.clamp(-1.0, 4.0))
    want_q, want_S = _quantized(torch.cat(vs, 1), out)
    got = codes.cpu().numpy()
    real = np.concatenate([np.arange(o, o + w) for o, w in zip(offs, widths)])
    assert np.array_equal(got[..., real], want_q[..., :len(real)]), "codes"
    pads = np.setdiff1d(np.arange(offs[-1] + (widths[-1] + 15) // 16 * 16), real)
    assert (got[..., pads] == 0).all(), "pad channels"
    assert (got[..., cstride - 32:] == 99).all(), "sentinels past the slices"
    assert np.array_equal(S.cpu().numpy(), want_S), "S"


@pytest.mark.parametrize("widths", [(16, 17), (32, 48, 5), (16, 64, 16, 130), (48, 16, 32, 16, 33)],
                         ids=lambda w: "-".join(map(str, w)))
@pytest.mark.parametrize("dw", [False, True])
@pytest.mark.parametrize("observers", [False, True])
def test_slices_share_codes_and_sums(widths, dw, observers):
    _slices(widths, dw, observers, seed=sum(widths))


# ---- the affine upsample ------------------------------------------------------------------------------------------------
def _upsample(N, Cn, H, W, OH, OW, ac, obs=(f32(-0.3), f32(2.2), 8), special=False, seed=0):
    from dfq_b200 import int8
    from dfq_b200.utils.quantize import QuantMeasure
    torch.manual_seed(seed)
    x = torch.randn(N, Cn, H, W, device="cuda") * 2
    if special:
        x.view(-1)[::7][:SPECIAL.size] = torch.from_numpy(SPECIAL).cuda()
    out, pre, post = (f32(-1.3), f32(2.9), 8), (-0.5, 2.5), (-1.0, 2.0)
    coff, cstride = 16, 16 + (Cn + 15) // 16 * 16 + 16
    up = int8.AffineInt8UpsampleBilinear(Cn, ac, out, (coff, cstride), pre, obs, post, sums=True)
    codes = torch.full((N, OH, OW, cstride), 99, dtype=torch.int8, device="cuda")
    S = torch.zeros((N, OH, OW), dtype=torch.int32, device="cuda")
    up(x, (OH, OW), out=(codes, S))
    v = F.interpolate(x, size=(OH, OW), mode="bilinear", align_corners=ac)
    v = torch.where(torch.isnan(v), v, v.clamp(*pre))
    if obs is not None:
        q = QuantMeasure(num_bits=obs[2]).cuda().eval()
        q.running_min.fill_(float(obs[0])); q.running_max.fill_(float(obs[1]))
        with torch.no_grad():
            v = q(v)
    v = torch.where(torch.isnan(v), v, v.clamp(*post))
    want_q, want_S = _quantized(v, out)
    got = codes.cpu().numpy()
    assert np.array_equal(got[..., coff:coff + Cn], want_q[..., :Cn])
    assert (got[..., coff + Cn:coff + (Cn + 15) // 16 * 16] == 0).all()
    assert (got[..., :coff] == 99).all() and (got[..., coff + (Cn + 15) // 16 * 16:] == 99).all()
    assert np.array_equal(S.cpu().numpy(), want_S)


@pytest.mark.parametrize("ac", [False, True])
@pytest.mark.parametrize("shape", [(2, 19, 1, 1, 33, 33), (1, 40, 33, 33, 129, 129), (2, 17, 7, 5, 19, 23),
                                   (1, 256, 9, 9, 33, 33), (2, 48, 10, 10, 10, 10)], ids=lambda s: "x".join(map(str, s)))
def test_affine_upsample_equals_quantmeasure_on_interpolate(ac, shape):
    _upsample(*shape, ac, seed=sum(shape))


@pytest.mark.parametrize("bits", [0, 1, 5])
def test_affine_upsample_special_values_and_observer_bits(bits):
    _upsample(2, 21, 6, 7, 13, 11, True, obs=None if bits == 0 else (f32(-0.3), f32(2.2), bits), special=True, seed=bits)
    _upsample(1, 16, 5, 5, 5, 5, False, obs=None if bits == 0 else (f32(-0.3), f32(2.2), bits), special=True, seed=bits)


def _resize_call(x, yq, S, **kw):
    from dfq_b200 import _lib
    g = np.zeros(1, _lib.I8_AFFINE_RESIZE_DT)
    d = dict(N=1, C=20, H=4, W=4, OH=8, OW=8, align_corners=1, coff=16, cstride=64, pre_lo=-INF, pre_hi=INF,
             obs_min=-1.0, obs_max=1.0, obs_bits=8, post_lo=-INF, post_hi=INF, out_min=-1.0, out_max=1.0, out_bits=8)
    d.update(kw)
    for k, v in d.items():
        g[0][k] = v
    return _lib.load().dfq_i8_affine_upsample_bilinear(_p(x), _p(yq), _p(S), _lib.table_ptr(g), _lib.stream_ptr())


def test_affine_upsample_refusals_leave_the_buffers_untouched():
    x = torch.randn(1, 20, 4, 4, device="cuda")
    yq = torch.full((64 * 64 + 16,), 99, dtype=torch.int8, device="cuda")
    S = torch.full((64 + 4,), -7, dtype=torch.int32, device="cuda")
    refused = [
        (dict(OH=0), -1), (dict(C=-1), -1), (dict(align_corners=2), -1), (dict(coff=8), -1), (dict(cstride=40), -1),
        (dict(coff=48), -1), (dict(pre_lo=2.0, pre_hi=1.0), -1), (dict(post_lo=math.nan), -1), (dict(obs_bits=-1), -1),
        (dict(obs_bits=9), -2), (dict(obs_max=INF), -1), (dict(out_bits=0), -1), (dict(out_bits=9), -2),
        (dict(out_min=math.nan), -1), (dict(out_min=-3e38, out_max=3e38, out_bits=1), -1),
    ]
    for kw, rc in refused:
        assert _resize_call(x, yq[:64 * 64], S[:64], **kw) == rc, kw
        torch.cuda.synchronize()
        assert (yq == 99).all() and (S == -7).all(), kw
    assert _resize_call(x, yq[1:], S[:64]) == -1                           # yq not 16-byte aligned
    assert _resize_call(None, yq[:64 * 64], S[:64]) == -1 and _resize_call(x, None, S[:64]) == -1
    xs = torch.zeros(64 * 64 // 4 + 64, device="cuda")                     # x overlapping the slice
    assert _resize_call(xs, xs.view(torch.int8)[:64 * 64], S[:64]) == -1
    torch.cuda.synchronize()
    assert (yq == 99).all() and (S == -7).all()
    S[:64].zero_()
    assert _resize_call(x, yq[:64 * 64], S[:64]) == 0
    torch.cuda.synchronize()
    assert (yq[64 * 64:] == 99).all() and (S[64:] == -7).all()


# ---- layout refusals ----------------------------------------------------------------------------------------------------
def test_layout_refusals_leave_the_buffers_untouched():
    from dfq_b200 import _lib, int8
    conv = _fake_quantized_conv(nn.Conv2d(16, 20, 3).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.0, 1.0)
    g = layer._geometry(1, 6, 6)                                            # 4 x 4 output
    xq, S, *_ = layer._input(torch.randn(1, 16, 6, 6, device="cuda"))
    yq = torch.full((16 * 64 + 16,), 99, dtype=torch.int8, device="cuda")
    S_out = torch.full((16 + 4,), -7, dtype=torch.int32, device="cuda")

    def call(lay=(16, 64, 1, 1, -3), out=(-1.0, 1.0, 8), pre=NONE, obs=None):
        d = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
        d[0] = (0, 0, yq.data_ptr(), S_out.data_ptr()) + tuple(out) + tuple(pre) + NONE
        lt = np.zeros(1, _lib.I8_AFFINE_LAYOUT_DT)
        lt[0] = lay
        o = None
        if obs is not None:
            o = np.zeros(1, _lib.I8_AFFINE_OBSERVE_DT)
            o[0] = tuple(obs) + (0.0, 0.0, 0)
        return _lib.load().dfq_i8_affine_conv_layout(_p(xq), _p(S), _p(layer.weight_codes), _p(layer.tap_table),
                                                     _lib.table_ptr(layer.constants), _p(layer.bias), _lib.table_ptr(d),
                                                     None if o is None else _lib.table_ptr(o), _lib.table_ptr(lt),
                                                     _lib.table_ptr(g), _lib.stream_ptr())
    refused = [
        (dict(lay=(8, 64, 1, 1, 0)), -1), (dict(lay=(16, 40, 1, 1, 0)), -1), (dict(lay=(48, 64, 1, 1, 0)), -1),
        (dict(lay=(-16, 64, 1, 1, 0)), -1), (dict(lay=(16, 64, 2, 1, 0)), -1), (dict(lay=(16, 64, 1, 2, 0)), -1),
        (dict(lay=(16, 64, 1, 1, 128)), -1), (dict(lay=(16, 64, 1, 1, -129)), -1), (dict(out=(-1.0, 1.0, 9)), -2),
        (dict(pre=(1.0, 0.0)), -1), (dict(obs=(0.0, 0.0, 0)), -1), (dict(obs=(-1.0, 1.0, 9)), -2),
    ]
    for kw, rc in refused:
        assert call(**kw) == rc, kw
        torch.cuda.synchronize()
        assert (yq == 99).all() and (S_out == -7).all(), kw
    assert call(lay=(16, 64, 0, 0, 200)) == 0                               # the code is only read when the pad is on
    S_out[:16].zero_()
    assert call() == 0 and call(obs=(-0.5, 0.5, 8)) == 0
    torch.cuda.synchronize()
    assert (yq[16 * 64:] == 99).all() and (S_out[16:] == -7).all()
    assert (yq[:16 * 64].view(16, 64)[:, :16] == 99).all() and (yq[:16 * 64].view(16, 64)[:, 48:] == 99).all()


# ---- models in the reference's evaluation state -------------------------------------------------------------------------
def _equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_equal(u, v) for u, v in zip(a, b))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_deeplab_evaluation_state_chained_through_pads_and_concatenations():
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
            ct = LT.module_tensor_op
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
            base = int8.chain_affine(model, residual=True)
            g = torch.Generator(device="cuda").manual_seed(2)
            for size in (129, 97):
                x = torch.randn(2, 3, size, size, device="cuda", generator=g).clamp_(-2.5, 2.5)
                with torch.no_grad():
                    ref, got, got_base = model(x), gm(x), base(x)
                assert _equal(ref, got) and _equal(ref, got_base), size
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
            convs = [n for n, m in gm.named_modules() if isinstance(m, int8.AffineInt8Conv2d)]
            carried = {q for _, q, _ in gm.requantized_edges}
            print("deeplab: folded %d, cats %d, upsamples %d, observers %d, edges %d, inputs carried %d of %d: not %s" % (
                len(gm.folded_pads), len(gm.fused_cats), len(gm.fused_upsamples), len(gm.fused_observers),
                len(gm.requantized_edges), len(carried), len(convs), sorted(set(convs) - carried)))
            assert len(gm.folded_pads) == 17 and all(tl in ((1, 1), (2, 2)) for _, _, tl in gm.folded_pads)
            assert (len(gm.fused_cats), len(gm.fused_upsamples), len(gm.fused_observers)) == (2, 2, 30)
            assert sorted(c[2] for c in gm.fused_cats) == [[0, 256], [0, 256, 512, 768, 1024]]
            assert not any(n.op == "call_function" and n.target in (F.pad, torch._C._nn.pad) for n in gm.graph.nodes)
            assert (len(carried), len(convs)) == DEEPLAB_CARRIED
            assert sorted(set(convs) - carried) == ["aspp.image_pool.1", "backbone.features.0.0"]
            # the same model without functional-op observers
            LT.restore_op()
            LT.module_tensor_op = None
            try:
                gm2 = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
                x = torch.randn(2, 3, 129, 129, device="cuda", generator=g).clamp_(-2.5, 2.5)
                with torch.no_grad():
                    assert _equal(model(x), gm2(x))
                assert (len(gm2.folded_pads), len(gm2.fused_cats), len(gm2.fused_upsamples), len(gm2.fused_observers)) \
                    == (17, 2, 2, 0)
            finally:
                LT.module_tensor_op = ct
                LT.replace_op()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


# convolution inputs carried as codes in the DeepLab above, of its convolutions, as measured on an H100: the two left read
# fp32 - the stem (the network's input) and the image-pooling branch's 1x1 convolution (behind an adaptive average pool)
DEEPLAB_CARRIED = (59, 61)


def test_ssd_evaluation_state_head_concatenations_stay():
    from dfq_b200 import int8
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
            x = torch.randn(2, 3, 300, 300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
            with torch.no_grad():
                assert _equal(model(x.clamp(-2.5, 2.5)), gm(x.clamp(-2.5, 2.5)))
            assert gm.fused_cats == [] and gm.fused_upsamples == []
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
