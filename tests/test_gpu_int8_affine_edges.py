"""The affine int8 scheme on the H100 off its 8-bit defaults (dfq_i8_affine_* in libdfq_sm90.so, dfq_b200.int8.convert_affine
and chain_affine): 1- to 8-bit activation and weight codes from both fake-quantization recipes, output pixels without an
in-image tap, the largest K whose int32 sums cannot overflow and the first one refused, the reference's own recipe end to
end (weights fake-quantized on the CPU, 8-bit biases, 8, 6 and 4-bit weights), and SSD-Lite in the reference's evaluation
state.  Kernels are checked bit for bit against tests/int8_affine_oracle.py, int8_affine_chain_oracle.py and
int8_affine_observe_oracle.py, into sentinel-filled buffers."""
import ctypes as C
import copy
import math
from collections import Counter, OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_calibrated
import affine_observed_state
import int8_affine_chain_oracle as AC
import int8_affine_observe_oracle as AO
import int8_affine_oracle as A
from oracle import dfq_oracle as D
from test_gpu_int8_affine import _fake_quantized_conv, _same_bits
from test_gpu_int8_affine_chain import _launch as _launch_fused
from test_gpu_int8_affine_observe import _launch as _launch_observed

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
BIAS = np.array([np.inf, -np.inf, -0.0, 1e-40, -1e-41, 0.0], f32)     # y = fp32(sum) + bias: no NaN, whose payload differs
Y_SENTINEL, P_SENTINEL, Q_SENTINEL, S_SENTINEL = 7.25, -2 ** 31, 99, -2 ** 31
TAIL = 64


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _low_bit_conv(Cin, O, k, s, p, d, g, w_bits, div_mode, seed, special_bias=False):
    """A seeded nn.Conv2d on the GPU whose weights quantize_targ_layer's recipe put on a w_bits-bit min / max grid: "div" on
    the CPU (true division, the reference's mains), "recip" on CUDA (reciprocal multiply)."""
    torch.manual_seed(seed)
    conv = nn.Conv2d(Cin, O, k, s, p, d, g)
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(D.quantize(conv.weight.numpy(), w_bits, div_mode=div_mode)))
        if special_bias:
            conv.bias[:min(O, BIAS.size)] = torch.from_numpy(BIAS[:min(O, BIAS.size)])
    return conv.cuda()


def _layer(conv, x, act_bits, w_bits):
    from dfq_b200 import int8
    return int8.AffineInt8Conv2d.from_conv(conv, f32(float(x.min()) * 0.8), f32(float(x.max()) * 0.8), act_bits, w_bits)


def _codes_and_terms(layer, conv, x):
    """(oracle input codes, oracle weight codes, (P, A, Wv, Nv)) at the layer's bits."""
    xo, _ = A.act_codes(x.cpu().numpy(), layer.act_min, layer.act_max, layer.act_bits)
    wo, bad = A.weight_codes(conv.weight.detach().cpu().numpy(), layer.w_min, layer.w_scale, layer.w_bits)
    assert bad == 0
    return xo, wo, A.terms(xo, wo, conv.stride, conv.padding, conv.dilation, conv.groups)


def _check_pack(layer, wo):
    """The packed codes (pad channels zero) and, dense, the tap prefix table."""
    kh, kw = layer.kernel_size
    Cin, Cout = layer.in_channels, layer.out_channels
    codes = layer.weight_codes.cpu().numpy()
    if layer.groups == 1:
        codes = codes.reshape(Cout, kh, kw, layer.cpad)
        assert np.array_equal(codes[..., :Cin], wo.transpose(0, 2, 3, 1)) and not codes[..., Cin:].any()
        assert np.array_equal(layer.tap_table.cpu().numpy().reshape(-1, kh + 1, kw + 1), A.tap_table(wo))
    else:
        codes = codes.reshape(kh * kw, layer.cpad)
        assert np.array_equal(codes[:, :Cin], wo.reshape(Cin, kh * kw).T) and not codes[:, Cin:].any()


def _run_into_sentinels(layer, x):
    """(input codes [N, H, W, cpad], S, y, P) of the per-layer entries (dfq_i8_affine_quantize, dfq_i8_affine_conv), y and P
    written into sentinel-filled buffers whose tails past the output must stay untouched."""
    from dfq_b200 import _lib
    xq, S, N, H, W = layer._input(x)
    g = layer._geometry(N, H, W)
    shape = (N, layer.out_channels, int(g[0]["OH"]), int(g[0]["OW"]))
    n = int(np.prod(shape))
    y = torch.full((n + TAIL,), Y_SENTINEL, device="cuda")
    P = torch.full((n + TAIL,), P_SENTINEL, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    _lib.check(lib.dfq_i8_affine_conv(_p(xq), _p(S), _p(layer.weight_codes), _p(layer.tap_table) if layer.groups == 1 else None,
                                      _lib.table_ptr(layer.constants), _p(layer.bias), _p(y), _p(P), _lib.table_ptr(g),
                                      _lib.stream_ptr()), "dfq_i8_affine_conv")
    y, P = y.cpu().numpy(), P.cpu().numpy()
    assert (y[n:] == Y_SENTINEL).all() and (P[n:] == P_SENTINEL).all(), "past the output"
    return xq.reshape(N, H, W, layer.cpad).cpu().numpy(), S.reshape(N, H, W).cpu().numpy(), y[:n].reshape(shape), \
        P[:n].reshape(shape)


def _per_layer(layer, conv, x):
    """Check the input codes and S, the packed weights, P and y of the per-layer path against the oracle; returns
    (oracle terms, y, P)."""
    xo, wo, terms = _codes_and_terms(layer, conv, x)
    xq, S, y, P = _run_into_sentinels(layer, x)
    Cin = layer.in_channels
    assert np.array_equal(xq[..., :Cin], xo.transpose(0, 2, 3, 1)) and not xq[..., Cin:].any(), "input codes"
    assert np.array_equal(S, xo.astype(np.int64).sum(axis=1)), "S"
    _check_pack(layer, wo)
    assert np.array_equal(P, terms[0]), "P"
    bias = layer.bias.cpu().numpy()
    assert _same_bits(y, A.epilogue(*terms, tuple(layer.constants[0]), bias)), "y"
    return terms, y, P


def _epilogue(layer, conv, x, out, residual=False, pre=NONE, post=NONE, obs=None, res=None, seed=0):
    """The layer through dfq_i8_affine_conv_fused (obs and res None) or dfq_i8_affine_conv_observed into sentinel-filled y,
    codes and S buffers; checks all three against the oracle and returns (v, codes [N, OH, OW, Opad], S)."""
    from dfq_b200 import _lib
    xq, S, N, H, W = layer._input(x)
    g = layer._geometry(N, H, W)
    OH, OW, O = int(g[0]["OH"]), int(g[0]["OW"]), layer.out_channels
    opad = (O + 15) // 16 * 16
    r = None
    if residual:
        rn = (np.random.default_rng(seed).standard_normal((N, O, OH, OW)) * 3).astype(f32)
        r = torch.from_numpy(rn).cuda()
    y = torch.full((N * O * OH * OW + TAIL,), Y_SENTINEL, device="cuda")
    yq = torch.full((N * OH * OW * opad + TAIL,), Q_SENTINEL, dtype=torch.int8, device="cuda")
    S_out = torch.full((N * OH * OW + TAIL,), S_SENTINEL, dtype=torch.int32, device="cuda")
    observed = obs is not None or res is not None
    if observed:
        rc = _launch_observed(layer, xq, S, g, r, y, yq, S_out, out, pre, post, obs or (0.0, 0.0, 0), res or (0.0, 0.0, 0))
    else:
        rc = _launch_fused(layer, xq, S, g, r, y, yq, S_out, out, pre, post)
    _lib.check(rc, "dfq_i8_affine_conv_observed" if observed else "dfq_i8_affine_conv_fused")
    _, _, terms = _codes_and_terms(layer, conv, x)
    args = (*terms, tuple(layer.constants[0]), layer.bias.cpu().numpy(), None if r is None else r.cpu().numpy(), pre, post,
            out)
    v_o, q_o, S_o = AO.observed(*args, obs, res) if observed else AC.fused(*args)
    y, yq, S_out = y.cpu().numpy(), yq.cpu().numpy(), S_out.cpu().numpy()
    n, m = N * O * OH * OW, N * OH * OW
    assert (y[n:] == Y_SENTINEL).all() and (yq[m * opad:] == Q_SENTINEL).all() and (S_out[m:] == S_SENTINEL).all()
    v, codes, s = y[:n].reshape(N, O, OH, OW), yq[:m * opad].reshape(N, OH, OW, opad), S_out[:m].reshape(N, OH, OW)
    assert _same_bits(v, v_o), "y vs oracle"
    assert np.array_equal(codes, AC.to_nhwc(q_o)), "codes vs oracle"
    assert np.array_equal(s, S_o), "S vs oracle"
    return v, codes, s


# ---- A. low-bit codes -----------------------------------------------------------------------------------------------------
# (N, Cin, H, W, Cout, k, s, p, d, groups), activation bits, weight bits: every width 1-8 on each side, on cases of
# tests/test_gpu_int8.py's DENSE, TILES and DW lists (unaligned C, O past the 64-channel tile, per-axis geometry)
LOW_BITS = [
    ((1, 24, 17, 16, 100, 7, 2, 3, 1, 1), 1, 8),
    ((1, 160, 9, 7, 24, 3, 1, 3, 2, 1), 2, 7),
    ((2, 17, 11, 13, 33, (3, 5), (2, 1), (1, 2), (1, 2), 1), 3, 6),
    ((5, 15, 7, 9, 65, 3, 1, 1, 1, 1), 4, 5),
    ((1, 65, 1, 1, 64, 1, 1, 0, 1, 1), 5, 4),
    ((2, 64, 6, 11, 129, 1, 1, 0, 1, 1), 6, 3),
    ((1, 144, 9, 9, 144, 3, 1, 2, 2, 144), 7, 2),
    ((2, 48, 11, 13, 48, (3, 5), (2, 1), (1, 2), (1, 2), 48), 8, 1),
    ((3, 19, 8, 8, 19, 5, 1, 2, 1, 19), 2, 4),
    ((1, 16, 13, 13, 100, 3, 2, 0, 6, 1), 8, 2),
]


def _low_id(v):
    return "x".join("-".join(map(str, e)) if isinstance(e, tuple) else str(e) for e in v) if isinstance(v, tuple) else str(v)


@pytest.mark.parametrize("div_mode", ["div", "recip"])
@pytest.mark.parametrize("case,act_bits,w_bits", LOW_BITS, ids=_low_id)
def test_low_bit_codes_per_layer_bit_exact(case, act_bits, w_bits, div_mode):
    """Codes of act_bits and w_bits bits: the input codes span [-128, 2^act_bits - 129] (the range is 0.8 of the input's)
    and the weight codes [-128, 2^w_bits - 129] (min and max of the tensor are on its grid); the grid search runs at
    qmax = 2^w_bits - 1 and the tap table sums those codes."""
    N, Cin, H, W, O, k, s, p, d, g = case
    conv = _low_bit_conv(Cin, O, k, s, p, d, g, w_bits, div_mode, seed=act_bits * 10 + w_bits)
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    layer = _layer(conv, x, act_bits, w_bits)
    assert layer.w_bits == w_bits and layer.act_bits == act_bits
    _per_layer(layer, conv, x)
    xo, wo, _ = _codes_and_terms(layer, conv, x)
    assert xo.min() == -128 and xo.max() == 2 ** act_bits - 129
    assert wo.min() == -128 and wo.max() == 2 ** w_bits - 129


@pytest.mark.parametrize("observed", [False, True], ids=["fused", "observed"])
@pytest.mark.parametrize("case,act_bits,w_bits", [LOW_BITS[i] for i in (0, 3, 5, 6, 7, 8)], ids=_low_id)
def test_low_bit_codes_through_the_epilogues(case, act_bits, w_bits, observed):
    """The same low-bit inputs and weights through dfq_i8_affine_conv_fused and dfq_i8_affine_conv_observed with a residual,
    the consumer's codes at other low bit widths."""
    N, Cin, H, W, O, k, s, p, d, g = case
    conv = _low_bit_conv(Cin, O, k, s, p, d, g, w_bits, "div" if act_bits % 2 else "recip", seed=act_bits + w_bits,
                         special_bias=True)
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    layer = _layer(conv, x, act_bits, w_bits)
    out = (f32(-1.1), f32(5.5), 9 - act_bits)
    kw = dict(obs=(f32(-0.3), f32(4.1), w_bits), res=(f32(-2.7), f32(3.3), act_bits)) if observed else {}
    _epilogue(layer, conv, x, out, residual=True, pre=(0.0, 6.0), seed=act_bits, **kw)


@pytest.mark.parametrize("I,O,act_bits,w_bits", [(1, 1, 8, 8), (1, 37, 3, 5), (17, 1, 6, 1), (17, 37, 2, 7), (1280, 1, 7, 4),
                                                 (1280, 37, 5, 2)])
def test_low_bit_linear_on_a_3d_input(I, O, act_bits, w_bits):
    """AffineInt8Linear on [B, T, I]: the leading dimensions are one batch of 1x1 convolutions; 1 and 17 input features
    leave the 16-channel chunk nearly empty, one output feature one weight row (with I = O = 1 a constant weight tensor,
    whose scale is quantize_targ_layer's floor)."""
    from dfq_b200 import int8
    torch.manual_seed(I * 100 + O)
    lin = nn.Linear(I, O)
    with torch.no_grad():
        lin.weight.copy_(torch.from_numpy(D.quantize(lin.weight.numpy(), w_bits, div_mode="div")))
    lin = lin.cuda()
    x = torch.randn(3, 5, I, device="cuda") * 1.5
    lo, hi = f32(-2.0), f32(1.7)
    layer = int8.AffineInt8Linear.from_linear(lin, lo, hi, act_bits, w_bits)
    y = layer(x)
    _, y_ref = A.conv(x.cpu().numpy().reshape(15, I, 1, 1), lo, hi, act_bits, lin.weight.detach().cpu().numpy().reshape(O, I, 1, 1),
                      layer.w_min, layer.w_scale, w_bits, lin.bias.detach().cpu().numpy())
    assert y.shape == (3, 5, O) and _same_bits(y.cpu().numpy(), y_ref.reshape(3, 5, O))


# ---- B. output pixels without an in-image tap -----------------------------------------------------------------------------
# (N, Cin, H, W, Cout, k, s, p, d): 1x1 padded by 2; 3x3 padded by 4 on 2x2; dilated 3x3 padded past its reach on each axis
# (reach 4 and 6, padding 5 and 7); SSD-Lite's tail maps: 3x3 padded by 1 on 1x1 and 2x2 (only the centre taps are in the
# image; stride 2 as in its extras)
EMPTY = [
    (2, 19, 3, 3, 70, 1, 1, 2, 1),
    (1, 24, 2, 2, 33, 3, 1, 4, 1),
    (1, 17, 4, 5, 20, 3, 1, (5, 7), (2, 3)),
    (2, 32, 1, 1, 40, 3, 1, 1, 1),
    (2, 32, 2, 2, 40, 3, 1, 1, 1),
    (1, 16, 2, 2, 24, 3, 2, 1, 1),
]


def _empty_windows(terms):
    """[N, OH, OW] mask of the output pixels with no in-image tap (Nv = 0 for every channel)."""
    Nv = terms[3]
    empty = Nv == 0
    assert (empty == empty[:, :1]).all()
    return empty[:, 0]


@pytest.mark.parametrize("depthwise", [False, True], ids=["dense", "depthwise"])
@pytest.mark.parametrize("case", EMPTY, ids=_low_id)
def test_empty_tap_windows_give_the_bias(case, depthwise):
    """Where no tap is in the image the prefix-table rectangle is empty, A = Wv = Nv = P = 0, and y = fp32(0) + bias[o] bit for
    bit (inf, -inf, -0.0 -> +0.0, subnormals); the fused epilogue writes the consumer's codes of that value and their sum."""
    N, Cin, H, W, O, k, s, p, d = case
    O, g = (Cin, Cin) if depthwise else (O, 1)
    conv = _low_bit_conv(Cin, O, k, s, p, d, g, 8, "div", seed=N + Cin + H + W + O, special_bias=True)
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    layer = _layer(conv, x, 8, 8)
    terms, y, P = _per_layer(layer, conv, x)
    empty = _empty_windows(terms)
    bias = layer.bias.cpu().numpy()
    want = (f32(0) + bias).astype(f32)
    if case[5] == 3 and case[7] == 1:
        assert not empty.any()                                 # the tail maps keep their centre taps
    else:
        assert empty.any() and not empty.all()
    for n, oh, ow in zip(*np.nonzero(empty)):
        assert not P[n, :, oh, ow].any()
        assert _same_bits(y[n, :, oh, ow], want)
    out = (f32(-0.9), f32(1.3), 8)
    _, codes, S = _epilogue(layer, conv, x, out)
    q_b, _ = A.act_codes(want.reshape(1, -1, 1, 1), *out)
    for n, oh, ow in zip(*np.nonzero(empty)):
        assert np.array_equal(codes[n, oh, ow, :O], q_b.reshape(-1)) and not codes[n, oh, ow, O:].any()
        assert S[n, oh, ow] == int(q_b.astype(np.int64).sum())


# ---- C. the int32 limit ---------------------------------------------------------------------------------------------------
def _limit_conv(Cn):
    """1x1, Cn inputs, 3 outputs, weights +-0.5 on the 8-bit grid [-0.5, 0.5]: channel 0 all at the minimum (code -128),
    channel 1 at the minimum but its last weight at the maximum (127), channel 2 at the maximum but its first weight at the
    minimum."""
    conv = nn.Conv2d(Cn, 3, 1).cuda()
    with torch.no_grad():
        w = torch.full((3, Cn, 1, 1), -0.5)
        w[1, -1] = 0.5
        w[2] = 0.5
        w[2, 0] = -0.5
        conv.weight.copy_(w)
    return _fake_quantized_conv(conv)


@pytest.mark.parametrize("Cn", [131071, 131056], ids=["K131071-Cpad131072", "K131056-aligned"])
def test_largest_accepted_k_sums_exactly(Cn):
    """Every input at the range's minimum (code -128), K = Cn: P = 16384 K on channel 0 (at K = 131071, 2^31 - 1 - 16383),
    16384 (K - 1) - 128 * 127 on channel 1, and -128 * 127 (K - 1) + 16384 (the most negative products) on channel 2 - against
    the closed form, the oracle, and through the fused epilogue."""
    from dfq_b200 import int8
    x = torch.full((1, Cn, 2, 2), -1.0, device="cuda")
    conv = _limit_conv(Cn)
    layer = int8.AffineInt8Conv2d.from_conv(conv, f32(-1), f32(1))
    _, _, P = _per_layer(layer, conv, x)
    K = Cn
    closed = [16384 * K, 16384 * (K - 1) - 128 * 127, -128 * 127 * (K - 1) + 16384]
    assert [int(v) for v in P[0, :, 0, 0]] == closed and (P == P[:, :, :1, :1]).all()
    if K == 131071:
        assert closed[0] == 2 ** 31 - 1 - 16383
    assert closed[2] > -2 ** 31
    _epilogue(layer, conv, x, (f32(-3e9), f32(3e9), 8), residual=True, seed=K)


def test_k_of_2_pow_17_is_refused():
    """K = 131072 = 2^17: convert_affine names the layer and replaces nothing (a Conv2d of 131072 inputs, a 2x4 kernel on
    16384, a Linear), and the four C entries return -2 with "131072" in dfq_last_error - their buffers hold the full K, so a
    launch could not reach past them, and stay untouched."""
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    for i, m in enumerate([Q.QuantNConv2d(131072, 2, 1), Q.QuantNConv2d(16384, 2, (2, 4)), Q.QuantNLinear(131072, 3)]):
        model = nn.Sequential(Q.QuantNConv2d(3, 4, 1), m).cuda().eval()
        before = [type(c) for c in model]
        with pytest.raises(_lib.DfqError, match=r"layer 1: K = kh \* kw \* C / groups = 131072 reaches 131072"):
            int8.convert_affine(model, OrderedDict((id(c), c) for c in model), targ)
        assert [type(c) for c in model] == before, i

    lib, st = _lib.load(), _lib.stream_ptr()
    small = int8.AffineInt8Conv2d.from_conv(_fake_quantized_conv(nn.Conv2d(16, 1, 1).cuda()), -1.0, 1.0)
    g = small._geometry(1, 1, 1)
    g[0]["C"] = g[0]["Cpad"] = 131072
    K = 131072
    w = torch.zeros(K, device="cuda")
    xq = torch.full((K,), Q_SENTINEL, dtype=torch.int8, device="cuda")
    wq = torch.full((K,), Q_SENTINEL, dtype=torch.int8, device="cuda")
    table = torch.full((4,), S_SENTINEL, dtype=torch.int32, device="cuda")
    S = torch.zeros(1, dtype=torch.int32, device="cuda")
    n_bad = torch.full((1,), S_SENTINEL, dtype=torch.int32, device="cuda")
    y = torch.full((16,), Y_SENTINEL, device="cuda")
    P = torch.full((16,), P_SENTINEL, dtype=torch.int32, device="cuda")
    yq = torch.full((16 + TAIL,), Q_SENTINEL, dtype=torch.int8, device="cuda")
    S_out = torch.full((16,), S_SENTINEL, dtype=torch.int32, device="cuda")
    small.weight_codes, small.tap_table = wq, table
    out, obs = (-1.0, 1.0, 8), (-1.0, 1.0, 8)
    calls = {
        "dfq_i8_affine_pack": lambda: lib.dfq_i8_affine_pack(_p(w), C.c_float(-1.0), C.c_float(0.01), 8, _p(wq), _p(table),
                                                             _p(n_bad), _lib.table_ptr(g), st),
        "dfq_i8_affine_conv": lambda: lib.dfq_i8_affine_conv(_p(xq), _p(S), _p(wq), _p(table), _lib.table_ptr(small.constants),
                                                             _p(small.bias), _p(y), _p(P), _lib.table_ptr(g), st),
        "dfq_i8_affine_conv_fused": lambda: _launch_fused(small, xq, S, g, None, y, yq[:16], S_out, out),
        "dfq_i8_affine_conv_observed": lambda: _launch_observed(small, xq, S, g, None, y, yq[:16], S_out, out, obs=obs),
    }
    for name, call in calls.items():
        assert call() == -2, name
        assert "131072" in lib.dfq_last_error().decode(), name
        torch.cuda.synchronize()
        assert (wq == Q_SENTINEL).all() and (table == S_SENTINEL).all() and (n_bad == S_SENTINEL).all(), name
        assert (y == Y_SENTINEL).all() and (P == P_SENTINEL).all() and (yq == Q_SENTINEL).all() and \
            (S_out == S_SENTINEL).all(), name


# ---- D. the reference's recipe end to end ---------------------------------------------------------------------------------
def _layer_ulps(names, twins, converted, seen):
    """Over the layers, each on the input its fake-quantized twin saw: (worst |int - fake quant| in ulp of the bound
    sum |x^| |w^| + |b|, worst |int - double| in ulp of the offset bound sum (|x^| + |ma|)(|w^| + |mw|) + |b|, worst
    |int - fake quant| / (16 ulp of the bound + 4 ulp of the offset bound)).  The integer sums are exact on the codes; x^ =
    fp32(fp32(q fa) + ma) and w^ are rounded at the magnitude of their offsets, so where the offsets dwarf the values the
    twin's fp32 sum of x^ w^ moves from the integer result by ulps of the offset bound, not of its own."""
    worst, worst64, within, worst_layer = 0.0, 0.0, 0.0, None
    for n in names:
        xin, yfq = seen[n]
        lay, twin = converted[n], twins[n]
        xh = twin.quant(xin)
        w = twin.weight
        y = lay(xin)
        if isinstance(twin, nn.Conv2d):
            conv = lambda a, b: F.conv2d(a, b, None, twin.stride, twin.padding, twin.dilation, twin.groups)
        else:
            conv = lambda a, b: F.linear(a, b)
        b = twin.bias.double().reshape((-1,) + (1,) * (y.dim() - 2))
        bound = conv(xh.abs().double(), w.abs().double()) + b.abs()
        y64 = conv(xh.double(), w.double()) + b
        ma, mw = abs(float(twin.quant.running_min)), abs(float(w.min()))
        bound64 = conv(xh.abs().double() + ma, w.abs().double() + mw) + b.abs()
        ulp = torch.from_numpy(np.spacing(bound.float().cpu().numpy())).cuda().double()
        ulp64 = torch.from_numpy(np.spacing(bound64.float().cpu().numpy())).cuda().double()
        diff = (y.double() - yfq.double()).abs()
        if float((diff / ulp).max()) > worst:
            worst, worst_layer = float((diff / ulp).max()), n
        worst64 = max(worst64, float(((y.double() - y64).abs() / ulp64).max()))
        within = max(within, float((diff / (16 * ulp + 4 * ulp64)).max()))
    print("  worst |int - fake quant| on %s" % worst_layer)
    return worst, worst64, within


def _record(model, names):
    """Forward hooks keeping (input, output) of the named layers; returns (dict, hooks)."""
    seen, mods = {}, dict(model.named_modules())
    hooks = [mods[n].register_forward_hook(lambda m, i, o, n=n: seen.__setitem__(n, (i[0].detach(), o.detach())))
             for n in names]
    return seen, hooks


@pytest.fixture
def no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("bits_weight", [8, 6, 4])
@pytest.mark.parametrize("net", ["resnet18", "mobilenet_v2"])
def test_reference_recipe_cpu_quantized_weights(net, bits_weight, no_tf32):
    """quantize_targ_layer before .cuda() as the reference's mains call it (weights fake-quantized with true division),
    bits_weight-bit weights and 8-bit biases: convert_affine(bits_weight=b) converts every layer, each within 16 ulp of the
    fake-quantized twin's output and 4 ulp of the double sum (the bounds of test_gpu_int8_affine.py), and chain_affine's
    logits equal the per-layer model's bit for bit with and without residual fusion.  Converting with a narrower grid than
    the weights' is refused.

    Measured on an H100 (8 / 6 / 4-bit weights): worst |int - fake quant| 6.0 / 9.25 / 10.0 ulp on ResNet-18 and 7.0 / 6.0 /
    5.5 on MobileNetV2, |int - double| at most 1.11 ulp; relative logit error against the fake-quantized model 5.7e-3 /
    5.7e-3 / 5.2e-3 (ResNet-18) and 3.0e-3 / 2.6e-3 / 2.7e-3 (MobileNetV2), asserted below 1e-2.  The error does not grow
    as the weight grid coarsens: both models run on the same weights, and what differs - fp32 rounding of the sums moving
    activations across the next quantizer's rounding boundaries - does not depend on the weights' bits."""
    from dfq_b200 import _lib, int8
    fq, qgraph, qtarg = affine_calibrated.calibrated(net, bits_weight=bits_weight, bits_bias=8, quantize_on_cpu=True)
    twins = {n: m for n, m in fq.named_modules() if type(m) in qtarg}
    aff = copy.deepcopy(fq)
    agraph = OrderedDict((id(m), m) for m in aff.modules() if type(m) in qtarg)
    if bits_weight == 8:
        with pytest.raises(_lib.DfqError, match="not on a 4-bit min / max grid"):
            int8.convert_affine(aff, agraph, qtarg, bits_weight=4)
        present = {id(m) for m in aff.modules()}
        assert all(type(m) in qtarg and id(m) in present for m in agraph.values())
    names = int8.convert_affine(aff, agraph, qtarg, bits_weight=bits_weight)
    amods = dict(aff.named_modules())
    assert sorted(names) == sorted(twins) and all(amods[n].w_bits == bits_weight for n in names)
    x = torch.randn(8, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
    seen, hooks = _record(fq, names)
    with torch.no_grad():
        ref = fq(x)
        for h in hooks:
            h.remove()
        worst, worst64, _ = _layer_ulps(names, twins, amods, seen)
        got = aff(x)
        chained = {"chained": int8.chain_affine(aff)(x), "residual": int8.chain_affine(aff, residual=True)(x)}
    err = float((got - ref).norm() / ref.norm())
    print("%s, %d-bit weights (CPU-quantized, 8-bit biases): %d layers, worst |int - fake quant| %.2f ulp, |int - double| "
          "%.2f ulp, relative logit error %.3g" % (net, bits_weight, len(names), worst, worst64, err))
    assert worst <= 16 and worst64 <= 4, (worst, worst64)
    assert err < 1e-2, err
    for k, v in chained.items():
        assert torch.equal(v.view(torch.int32), got.view(torch.int32)), k


# ---- E. SSD-Lite and the layer-by-layer bound in the evaluation state -----------------------------------------------------
SSD_COUNTS = (53, 85, 10, 20)   # (chain_affine edges, chain_affine(residual=True) edges, fused adds, fused observers)


def test_ssd_lite_evaluation_state_chained_equals_per_layer(no_tf32):
    """main_ssd.py --quantize's model at 300x300: records of 10 adds, two 6-way cats and a softmax; both outputs of
    chain_affine, with and without residual fusion, equal the per-layer affine model's bit for bit.  The cat operands'
    observers stay in torch: every head permutes before the cat."""
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
        ct = LT.module_tensor_op
        ops = Counter((name.rsplit("_", 2)[0], int(name.rsplit("_", 1)[1])) for _, name in ct.name_tensor_op)
        assert ops == {("add", 2): 10, ("torch_cat", 6): 2, ("F_softmax", 1): 1}, ops
        int8.convert_affine(model, qgraph, qtarg)
        chained, gm = int8.chain_affine(model), int8.chain_affine(model, residual=True)
        x = torch.randn(4, 3, 300, 300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
        with torch.no_grad():
            ref = model(x)
            got = {"chained": chained(x), "residual": gm(x)}
        counts = (len(chained.requantized_edges), len(gm.requantized_edges), len(gm.fused_adds), len(gm.fused_observers))
        print("ssd: edges %d / %d, adds %d, fused observers %d %s" % (counts + (sorted({w for _, w, _ in gm.fused_observers}),)))
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
        for k, v in got.items():
            assert len(v) == 2 and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(ref, v)), k
        assert counts == SSD_COUNTS


@pytest.mark.parametrize("net,size", [("ssd", 300), ("deeplab", 129)])
def test_evaluation_state_layer_by_layer_bounds(net, size, no_tf32):
    """Every converted layer of SSD-Lite (1x1 and 2x2 tail maps) and the padded DeepLab (dilated and fixed-padded layers),
    on the inputs the twins saw in the evaluation state: within 4 ulp of the offset bound of the double sum, and within 16
    ulp of the bound plus 4 ulp of the offset bound of its fake-quantized twin.

    Measured on an H100: |int - double| 1.24 ulp (SSD-Lite) and 1.03 ulp (DeepLab); |int - fake quant| 15.0 ulp of the
    bound on SSD-Lite, 131.25 on DeepLab.  There the twin's fp32 output agrees with the double sum of its x^ w^ to 1e-11
    and the integer result differs from both by 1.6e-8, 0.02 ulp of the offset bound: the inputs of the backbone's 1x1
    expansions span zero with offsets of -0.5 to -1.2, and their outputs (1.6e-4 against a bound of 1.7e-3 on
    backbone.features.12.conv.0) cancel far below the offsets' rounding - the 16-ulp bound of the classifiers does not
    apply to such layers.  The combined twin bound was met at 0.2 (SSD-Lite) and 0.17 (DeepLab) of its width."""
    from dfq_b200 import int8
    with affine_observed_state.evaluation_state(net, size=size, batch=4) as (model, qgraph, qtarg):
        twins = {n: m for n, m in model.named_modules() if type(m) in qtarg}
        x = torch.randn(4, 3, size, size, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
        seen, hooks = _record(model, list(twins))
        with torch.no_grad():
            model(x)
        for h in hooks:
            h.remove()
        names = int8.convert_affine(model, qgraph, qtarg)
        assert sorted(names) == sorted(twins)
        with torch.no_grad():
            worst, worst64, within = _layer_ulps(names, twins, dict(model.named_modules()), seen)
    print("%s: %d layers, worst |int - fake quant| %.2f ulp (%.3g of 16 ulp + 4 offset ulp), |int - double| %.2f ulp"
          % (net, len(names), worst, within, worst64))
    assert worst64 <= 4 and within <= 1, (worst64, within)
