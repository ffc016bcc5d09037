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


def _channel_scales(w, seed):
    """One weight scale per output channel, all different: 128 / max|W[o]| times a factor in [0.5, 1.5].  Channel 0 gets
    scale 0 (codes 0, dq 0: its output is the bias) and channel 1 four times its range scale (codes saturate at +-127)."""
    m = w.detach().abs().flatten(1).amax(1).double().cpu().numpy()
    ws = 128. / m * np.random.default_rng(seed).uniform(0.5, 1.5, m.size)
    ws[0] = 0
    if ws.size > 1:
        ws[1] *= 4
    return ws.astype(f32)


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _seed(c):
    return sum(v if isinstance(v, int) else sum(v) for v in c)


def _case_id(c):
    return "x".join("-".join(map(str, v)) if isinstance(v, tuple) else str(v) for v in c)


def _oracle(x, conv, a, ws):
    """(acc, y) of the int8 layer by the oracle, from the fp32 input and the module's fp32 weights; ws: one scale, or one per
    output channel."""
    w = conv.weight.detach().cpu().numpy()
    ws = np.broadcast_to(np.asarray(ws, f32), (w.shape[0],))
    xq = O.i8_quantize(x.detach().cpu().numpy(), a)
    acc = O.i8_conv(xq, O.i8_quantize(w, ws.reshape(-1, 1, 1, 1)), conv.stride, conv.padding, conv.dilation, conv.groups)
    b = None if conv.bias is None else conv.bias.detach().cpu().numpy()
    return acc, O.i8_dequant(acc, a, ws, b)


def _packed_codes(layer):
    """The packed weight codes as [O, C/groups, kh, kw]; asserts the channel padding is zero."""
    kh, kw = layer.kernel_size
    codes = layer.weight_codes.cpu().numpy()
    if layer.groups == 1:
        codes = codes.reshape(layer.out_channels, kh, kw, layer.cpad)
        assert not codes[..., layer.in_channels:].any()
        return codes[..., :layer.in_channels].transpose(0, 3, 1, 2)
    codes = codes.reshape(kh * kw, layer.cpad)
    assert not codes[:, layer.in_channels:].any()
    return codes[:, :layer.in_channels].T.reshape(layer.out_channels, 1, kh, kw)


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32))


def _run_conv(N, Cin, H, W, Cout, k, s, p, d, g=1, seed=0, x=None, conv=None, a=None, ws=None):
    """Convert, run with the int32 sums, and check codes, sums and outputs against the oracle.  a / ws default to
    128 / max|x| and one 128 / max|W| for the layer."""
    from dfq_b200 import int8
    torch.manual_seed(seed)
    conv = conv or nn.Conv2d(Cin, Cout, k, s, p, d, g).cuda()
    x = torch.randn(N, Cin, H, W, device="cuda") * 2 if x is None else x
    a = _ascale(x) if a is None else a
    ws = _wscale(conv.weight) if ws is None else ws
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    y, acc = layer.run(x, with_acc=True)
    acc_ref, y_ref = _oracle(x, conv, a, ws)
    w = conv.weight.detach().cpu().numpy()
    assert np.array_equal(_packed_codes(layer), O.i8_quantize(w, np.broadcast_to(np.asarray(ws, f32), (Cout,)).reshape(-1, 1, 1, 1))), "codes"
    assert np.array_equal(acc.cpu().numpy(), acc_ref), "acc"
    assert _same_bits(y.cpu().numpy(), y_ref), "y"
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


DENSE = [  # (N, Cin, H, W, Cout, k, stride, pad, dil); k / stride / pad / dil: an int, or (h, w)
    (1, 3, 15, 15, 8, 3, 1, 1, 1), (3, 16, 8, 9, 24, 1, 2, 0, 1), (1, 24, 17, 16, 100, 7, 2, 3, 1),
    (3, 96, 10, 10, 1000, 1, 1, 0, 1), (1, 160, 9, 7, 24, 3, 1, 3, 2), (1, 512, 7, 7, 100, 3, 2, 1, 1),
    (3, 3, 30, 31, 24, 7, 2, 3, 1), (1, 16, 20, 20, 8, 3, 1, 3, 6), (1, 24, 5, 5, 8, 3, 1, 0, 1),
    (3, 512, 1, 1, 1000, 1, 1, 0, 1), (1, 96, 7, 7, 24, 7, 1, 0, 1), (1, 160, 11, 12, 8, 3, 2, 1, 2),
    (3, 24, 14, 13, 1000, 3, 1, 1, 1), (1, 3, 224, 224, 24, 3, 2, 1, 1), (3, 512, 6, 5, 8, 1, 2, 0, 1),
    (1, 16, 13, 13, 100, 3, 2, 0, 6), (3, 160, 4, 4, 100, 7, 1, 3, 1),
    # off the square: load_tile splits a tap as (tap / kw, tap % kw); the pairs below differ per axis
    (2, 16, 9, 12, 24, (1, 7), 1, (0, 3), 1),                        # 1x7
    (1, 24, 12, 9, 40, (7, 1), 1, (3, 0), 1),                        # 7x1
    (2, 17, 11, 13, 33, (3, 5), (2, 1), (1, 2), (1, 2)),             # 3x5, stride / pad / dilation per axis
    (1, 32, 13, 14, 16, (5, 3), (1, 3), 0, (2, 1)),                  # 5x3
]


@pytest.mark.parametrize("case", DENSE, ids=_case_id)
def test_dense_conv_acc_and_output_bit_exact(case):
    _run_conv(*case, seed=_seed(case))


# Tiles of k_i8_conv_mma (BM x BN x BK = 128 x 64 x 64, STAGES = 3; pinned in tests/test_boundary_guards.py): cases on both
# sides of each size.  M = N*OH*OW output pixels, KT = ceil(kh*kw*Cpad / BK) K tiles (KT = 2 = STAGES - 1 fills the ring
# exactly).  test_boundary_guards.py checks that the list covers every edge below.
TILE_EDGES = dict(M={1, 31, 127, 128, 129}, O={1, 7, 9, 63, 64, 65, 129}, C={1, 15, 16, 17, 64, 65}, KT={1, 2, 3, 4})
TILES = [  # (N, Cin, H, W, Cout, k, stride, pad, dil)
    (1, 65, 1, 1, 64, 1, 1, 0, 1),                 # M 1, O 64 = BN, C 65 (Cpad 80), KT 2
    (1, 1, 1, 31, 129, (1, 3), 1, (0, 1), 1),      # M 31, O 129 = 2 BN + 1, C 1, KT 1
    (1, 15, 127, 1, 7, (5, 1), 1, (2, 0), 1),      # M 127 = BM - 1, O 7, C 15, KT 2
    (2, 16, 8, 8, 63, 3, 1, 1, 1),                 # M 128 = BM with an image boundary at m = 64, O 63, C 16, KT 3
    (1, 64, 4, 44, 1, 2, 1, 0, 1),                 # M 129 = BM + 1, O 1, C 64, KT 4
    (3, 17, 1, 43, 9, 1, 1, 0, 1),                 # M 129 over three images (boundaries at 43 and 86), O 9, C 17, KT 1
    (5, 15, 7, 9, 65, 3, 1, 1, 1),                 # M 315: three M tiles, images straddling them, O 65 = BN + 1, KT 3
    (2, 64, 6, 11, 129, 1, 1, 0, 1),               # M 132, O 129, C 64 = BK, KT 1
    (1, 16, 9, 15, 65, 4, 1, 0, 1),                # KT 4 from 16 taps of 16 channels, M 72, O 65
    (1, 64, 8, 16, 64, (1, 2), 1, 0, 1),           # K 128: KT 2 exactly, M 120
]


def tile_geometry(case):
    """(M, O, C, KT) of a TILES case."""
    N, Cn, H, W, Oc, k, s, p, d = case
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    OH, OW = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    return N * OH * OW, Oc, Cn, -(-kh * kw * ((Cn + 15) // 16 * 16) // 64)


@pytest.mark.parametrize("case", TILES, ids=_case_id)
def test_dense_conv_tile_edges_bit_exact(case):
    _run_conv(*case, seed=sum(tile_geometry(case)))


DW = [  # (N, C, H, W, k, stride, pad, dil); k / stride / pad / dil: an int, or (h, w)
    (1, 32, 15, 15, 3, 1, 1, 1), (3, 96, 14, 13, 3, 2, 1, 1), (1, 144, 9, 9, 3, 1, 2, 2), (1, 24, 17, 16, 3, 2, 4, 4),
    (3, 19, 8, 8, 5, 1, 2, 1), (1, 960, 7, 7, 3, 1, 1, 1), (1, 40, 3, 3, 3, 1, 0, 1), (1, 16, 11, 10, 7, 2, 3, 2),
    # off the square: k_i8_conv_dw walks rows with stride_h / dil_h and columns with stride_w / dil_w
    (2, 32, 9, 12, (1, 7), 1, (0, 3), 1),                            # 1x7
    (1, 40, 12, 9, (7, 1), 1, (3, 0), 1),                            # 7x1
    (2, 48, 11, 13, (3, 5), (2, 1), (1, 2), (1, 2)),                 # 3x5, stride / pad / dilation per axis
    (1, 24, 13, 14, (5, 3), (1, 3), 0, (2, 1)),                      # 5x3
    (2, 33, 6, 7, 1, (1, 2), 0, 1),                                  # 1x1 depthwise, stride per axis
]


@pytest.mark.parametrize("case", DW, ids=_case_id)
def test_depthwise_conv_acc_and_output_bit_exact(case):
    N, Cn, H, W, k, s, p, d = case
    _run_conv(N, Cn, H, W, Cn, k, s, p, d, g=Cn, seed=_seed(case))


PER_CHANNEL = [  # (N, Cin, H, W, Cout, k, stride, pad, dil, groups) with _channel_scales: one weight scale per channel
    (2, 24, 9, 9, 72, 3, 1, 1, 1, 1),             # dense: O 72 spans an N tile of 64 and the next
    (1, 40, 7, 6, 9, (1, 3), 1, (0, 1), 1, 1),    # dense, a single N tile
    (2, 40, 9, 9, 40, 3, 1, 1, 1, 40),            # depthwise: three 16-channel chunks, the last one partial
    (1, 144, 8, 8, 144, 3, 2, 1, 1, 144),         # depthwise, nine full chunks
]


@pytest.mark.parametrize("case", PER_CHANNEL, ids=_case_id)
def test_per_channel_weight_scales_bit_exact(case):
    """Packed codes, sums and outputs with a different scale in every channel, a zero one and a saturating one."""
    N, Cn, H, W, Oc, k, s, p, d, g = case
    torch.manual_seed(Oc)
    conv = nn.Conv2d(Cn, Oc, k, s, p, d, g).cuda()
    ws = _channel_scales(conv.weight, Oc)
    layer, x, y = _run_conv(N, Cn, H, W, Oc, k, s, p, d, g=g, conv=conv, ws=ws)
    codes = _packed_codes(layer)
    assert not codes[0].any() and np.abs(codes[1]).max() == 127
    assert np.array_equal(y[:, 0].cpu().numpy(), np.broadcast_to(conv.bias[0].item(), y[:, 0].shape).astype(f32))
    assert np.array_equal(layer.dq.cpu().numpy()[0], f32(0))


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


def _as_conv(lin):
    conv = nn.Conv2d(lin.in_features, lin.out_features, 1).cuda()
    with torch.no_grad():
        conv.weight.copy_(lin.weight.reshape(conv.weight.shape)); conv.bias.copy_(lin.bias)
    return conv


def test_linear_on_a_3d_input_with_per_channel_scales():
    """Int8Linear on [B, T, I] with I = 100 (Cpad 112, not a multiple of 16) and one weight scale per output feature."""
    from dfq_b200 import int8
    torch.manual_seed(11)
    lin = nn.Linear(100, 37).cuda()
    x = torch.randn(3, 5, 100, device="cuda")
    a, ws = _ascale(x), _channel_scales(lin.weight, 11)
    layer = int8.Int8Linear.from_linear(lin, a, ws)
    y = layer(x)
    _, y_ref = _oracle(x.reshape(15, 100, 1, 1), _as_conv(lin), a, ws)
    assert y.shape == (3, 5, 37) and _same_bits(y.cpu().numpy(), y_ref.reshape(3, 5, 37))
    assert np.array_equal(_packed_codes(layer).reshape(37, 100), O.i8_quantize(lin.weight.detach().cpu().numpy(), ws[:, None]))


# ---- grid-stride loops: more work items than one launch has threads ---------------------------------------------------
Q_SENTINEL, ACC_SENTINEL = -128, -2 ** 31          # never a code (the clamp is +-127), never a sum of these layers


def _launch_cap():
    """grid_for() in int8_conv.cu: at most sm_count * 32 blocks of 256 threads per launch."""
    from dfq_b200 import _lib
    sm = C.c_int()
    _lib.check(_lib.load().dfq_device_info(C.byref(sm), None), "dfq_device_info")
    return sm.value * 32 * 256


def _quantize_abi(x, a, cpad):
    """dfq_i8_quantize_nhwc into a buffer prefilled with Q_SENTINEL; returns [N, H, W, Cpad]."""
    from dfq_b200 import _lib
    N, Cn, H, W = x.shape
    q = torch.full((N * H * W * cpad,), Q_SENTINEL, dtype=torch.int8, device="cuda")
    _lib.check(_lib.load().dfq_i8_quantize_nhwc(C.c_void_p(x.data_ptr()), C.c_void_p(q.data_ptr()), N, Cn, H, W, cpad,
                                                C.c_float(a), _lib.stream_ptr()), "dfq_i8_quantize_nhwc")
    return q.reshape(N, H, W, cpad)


def test_quantizer_grid_stride_loop_covers_every_item():
    N, Cn, H, W = 5, 72, 224, 224                   # 5 * 5 chunks * 224 * 224 = 1,254,400 items
    items = N * ((Cn + 15) // 16) * H * W
    assert items > _launch_cap(), "the case no longer takes a second trip through the loop"
    torch.manual_seed(5)
    x = torch.randn(N, Cn, H, W, device="cuda") * 3
    q = _quantize_abi(x, f32(20.0), 80).cpu().numpy()
    assert np.array_equal(q[..., :Cn], O.i8_quantize(x.cpu().numpy(), f32(20.0)).transpose(0, 2, 3, 1))
    assert not q[..., Cn:].any()


def test_dense_packer_grid_stride_loop_covers_every_item():
    """512 x 256 x 3 x 3 packs 512 * 9 * 256 = 1,179,648 codes; then the layer runs on a small image."""
    from dfq_b200 import _lib, int8
    torch.manual_seed(6)
    conv = nn.Conv2d(256, 512, 3, 1, 1).cuda()
    assert 512 * 9 * 256 > _launch_cap(), "the case no longer takes a second trip through the loop"
    ws = _channel_scales(conv.weight, 6)
    layer = _run_conv(2, 256, 3, 4, 512, 3, 1, 1, 1, conv=conv, ws=ws)[0]
    out = torch.full_like(layer.weight_codes, Q_SENTINEL)
    g = layer._geometry(1, 3, 3, stride=(1, 1), padding=(0, 0))
    w = conv.weight.detach().contiguous()
    _lib.check(_lib.load().dfq_i8_pack_weights(C.c_void_p(w.data_ptr()), C.c_void_p(layer.w_scale.data_ptr()),
                                               C.c_void_p(out.data_ptr()), _lib.table_ptr(g), _lib.stream_ptr()), "pack")
    assert torch.equal(out, layer.weight_codes)


def test_depthwise_grid_stride_loop_covers_every_item():
    """N 48, C 144, 56 x 56: 48 * 9 chunks * 3136 pixels = 1,354,752 items for the quantizer and for k_i8_conv_dw; every
    output, sum and code buffer is prefilled with a sentinel."""
    from dfq_b200 import _lib, int8
    N, Cn, H, W = 48, 144, 56, 56
    assert N * (Cn // 16) * H * W > _launch_cap(), "the case no longer takes a second trip through the loop"
    torch.manual_seed(7)
    conv = nn.Conv2d(Cn, Cn, 3, 1, 1, groups=Cn).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda")
    a, ws = _ascale(x), _channel_scales(conv.weight, 7)
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    xq = _quantize_abi(x, a, layer.cpad)
    y = torch.full((N, Cn, H, W), float("nan"), device="cuda")
    acc = torch.full((N, Cn, H, W), ACC_SENTINEL, dtype=torch.int32, device="cuda")
    _lib.check(_lib.load().dfq_i8_conv(C.c_void_p(xq.data_ptr()), C.c_void_p(layer.weight_codes.data_ptr()),
                                       C.c_void_p(layer.dq.data_ptr()), C.c_void_p(layer.bias.data_ptr()),
                                       C.c_void_p(y.data_ptr()), C.c_void_p(acc.data_ptr()),
                                       _lib.table_ptr(layer._geometry(N, H, W)), _lib.stream_ptr()), "dfq_i8_conv")
    acc_ref, y_ref = _oracle(x, conv, a, ws)
    assert np.array_equal(xq.cpu().numpy(), O.i8_quantize(x.cpu().numpy(), a).transpose(0, 2, 3, 1))
    assert np.array_equal(acc.cpu().numpy(), acc_ref)
    assert _same_bits(y.cpu().numpy(), y_ref)


# ---- special values ------------------------------------------------------------------------------------------------
def _inject(x, values, seed):
    flat = x.reshape(-1)
    idx = torch.from_numpy(np.random.default_rng(seed).choice(flat.numel(), len(values), replace=False)).cuda()
    flat[idx] = torch.tensor(values, device="cuda")
    return x


@pytest.mark.parametrize("groups", [1, 24])
def test_non_finite_and_overflowing_activations(groups):
    """NaN -> -127 (DESIGN.md section 3.8), +-inf and products past fp32's range -> +-127, next to ordinary values."""
    torch.manual_seed(8)
    x = _inject(torch.randn(2, 24, 9, 10, device="cuda") * 2, [float("nan")] * 6 + [float("inf")] * 5 +
                [float("-inf")] * 5 + [3e38, -3e38, 1e37, -1e37], 8)
    layer, _, y = _run_conv(2, 24, 9, 10, 24, 3, 1, 1, 1, g=groups, x=x, a=f32(40.0))
    q = _quantize_abi(x, f32(40.0), layer.cpad).cpu().numpy()[..., :24].transpose(0, 3, 1, 2)
    assert np.all(q[np.isnan(x.cpu().numpy())] == -127) and np.all(q[x.cpu().numpy() >= 1e37] == 127)
    assert np.all(q[x.cpu().numpy() <= -1e37] == -127)


def test_subnormal_activations_are_not_flushed():
    """x ~ 3e-38 (a third of it subnormal) at a = 2e38: the codes come from the subnormal products, and dq = 1 / (a * 1)
    is itself subnormal."""
    torch.manual_seed(9)
    conv = nn.Conv2d(16, 8, 3, 1, 1).cuda()
    with torch.no_grad():
        conv.weight.mul_(200.0)
    x = torch.randn(1, 16, 7, 7, device="cuda") * 3e-38
    assert int((x.abs() < 1.1754944e-38).sum()) > 100 and float(x.abs().max()) < 1e-36
    _, _, y = _run_conv(1, 16, 7, 7, 8, 3, 1, 1, 1, x=x, conv=conv, a=f32(2e38), ws=f32(1.0))
    q = O.i8_quantize(x.cpu().numpy(), f32(2e38))
    assert np.abs(q[np.abs(x.cpu().numpy()) < 1.1754944e-38]).max() >= 2


@pytest.mark.parametrize("groups", [1, 16])
def test_zero_activation_scale_with_finite_and_infinite_input(groups):
    """a = 0 (a zero range): finite inputs quantize to 0; an infinite one gives inf * 0 = NaN -> -127, which the sums carry,
    while dq = 0 leaves the bias as the output."""
    torch.manual_seed(10)
    x = torch.randn(2, 16, 6, 6, device="cuda")
    layer, _, y = _run_conv(2, 16, 6, 6, 16, 3, 1, 1, 1, g=groups, x=x, a=f32(0.0))
    assert not layer.run(x, with_acc=True)[1].any()
    x = _inject(x.clone(), [float("inf")] * 3 + [float("-inf")] * 3, 10)
    layer, _, y = _run_conv(2, 16, 6, 6, 16, 3, 1, 1, 1, g=groups, x=x, a=f32(0.0), conv=None)
    acc = layer.run(x, with_acc=True)[1]
    assert acc.any()
    b = layer.bias.cpu().numpy().reshape(1, -1, 1, 1)
    assert np.array_equal(y.cpu().numpy(), np.broadcast_to(b, y.shape))


@pytest.mark.parametrize("ws", [0.0, 1.0])
@pytest.mark.parametrize("groups", [1, 24])
def test_all_zero_weights(groups, ws):
    """A layer of zero weights: codes 0, sums 0, output = bias (ws 0 is what convert_to_int8 gives a zero range)."""
    conv = nn.Conv2d(24, 24, 3, 1, 1, groups=groups).cuda()
    with torch.no_grad():
        conv.weight.zero_()
    layer, x, y = _run_conv(1, 24, 8, 8, 24, 3, 1, 1, 1, g=groups, conv=conv, ws=f32(ws))
    assert not layer.weight_codes.any() and not layer.run(x, with_acc=True)[1].any()
    b = conv.bias.detach().cpu().numpy().reshape(1, -1, 1, 1)
    assert np.array_equal(y.cpu().numpy(), np.broadcast_to(b, y.shape))


# ---- Python entry edges --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [1, 24])
def test_channels_last_sliced_side_stream_and_with_acc_give_the_same_output(groups):
    from dfq_b200 import int8
    torch.manual_seed(12)
    conv = nn.Conv2d(24, 24, 3, 1, 1, groups=groups).cuda()
    big = torch.randn(2, 30, 20, 36, device="cuda") * 2
    x = big[:, 3:27, :, ::2]                                            # sliced: not contiguous
    assert not x.is_contiguous()
    a, ws = _ascale(x), _channel_scales(conv.weight, 12)
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    y, acc = layer.run(x, with_acc=True)
    acc_ref, y_ref = _oracle(x.contiguous(), conv, a, ws)
    assert np.array_equal(acc.cpu().numpy(), acc_ref) and _same_bits(y.cpu().numpy(), y_ref)
    cl = x.contiguous().to(memory_format=torch.channels_last)
    assert not cl.is_contiguous()
    assert torch.equal(layer(cl), y)
    y2, none = layer.run(x, with_acc=False)
    assert none is None and torch.equal(y2, y)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        y3, acc3 = layer.run(x, with_acc=True)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(y3, y) and torch.equal(acc3, acc)


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


# ---- the reference's int8 MobileNetV2 end to end ----------------------------------------------------------------------
REF_IMAGES = 3
# Thresholds measured on the CPU (tests/test_int8_host.py runs the same comparison through the oracle-backed library) on
# these 3 seeded N(0, 1) images: the int8 logits are 0.272 (reference codes) and 0.265 (this calibration) from the calibrated
# fp32 model's, relative 2-norm, and this calibration is 0.100 from the reference codes.  That divergence is rounding flips in
# the activation codes that grow layer by layer (6e-7 after the first layer, 0.2 before the classifier), not a wrong layer.
# Every image predicted the same class in every arm, with fp32 top-1 margins of 0.78-0.92.  On an H100 the calibration is
# the reference's to the bit, so this calibration's logits equal the reference codes' (0.0) and are 0.272 from fp32.
INT8_VS_FP32_REL, PKG_VS_REF_REL, TOP1_AGREE = 0.4, 0.2, 2 / 3


def _ref_images(n=REF_IMAGES):
    return torch.randn(n, 3, 224, 224, generator=torch.Generator().manual_seed(0))


def _ref_net():
    import ncnn_int8_case as case
    if case.paths() is None:
        pytest.skip("reference int8 model not staged in oracle/_ref")
    return case, case.Int8Net()


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _gpu_executor(case, net):
    """Int8Conv2d / Int8Linear of each layer, built from codes / w_scale in fp32 with the .bin's per-channel weight scales,
    input scale and bias; their packed codes must equal the .bin's."""
    from dfq_b200 import int8
    mods = []
    for s in net.specs:
        w = torch.from_numpy(case.spec_weight(s)).cuda()
        b = None if s["bias"] is None else torch.from_numpy(s["bias"]).cuda()
        if s["type"] == "InnerProduct":
            m = int8.Int8Linear(w, b, s["in_scale"], s["w_scales"])
        else:
            m = int8.Int8Conv2d(w, b, s["in_scale"], s["w_scales"], s["stride"], s["pad"], s["dilation"], s["groups"])
        assert np.array_equal(_packed_codes(m), s["codes"]), s["name"]
        mods.append(m)
    return lambda s, x: mods[s["index"]].run(x)[0]


def test_reference_int8_mobilenetv2_end_to_end_against_the_oracle():
    """The reference's deployed int8 model through the interpreter (tests/ncnn_int8_case.py), executed by the GPU kernels
    and by the oracle: bit for bit up to the last ReLU, a few ulp after torch's global mean, and bit for bit again through
    the classifier fed the GPU's pooled vector."""
    case, net = _ref_net()
    x = _ref_images()
    with torch.no_grad():
        gpu = net.forward(x.cuda(), _gpu_executor(case, net))
        ref = net.forward(x, case.oracle_executor)
    names = list(ref)
    last_relu = [l for l in net.layers if l["type"] == "ReLU"][-1]["tops"][0]
    for n in names[:names.index(last_relu) + 1]:
        assert _same_bits(gpu[n].cpu().numpy(), ref[n].numpy()), n
    pool = [l for l in net.layers if l["type"] == "Reduction"][0]["tops"][0]
    pg, pr = gpu[pool].cpu().numpy(), ref[pool].numpy()
    assert np.all(np.abs(pg - pr) <= 4 * np.spacing(np.abs(pr))), float(np.abs(pg - pr).max())
    fc = net.specs[-1]
    logits = [l for l in net.layers if l["type"] == "InnerProduct"][0]["tops"][0]
    y_ref = case.oracle_executor(fc, torch.from_numpy(pg).reshape(REF_IMAGES, -1, 1, 1)).reshape(REF_IMAGES, -1)
    assert _same_bits(gpu[logits].cpu().numpy(), y_ref.numpy())


def test_cuda_calibration_in_the_reference_int8_mobilenetv2(monkeypatch):
    """This package's calibration of the bundled checkpoint (BN fold and signed equalization on the GPU), converted with the
    table's activation scales, in the same interpreter: close to the reference codes' logits, and to the calibrated fp32
    model's (TF32 off) with the same top-1."""
    import ncnn_table_case
    from dfq_b200 import int8
    case, net = _ref_net()
    if ncnn_table_case.checkpoint_path() is None:
        pytest.skip("checkpoint not staged in oracle/_ref")
    graph, targ = case.calibrated_graph(monkeypatch)
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    holder = nn.ModuleList(layers).cuda()
    rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
    int8.convert_to_int8(holder, graph, targ, act_scales=list(rows["activation_scales"]))
    x = _ref_images().cuda()
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            fp32 = net.forward(x, case.fp32_executor([l.cuda() for l in layers]))["781"]
            ours = net.forward(x, lambda s, v: holder[s["index"]].run(v)[0])["781"]
            theirs = net.forward(x, _gpu_executor(case, net))["781"]
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    e_ref, e_fp = _rel(ours, theirs), _rel(ours, fp32)
    agree = float((ours.argmax(1) == fp32.argmax(1)).float().mean())
    print("int8 (this calibration) vs reference codes %.4g, vs fp32 %.4g; top-1 agreement %.2f" % (e_ref, e_fp, agree))
    assert e_ref < PKG_VS_REF_REL and e_fp < INT8_VS_FP32_REL and agree >= TOP1_AGREE
