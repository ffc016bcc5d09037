"""Layout copies removed on the H100: dfq_i8_conv_nhwc bit for bit against dfq_i8_conv_fused's fp32 output permuted, its
writes confined to its rows and its refusals; zero pads folded into convolutions; and chain_int8(..., layout=True) on the
networks written after the reference's DeepLab-v3+ (MobileNetV2, fixed padding) and MobileNetV2-SSD-Lite, bit for bit
against the per-layer path."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from deeplab_mobilenet_padded import DeepLabMobileNetPadded
from ssd_lite_like import SSDLiteLike
from test_gpu_int8_upsample import _convert

pytestmark = pytest.mark.gpu
INF = math.inf
NONE = (-INF, INF)
SENTINEL = 0x7FA5A5A5


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _layer(Cn, O, k, groups, seed, stride=1, padding=1, dilation=1):
    """An Int8Conv2d whose bias holds NaN, +-inf and -0.0 on its first channels (they reach the epilogue as they are)."""
    from dfq_b200 import int8
    torch.manual_seed(seed)
    conv = nn.Conv2d(Cn, O, k, stride, padding, dilation, groups=groups)
    with torch.no_grad():
        conv.bias.mul_(4)
        special = torch.tensor([math.nan, INF, -INF, -0.0])[:O]
        conv.bias[:len(special)] = special
    return int8.Int8Conv2d.from_conv(conv.cuda(), 9.0, 128. / float(conv.weight.abs().max())).cuda()


CLAMPS = [(NONE, NONE), ((0.0, 6.0), NONE), ((-1.0, INF), (-INF, 0.5)), ((-INF, -0.0), NONE)]


def _check_rows(layer, x, clamps, off, gap):
    """Two slices of the same layer's rows, at off and off + extent + gap of each image, against the fused fp32 output."""
    from dfq_b200 import int8
    pre, post = clamps
    fused = layer.chained(epilogue=int8.Epilogue(None, pre, post, False, True))(x)
    N, O, OH, OW = fused.shape
    want = fused.permute(0, 2, 3, 1).reshape(N, -1).view(torch.int32)
    ext = OH * OW * O
    stride = off + 2 * ext + gap + 5
    buf = torch.full((N, stride), SENTINEL, dtype=torch.int32, device="cuda")
    rows = layer.chained(epilogue=int8.Epilogue(None, pre, post, False, True), rows=True)
    rows(x, out=buf.view(torch.float32), off=off)
    rows(x, out=buf.view(torch.float32), off=off + ext + gap)
    for o in (off, off + ext + gap):
        assert torch.equal(buf[:, o:o + ext], want), (O, off, clamps)
    keep = torch.ones(stride, dtype=torch.bool, device="cuda")
    keep[off:off + ext] = False
    keep[off + ext + gap:off + 2 * ext + gap] = False
    assert bool((buf[:, keep] == SENTINEL).all())
    alone = rows(x)                                              # a tensor of its own: the permuted output
    assert tuple(alone.shape) == (N, OH * OW, O) and torch.equal(alone.reshape(N, -1).view(torch.int32), want)


@pytest.mark.parametrize("O", [1, 3, 24, 63, 64, 65, 126, 130])
def test_dense_rows_are_the_fused_output_permuted(O):
    # 7x9 (63 pixels, not a multiple of 8) x 3 images: M = 189, a tail past one 128-pixel tile; 13x11 x 2: 286
    for i, (N, H, W, off, gap) in enumerate([(3, 7, 9, 0, 0), (2, 13, 11, 7, 3), (1, 5, 6, 64, 1)]):
        layer = _layer(37, O, 3, 1, O * 10 + i)
        x = (torch.randn(N, 37, H, W, device="cuda") * 3)
        _check_rows(layer, x, CLAMPS[i % len(CLAMPS)], off, gap)
        _check_rows(layer, x, CLAMPS[(i + 2) % len(CLAMPS)], off + 1, gap)


@pytest.mark.parametrize("O", [3, 24, 63, 64, 65, 126, 130])
def test_depthwise_rows_are_the_fused_output_permuted(O):
    for i, (N, H, W, off, gap) in enumerate([(3, 7, 9, 0, 0), (2, 13, 11, 9, 2)]):
        layer = _layer(O, O, 3, O, O * 10 + i, stride=1 + i, dilation=1 + i)
        x = torch.randn(N, O, H, W, device="cuda") * 3
        for j, clamps in enumerate(CLAMPS):
            _check_rows(layer, x, clamps, off + j, gap)


def test_refusals_leave_the_buffers_untouched():
    from dfq_b200 import _lib
    lib = _lib.load()
    layer = _layer(16, 8, 1, 1, 0, padding=0)
    N, H, W = 2, 4, 4
    x = torch.randn(N, 16, H, W, device="cuda")
    xq = torch.empty(N * H * W * 16, dtype=torch.int8, device="cuda")
    _lib.check(lib.dfq_i8_quantize_nhwc(_vp(x), _vp(xq), N, 16, H, W, 16, C.c_float(9.0), _lib.stream_ptr()), "quantize")
    y = torch.full((N * 200,), SENTINEL, dtype=torch.int32, device="cuda")
    g = layer._geometry(N, H, W)
    ext = H * W * 8

    def call(off=0, stride=200, geo=g, **e):
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0, y.data_ptr(), 0, 0.0, -INF, INF, -INF, INF)
        for k, v in e.items():
            d[0][k] = v
        return lib.dfq_i8_conv_nhwc(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias), _lib.table_ptr(d),
                                    off, stride, _lib.table_ptr(geo), _lib.stream_ptr())
    cases = [(dict(y=0), "no output"), (dict(y=y.data_ptr() + 2), "4-byte"), (dict(residual=y.data_ptr()), "must be NULL"),
             (dict(yq=xq.data_ptr()), "must be NULL"), (dict(off=-1), "off must be non-negative"),
             (dict(stride=ext - 1), "img_stride"), (dict(off=73, stride=200), "img_stride"),
             (dict(pre_lo=math.nan), "bounds"), (dict(post_lo=1.0, post_hi=0.0), "bounds"),
             (dict(y=xq.data_ptr() + 16), "overlaps xq")]
    for e, what in cases:
        off, stride = e.pop("off", 0), e.pop("stride", 200)
        rc = call(off, stride, **e)
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (what, lib.dfq_last_error())
    bad = g.copy()
    bad[0]["groups"] = 2
    assert call(geo=bad) == -2 and b"grouping" in lib.dfq_last_error()
    torch.cuda.synchronize()
    assert bool((y == SENTINEL).all())
    assert call(off=200 - ext) == 0                              # the last fitting offset
    torch.cuda.synchronize()
    assert bool((y.view(N, 200)[:, :200 - ext] == SENTINEL).all())


# ---- zero padding folded into the next convolution ---------------------------------------------------------------------------
class _Pad(nn.Module):
    def __init__(self, b, pad):
        super().__init__()
        self.a, self.b, self.pad = nn.Conv2d(3, 16, 3, 1, 1), b, pad

    def forward(self, x):
        return self.b(F.pad(F.relu(self.a(x)), self.pad))


@pytest.mark.parametrize("b, pad", [
    (nn.Conv2d(16, 8, 1), (1, 1, 1, 1)), (nn.Conv2d(16, 8, 1), (2, 2, 2, 2)),
    (nn.Conv2d(16, 24, 3, 1, 0, 2), (2, 2, 2, 2)), (nn.Conv2d(16, 16, 3, 1, 0, 2, groups=16), (2, 2, 2, 2)),
    (nn.Conv2d(16, 8, 3, 2), (1, 1, 1, 1)), (nn.Conv2d(16, 16, 3, 2, 0, groups=16), (1, 1, 0, 0)),
], ids=["1x1_pad1", "1x1_pad2", "dense_dil2", "dw_dil2", "dense_s2", "dw_s2_lr"])
def test_folded_pad_is_the_conv_of_the_padded_input(b, pad):
    from dfq_b200 import int8
    torch.manual_seed(1)
    model = _Pad(b, pad).cuda().eval()
    x = torch.randn(2, 3, 13, 11, device="cuda")
    _convert(model, x)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
        assert [(p, c) for p, c, _ in gm.folded_pads] == [("pad", "b")]
        for xx in (x, torch.randn(1, 3, 9, 7, device="cuda") * 5):
            ref, got = model(xx), gm(xx)
            assert got.shape == ref.shape and torch.equal(got.view(torch.int32), ref.view(torch.int32))


# ---- the reference's networks ----------------------------------------------------------------------------------------------------
def _net(net, batch, size, is_test=False):
    torch.manual_seed(0)
    model = (DeepLabMobileNetPadded(21) if net == "deeplab" else SSDLiteLike(21, is_test=is_test)).cuda().eval()
    x = torch.randn(batch, 3, size, size, device="cuda")
    return _convert(model, x), x


def _same(got, ref):
    got, ref = (t if isinstance(t, tuple) else (t,) for t in (got, ref))
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        assert a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("batch, size", [(2, 129), (1, 513)])
def test_deeplab_mobilenet_folds_its_pads_bit_identically(batch, size):
    from dfq_b200 import int8
    model, x = _net("deeplab", batch, size)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
        base = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
        assert sum(isinstance(m, int8.Int8Conv2d) for m in model.modules()) == 61
        assert len(gm.folded_pads) == 17 and gm.fused_heads == [] and len(gm.fused_cats) == 2
        assert len({q for _, q, _ in gm.requantized_edges}) == 59
        assert len({q for _, q, _ in base.requantized_edges}) == 42
        assert not [n for n in gm.graph.nodes if n.op == "call_function" and n.target is F.pad]
        ref, got = model(x), gm(x)
    assert tuple(got.shape) == (batch, 21, size, size)
    _same(got, ref)


@pytest.mark.parametrize("is_test", [False, True])
def test_ssd_lite_writes_its_heads_into_the_cats_bit_identically(is_test):
    from dfq_b200 import int8
    model, x = _net("ssd", 4, 300, is_test)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
        base = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
        assert sum(isinstance(m, int8.Int8Conv2d) for m in model.modules()) == 86
        assert [(c, len(p), k) for c, p, k in gm.fused_heads] == [("cat", 6, 21), ("cat_1", 6, 4)]
        assert len({q for _, q, _ in gm.requantized_edges}) == len({q for _, q, _ in base.requantized_edges}) == 85
        left = {str(n.target) for n in gm.graph.nodes if n.op in ("call_method", "call_function")}
        assert not left & {"permute", "contiguous", "view", "size"} and torch.cat not in \
            {n.target for n in gm.graph.nodes}
        ref, got = model(x), gm(x)
        assert tuple(got[0].shape) == (4, 3000, 21) and tuple(got[1].shape) == (4, 3000, 4)
        _same(got, ref)
        x2 = torch.randn(2, 3, 240, 320, device="cuda")          # the same module at another size: R follows the input
        ref2, got2 = model(x2), gm(x2)
        assert got2[0].shape[1] != got[0].shape[1]
        _same(got2, ref2)
