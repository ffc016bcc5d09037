"""Int8 bilinear upsampling on the H100: dfq_i8_upsample_bilinear bit for bit against torch's F.interpolate and byte for byte
against the oracle (tests/int8_upsample_oracle.py), its channel-slice writes and refusals, and
chain_int8(..., residual=True, pool_cat=True, upsample=True) on two DeepLab networks bit for bit against the per-layer
path."""
import ctypes as C
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_oracle as O
import int8_upsample_oracle as UO
import test_gpu_int8 as G
from deeplab_v3plus_like import DeepLabV3PlusLike
from test_gpu_int8_pool_cat import _special

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
SENTINEL = -128
Y_SENTINEL = 0x7FA5A5A5


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _resize(N, Cn, H, W, OH, OW, ac, coff=0, cstride=None, scale=0.0, lo=-INF, hi=INF):
    from dfq_b200 import _lib
    g = np.zeros(1, _lib.I8_RESIZE_DT)
    g[0] = (N, Cn, H, W, OH, OW, int(ac), coff, cstride or (Cn + 15) // 16 * 16, scale, lo, hi)
    return g


def _upsample(g, x, y=None, yq=None):
    from dfq_b200 import _lib
    return _lib.load().dfq_i8_upsample_bilinear(_vp(x), _vp(y), _vp(yq), _lib.table_ptr(g), _lib.stream_ptr())


# (H, W, OH, OW): the ASPP's 1x1 image pool, the decoder's 4x, non-integer ratios, downsampling, a single output row or
# column, a single input row or column, the same-size copy
GRID = [(1, 1, 33, 33), (33, 33, 129, 129), (9, 11, 33, 17), (13, 7, 20, 30), (33, 33, 17, 17), (7, 5, 1, 9),
        (7, 5, 6, 1), (1, 5, 4, 9), (6, 1, 4, 9), (1, 1, 1, 1), (13, 11, 13, 11)]


@pytest.mark.parametrize("ac", [False, True], ids=["align_corners=False", "align_corners=True"])
@pytest.mark.parametrize("clamp", [(-INF, INF), (0.0, 6.0)], ids=["no_clamp", "relu6"])
def test_kernel_is_torch_and_the_oracle_bit_for_bit(ac, clamp):
    """y bit for bit F.interpolate (NaN bits included: both are H100 arithmetic), codes byte for byte the oracle's and
    q(clamp(F.interpolate(x))); C = 37 is not a multiple of 16; NaN, +-inf, -0.0 and subnormal inputs."""
    from dfq_b200 import _lib
    N, Cn, scale = 2, 37, f32(9.5)
    for H, W, OH, OW in GRID:
        x = _special(N, Cn, H, W, H * 100 + W)
        xd = torch.from_numpy(x).cuda()
        ref = F.interpolate(xd, size=(OH, OW), mode="bilinear", align_corners=ac)
        want = UO.i8_upsample_bilinear(x, OH, OW, ac)
        r = ref.cpu().numpy()
        assert np.array_equal(want.view(np.uint32), r.view(np.uint32)), ("oracle vs torch", H, W, OH, OW)
        n = N * Cn * OH * OW
        y = torch.from_numpy(np.full(n + 32, Y_SENTINEL, np.uint32).view(f32)).cuda()
        nq = N * OH * OW * 48
        yq = torch.full((nq + 64,), SENTINEL, dtype=torch.int8, device="cuda")
        _lib.check(_upsample(_resize(N, Cn, H, W, OH, OW, ac, scale=scale, lo=clamp[0], hi=clamp[1]), xd, y, yq),
                   "dfq_i8_upsample_bilinear")
        got_y, got_q = y.cpu().numpy().view(np.uint32), yq.cpu().numpy()
        assert np.array_equal(got_y[:n], r.reshape(-1).view(np.uint32)), (H, W, OH, OW)
        assert np.all(got_y[n:] == Y_SENTINEL)
        codes = UO.i8_upsample_codes(want, scale, *clamp)
        assert np.array_equal(got_q[:nq], codes.reshape(-1)), (H, W, OH, OW)
        assert np.array_equal(codes, UO.CO.to_nhwc_codes(O.i8_quantize(UO.CO.i8_clamp(r, *clamp), scale)))
        assert np.all(got_q[nq:] == SENTINEL)


@pytest.mark.parametrize("outs", ["fp32", "codes"])
def test_each_output_alone(outs):
    from dfq_b200 import _lib
    N, Cn, H, W, OH, OW = 1, 20, 9, 11, 33, 17
    x = _special(N, Cn, H, W, 7)
    xd = torch.from_numpy(x).cuda()
    want = UO.i8_upsample_bilinear(x, OH, OW, False)
    y = torch.empty(N, Cn, OH, OW, device="cuda") if outs == "fp32" else None
    yq = torch.full((N, OH, OW, 32), SENTINEL, dtype=torch.int8, device="cuda") if outs == "codes" else None
    _lib.check(_upsample(_resize(N, Cn, H, W, OH, OW, False, scale=3.0), xd, y, yq), "dfq_i8_upsample_bilinear")
    if y is not None:
        assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
    else:
        assert np.array_equal(yq.cpu().numpy(), UO.i8_upsample_codes(want, f32(3.0)))


def test_grid_stride_loop_covers_every_item():
    from dfq_b200 import _lib
    N, Cn, H, W, OH, OW = 8, 256, 33, 33, 129, 129
    assert N * (Cn // 16) * OH * OW > G._launch_cap()
    torch.manual_seed(5)
    x = torch.randn(N, Cn, H, W, device="cuda") * 4
    yq = torch.full((N, OH, OW, Cn), SENTINEL, dtype=torch.int8, device="cuda")
    y = torch.empty(N, Cn, OH, OW, device="cuda")
    _lib.check(_upsample(_resize(N, Cn, H, W, OH, OW, True, scale=20.0), x, y, yq), "dfq_i8_upsample_bilinear")
    ref = F.interpolate(x, size=(OH, OW), mode="bilinear", align_corners=True)
    assert torch.equal(y.view(torch.int32), ref.view(torch.int32))
    want = O.i8_quantize(ref.cpu().numpy(), f32(20.0)).transpose(0, 2, 3, 1)
    assert np.array_equal(yq.cpu().numpy(), want)


def test_slice_writes_only_its_channels():
    """Codes into channels [coff, coff + 48) of a wider tensor: sentinel neighbours untouched, pad channels 0."""
    from dfq_b200 import _lib
    N, Cn, H, W, OH, OW = 2, 37, 5, 6, 9, 11
    x = _special(N, Cn, H, W, 3)
    codes = UO.i8_upsample_codes(UO.i8_upsample_bilinear(x, OH, OW, True), f32(4.0), 0.0, INF).reshape(-1, 48)
    px = N * OH * OW
    for coff, cstride in [(0, 48), (16, 64), (32, 96), (64, 112)]:
        buf = torch.full((px, cstride), SENTINEL, dtype=torch.int8, device="cuda")
        g = _resize(N, Cn, H, W, OH, OW, True, coff, cstride, 4.0, 0.0, INF)
        _lib.check(_upsample(g, torch.from_numpy(x).cuda(), yq=buf), "dfq_i8_upsample_bilinear")
        b = buf.cpu().numpy()
        assert np.array_equal(b[:, coff:coff + 48], codes), (coff, cstride)
        assert np.all(b[:, coff + Cn:coff + 48] == 0)
        assert np.all(b[:, :coff] == SENTINEL) and np.all(b[:, coff + 48:] == SENTINEL)


def test_refusals():
    from dfq_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(2 * 16 * 4 * 4, device="cuda")
    y = torch.full((2 * 16 * 8 * 8,), 7.0, device="cuda")
    yq = torch.full((2 * 8 * 8 * 64 + 64,), SENTINEL, dtype=torch.int8, device="cuda")
    good = dict(N=2, Cn=16, H=4, W=4, OH=8, OW=8, ac=False)
    cases = [(dict(OH=0), dict(y=y), "empty dimension"), (dict(W=-1), dict(y=y), "empty dimension"),
             (dict(ac=2), dict(y=y), "align_corners"), (dict(coff=8, cstride=64), dict(yq=yq), "multiples of 16"),
             (dict(cstride=40), dict(yq=yq), "multiples of 16"), (dict(coff=16, cstride=16), dict(yq=yq), "exceeds cstride"),
             ({}, {}, "no output"), ({}, dict(yq=yq[1:]), "16-byte aligned"), ({}, dict(y=y[1:].view(torch.int8)[1:]), "4-byte"),
             ({}, dict(x=x.view(torch.int8)[2:], y=y), "4-byte"),
             (dict(scale=INF), dict(yq=yq), "out_scale"), (dict(scale=-1.0), dict(yq=yq), "out_scale"),
             (dict(lo=1.0, hi=0.0), dict(y=y), "bounds"), (dict(lo=float("nan")), dict(y=y), "bounds"),
             ({}, dict(x=y, y=y), "x overlaps"), ({}, dict(x=yq[64:].view(torch.float32), yq=yq), "x overlaps"),
             ({}, dict(y=yq[:4096].view(torch.float32), yq=yq[4096:]), "y overlaps")]
    for geo, bufs, what in cases:
        a = dict(good, **geo)
        g = _resize(a["N"], a["Cn"], a["H"], a["W"], a["OH"], a["OW"], a["ac"], a.get("coff", 0), a.get("cstride"),
                    a.get("scale", 1.0), a.get("lo", -INF), a.get("hi", INF))
        g[0]["align_corners"] = a["ac"]
        xx = bufs.pop("x", x)
        rc = _upsample(g, xx, bufs.get("y"), bufs.get("yq"))
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (what, lib.dfq_last_error())
    torch.cuda.synchronize()
    assert bool((yq == SENTINEL).all()) and bool((y == 7.0).all())


# ---- whole models -----------------------------------------------------------------------------------------------------------
def _convert(model, x):
    """BN folded by trace_graph + merge_batchnorm, every Conv2d / Linear converted at 128 / max|input| of a forward pass
    (test_gpu_int8_pool_cat.py's _model)."""
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm
    graph, bottoms = trace_graph(model)
    merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
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
    return model


def _model(net, batch=2, size=129):
    import torchvision
    torch.manual_seed(0)
    if net == "deeplab_v3plus_like":
        model = DeepLabV3PlusLike(num_classes=21)
    else:
        model = torchvision.models.segmentation.deeplabv3_resnet50(weights=None, weights_backbone=None, aux_loss=False)
    model = model.cuda().eval()
    x = torch.randn(batch, 3, size, size, device="cuda")
    return _convert(model, x), x


@pytest.mark.parametrize("net, convs, carried, carried_pool_cat, cats, ups", [
    ("deeplab_v3plus_like", 34, 32, 30, 2, [("interpolate", "aspp.pool.1", "slice", True),
                                            ("interpolate_1", "aspp.project.0", "slice", True)]),
    ("deeplabv3_resnet50", 61, 59, 58, 1, [("interpolate", "classifier.0.convs.4.1", "slice", False)]),
])
def test_upsample_chained_model_is_bit_identical_to_the_per_layer_path(net, convs, carried, carried_pool_cat, cats, ups):
    from dfq_b200 import int8
    model, x = _model(net)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
        base = int8.chain_int8(model, residual=True, pool_cat=True)
        assert sum(isinstance(m, int8.Int8Conv2d) for m in model.modules()) == convs
        assert len({q for _, q, _ in gm.requantized_edges}) == carried
        assert len({q for _, q, _ in base.requantized_edges}) == carried_pool_cat
        assert len(gm.fused_cats) == cats and base.fused_cats == [] and gm.fused_upsamples == ups
        ref, got = model(x), gm(x)
    ref, got = (t["out"] if isinstance(t, dict) else t for t in (ref, got))
    assert tuple(got.shape) == (2, 21, 129, 129)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), net
