"""Int8 max pooling and channel-slice writes on the H100: dfq_i8_maxpool and dfq_i8_conv_slice against the oracle
(tests/int8_pool_cat_oracle.py) byte for byte and bit for bit, and chain_int8(..., residual=True, pool_cat=True) on whole
torchvision models bit for bit against the per-layer path."""
import ctypes as C
import itertools
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_chain_oracle as CO
import int8_oracle as O
import int8_pool_cat_oracle as PO
import test_gpu_int8 as G
import test_gpu_int8_residual as GR

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
SENTINEL = -128


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _pool_geometry(N, Cn, H, W, k, s, p, d, ceil, Cpad=None):
    from dfq_b200 import _lib
    g = np.zeros(1, _lib.I8_POOL_DT)
    g[0] = (N, Cn, H, W, k, k, s, s, p, p, d, d, int(ceil), PO.pool_extent(H, k, p, s, d, ceil),
            PO.pool_extent(W, k, p, s, d, ceil), Cpad or (Cn + 15) // 16 * 16)
    return g


def _maxpool(g, xq=None, x=None, y=None, yq=None, scale=0.0):
    from dfq_b200 import _lib
    return _lib.load().dfq_i8_maxpool(_vp(xq), _vp(x), _vp(y), _vp(yq), C.c_float(scale), _lib.table_ptr(g),
                                      _lib.stream_ptr())


GEOMS = [(k, s, p, d, ceil) for k, s, p, d, ceil in itertools.product((1, 2, 3), (1, 2), (0, 1), (1, 2), (False, True))
         if p <= k // 2 and p <= (d * (k - 1) + 1) // 2]


@pytest.mark.parametrize("N, Cn, H, W", [(2, 37, 13, 11), (1, 16, 1, 3)])
def test_codes_pool_matches_the_oracle_and_torch(N, Cn, H, W):
    """Every kernel / stride / padding / dilation / ceil_mode combination torch accepts, C not a multiple of 16, odd sizes
    where ceil_mode adds a window: byte for byte the oracle, and q8(F.max_pool2d(x)) for NaN-free x."""
    from dfq_b200 import _lib
    torch.manual_seed(N * 100 + Cn)
    x = torch.randn(N, Cn, H, W, device="cuda") * 3
    a = G._ascale(x)
    cp = (Cn + 15) // 16 * 16
    xq = np.zeros((N, H, W, cp), np.int8)
    xq[..., :Cn] = O.i8_quantize(x.cpu().numpy(), a).transpose(0, 2, 3, 1)
    xq_d = torch.from_numpy(xq).cuda()
    extra = 0
    for k, s, p, d, ceil in GEOMS:
        g = _pool_geometry(N, Cn, H, W, k, s, p, d, ceil)
        OH, OW = int(g[0]["OH"]), int(g[0]["OW"])
        if OH <= 0 or OW <= 0:
            continue
        extra += ceil and OH != PO.pool_extent(H, k, p, s, d, False)
        yq = torch.full((N * OH * OW * cp + 64,), SENTINEL, dtype=torch.int8, device="cuda")
        _lib.check(_maxpool(g, xq=xq_d, yq=yq), "dfq_i8_maxpool")
        got = yq.cpu().numpy()
        want = PO.i8_maxpool_codes(xq, Cn, (k, k), (s, s), (p, p), (d, d), ceil)
        assert np.array_equal(got[:want.size], want.reshape(-1)), (k, s, p, d, ceil)
        assert np.all(got[want.size:] == SENTINEL)
        ref = F.max_pool2d(x, k, s, p, d, ceil)
        if not torch.isinf(ref).any():
            assert np.array_equal(want[..., :Cn], O.i8_quantize(ref.cpu().numpy(), a).transpose(0, 2, 3, 1)), (k, s, p, d)
    assert extra > 0 or H < 3, "no geometry where ceil_mode adds a window"


def test_codes_pool_grid_stride_loop_covers_every_item():
    from dfq_b200 import _lib
    N, Cn, H, W = 96, 64, 112, 112
    g = _pool_geometry(N, Cn, H, W, 3, 2, 1, 1, False)
    OH, OW = int(g[0]["OH"]), int(g[0]["OW"])
    assert N * (Cn // 16) * OH * OW > G._launch_cap()
    torch.manual_seed(3)
    xq = torch.randint(-127, 128, (N, H, W, Cn), dtype=torch.int8, device="cuda")
    yq = torch.full((N, OH, OW, Cn), SENTINEL, dtype=torch.int8, device="cuda")
    _lib.check(_maxpool(g, xq=xq, yq=yq), "dfq_i8_maxpool")
    want = F.max_pool2d(xq.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1).to(torch.int8)
    assert torch.equal(yq, want)


def _special(N, Cn, H, W, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((N, Cn, H, W)) * 2).astype(f32)
    flat = x.reshape(-1)
    idx = rng.permutation(flat.size)
    parts = np.array_split(idx[: flat.size // 3], 6)
    flat[parts[0]] = np.nan
    flat[parts[1]] = np.inf
    flat[parts[2]] = -np.inf
    flat[parts[3]] = -0.0
    flat[parts[4]] = 0.0
    flat[parts[5]] = np.float32(1e-40)                          # subnormal
    return x


@pytest.mark.parametrize("outs", ["both", "fp32", "codes"])
def test_fp32_pool_is_torch_bit_for_bit(outs):
    from dfq_b200 import _lib
    N, Cn, H, W = 2, 21, 15, 13
    x = _special(N, Cn, H, W, 5)
    x_d = torch.from_numpy(x).cuda()
    for k, s, p, d, ceil in [(3, 2, 1, 1, False), (3, 2, 0, 1, True), (2, 1, 1, 2, True), (1, 1, 0, 1, False)]:
        g = _pool_geometry(N, Cn, H, W, k, s, p, d, ceil)
        OH, OW = int(g[0]["OH"]), int(g[0]["OW"])
        ref = F.max_pool2d(x_d, k, s, p, d, ceil)
        want = PO.i8_maxpool(x, (k, k), (s, s), (p, p), (d, d), ceil)
        assert np.array_equal(np.isnan(want), torch.isnan(ref).cpu().numpy())
        fin = ~np.isnan(want)
        assert np.array_equal(want[fin].view(np.uint32), ref.cpu().numpy()[fin].view(np.uint32)), "oracle vs torch"
        y = torch.from_numpy(np.full(N * Cn * OH * OW + 32, GR.Y_SENTINEL, np.uint32).view(f32)).cuda()
        yq = torch.full((N * OH * OW * 32 + 64,), SENTINEL, dtype=torch.int8, device="cuda")
        scale = f32(9.5)
        _lib.check(_maxpool(g, x=x_d, y=y if outs != "codes" else None, yq=yq if outs != "fp32" else None, scale=scale),
                   "dfq_i8_maxpool")
        got_y, got_q = y.cpu().numpy().view(np.uint32), yq.cpu().numpy()
        n = ref.numel()
        if outs != "codes":
            r = ref.cpu().numpy().reshape(-1)
            assert np.array_equal(np.isnan(got_y[:n].view(f32)), np.isnan(r))
            assert np.array_equal(got_y[:n][~np.isnan(r)], r[~np.isnan(r)].view(np.uint32)), (k, s, p, d, ceil)
        assert np.all(got_y[n if outs != "codes" else 0:] == GR.Y_SENTINEL)
        nq = N * OH * OW * 32
        if outs != "fp32":
            q = np.zeros((N, OH, OW, 32), np.int8)
            q[..., :Cn] = O.i8_quantize(ref.cpu().numpy(), scale).transpose(0, 2, 3, 1)
            assert np.array_equal(got_q[:nq], q.reshape(-1))
        assert np.all(got_q[nq if outs != "fp32" else 0:] == SENTINEL)


def test_fp32_pool_keeps_the_first_of_tied_zeros():
    """max(-0.0, +0.0) keeps the first in window order, as torch: the sign shows through 1 / y."""
    from dfq_b200 import _lib
    x = torch.tensor([[[[-0.0, 0.0], [0.0, -0.0]]]], device="cuda")
    g = _pool_geometry(1, 1, 2, 2, 2, 2, 0, 1, False)
    y = torch.empty(1, 1, 1, 1, device="cuda")
    _lib.check(_maxpool(g, x=x, y=y), "dfq_i8_maxpool")
    assert torch.equal(y.view(torch.int32), F.max_pool2d(x, 2).view(torch.int32)) and float(1 / y) == -INF


def test_codes_mode_documented_exceptions():
    """A window holding a NaN: -127 per layer, the max of the other codes here.  Scale 0 with an infinite input: per layer
    q8(inf * 0) = -127, here the max of the codes (0)."""
    from dfq_b200 import _lib
    x = np.array([[[[np.nan, 1.0], [2.0, -1.0]]]], f32)
    xq = np.zeros((1, 2, 2, 16), np.int8)
    xq[..., 0] = O.i8_quantize(x, f32(10)).transpose(0, 2, 3, 1)[..., 0]
    g = _pool_geometry(1, 1, 2, 2, 2, 2, 0, 1, False)
    yq = torch.zeros(16, dtype=torch.int8, device="cuda")
    _lib.check(_maxpool(g, xq=torch.from_numpy(xq).cuda(), yq=yq), "dfq_i8_maxpool")
    assert int(yq[0]) == 20 and int(O.i8_quantize(F.max_pool2d(torch.from_numpy(x), 2).numpy(), f32(10)).item()) == -127
    x = np.array([[[[np.inf, 1.0], [2.0, -1.0]]]], f32)
    xq[..., 0] = O.i8_quantize(x, f32(0)).transpose(0, 2, 3, 1)[..., 0]
    _lib.check(_maxpool(g, xq=torch.from_numpy(xq).cuda(), yq=yq), "dfq_i8_maxpool")
    assert int(yq[0]) == 0 and int(O.i8_quantize(np.array([np.inf], f32), f32(0))[0]) == -127


def test_pool_refusals():
    from dfq_b200 import _lib
    lib = _lib.load()
    xq = torch.zeros(4 * 4 * 16, dtype=torch.int8, device="cuda")
    x = torch.zeros(16, device="cuda")
    yq = torch.full((64,), SENTINEL, dtype=torch.int8, device="cuda")
    good = _pool_geometry(1, 1, 4, 4, 2, 2, 0, 1, False)
    bad_oh = good.copy(); bad_oh[0]["OH"] = 3
    bad_pad = _pool_geometry(1, 1, 4, 4, 2, 2, 0, 1, False); bad_pad[0]["pad_h"] = 2
    bad_cpad = good.copy(); bad_cpad[0]["Cpad"] = 8
    for g, kw, what in [(bad_oh, dict(xq=xq, yq=yq), "OH / OW"), (bad_pad, dict(xq=xq, yq=yq), "padding"),
                        (bad_cpad, dict(xq=xq, yq=yq), "Cpad"), (good, dict(xq=xq, x=x, yq=yq), "exactly one input"),
                        (good, dict(yq=yq), "exactly one input"), (good, dict(xq=xq, yq=yq, y=x), "codes out only"),
                        (good, dict(x=x), "no output"), (good, dict(x=x, yq=yq, scale=INF), "out_scale"),
                        (good, dict(xq=xq, yq=xq), "overlaps")]:
        rc = _maxpool(g, **kw)
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (what, lib.dfq_last_error())
    torch.cuda.synchronize()
    assert bool((yq == SENTINEL).all())


# ---- slice writes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dense", "depthwise"])
@pytest.mark.parametrize("epi", ["requant", "fused"])
def test_slice_writes_only_its_channels(kind, epi):
    """Codes of dfq_i8_conv_slice at (coff, cstride) equal those of dfq_i8_conv_requant / dfq_i8_conv_fused, written only
    into the slice: sentinel neighbours untouched, pad channels only inside the slice."""
    from dfq_b200 import _lib, int8
    torch.manual_seed(11)
    Cn, O_ = (24, 40) if kind == "dense" else (40, 40)
    conv = nn.Conv2d(Cn, O_, 3, 1, 1, groups=1 if kind == "dense" else Cn).cuda()
    layer = int8.Int8Conv2d.from_conv(conv, 4.0, G._channel_scales(conv.weight, 11))
    N, H, W = 2, 9, 7
    g = layer._geometry(N, H, W)
    xq = torch.randint(-127, 128, (N, H, W, layer.cpad), dtype=torch.int8, device="cuda")
    cpad, px = 48, N * H * W
    pre, post, scale = (0.0, 6.0), ((-INF, INF) if epi == "requant" else (0.0, 5.0)), f32(20.0)
    ref = torch.empty((px, cpad), dtype=torch.int8, device="cuda")
    y = torch.empty(N * O_ * H * W, device="cuda")
    d = GR._epilogue(y=0 if epi == "requant" else y.data_ptr(), yq=ref.data_ptr(), out_scale=scale, pre=pre, post=post)
    lib = _lib.load()
    _lib.check(lib.dfq_i8_conv_fused(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias), _lib.table_ptr(d),
                                     _lib.table_ptr(g), _lib.stream_ptr()), "fused")
    for coff, cstride in [(0, 48), (16, 64), (32, 96), (64, 112)]:
        buf = torch.full((px, cstride), SENTINEL, dtype=torch.int8, device="cuda")
        y2 = torch.empty_like(y)
        d = GR._epilogue(y=0 if epi == "requant" else y2.data_ptr(), yq=buf.data_ptr(), out_scale=scale, pre=pre, post=post)
        _lib.check(lib.dfq_i8_conv_slice(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias),
                                         _lib.table_ptr(d), coff, cstride, _lib.table_ptr(g), _lib.stream_ptr()), "slice")
        assert torch.equal(buf[:, coff:coff + cpad], ref), (coff, cstride)
        assert bool((buf[:, :coff] == SENTINEL).all()) and bool((buf[:, coff + cpad:] == SENTINEL).all())
        assert bool((buf[:, coff + O_:coff + cpad] == 0).all())
        if epi == "fused":
            assert torch.equal(y2.view(torch.int32), y.view(torch.int32))


def test_slice_refusals():
    from dfq_b200 import _lib, int8
    lib = _lib.load()
    layer = int8.Int8Conv2d.from_conv(nn.Conv2d(16, 24, 1).cuda(), 1.0, 1.0)
    N, H, W = 1, 4, 4
    g = layer._geometry(N, H, W)
    xq = torch.zeros(N * H * W * 16, dtype=torch.int8, device="cuda")
    buf = torch.full((N * H * W, 64), SENTINEL, dtype=torch.int8, device="cuda")
    y = torch.zeros(N * 24 * H * W, device="cuda")
    b = buf.data_ptr()
    for coff, cstride, kw, what in [(8, 64, {}, "multiples of 16"), (0, 40, {}, "multiples of 16"),
                                    (48, 64, {}, "exceeds cstride"), (16, 32, {}, "exceeds cstride"),
                                    (0, 64, dict(r=b + 64 * 15 + 16), "residual overlaps the slice"),
                                    (0, 64, dict(y=b + 64 * 3), "y overlaps the slice"),
                                    (0, 64, dict(yq=0), "no codes")]:
        d = GR._epilogue(**dict(dict(yq=b, out_scale=1.0), **kw))
        rc = lib.dfq_i8_conv_slice(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias), _lib.table_ptr(d),
                                   coff, cstride, _lib.table_ptr(g), _lib.stream_ptr())
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (what, lib.dfq_last_error())
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL).all())


# ---- whole models ---------------------------------------------------------------------------------------------------------
def _model(net, batch=2):
    """torchvision `net` (seeded), BN folded by trace_graph + merge_batchnorm, every Conv2d / Linear converted at 128 / max
    |input| of a forward pass (tools/bench_int8.py's scales)."""
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm
    torch.manual_seed(0)
    kw = dict(aux_logits=False, init_weights=True) if net == "googlenet" else {}
    model = getattr(torchvision.models, net)(num_classes=1000, **kw).cuda().eval()
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


@pytest.mark.parametrize("net, carried, cats, pools", [("squeezenet1_1", 25, 8, 3), ("googlenet", 56, 8, 13),
                                                       ("resnet18", 19, 0, 1)])
def test_pool_cat_chained_model_is_bit_identical_to_the_per_layer_path(net, carried, cats, pools):
    from dfq_b200 import int8
    model, x = _model(net)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True)
        assert len({q for _, q, _ in gm.requantized_edges}) == carried
        assert len(gm.fused_cats) == cats and len(gm.fused_pools) == pools
        ref = model(x)
        got = gm(x)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), net


def test_cat_with_consumers_one_ulp_apart_stays_fp32_and_bit_identical():
    from dfq_b200 import int8

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.s, self.a, self.b = nn.Conv2d(3, 16, 3, 1, 1), nn.Conv2d(16, 16, 1), nn.Conv2d(16, 24, 3, 1, 1)
            self.z1, self.z2 = nn.Conv2d(40, 8, 1), nn.Conv2d(40, 8, 1)

        def forward(self, x):
            s = F.relu(self.s(x))
            c = torch.cat([F.relu(self.a(s)), F.relu(self.b(s))], 1)
            return self.z1(c) + self.z2(c)
    torch.manual_seed(4)
    model = M().cuda().eval()
    x = torch.randn(2, 3, 17, 19, device="cuda")
    acts = [4.0, 3.0, 3.0, 2.0, float(np.nextafter(f32(2.0), f32(3)))]
    int8.convert_to_int8(model, OrderedDict((id(m), m) for m in model.modules() if isinstance(m, nn.Conv2d)), [nn.Conv2d],
                         act_scales=acts)
    with torch.no_grad():
        gm = int8.chain_int8(model, residual=True, pool_cat=True)
        assert gm.fused_cats == []
        assert torch.equal(gm(x).view(torch.int32), model(x).view(torch.int32))
