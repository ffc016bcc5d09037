"""dfq_b200.int8.chain_int8(..., layout=True) on the CPU: which zero pads are folded into convolutions and which detection-head
concatenations are written in place, and that the chained module computes what the per-layer one does - through the host
twins of the library (tests/int8_layout_oracle.py), with torch told that CPU tensors are on the GPU.  Also the two networks
written after the reference's DeepLab-v3+ and MobileNetV2-SSD-Lite against the reference's traced topologies."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_layout_oracle as LO
from deeplab_mobilenet_padded import DeepLabMobileNetPadded
from ssd_lite_like import SSDLiteLike
from test_int8_chain_host import _identity_bns, _x
from test_int8_pool_cat_host import _scales_through_pools
from test_int8_upsample_host import _convert, _gpu_interpolate

f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _chain(monkeypatch, model, x, acts=None):
    """The chained module (layout=True) of `model` converted at `acts` (default: _scales_through_pools), checked bit for bit
    against the per-layer model on x through the twins; (gm, fake)."""
    from dfq_b200 import int8
    fake = LO.install(monkeypatch)
    torch.manual_seed(0)
    model = model.eval()
    _convert(model, acts or _scales_through_pools(model))
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    _gpu_interpolate(monkeypatch)
    with torch.no_grad():
        fake.calls.clear()
        y = gm(x)
        ref = model(x)
    ys, refs = (t if isinstance(t, tuple) else (t,) for t in (y, ref))
    for a, b in zip(ys, refs):
        assert a.dtype == torch.float32 and a.shape == b.shape
        assert np.array_equal(a.numpy().view(np.int32), b.numpy().view(np.int32))
    return gm, fake


def _ops(gm, *names):
    return [n for n in gm.graph.nodes if (n.op == "call_method" and n.target in names) or
            (n.op == "call_function" and getattr(n.target, "__name__", None) in names)]


# ---- (a) zero padding folded into the next convolution ------------------------------------------------------------------------
class _Pad(nn.Module):
    """a -> relu -> F.pad(**pad) -> b (-> after)"""

    def __init__(self, b=None, pad=(1, 1, 1, 1), kw=None, extra=None):
        super().__init__()
        self.a = nn.Conv2d(3, 16, 3, 1, 1)
        self.b = b or nn.Conv2d(16, 8, 3)
        self.pad, self.kw, self.extra = pad, kw or {}, extra

    def forward(self, x):
        p = F.pad(F.relu(self.a(x)), self.pad, **self.kw)
        y = self.b(p)
        return y if self.extra is None else (y, self.extra(p))


@pytest.mark.parametrize("b, pad, kw, tl", [
    (nn.Conv2d(16, 8, 3), (1, 1, 1, 1), {}, (1, 1)),
    (nn.Conv2d(16, 8, 1), (1, 1, 1, 1), {}, (1, 1)),                          # 1x1: the border is the bias
    (nn.Conv2d(16, 8, 1), (2, 2, 2, 2), dict(mode="constant", value=0.0), (2, 2)),
    (nn.Conv2d(16, 16, 3, 1, 0, 2, groups=16), (2, 2, 2, 2), {}, (2, 2)),    # depthwise, dilation 2
    (nn.Conv2d(16, 8, 3, 2, 1), (1, 1), dict(value=0), (0, 1)),              # (l, r) only; stride 2 and its own padding
    (nn.Conv2d(16, 8, 3, 2), (0, 0, 3, 3), {}, (3, 0)),
], ids=["3x3", "1x1_pad1", "1x1_pad2_kwargs", "dw_dilation2", "lr_stride2", "tb_only"])
def test_zero_pad_is_folded(monkeypatch, b, pad, kw, tl):
    from dfq_b200 import int8
    conv_pad = b.padding
    gm, fake = _chain(monkeypatch, _Pad(b, pad, kw), _x())
    assert gm.folded_pads == [("pad", "b", tl)]
    assert gm.get_submodule("b").padding == (conv_pad[0] + tl[0], conv_pad[1] + tl[1])
    assert ("a", "b", (0.0, INF)) in gm.requantized_edges                   # a direct edge for the chain rules
    assert not _ops(gm, "pad") and "dfq_i8_quantize_nhwc" in fake.calls
    with torch.no_grad():
        plain = int8.chain_int8(_Pad(b, pad, kw).eval(), residual=True, pool_cat=True, upsample=True)
    assert not hasattr(plain, "folded_pads")


@pytest.mark.parametrize("pad, kw, extra, b", [
    ((1, 2, 1, 1), {}, None, None),                                 # asymmetric
    ((1, 1, 2, 1), {}, None, None),
    ((-1, -1, 0, 0), {}, None, nn.Conv2d(16, 8, 1)),                # negative
    ((1, 1, 1, 1), dict(mode="reflect"), None, None),
    ((1, 1, 1, 1), dict(mode="replicate"), None, None),
    ((1, 1, 1, 1), dict(value=1.0), None, None),                    # not zero
    ((1, 1, 1, 1, 0, 0), {}, None, None),                           # a third (channel) dimension
    ((1, 1, 1, 1), {}, "second_user", None),
    ((1, 1, 1, 1), {}, "relu_between", None),
], ids=["asym_lr", "asym_tb", "negative", "reflect", "replicate", "value1", "3d", "second_user", "relu_between"])
def test_other_pads_stay_in_torch(monkeypatch, pad, kw, extra, b):
    if extra == "relu_between":
        class M(_Pad):
            def forward(self, x):
                return self.b(F.relu(F.pad(self.a(x), self.pad, **self.kw)))
        model = M(b, pad, kw)
    else:
        model = _Pad(b, pad, kw, (lambda p: p.sum()) if extra == "second_user" else None)
    gm, _ = _chain(monkeypatch, model, _x())
    assert gm.folded_pads == [] and len(_ops(gm, "pad")) == 1


def test_zeropad2d_and_multi_site_convolutions_keep_their_pads(monkeypatch):
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.b = nn.Conv2d(3, 16, 3, 1, 1), nn.Conv2d(16, 16, 3)
            self.zp = nn.ZeroPad2d(1)

        def forward(self, x):
            y = self.b(self.zp(F.relu(self.a(x))))
            return self.b(F.pad(y, (1, 1, 1, 1)))                          # b runs at two sites
    gm, _ = _chain(monkeypatch, M(), _x())
    assert gm.folded_pads == [] and len(_ops(gm, "pad")) == 1


def test_pad_folds_in_a_residual_block_and_the_fan_out_follows(monkeypatch):
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.b, self.c = nn.Conv2d(3, 16, 3, 1, 1), nn.Conv2d(16, 16, 3), nn.Conv2d(16, 8, 1)

        def forward(self, x):
            h = F.relu(self.a(x))
            h = h + self.b(F.pad(h, (1, 1, 1, 1)))
            return self.c(h)
    gm, _ = _chain(monkeypatch, M(), _x())
    assert gm.folded_pads == [("pad", "b", (1, 1))]
    assert ("a", "b", (0.0, INF)) in gm.requantized_edges and ("b", "c", NONE) in gm.requantized_edges
    assert gm.fused_adds and gm.fused_adds[0][:2] == ("b", "add")


# ---- (b) detection heads written into their concatenation ----------------------------------------------------------------------
class _Heads(nn.Module):
    """two sources, each with a k-wide head: cat(view(permute(head(x))), 1); `form` varies how the layout is spelled"""

    def __init__(self, form="ref", k=6, k2=None):
        super().__init__()
        self.s1, self.s2 = nn.Conv2d(3, 16, 3, 1, 1), nn.Conv2d(16, 16, 3, 2, 1)
        self.h1, self.h2 = nn.Conv2d(16, 2 * k, 3, 1, 1), nn.Conv2d(16, 3 * (k2 or k), 1)
        self.form, self.k, self.k2 = form, k, k2 or k

    def _lay(self, y, k):
        f = self.form
        if f == "reshape":
            return y.permute(0, 2, 3, 1).reshape(y.shape[0], -1, k)
        t = y.permute(0, 2, 3, 1).contiguous()
        if f == "const_n":
            return t.view(2, -1, k)
        if f == "tuple":
            return t.view((t.size(0), -1, k))
        if f == "shape0":
            return t.view(t.shape[0], -1, k)
        if f == "size_index":
            return t.view(t.size()[0], -1, k)
        if f == "bad_perm":
            return y.permute(0, 3, 2, 1).contiguous().view(t.size(0), -1, k)
        if f == "bad_n":
            return t.view(t.size(1) // t.size(1) * t.size(0), -1, k)
        if f == "flat":
            return t.view(-1, k)
        return t.view(t.size(0), -1, k)

    def forward(self, x):
        a = F.relu(self.s1(x))
        b = F.relu(self.s2(a))
        h1 = self.h1(a)
        if self.form == "relu":
            h1 = F.relu6(h1)
        h2 = self.h2(b)
        outs = [self._lay(h1, self.k), self._lay(h2, self.k2)]
        if self.form == "flat":
            return torch.cat(outs, 0)
        if self.form == "second_user":
            return torch.cat(outs, 1), h1.mean()
        return torch.cat(outs, 1)


@pytest.mark.parametrize("form", ["ref", "reshape", "const_n", "tuple", "shape0", "size_index", "relu"])
def test_heads_write_their_rows_of_the_cat(monkeypatch, form):
    from dfq_b200 import int8
    gm, fake = _chain(monkeypatch, _Heads(form), _x())
    assert gm.fused_heads == [("cat", ["h1", "h2"], 6)]
    assert fake.calls.count("dfq_i8_conv_nhwc") == 2
    assert not _ops(gm, "permute", "contiguous", "view", "reshape", "size", "cat", "getitem", "getattr")
    h1 = gm.get_submodule("h1")
    assert h1.rows and h1.epilogue == (None, (0.0, 6.0) if form == "relu" else NONE, NONE, False, True)
    assert gm.get_submodule("h2").codes_in                                  # s2 -> h2 still carries codes
    cat = gm.get_submodule("int8_heads_cat")
    assert isinstance(cat, int8.Int8HeadConcat) and cat.batch == (2 if form == "const_n" else None)


def test_rows_follow_the_input_size_and_refuse_a_wrong_constant_batch(monkeypatch):
    from dfq_b200 import _lib
    gm, _ = _chain(monkeypatch, _Heads(), _x())
    for shape in [(1, 3, 7, 5), (3, 3, 16, 16)]:
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(4))
        with torch.no_grad():
            y = gm(x)
        assert y.shape[:2] == (shape[0], 2 * shape[2] * shape[3] + 3 * ((shape[2] + 1) // 2) * ((shape[3] + 1) // 2))
    gm, _ = _chain(monkeypatch, _Heads("const_n"), _x())
    with pytest.raises(_lib.DfqError, match="batch"):
        gm(torch.randn(3, 3, 9, 11))


@pytest.mark.parametrize("form", ["bad_perm", "bad_n", "flat", "second_user"])
def test_other_cats_stay_in_torch(monkeypatch, form):
    gm, _ = _chain(monkeypatch, _Heads(form), _x())
    assert gm.fused_heads == [] and len(_ops(gm, "cat")) == 1
    assert gm.fused_cats == []                                              # nor is it a channel concatenation


def test_one_operand_not_from_a_head_keeps_the_cat(monkeypatch):
    class M(_Heads):
        def forward(self, x):
            a = F.relu(self.s1(x))
            h1 = self._lay(self.h1(a), 6)
            return torch.cat([h1, self._lay(self.h2(a) * 2, 6)], 1)
    gm, _ = _chain(monkeypatch, M(), _x(), dict(s1=7.0, s2=5.0, h1=3.0, h2=3.0))
    assert gm.fused_heads == []


def test_rows_mode_of_a_layer_and_its_refusals(monkeypatch):
    from dfq_b200 import _lib, int8
    LO.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    torch.manual_seed(0)
    conv = nn.Conv2d(3, 5, 3, 1, 1)
    layer = int8.Int8Conv2d.from_conv(conv, 9.0, 128. / float(conv.weight.abs().max()))
    x = _x()
    y, acc = layer.chained().run(x, with_acc=True)
    rows = layer.chained(epilogue=int8.Epilogue(None, (0.0, INF), (-INF, 1.5), fp32=True), rows=True)
    got = rows(x)
    assert tuple(got.shape) == (2, 99, 5)
    want = LO.i8_rows(y.numpy(), (0.0, INF), (-INF, 1.5)).reshape(2, 99, 5)
    assert np.array_equal(got.numpy().view(np.int32), want.view(np.int32))
    buf = torch.full((2, 600), 7.0)
    rows(x, out=buf, off=101)
    b = buf.numpy()
    assert np.array_equal(b[:, 101:596], want.reshape(2, -1)) and (b[:, :101] == 7).all() and (b[:, 596:] == 7).all()
    with pytest.raises(_lib.DfqError, match="do not fit"):
        rows(x, out=buf, off=106)
    with pytest.raises(_lib.DfqError, match="exclude codes"):
        layer.chained(requant=(1.0, 0.0, INF), rows=True)
    with pytest.raises(_lib.DfqError, match="exclude codes"):
        layer.chained(epilogue=int8.Epilogue(2.0, fp32=True), rows=True)
    with pytest.raises(_lib.DfqError, match="int32 sums"):
        rows.run(x, with_acc=True)


def test_twin_refusals(monkeypatch):
    """The host twin refuses what the library refuses (tests/test_gpu_int8_layout.py checks the library's)."""
    from dfq_b200 import _lib
    fake = LO.install(monkeypatch)
    g = np.zeros(1, _lib.I8_CONV_DT)
    g[0] = (1, 16, 4, 4, 8, 1, 1, 1, 1, 0, 0, 1, 1, 1, 4, 4, 16, 0)
    xq = np.zeros(256 + 16, np.int8)
    xa = xq.ctypes.data + (-xq.ctypes.data) % 16
    y = np.zeros(512, f32)

    def call(off=0, stride=128, **e):
        d = np.zeros(1, _lib.I8_EPILOGUE_DT)
        d[0] = (0, y.ctypes.data, 0, 0.0, -INF, INF, -INF, INF)
        for k, v in e.items():
            d[0][k] = v
        return fake.dfq_i8_conv_nhwc(xa, xa, y.ctypes.data, None, d.ctypes.data, off, stride, g.ctypes.data, None)
    for bad in [dict(y=0), dict(y=y.ctypes.data + 2), dict(residual=y.ctypes.data), dict(yq=xa), dict(off=-1),
                dict(stride=127), dict(off=1, stride=128), dict(pre_lo=np.nan), dict(post_lo=1.0, post_hi=0.0),
                dict(y=xa)]:
        off, stride = bad.pop("off", 0), bad.pop("stride", 128)
        assert call(off, stride, **bad) == LO.E_ARG, bad


# ---- the reference's networks ----------------------------------------------------------------------------------------------------
def _conv_bn_args(model, x):
    out = []

    def hook(m, i, o):
        if isinstance(m, nn.Conv2d):
            out.append(("Conv2d", dict(in_channels=m.in_channels, out_channels=m.out_channels,
                                       kernel_size=list(m.kernel_size), stride=list(m.stride), padding=list(m.padding),
                                       dilation=list(m.dilation), groups=m.groups, bias=m.bias is not None)))
        else:
            out.append(("BatchNorm2d", dict(num_features=m.num_features, eps=m.eps)))
    hs = [m.register_forward_hook(hook) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.BatchNorm2d))]
    with torch.no_grad():
        model.eval()(x)
    for h in hs:
        h.remove()
    return out


@pytest.mark.parametrize("name", ["deeplab", "ssd"])
def test_networks_match_the_reference_topology(name):
    with open(os.path.join(GOLD, "topology_%s.json" % name)) as f:
        topo = json.load(f)
    want = [(n["type"], n["args"]) for n in topo["nodes"] if n["type"] in ("Conv2d", "BatchNorm2d")]
    model, x = (DeepLabMobileNetPadded(), torch.randn(1, 3, 65, 65)) if name == "deeplab" else \
        (SSDLiteLike(), torch.randn(1, 3, 300, 300))
    assert _conv_bn_args(model, x) == want
    if name == "deeplab":
        import torch.fx as fx
        pads = [n for n in fx.symbolic_trace(model).graph.nodes if n.op == "call_function" and n.target is F.pad]
        assert len(pads) == 17 == sum(n["key"].startswith("F.pad") for n in topo["nodes"])


def test_deeplab_mobilenet_folds_its_17_pads_and_runs_bit_identically(monkeypatch):
    model = _identity_bns(DeepLabMobileNetPadded(num_classes=5))
    gm, fake = _chain(monkeypatch, model, torch.randn(1, 3, 33, 29, generator=torch.Generator().manual_seed(2)))
    assert len(gm.folded_pads) == 17 and not _ops(gm, "pad")
    assert [t for _, _, t in gm.folded_pads] == [(1, 1)] * 16 + [(2, 2)]
    assert gm.folded_pads[0][1] == "backbone.features.1.conv.0"            # the first block's depthwise convolution
    assert [c[0] for c in gm.fused_cats] == ["cat", "cat_1"] and gm.fused_heads == []


@pytest.mark.parametrize("is_test", [False, True])
def test_ssd_lite_fuses_its_12_heads_and_runs_bit_identically(monkeypatch, is_test):
    model = _identity_bns(SSDLiteLike(num_classes=5, is_test=is_test))
    gm, fake = _chain(monkeypatch, model, torch.randn(1, 3, 96, 96, generator=torch.Generator().manual_seed(3)))
    assert [(c, len(p), k) for c, p, k in gm.fused_heads] == [("cat", 6, 5), ("cat_1", 6, 4)]
    assert fake.calls.count("dfq_i8_conv_nhwc") == 12
    assert not _ops(gm, "permute", "contiguous", "view", "cat")
    assert len(_ops(gm, "softmax")) == int(is_test)
