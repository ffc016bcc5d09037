"""dfq_b200.int8.chain_affine on the CPU: the oracle of the affine residual epilogue (tests/int8_affine_chain_oracle.py)
against the per-layer path's quantizer, and which edges, fan-outs and residual adds chain_affine fuses, with which ranges,
clamps and sums - through the host twin of dfq_i8_affine_conv_fused (tests/fakelib_int8_affine_chain.py), with torch told
that CPU tensors are on the GPU, so the chained module is checked bit for bit against the per-layer one."""
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

import fakelib_int8_affine_chain
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A

f32 = np.float32
INF = math.inf
NONE = (-INF, INF)


# ---- the oracle ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 4, 8])
@pytest.mark.parametrize("lo", [-1.5, 0.25])
@pytest.mark.parametrize("residual", [False, True])
def test_oracle_codes_are_the_quantizer_codes_of_the_per_layer_value(bits, lo, residual):
    """codes and S of the epilogue == act_codes(clamp(clamp(y) + r)) of the per-layer fp32 value, with NaN, +-inf, -0.0
    and subnormals through the bias and the residual."""
    rng = np.random.default_rng(bits * 7 + int(residual))
    xq = rng.integers(-128, 128, (2, 5, 6, 7)).astype(np.int8)
    wq = rng.integers(-128, 128, (19, 5, 3, 3)).astype(np.int8)
    P, Ax, Wv, Nv = A.terms(xq, wq, (1, 1), (1, 1))
    k = A.constants(f32(-0.7), f32(0.011), f32(-0.2), f32(0.0016))
    bias = rng.standard_normal(19).astype(f32)
    bias[:4] = (np.nan, np.inf, -np.inf, -0.0)
    r = (rng.standard_normal(P.shape) * 2).astype(f32) if residual else None
    if residual:
        r[0, 5, :2, :2] = (np.nan, 1e-40), (-np.inf, -0.0)
    out = (f32(lo), f32(lo + 3.5), bits)
    pre, post = (0.0, 6.0), (0.0, INF)
    v, q, S = AC.fused(P, Ax, Wv, Nv, k, bias, r, pre, post, out, gpu_nan=False)
    y = A.epilogue(P, Ax, Wv, Nv, k, bias)
    ref = np.clip(y, 0, 6)                                      # no NaN survives to here except the bias's
    ref = np.where(np.isnan(y), y, ref)
    if residual:
        ref = (ref + r).astype(f32)
    ref = np.where(ref < 0, f32(0), ref).astype(f32)
    assert np.array_equal(v.view(np.int32), ref.view(np.int32))
    q_ref, S_ref = A.act_codes(ref, *out)
    assert np.array_equal(q, q_ref) and np.array_equal(S, S_ref)
    assert np.array_equal(S, q.astype(np.int64).sum(axis=1))
    assert q[:, 0].min() == -128 and (q == -128).any()                # NaN -> code 0 (stored -128)
    assert q[:, 1].max() == 2 ** bits - 1 - 128                          # +inf saturates
    nhwc = AC.to_nhwc(q)
    assert nhwc.shape == (2, 6, 7, 32) and not nhwc[..., 19:].any()


# ---- chain_affine through the host twin ----------------------------------------------------------------------------------
def _qconv(cin, cout, k, lo, hi, groups=1, bits=8, padding=None, stride=1):
    from dfq_b200.utils import quantize as Q
    c = Q.QuantNConv2d(cin, cout, k, stride, k // 2 if padding is None else padding, groups=groups)
    with torch.no_grad():
        c.weight.copy_(torch.from_numpy(A.fake_quant_weights(c.weight.numpy(), 8)))
        c.bias.copy_(torch.randn(cout) * 0.1)
    c.quant.running_min.fill_(lo)
    c.quant.running_max.fill_(hi)
    c.quant.num_bits = bits
    return c


def _chain(monkeypatch, model, x, residual):
    """(chained module, fake): converts `model` with convert_affine, chains it, and checks that it computes what the
    per-layer model computes bit for bit and that the per-layer model is left as it was."""
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    fake = fakelib_int8_affine_chain.install(monkeypatch)
    model = model.eval()
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (Q.QuantNConv2d, Q.QuantNLinear)))
    int8.convert_affine(model, graph, [Q.QuantNConv2d, Q.QuantNLinear])
    layers = {n: m for n, m in model.named_modules() if isinstance(m, int8._AffineInt8Layer)}
    gm = int8.chain_affine(model, residual=residual)
    for n, m in model.named_modules():
        if isinstance(m, int8._AffineInt8Layer):
            assert layers[n] is m and not m.codes_in and m.epilogue is None and not m.sums, n
    for n, m in gm.named_modules():
        if isinstance(m, int8._AffineInt8Layer) and n in layers:
            assert m.weight_codes is layers[n].weight_codes and m.bias is layers[n].bias, n
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with torch.no_grad():
        fake.calls.clear()
        y = gm(x)
        calls = list(fake.calls)
        ref = model(x)
    assert y.dtype == torch.float32 and np.array_equal(y.numpy().view(np.int32), ref.numpy().view(np.int32))
    fused = [m for m in gm.modules() if isinstance(m, int8._AffineInt8Layer) and m.epilogue is not None]
    assert calls.count("dfq_i8_affine_conv_fused") == len(fused)
    codes_in = [m for m in gm.modules() if isinstance(m, int8._AffineInt8Layer) and m.codes_in]
    n_layers = sum(isinstance(m, int8._AffineInt8Layer) for m in gm.modules())
    assert calls.count("dfq_i8_affine_quantize") == n_layers - len(codes_in)
    return gm, fake


class _Line(nn.Module):
    """dense -> relu -> depthwise -> relu6 -> dense -> relu -> dense, then a Linear (opaque)."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a = _qconv(3, 16, 3, -2.5, 2.5)
        self.b = _qconv(16, 16, 3, 0.0, 4.0, groups=16)
        self.c = _qconv(16, 24, 1, 0.0, 6.0)
        self.d = _qconv(24, 8, 3, 0.0, 3.0)
        self.relu, self.relu6 = nn.ReLU(), nn.ReLU6()
        from dfq_b200.utils import quantize as Q
        self.fc = Q.QuantNLinear(8 * 25, 10)
        with torch.no_grad():
            self.fc.weight.copy_(torch.from_numpy(A.fake_quant_weights(self.fc.weight.numpy(), 8)))
        self.fc.quant.running_min.fill_(0.0)
        self.fc.quant.running_max.fill_(2.0)

    def forward(self, x):
        x = self.relu(self.d(self.relu(self.c(self.relu6(self.b(self.relu(self.a(x))))))))
        return self.fc(x.flatten(1))


@pytest.mark.parametrize("residual", [False, True])
def test_single_user_edges_carry_codes_and_sums_only_for_dense_consumers(monkeypatch, residual):
    gm, _ = _chain(monkeypatch, _Line(), torch.randn(2, 3, 5, 5) * 2, residual)
    assert gm.requantized_edges == [("a", "b", (0.0, INF)), ("b", "c", (0.0, 6.0)), ("c", "d", (0.0, INF))]
    assert (gm.a.sums, gm.b.sums, gm.c.sums) == (False, True, True)          # b is depthwise: it reads no S
    assert [gm.a.codes_in, gm.b.codes_in, gm.c.codes_in, gm.d.codes_in] == [False, True, True, True]
    assert gm.a.epilogue.out_scale == (0.0, 4.0, 8) and gm.c.epilogue.out_scale == (0.0, 3.0, 8)
    assert not any(m.fp32 for m in (gm.a.epilogue, gm.b.epilogue, gm.c.epilogue))
    assert gm.d.epilogue is None and type(gm.fc).__name__ == "AffineInt8Linear"      # the Linear stays opaque
    left = [n.name for n in gm.graph.nodes if n.op == "call_module" and n.target in ("relu", "relu6")]
    assert left == ["relu_2"]                                        # d -> relu -> the Linear stays in torch
    if residual:
        assert gm.fused_adds == []


class _FanOut(nn.Module):
    """a -> relu -> {b, c (b's range), d (another range), e (b's range at 7 bits), mean}"""

    def __init__(self, depthwise_first=False):
        super().__init__()
        torch.manual_seed(1)
        self.a = _qconv(3, 16, 3, -2.0, 2.0)
        self.b = _qconv(16, 16, 3, 0.0, 3.0, groups=16 if depthwise_first else 1)
        self.c = _qconv(16, 8, 1, 0.0, 3.0)
        self.d = _qconv(16, 8, 1, 0.0, 2.5)
        self.e = _qconv(16, 8, 1, 0.0, 3.0, bits=7)

    def forward(self, x):
        t = torch.relu(self.a(x))
        return self.b(t).sum() + self.c(t).sum() + self.d(t).sum() + self.e(t).sum() + t.mean()


@pytest.mark.parametrize("depthwise_first", [False, True])
def test_fan_out_by_range_key(monkeypatch, depthwise_first):
    """b and c read a's codes at their range; d (another range) and e (same range, 7 bits) and the mean take a's fp32
    output of the same launch.  S is written whenever a dense consumer takes the codes."""
    gm, _ = _chain(monkeypatch, _FanOut(depthwise_first), torch.randn(2, 3, 6, 6) * 2, True)
    assert gm.requantized_edges == [("a", "b", (0.0, INF)), ("a", "c", (0.0, INF))]
    assert gm.a.epilogue.out_scale == (0.0, 3.0, 8) and gm.a.epilogue.fp32 and gm.a.sums
    assert not gm.d.codes_in and not gm.e.codes_in and gm.b.codes_in and gm.c.codes_in
    assert gm.fused_adds == []
    gm, _ = _chain(monkeypatch, _FanOut(depthwise_first), torch.randn(2, 3, 6, 6) * 2, False)
    assert gm.requantized_edges == []                               # a has several users: no single-user edge


def test_fan_out_to_depthwise_consumers_only_writes_no_sums(monkeypatch):
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(2)
            self.a = _qconv(3, 16, 1, -2.0, 2.0)
            self.b = _qconv(16, 16, 3, 0.0, 3.0, groups=16)
            self.c = _qconv(16, 16, 5, 0.0, 3.0, groups=16)

        def forward(self, x):
            t = torch.relu(self.a(x))
            return self.b(t) + self.c(t)

    gm, _ = _chain(monkeypatch, M(), torch.randn(1, 3, 7, 7) * 2, True)
    assert [e[:2] for e in gm.requantized_edges] == [("a", "b"), ("a", "c")]
    assert not gm.a.sums and not gm.a.epilogue.fp32


class _Block(nn.Module):
    """ResNet's BasicBlock on affine layers: relu(conv2(relu(conv1(x))) + shortcut(x)), the shortcut a 1x1 downsample
    computed after conv2 (as torchvision does) or the identity; then a consumer of the sum."""

    def __init__(self, downsample):
        super().__init__()
        torch.manual_seed(3)
        self.stem = _qconv(3, 16, 3, -2.0, 2.0)
        self.conv1 = _qconv(16, 16, 3, 0.0, 3.0, stride=2 if downsample else 1)
        self.conv2 = _qconv(16, 16, 3, 0.0, 2.0)
        self.ds = _qconv(16, 16, 1, 0.0, 3.0, stride=2, padding=0) if downsample else None
        self.bn = nn.BatchNorm2d(16, eps=1e-10).eval()            # an identity BN, as merge_batchnorm leaves it
        self.head = _qconv(16, 8, 1, 0.0, 4.0)

    def forward(self, x):
        x = torch.relu(self.stem(x))
        out = self.bn(self.conv2(torch.relu(self.conv1(x))))
        sc = self.ds(x) if self.ds is not None else x
        return self.head(torch.relu(out + sc))


@pytest.mark.parametrize("downsample", [False, True])
def test_residual_add_fused_into_the_producer_with_downsample_ordering(monkeypatch, downsample):
    gm, _ = _chain(monkeypatch, _Block(downsample), torch.randn(2, 3, 8, 8) * 2, True)
    r = "ds" if downsample else "relu"
    (p, add, r_name, pre, post), = gm.fused_adds
    assert (p, r_name, pre, post) == ("conv2", r, NONE, (0.0, INF))
    assert ("conv2", "head", (0.0, INF)) in gm.requantized_edges and ("conv1", "conv2", (0.0, INF)) in gm.requantized_edges
    assert gm.conv2.epilogue.residual and gm.conv2.epilogue.out_scale == (0.0, 4.0, 8) and gm.conv2.sums
    assert not gm.conv2.epilogue.fp32
    order = [n.target for n in gm.graph.nodes if n.op == "call_module"]
    if downsample:
        assert order.index("ds") < order.index("conv2")             # the producer moved to the add's position
        assert ("stem", "conv1", (0.0, INF)) in gm.requantized_edges and ("stem", "ds", (0.0, INF)) in gm.requantized_edges
        assert gm.stem.epilogue.fp32 is False
    else:
        assert gm.stem.epilogue.fp32                                 # the identity shortcut is fp32


def test_residual_of_another_shape_is_refused_naming_the_layer(monkeypatch):
    from dfq_b200 import _lib, int8

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(4)
            self.a = _qconv(3, 16, 3, -2.0, 2.0)
            self.b = _qconv(16, 16, 3, 0.0, 3.0)

        def forward(self, x):
            t = torch.relu(self.a(x))
            return self.b(t) + t[:, :1]

    fakelib_int8_affine_chain.install(monkeypatch)
    model = M().eval()
    from dfq_b200.utils import quantize as Q
    int8.convert_affine(model, OrderedDict((id(m), m) for m in model.modules() if isinstance(m, Q.QuantNConv2d)),
                        [Q.QuantNConv2d])
    gm = int8.chain_affine(model, residual=True)
    assert len(gm.fused_adds) == 1
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(_lib.DfqError, match="layer b: the residual must be fp32"):
        gm(torch.randn(1, 3, 5, 5))


def test_ncnn_layers_stay_opaque(monkeypatch):
    """An Int8Conv2d between affine layers ends both chains: no edge crosses the two schemes."""
    import fakelib_int8
    from dfq_b200 import int8
    fakelib_int8_affine_chain.install(monkeypatch)
    torch.manual_seed(5)
    m = nn.Sequential(_qconv(3, 16, 3, -2.0, 2.0), nn.ReLU(), nn.Conv2d(16, 16, 3, padding=1), nn.ReLU(),
                      _qconv(16, 8, 3, 0.0, 3.0), nn.ReLU(), _qconv(8, 8, 1, 0.0, 2.0)).eval()
    from dfq_b200.utils import quantize as Q
    int8.convert_affine(m, OrderedDict((id(x), x) for x in m.modules() if isinstance(x, Q.QuantNConv2d)), [Q.QuantNConv2d])
    m[2] = int8.Int8Conv2d.from_conv(m[2], 30.0, [40.0] * 16)
    for residual in (False, True):
        gm = int8.chain_affine(m, residual=residual)
        assert gm.requantized_edges == [("4", "6", (0.0, INF))]
        assert getattr(gm, "2") is m[2]


def test_chained_refusals():
    """chained() refuses output ranges and bits the quantizer refuses and epilogues that return nothing."""
    from dfq_b200 import _lib, int8
    layer = int8._AffineInt8Layer.__new__(int8.AffineInt8Conv2d)
    nn.Module.__init__(layer)
    for k, v in dict(out_channels=4, in_channels=4, groups=1, kernel_size=(1, 1), stride=(1, 1), padding=(0, 0),
                     dilation=(1, 1), cpad=16, act_bits=8, w_bits=8, act_min=0.0, act_max=1.0, w_min=0.0, w_scale=1.0,
                     constants=None, layer_name="L").items():
        setattr(layer, k, v)
    for out, match in (((0.0, 1.0, 9), "9 bits"), ((0.0, 1.0, 0), "0 bits"), ((0.0, math.inf, 8), "output range"),
                       ((-3e38, 3e38, 1), "output range")):
        with pytest.raises(_lib.DfqError, match=match):
            layer.chained(requant=(out, 0.0, INF))
    with pytest.raises(_lib.DfqError, match="neither codes nor fp32"):
        layer.chained(epilogue=int8.Epilogue(None))
    with pytest.raises(_lib.DfqError, match="two output modes"):
        layer.chained(requant=((0.0, 1.0, 8), 0.0, INF), epilogue=int8.Epilogue(None, fp32=True))
    with pytest.raises(_lib.DfqError, match="pre-add"):
        layer.chained(requant=((0.0, 1.0, 8), 1.0, 0.0))
    new = layer.chained(epilogue=int8.Epilogue((f32(0.1), 1.0, 3), fp32=True), sums=True, codes_in=True)
    assert new.epilogue.out_scale == (float(f32(0.1)), 1.0, 3) and new.sums and new.codes_in and layer.epilogue is None
    assert not layer.chained(epilogue=int8.Epilogue(None, fp32=True), sums=True).sums     # no codes, no sums


def test_fake_library_refusals(monkeypatch):
    """The entry's refusals as the stand-in states them (the -m gpu tests check the library itself)."""
    from dfq_b200 import _lib, int8
    fake = fakelib_int8_affine_chain.install(monkeypatch)
    layer = int8.AffineInt8Conv2d.from_conv(_qconv(16, 8, 3, -1.0, 1.0), -1.0, 1.0)
    g = layer._geometry(1, 4, 4)
    xq, S = torch.zeros(16 * 16, dtype=torch.int8), torch.zeros(16, dtype=torch.int32)
    y, r = torch.zeros(128), torch.zeros(128)
    yq, S_out = torch.zeros(256, dtype=torch.int8), torch.zeros(16, dtype=torch.int32)

    def call(**kw):
        d = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
        e = dict(residual=0, y=y.data_ptr(), yq=yq.data_ptr(), S=S_out.data_ptr(), out_min=-1.0, out_max=1.0, out_bits=8,
                 pre_lo=-INF, pre_hi=INF, post_lo=-INF, post_hi=INF)
        e.update(kw)
        for k, v in e.items():
            d[0][k] = v
        return fake.dfq_i8_affine_conv_fused(xq.data_ptr(), S.data_ptr(), layer.weight_codes.data_ptr(),
                                             layer.tap_table.data_ptr(), layer.constants.ctypes.data, layer.bias.data_ptr(),
                                             d.ctypes.data, g.ctypes.data, None)

    assert call() == 0 and call(y=0) == 0 and call(yq=0, S=0) == 0 and call(S=0) == 0
    assert call(y=0, yq=0, S=0) == -1 and call(yq=0) == -1                   # nothing asked; S without yq
    assert call(out_bits=9) == -2 and call(out_bits=0) == -1 and call(out_max=math.nan) == -1
    assert call(out_min=-3e38, out_max=3e38, out_bits=1) == -1
    assert call(pre_lo=1.0, pre_hi=0.0) == -1 and call(post_hi=math.nan) == -1
    assert call(residual=y.data_ptr()) == -1 and call(S=yq.data_ptr()) == -1 and call(yq=yq.data_ptr() + 1) == -1
    assert call(residual=r.data_ptr()) == 0
