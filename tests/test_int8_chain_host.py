"""dfq_b200.int8.chain_int8 on the CPU: which edges between converted convolutions are fused, the clamp each one carries, and
that the chained module computes what the per-layer one does - through the host twins of the library
(tests/int8_chain_oracle.py), with torch told that CPU tensors are on the GPU."""
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_chain_oracle as CO

INF = math.inf


def _identity_bn(c):
    """A BatchNorm2d as merge_batchnorm leaves it: eval, weight 1, bias 0, mean 0, var 1, fp32(1 + eps) == 1."""
    from dfq_b200.utils.layer_transform import _identity_bn_eps
    bn = nn.BatchNorm2d(c, eps=_identity_bn_eps()).eval()
    return bn


def _convert(model, seed=0):
    """convert_to_int8 on every Conv2d / Linear with made-up activation scales; returns the converted names."""
    from dfq_b200 import int8
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    acts = np.random.default_rng(seed).uniform(4.0, 40.0, len(graph)).tolist()
    return int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=acts)


def _chain(monkeypatch, model, x=None):
    """(chained module, fused edges); with an input x, also checks that it computes model(x) bit for bit and that model
    itself is unchanged."""
    from dfq_b200 import int8
    fake = CO.install(monkeypatch)
    torch.manual_seed(0)
    model = model.eval()
    _convert(model)
    layers = {n: m for n, m in model.named_modules() if isinstance(m, int8._Int8Layer)}
    gm = int8.chain_int8(model)
    for n, m in model.named_modules():
        if isinstance(m, int8._Int8Layer):
            assert layers[n] is m and not m.codes_in and m.requant is None, n
    if x is not None:
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        with torch.no_grad():
            fake.calls.clear()
            y = gm(x)
            assert fake.calls.count("dfq_i8_conv_requant") == len(gm.requantized_edges)
            ref = model(x)
        assert y.dtype == torch.float32 and np.array_equal(y.numpy().view(np.int32), ref.numpy().view(np.int32))
    return gm, gm.requantized_edges


class _Two(nn.Module):
    """conv a -> `mid` (a function of the tensor) -> conv b"""

    def __init__(self, mid, cin=3, c=24, cout=8, b_groups=1):
        super().__init__()
        self.a = nn.Conv2d(cin, c, 3, 1, 1)
        self.b = nn.Conv2d(c, cout if b_groups == 1 else c, 3, 2, 1, groups=b_groups)
        self.mid = mid

    def forward(self, x):
        return self.b(self.mid(self.a(x)))


def _x(c=3):
    return torch.randn(2, c, 9, 11, generator=torch.Generator().manual_seed(1)) * 2


# ---- the fusion rule, one case per item -------------------------------------------------------------------------------
def test_conv_relu_conv(monkeypatch):
    _, edges = _chain(monkeypatch, nn.Sequential(nn.Conv2d(3, 24, 3, 1, 1), nn.ReLU(), nn.Conv2d(24, 8, 1)), _x())
    assert edges == [("0", "2", (0.0, INF))]


def test_conv_conv_and_depthwise_consumer(monkeypatch):
    m = nn.Sequential(nn.Conv2d(3, 24, 3, 1, 1), nn.Conv2d(24, 24, 3, 1, 1, groups=24), nn.Conv2d(24, 5, 1))
    _, edges = _chain(monkeypatch, m, _x())
    assert edges == [("0", "1", (-INF, INF)), ("1", "2", (-INF, INF))]


def test_identity_bn_then_relu6(monkeypatch):
    m = nn.Sequential(nn.Conv2d(3, 24, 3, 1, 1), _identity_bn(24), nn.ReLU6(inplace=True), nn.Conv2d(24, 8, 1))
    gm, edges = _chain(monkeypatch, m, _x())
    assert edges == [("0", "3", (0.0, 6.0))]
    assert not any(n.op == "call_module" and n.target in ("1", "2") for n in gm.graph.nodes)


@pytest.mark.parametrize("fn, clamp", [(F.relu, (0.0, INF)), (torch.relu, (0.0, INF)), (lambda t: t.relu(), (0.0, INF)),
                                       (F.relu6, (0.0, 6.0)), (lambda t: F.hardtanh(t, -1.0, 2.5), (-1.0, 2.5)),
                                       (nn.Hardtanh(-1.0, 2.5), (-1.0, 2.5)), (nn.Identity(), (-INF, INF))],
                         ids=["F.relu", "torch.relu", "method_relu", "F.relu6", "F.hardtanh", "nn.Hardtanh", "nn.Identity"])
def test_functional_and_method_activations(monkeypatch, fn, clamp):
    class M(_Two):
        def forward(self, x):
            return self.b(fn(self.a(x)))
    m = M(None)
    if isinstance(fn, nn.Module):
        m.mid = fn
        m.forward = _Two.forward.__get__(m)
    _, edges = _chain(monkeypatch, m, _x())
    assert edges == [("a", "b", clamp)]


def test_nested_clamps_compose(monkeypatch):
    class M(_Two):
        def forward(self, x):
            return self.b(F.relu(nn.functional.relu6(F.hardtanh(self.a(x), -1.0, 2.5))))
    _, edges = _chain(monkeypatch, M(None), _x())
    assert edges == [("a", "b", (0.0, 2.5))]

    class Disjoint(_Two):                                       # clamp(clamp(v, -3, -1), 0, inf) is 0 everywhere
        def forward(self, x):
            return self.b(F.relu(F.hardtanh(self.a(x), -3.0, -1.0)))
    _, edges = _chain(monkeypatch, Disjoint(None), _x())
    assert edges == [("a", "b", (0.0, 0.0))]


def test_dropout_in_eval_fuses_and_in_training_does_not(monkeypatch):
    m = _Two(nn.Sequential(nn.Dropout(0.3), nn.ReLU()))
    _, edges = _chain(monkeypatch, m, _x())
    assert edges == [("a", "b", (0.0, INF))]
    m = _Two(nn.Sequential(nn.Dropout(0.3), nn.ReLU()))
    CO.install(monkeypatch)
    _convert(m.eval())
    m.mid[0].train()
    from dfq_b200 import int8
    assert int8.chain_int8(m).requantized_edges == []


def test_the_consumer_takes_the_requantized_codes_of_the_next_scale(monkeypatch):
    """The producer's output is the consumer's codes: i8_requantize of the producer's sums at the consumer's act_scale."""
    from dfq_b200 import _lib
    gm, _ = _chain(monkeypatch, nn.Sequential(nn.Conv2d(3, 20, 3, 1, 1), nn.ReLU6(), nn.Conv2d(20, 8, 1)))
    p, q = gm.get_submodule("0"), gm.get_submodule("2")
    assert p.requant == (q.act_scale, 0.0, 6.0) and q.codes_in and not p.codes_in and q.requant is None
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    x = _x()
    yq, none = p.run(x)
    assert none is None and yq.dtype == torch.int8 and tuple(yq.shape) == (2, 9, 11, 32)
    plain = p.chained()                                         # the same buffers, fp32 out
    _, acc = plain.run(x, with_acc=True)
    ref = CO.i8_requantize(acc.numpy(), p.act_scale, p.w_scale.numpy(), p.bias.numpy(), q.act_scale, 0.0, 6.0)
    assert np.array_equal(yq.numpy(), CO.to_nhwc_codes(ref))
    with pytest.raises(_lib.DfqError, match="int32 sums"):
        p.run(x, with_acc=True)
    with pytest.raises(_lib.DfqError, match="int8 codes"):
        q.run(x)
    with pytest.raises(_lib.DfqError, match="expects fp32"):
        plain.run(yq)


# ---- what must not fuse ---------------------------------------------------------------------------------------------
def test_non_identity_or_training_batchnorm_is_not_fused(monkeypatch):
    bn = _identity_bn(24)
    with torch.no_grad():
        bn.weight[3] = 2.0
    _, edges = _chain(monkeypatch, _Two(nn.Sequential(bn, nn.ReLU())), _x())
    assert edges == []
    _, edges = _chain(monkeypatch, _Two(nn.Sequential(nn.BatchNorm2d(24).eval(), nn.ReLU())), _x())   # eps 1e-5
    assert edges == []
    m = _Two(nn.Sequential(_identity_bn(24), nn.ReLU()))
    CO.install(monkeypatch)
    _convert(m.eval())
    m.mid[0].train()
    from dfq_b200 import int8
    assert int8.chain_int8(m).requantized_edges == []


def test_second_user_is_not_fused(monkeypatch):
    class M(_Two):
        def forward(self, x):
            r = F.relu(self.a(x))
            return self.b(r) + r.mean()
    _, edges = _chain(monkeypatch, M(None, b_groups=24), _x())
    assert edges == []

    class Producer(_Two):                                       # the producer's output itself used twice
        def forward(self, x):
            y = self.a(x)
            return self.b(y) + y.sum()
    _, edges = _chain(monkeypatch, Producer(None), _x())
    assert edges == []


def test_maxpool_in_between_is_not_fused(monkeypatch):
    _, edges = _chain(monkeypatch, _Two(nn.Sequential(nn.ReLU(), nn.MaxPool2d(2))), _x())
    assert edges == []


def test_linear_consumer_is_not_fused(monkeypatch):
    m = nn.Sequential(nn.Conv2d(4, 8, 1), nn.ReLU(), nn.Linear(16, 3))
    x = torch.randn(1, 4, 5, 16, generator=torch.Generator().manual_seed(2))
    _, edges = _chain(monkeypatch, m, x)
    assert edges == []


# ---- other host-side checks -----------------------------------------------------------------------------------------
class _Block(nn.Module):
    """torchvision's BasicBlock pattern: one self.relu called after bn1 and again after the residual add."""

    def __init__(self, c=16):
        super().__init__()
        self.conv1, self.bn1 = nn.Conv2d(c, c, 3, 1, 1), _identity_bn(c)
        self.conv2, self.bn2 = nn.Conv2d(c, c, 3, 1, 1), _identity_bn(c)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return self.relu(out + x)


def test_shared_relu_module_loses_only_the_call_between_the_convolutions(monkeypatch):
    gm, edges = _chain(monkeypatch, _Block(), _x(16))
    assert edges == [("conv1", "conv2", (0.0, INF))]
    relus = [n for n in gm.graph.nodes if n.op == "call_module" and n.target == "relu"]
    assert len(relus) == 1 and relus[0].args[0].target is __import__("operator").add
    assert isinstance(gm.relu, nn.ReLU)


def test_a_model_without_a_qualifying_edge_computes_the_same(monkeypatch):
    gm, edges = _chain(monkeypatch, nn.Sequential(nn.Conv2d(3, 8, 3), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(128, 4)),
                       torch.randn(2, 3, 10, 10, generator=torch.Generator().manual_seed(3)))
    assert edges == []


def _identity_bns(model):
    from dfq_b200.utils.layer_transform import _identity_bn_eps
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.fill_(1); m.bias.fill_(0); m.running_mean.fill_(0); m.running_var.fill_(1)
                m.eps = _identity_bn_eps()
    return model.eval()


@pytest.mark.parametrize("net, relu6, fused", [("mobilenet_v2", True, 36), ("mobilenet_v2", False, 36), ("resnet18", True, 8)],
                         ids=["mobilenet_v2", "mobilenet_v2_relu", "resnet18"])
def test_torchvision_edge_counts(monkeypatch, net, relu6, fused):
    """BN folded to the identity (what merge_batchnorm leaves): MobileNetV2 fuses 36 of its 52 convolution inputs, ResNet-18
    the conv1 -> conv2 edge of each of its 8 basic blocks.  Tracing only, no forward."""
    import torchvision
    from dfq_b200 import int8
    CO.install(monkeypatch)
    torch.manual_seed(0)
    model = _identity_bns(getattr(torchvision.models, net)(num_classes=10))
    if not relu6:
        for m in model.modules():
            for k, c in m.named_children():
                if isinstance(c, nn.ReLU6):
                    setattr(m, k, nn.ReLU())
    _convert(model)
    gm = int8.chain_int8(model)
    assert len(gm.requantized_edges) == fused
    clamps = {c for _, _, c in gm.requantized_edges}
    if net == "resnet18":
        assert clamps == {(0.0, INF)}
        assert [(p, q) for p, q, _ in gm.requantized_edges] == [("layer%d.%d.conv1" % (i, j), "layer%d.%d.conv2" % (i, j))
                                                                 for i in range(1, 5) for j in range(2)]
    else:                                                       # the linear bottlenecks carry no clamp
        assert clamps == {(0.0, 6.0 if relu6 else INF), (-INF, INF)}
