"""dfq_b200.int8.chain_int8(..., residual=True, pool_cat=True) on the CPU: which max pools and channel concatenations are
fused, and that the chained module computes what the per-layer one does - through the host twins of the library
(tests/int8_pool_cat_oracle.py), with torch told that CPU tensors are on the GPU."""
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_pool_cat_oracle as PO
from test_int8_chain_host import _identity_bns, _x
from test_int8_residual_host import _input_scales

INF = math.inf
NONE = (-INF, INF)


def _convert(model, acts):
    from dfq_b200 import int8
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    names = {id(m): n for n, m in model.named_modules()}
    int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=[acts[names[k]] for k in graph])


def _chain(monkeypatch, model, x, acts):
    """The chained module (residual=True, pool_cat=True) of `model` converted at `acts`, checked bit for bit against the
    per-layer model on x through the twins."""
    from dfq_b200 import int8
    fake = PO.install(monkeypatch)
    torch.manual_seed(0)
    model = model.eval()
    _convert(model, acts)
    gm = int8.chain_int8(model, residual=True, pool_cat=True)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with torch.no_grad():
        fake.calls.clear()
        y = gm(x)
        ref = model(x)
    assert y.dtype == torch.float32 and np.array_equal(y.numpy().view(np.int32), ref.numpy().view(np.int32))
    return gm, fake


class _Fire(nn.Module):
    """stem -> relu -> pool -> squeeze -> relu -> cat(e1 -> relu, e3 -> relu) -> pool -> z."""

    def __init__(self, e1=16, e3=24, pool=None, pool2=None):
        super().__init__()
        self.stem = nn.Conv2d(3, 16, 3, 1, 1)
        self.pool = pool or nn.MaxPool2d(3, 2, ceil_mode=True)
        self.squeeze = nn.Conv2d(16, 8, 1)
        self.e1, self.e3 = nn.Conv2d(8, e1, 1), nn.Conv2d(8, e3, 3, 1, 1)
        self.pool2 = pool2 or nn.MaxPool2d(2, 1, padding=1, dilation=2)
        self.z = nn.Conv2d(e1 + e3, 8, 1)

    def cat(self, s):
        return torch.cat([F.relu(self.e1(s)), F.relu(self.e3(s))], 1)

    def forward(self, x):
        s = F.relu(self.squeeze(self.pool(F.relu(self.stem(x)))))
        return self.z(self.pool2(self.cat(s))).mean((2, 3))


ACTS = {"stem": 7.0, "squeeze": 3.0, "e1": 5.0, "e3": 5.0, "z": 2.0, "z2": 2.0}


def test_pools_and_cat_fuse_and_run_bit_identically(monkeypatch):
    gm, fake = _chain(monkeypatch, _Fire(), _x(), ACTS)
    assert [c[0] for c in gm.fused_cats] == ["cat"] and gm.fused_cats[0][1:] == (["e1", "e3"], [0, 16])
    assert [(p[0], p[1]) for p in gm.fused_pools] == [("pool", "codes"), ("pool2", "codes")]
    assert {q for _, q, _ in gm.requantized_edges} == {"squeeze", "e1", "e3", "z"}
    assert gm.get_submodule("e1").out_slice == (0, 48) and gm.get_submodule("e3").out_slice == (16, 48)
    assert gm.get_submodule("e3").requant == (2.0, 0.0, INF)
    assert not any(n.op == "call_function" and n.target is torch.cat for n in gm.graph.nodes)
    assert fake.calls.count("dfq_i8_conv_slice") == 2 and fake.calls.count("dfq_i8_maxpool") == 2


def test_functional_pool_and_identity_after_a_pool(monkeypatch):
    class M(_Fire):
        def __init__(self):
            super().__init__()
            self.drop = nn.Dropout()

        def forward(self, x):
            t = F.max_pool2d(F.relu(self.stem(x)), 3, 2, 1, 1, True)
            s = F.relu(self.squeeze(self.drop(t)))
            return self.z(self.cat(s)).mean((2, 3))
    gm, _ = _chain(monkeypatch, M(), _x(), ACTS)
    assert [p[:2] for p in gm.fused_pools] == [("max_pool2d", "codes")]
    assert not any(n.op == "call_module" and n.target == "drop" for n in gm.graph.nodes)


@pytest.mark.parametrize("what", ["operand_40", "second_user", "dim2", "fp32_user", "scale_ulp"])
def test_cats_that_stay_fp32(monkeypatch, what):
    acts = dict(ACTS)
    if what == "operand_40":
        model = _Fire(e1=40)
    elif what == "scale_ulp":
        class M(_Fire):
            def __init__(self):
                super().__init__()
                self.z2 = nn.Conv2d(40, 8, 1)

            def forward(self, x):
                c = self.cat(F.relu(self.squeeze(F.relu(self.stem(x)))))
                return self.z(c).mean((2, 3)) + self.z2(c).mean((2, 3))
        model = M()
        acts["z2"] = float(np.nextafter(np.float32(2.0), np.float32(9)))
    else:
        acts["z2"] = 2.0
        class M(_Fire):
            def __init__(self):
                super().__init__(e3=24 if what != "dim2" else 16)
                self.z2 = nn.Conv2d(16, 8, 1)

            def forward(self, x):
                s = F.relu(self.squeeze(F.relu(self.stem(x))))
                a, b = F.relu(self.e1(s)), F.relu(self.e3(s))
                if what == "second_user":
                    return self.z(torch.cat([a, b], 1)).mean((2, 3)) + a.mean()
                if what == "dim2":
                    return self.z2(torch.cat([a, b], 2)).mean((2, 3))
                c = torch.cat([a, b], 1)
                return self.z(c).mean((2, 3)) + c.mean()
        model = M()
    gm, _ = _chain(monkeypatch, model, _x(), acts)
    assert gm.fused_cats == []


@pytest.mark.parametrize("what", ["avg", "clamp_after", "fp32_user_of_a_fan_out"])
def test_pools_that_stay_fp32(monkeypatch, what):
    acts = dict(ACTS)
    if what == "avg":
        model = _Fire(pool=nn.AvgPool2d(2))
    else:
        class M(_Fire):
            def __init__(self):
                super().__init__(e3=24 if what != "dim2" else 16)
                self.z2 = nn.Conv2d(16, 8, 1)

            def forward(self, x):
                t = self.pool(F.relu(self.stem(x)))
                if what == "clamp_after":
                    t = F.relu(t)
                out = self.z(self.cat(F.relu(self.squeeze(t)))).mean((2, 3))
                if what == "fp32_user_of_a_fan_out":
                    out = out + self.stem(x).mean() * 0
                return out
        model = M()
    gm, _ = _chain(monkeypatch, model, _x(), acts)
    assert "pool" not in [p[0] for p in gm.fused_pools]


def test_pool_node_predicate():
    import torch.fx as fx
    from dfq_b200 import int8
    m = nn.Sequential(nn.MaxPool2d(2, return_indices=True))
    g = fx.symbolic_trace(m).graph
    mods = dict(m.named_modules())
    assert all(int8._max_pool(n, mods) is None for n in g.nodes if n.op == "call_module")

    class P(nn.Module):
        def forward(self, x):
            return F.max_pool2d(x, 2, return_indices=True)[0] + F.max_pool2d(x, 2) + F.avg_pool2d(x, 2)
    g = fx.symbolic_trace(P()).graph
    hits = [n for n in g.nodes if n.op == "call_function" and int8._max_pool(n, {}) is not None]
    assert len(hits) == 1 and hits[0].kwargs["return_indices"] is False


def test_resnet_style_stem_pools_in_fp32_mode(monkeypatch):
    """conv -> relu -> maxpool -> {conv a, residual of a's block}: the producer writes fp32, the pool fp32 for the add and
    codes for a."""
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem, self.pool = nn.Conv2d(3, 16, 3, 2, 1), nn.MaxPool2d(3, 2, 1)
            self.a, self.b, self.z = nn.Conv2d(16, 16, 3, 1, 1), nn.Conv2d(16, 16, 3, 1, 1), nn.Conv2d(16, 8, 1)

        def forward(self, x):
            t = self.pool(F.relu(self.stem(x)))
            return self.z(F.relu(self.b(F.relu(self.a(t))) + t)).mean((2, 3))
    gm, _ = _chain(monkeypatch, M(), _x(), {"stem": 7.0, "a": 3.0, "b": 4.0, "z": 2.0})
    assert gm.fused_pools == [("pool", "fp32", ("fp32", "codes"))]
    assert ("pool", "a", (0.0, INF)) in gm.requantized_edges
    assert gm.get_submodule("stem").epilogue == (None, (0.0, INF), NONE, False, True)
    assert [a[:3] for a in gm.fused_adds] == [("b", "add", "pool")]


def test_fp32_pool_whose_codes_consumer_adds_the_pool_as_its_residual(monkeypatch):
    """conv -> relu -> maxpool -> {b, residual of b's own add}: b reads the pool's codes and adds its fp32 output.  Only
    b's input may become the codes: its residual, the same pool node, stays the pool's fp32 output."""
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem, self.pool = nn.Conv2d(3, 16, 3, 1, 1), nn.MaxPool2d(2, 2)
            self.b, self.z = nn.Conv2d(16, 16, 3, 1, 1), nn.Conv2d(16, 8, 1)

        def forward(self, x):
            t = self.pool(F.relu(self.stem(x)))
            return self.z(torch.relu(F.relu6(self.b(t)) + t))
    gm, _ = _chain(monkeypatch, M(), _x(), {"stem": 7.0, "b": 3.0, "z": 2.0})
    assert gm.fused_pools == [("pool", "fp32", ("fp32", "codes"))]
    assert ("pool", "b", (0.0, INF)) in gm.requantized_edges
    assert [a[:3] for a in gm.fused_adds] == [("b", "add", "pool")]


def test_pool_cat_needs_residual():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="pool_cat=True builds on residual=True"):
        int8.chain_int8(_Fire(), pool_cat=True)


# ---- torchvision ----------------------------------------------------------------------------------------------------------
def _scales_through_pools(model):
    """_input_scales with a pool's users given the scale of the pool's input."""
    import torch.fx as fx
    from dfq_b200 import int8
    g = int8._Int8Tracer().trace(model)
    mods = dict(model.named_modules())
    rng, by_input, acts = np.random.default_rng(0), {}, {}
    for n in g.nodes:
        if n.op == "call_module" and isinstance(mods[n.target], (nn.Conv2d, nn.Linear)):
            src = n.args[0]
            while isinstance(src, fx.Node) and (int8._max_pool(src, mods) is not None or (
                    src.op == "call_module" and type(mods[src.target]) in (nn.BatchNorm2d, nn.Dropout))):
                src = src.args[0]
            acts[n.target] = by_input.setdefault(src, float(rng.uniform(4.0, 40.0)))
    return acts


@pytest.mark.parametrize("net, carried, convs, cats, pools, pool_mode", [
    ("squeezenet1_1", 25, 26, (8, 8), (3, 3), "codes"),
    ("googlenet", 56, 57, (8, 9), (13, 13), "codes"),
    ("resnet18", 19, 20, (0, 0), (1, 1), "fp32"),
])
def test_torchvision_counts(monkeypatch, net, carried, convs, cats, pools, pool_mode):
    import torchvision
    from dfq_b200 import int8
    PO.install(monkeypatch)
    torch.manual_seed(0)
    kw = dict(aux_logits=False, init_weights=True) if net == "googlenet" else {}
    model = _identity_bns(getattr(torchvision.models, net)(num_classes=10, **kw)).eval()
    _convert(model, _scales_through_pools(model))
    gm = int8.chain_int8(model, residual=True, pool_cat=True)
    all_convs = [n for n, m in model.named_modules() if isinstance(m, int8.Int8Conv2d)]
    got = {q for _, q, _ in gm.requantized_edges}
    assert (len(got), len(all_convs)) == (carried, convs)
    assert len(gm.fused_cats) == cats[0] and len(gm.fused_pools) == pools[0]
    assert {p[1] for p in gm.fused_pools} == {pool_mode}
    if net == "resnet18":
        base = int8.chain_int8(model, residual=True)
        assert got == {q for _, q, _ in base.requantized_edges} | {"layer1.0.conv1"}
        assert gm.fused_adds == base.fused_adds


def test_mobilenet_v2_is_what_residual_gives(monkeypatch):
    import torchvision
    from dfq_b200 import int8
    PO.install(monkeypatch)
    torch.manual_seed(0)
    model = _identity_bns(torchvision.models.mobilenet_v2(num_classes=10)).eval()
    _convert(model, _input_scales(model))
    a, b = int8.chain_int8(model, residual=True), int8.chain_int8(model, residual=True, pool_cat=True)
    assert a.requantized_edges == b.requantized_edges and a.fused_adds == b.fused_adds
    assert b.fused_cats == [] and b.fused_pools == []
    assert str(a.graph) == str(b.graph)


def test_small_squeezenet_forward_through_the_twins(monkeypatch):
    """torchvision's SqueezeNet 1.1 at 48x48, identity BNs: bit-identical to the per-layer model through the twins."""
    import torchvision
    model = torchvision.models.squeezenet1_1(num_classes=10)
    acts = _scales_through_pools(model)
    gm, fake = _chain(monkeypatch, model, torch.randn(1, 3, 48, 48), acts)
    assert len(gm.fused_cats) == 8 and fake.calls.count("dfq_i8_conv_slice") == 16
