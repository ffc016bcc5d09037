"""dfq_b200.int8.chain_int8(..., residual=True) on the CPU: which fan-out edges and residual adds are fused, the clamps and
scales they carry, and that the chained module computes what the per-layer one does - through the host twins of the library
(tests/int8_residual_oracle.py), with torch told that CPU tensors are on the GPU."""
import math
import operator

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_residual_oracle as RO
from test_int8_chain_host import _convert, _identity_bn, _identity_bns, _x

INF = math.inf
NONE = (-INF, INF)


def _chain(monkeypatch, model, x, acts=None):
    """(chained module, edges, fused adds): converts `model` (act_scales `acts` by layer name, else made-up ones), chains it
    with residual=True and checks that it computes model(x) bit for bit and that model itself is unchanged."""
    from dfq_b200 import int8
    fake = RO.install(monkeypatch)
    torch.manual_seed(0)
    model = model.eval()
    if acts is None:
        _convert(model)
    else:
        from collections import OrderedDict
        graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
        names = {id(m): n for n, m in model.named_modules()}
        int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=[acts[names[k]] for k in graph])
    layers = {n: m for n, m in model.named_modules() if isinstance(m, int8._Int8Layer)}
    gm = int8.chain_int8(model, residual=True)
    for n, m in model.named_modules():
        if isinstance(m, int8._Int8Layer):
            assert layers[n] is m and not m.codes_in and m.requant is None and m.epilogue is None, n
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with torch.no_grad():
        fake.calls.clear()
        y = gm(x)
        ref = model(x)
    assert y.dtype == torch.float32 and np.array_equal(y.numpy().view(np.int32), ref.numpy().view(np.int32))
    fused = [m for m in gm.modules() if isinstance(m, int8._Int8Layer) and m.epilogue is not None]
    assert fake.calls.count("dfq_i8_conv_fused") == len(fused)
    return gm, gm.requantized_edges, gm.fused_adds


def _calls(gm, op):
    return [n for n in gm.graph.nodes if n.op == "call_function" and n.target is op]


# ---- fan-out ------------------------------------------------------------------------------------------------------------
class _FanOut(nn.Module):
    """conv a -> relu -> {conv b, conv c, mean}: b and c take codes at one scale, the mean takes a's fp32 output."""

    def __init__(self):
        super().__init__()
        self.a = nn.Conv2d(3, 24, 3, 1, 1)
        self.b = nn.Conv2d(24, 8, 1)
        self.c = nn.Conv2d(24, 24, 3, 2, 1, groups=24)

    def forward(self, x):
        t = F.relu(self.a(x))
        return self.b(t).sum() + self.c(t).sum() + t.mean()


def test_fan_out_takes_codes_and_fp32_from_one_launch(monkeypatch):
    gm, edges, adds = _chain(monkeypatch, _FanOut(), _x(), acts=dict(a=9.0, b=5.0, c=5.0))
    assert edges == [("a", "b", (0.0, INF)), ("a", "c", (0.0, INF))] and adds == []
    a = gm.get_submodule("a")
    assert a.epilogue == (5.0, (0.0, INF), NONE, False, True) and a.requant is None
    assert gm.get_submodule("b").codes_in and gm.get_submodule("c").codes_in
    assert not any(n.op == "call_function" and n.target is F.relu for n in gm.graph.nodes)
    assert len(_calls(gm, operator.getitem)) == 2


def test_fan_out_consumer_at_another_scale_takes_fp32(monkeypatch):
    gm, edges, _ = _chain(monkeypatch, _FanOut(), _x(), acts=dict(a=9.0, b=5.0, c=np.nextafter(np.float32(5.0), 9)))
    assert edges == [("a", "b", (0.0, INF))]
    assert not gm.get_submodule("c").codes_in


def test_fan_out_of_convolutions_only_requantizes(monkeypatch):
    class M(_FanOut):
        def forward(self, x):
            t = self.a(x)
            return self.b(t).sum() + self.c(t).sum()
    gm, edges, _ = _chain(monkeypatch, M(), _x(), acts=dict(a=9.0, b=5.0, c=5.0))
    assert edges == [("a", "b", NONE), ("a", "c", NONE)]
    assert gm.get_submodule("a").requant == (5.0, -INF, INF) and gm.get_submodule("a").epilogue is None


# ---- residual adds ------------------------------------------------------------------------------------------------------
class _Inverted(nn.Module):
    """MobileNetV2's pattern: x = conv p (fan-out); out = x + q(relu(e(x))) with clamps before and after the add; then
    conv z."""

    def __init__(self, pre=nn.Identity(), post=nn.Identity(), c=24):
        super().__init__()
        self.p = nn.Conv2d(3, c, 3, 1, 1)
        self.e = nn.Conv2d(c, 2 * c, 1)
        self.q = nn.Conv2d(2 * c, c, 1)
        self.z = nn.Conv2d(c, 8, 1)
        self.pre, self.post = pre, post

    def forward(self, x):
        x = self.p(x)
        out = x + self.pre(self.q(F.relu6(self.e(x))))
        return self.z(self.post(out))


def test_x_plus_conv_of_x_where_x_is_a_fan_out(monkeypatch):
    gm, edges, adds = _chain(monkeypatch, _Inverted(), _x())
    assert edges == [("p", "e", NONE), ("e", "q", (0.0, 6.0)), ("q", "z", NONE)]
    assert adds == [("q", "add", "p", NONE, NONE)]
    assert gm.get_submodule("p").epilogue == (gm.get_submodule("e").act_scale, NONE, NONE, False, True)
    assert gm.get_submodule("q").epilogue == (gm.get_submodule("z").act_scale, NONE, NONE, True, False)
    assert not _calls(gm, operator.add)


def test_add_with_pre_and_post_clamps(monkeypatch):
    gm, edges, adds = _chain(monkeypatch, _Inverted(pre=nn.Sequential(_identity_bn(24), nn.Hardtanh(-1.0, 2.5)),
                                                    post=nn.Sequential(nn.ReLU(), nn.ReLU6())), _x())
    assert adds == [("q", "add", "p", (-1.0, 2.5), (0.0, 6.0))]
    assert edges[-1] == ("q", "z", (0.0, 6.0))


class _Basic(nn.Module):
    """torchvision's BasicBlock with a downsample branch, computed after conv2 in graph order; identity BNs."""

    def __init__(self, c=16):
        super().__init__()
        self.stem = nn.Conv2d(3, c, 3, 1, 1)
        self.conv1, self.bn1 = nn.Conv2d(c, 2 * c, 3, 2, 1), _identity_bn(2 * c)
        self.conv2, self.bn2 = nn.Conv2d(2 * c, 2 * c, 3, 1, 1), _identity_bn(2 * c)
        self.downsample = nn.Sequential(nn.Conv2d(c, 2 * c, 1, 2), _identity_bn(2 * c))
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        x = self.relu(self.stem(x))
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        identity = self.downsample(x)
        out += identity
        return self.relu(out).mean((2, 3))


def test_residual_through_identity_bn_and_node_moved_past_a_later_branch(monkeypatch):
    gm, edges, adds = _chain(monkeypatch, _Basic(), _x(), acts={"stem": 7.0, "conv1": 3.0, "downsample.0": 3.0, "conv2": 4.0})
    assert edges == [("stem", "conv1", (0.0, INF)), ("stem", "downsample.0", (0.0, INF)), ("conv1", "conv2", (0.0, INF))]
    assert adds == [("conv2", "add", "downsample_0", NONE, (0.0, INF))]
    nodes = list(gm.graph.nodes)
    pos = {n.target: i for i, n in enumerate(nodes) if n.op == "call_module"}
    assert pos["downsample.0"] < pos["conv2"]
    assert "downsample.1" not in pos and "bn2" not in pos
    conv2 = nodes[pos["conv2"]]
    assert conv2.args[1] is nodes[pos["downsample.0"]]


def test_residual_keeps_a_clamp_on_its_operand_in_torch(monkeypatch):
    class M(_Inverted):
        def forward(self, x):
            x = self.p(x)
            return self.z(F.relu(x) + self.q(F.relu6(self.e(x))))
    gm, edges, adds = _chain(monkeypatch, M(), _x())
    assert adds == [("q", "add", "relu", NONE, NONE)]
    assert len([n for n in gm.graph.nodes if n.op == "call_function" and n.target is F.relu]) == 1


# ---- what must not fuse -------------------------------------------------------------------------------------------------
def test_x_plus_x_and_alpha_are_not_fused(monkeypatch):
    class Twice(_Inverted):
        def forward(self, x):
            y = self.q(self.e(self.p(x)))
            return self.z(y + y)
    gm, _, adds = _chain(monkeypatch, Twice(), _x())
    assert adds == [] and len(_calls(gm, operator.add)) == 1

    class Alpha(_Inverted):
        def forward(self, x):
            x = self.p(x)
            return self.z(torch.add(x, self.q(self.e(x)), alpha=2.0))
    gm, _, adds = _chain(monkeypatch, Alpha(), _x())
    assert adds == [] and len(_calls(gm, torch.add)) == 1


def test_clamp_with_a_second_user_on_the_fused_operand_is_not_fused(monkeypatch):
    class M(_Inverted):
        def forward(self, x):
            x = self.p(x)
            t = F.relu(self.q(self.e(x)))
            return self.z(x + t) * t.mean()
    gm, edges, adds = _chain(monkeypatch, M(), _x())
    assert adds == [] and ("q", "z", (0.0, INF)) not in edges and len(_calls(gm, operator.add)) == 1


def test_multi_site_layer_is_not_fused(monkeypatch):
    class M(_Inverted):
        def forward(self, x):
            x = self.p(x)
            return self.z(x + self.q(self.e(x))) + self.z(x).mean()
    gm, edges, adds = _chain(monkeypatch, M(), _x())
    assert adds == [("q", "add", "p", NONE, NONE)]
    assert all("z" not in (p, q) for p, q, _ in edges)


def test_non_identity_bn_is_not_fused(monkeypatch):
    bn = _identity_bn(24)
    with torch.no_grad():
        bn.bias[2] = 0.5
    gm, edges, adds = _chain(monkeypatch, _Inverted(pre=bn), _x())
    assert adds == [] and ("q", "z", NONE) not in edges


def test_residual_of_another_shape_is_refused_naming_the_layer(monkeypatch):
    from dfq_b200 import _lib, int8
    gm, _, _ = _chain(monkeypatch, _Inverted(), _x())
    q = gm.get_submodule("q")
    assert q.codes_in and q.layer_name == "q"
    q = q.chained(epilogue=q.epilogue, name="q")                # fp32 in
    x = torch.zeros(2, 48, 9, 11)
    with pytest.raises(_lib.DfqError, match=r"layer q: the residual must be fp32 \[2, 24, 9, 11\] on cpu"):
        q.run(x, residual=torch.zeros(2, 24, 1, 1))
    with pytest.raises(_lib.DfqError, match="layer q: the residual must be fp32 .* on cpu, got torch.float32 .* on meta"):
        q.run(x, residual=torch.zeros(2, 24, 9, 11, device="meta"))        # another device than the input's
    with pytest.raises(_lib.DfqError, match="layer q: the residual must be fp32"):
        q.run(x, residual=torch.zeros(2, 24, 9, 11, dtype=torch.float64))
    with pytest.raises(_lib.DfqError, match="takes a residual input"):
        q.run(x)
    with pytest.raises(_lib.DfqError, match="neither codes nor fp32"):
        q.chained(epilogue=int8.Epilogue())
    with pytest.raises(_lib.DfqError, match="post-add bounds"):
        q.chained(epilogue=int8.Epilogue(1.0, post=(2.0, 1.0)))


# ---- torchvision ----------------------------------------------------------------------------------------------------------
def _input_scales(model):
    """Activation scales by layer name, equal for layers that read the same tensor (as calibration gives them)."""
    import torch.fx as fx
    from dfq_b200 import int8
    g = int8._Int8Tracer().trace(model)
    mods = dict(model.named_modules())
    rng, by_input, acts = np.random.default_rng(0), {}, {}
    for n in g.nodes:
        if n.op == "call_module" and isinstance(mods[n.target], (nn.Conv2d, nn.Linear)):
            src = n.args[0]
            while isinstance(src, fx.Node) and src.op == "call_module" and type(mods[src.target]) is nn.BatchNorm2d:
                src = src.args[0]
            acts[n.target] = by_input.setdefault(src, float(rng.uniform(4.0, 40.0)))
    return acts


@pytest.mark.parametrize("net, relu6, edges, adds, perturb", [
    ("mobilenet_v2", True, 51, 10, False), ("mobilenet_v2", False, 51, 10, False), ("resnet18", True, 18, 8, False),
    ("resnet18", True, 15, 8, True)], ids=["mobilenet_v2", "mobilenet_v2_relu", "resnet18", "resnet18_downsample_scale"])
def test_torchvision_counts(monkeypatch, net, relu6, edges, adds, perturb):
    """BN folded to the identity: MobileNetV2 carries every convolution input but the stem's and fuses its 10 residual adds;
    ResNet-18 carries 7 conv1, 3 downsample and 8 conv2 inputs and fuses its 8 adds - 15 edges when the downsample branches
    read the block input at another scale.  Tracing only, no forward."""
    import torchvision
    from dfq_b200 import int8
    RO.install(monkeypatch)
    torch.manual_seed(0)
    model = _identity_bns(getattr(torchvision.models, net)(num_classes=10))
    if not relu6:
        for m in model.modules():
            for k, c in m.named_children():
                if isinstance(c, nn.ReLU6):
                    setattr(m, k, nn.ReLU())
    acts = _input_scales(model)
    if perturb:
        for k in acts:
            if k.endswith("downsample.0"):
                acts[k] = float(np.nextafter(np.float32(acts[k]), np.float32(INF)))
    from collections import OrderedDict
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    names = {id(m): n for n, m in model.named_modules()}
    int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=[acts[names[k]] for k in graph])
    gm = int8.chain_int8(model, residual=True)
    assert len(gm.requantized_edges) == edges and len(gm.fused_adds) == adds
    carried = {q for _, q, _ in gm.requantized_edges}
    convs = [n for n, m in model.named_modules() if isinstance(m, int8.Int8Conv2d)]
    if net == "mobilenet_v2":
        assert [c for c in convs if c not in carried] == ["features.0.0"]
    else:
        kinds = [q.rsplit(".", 1)[-1] if not q.endswith("downsample.0") else "downsample" for _, q, _ in gm.requantized_edges]
        assert (kinds.count("conv1"), kinds.count("downsample"), kinds.count("conv2")) == ((7, 0, 8) if perturb else (7, 3, 8))
        assert [a[0] for a in gm.fused_adds] == ["layer%d.%d.conv2" % (i, j) for i in range(1, 5) for j in range(2)]
        assert {a[4] for a in gm.fused_adds} == {(0.0, INF)}
    plain = int8.chain_int8(model)                              # residual=False: exactly the single-user edges
    assert not hasattr(plain, "fused_adds") and len(plain.requantized_edges) == (36 if net == "mobilenet_v2" else 8)


def test_small_residual_network_forward_through_the_twin(monkeypatch):
    """A two-block residual stack with a fan-out between them runs bit-identically through the twins."""
    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.stem = nn.Conv2d(3, 16, 3, 1, 1)
            self.b1, self.b2 = _Inverted(c=16), _Inverted(c=16)

        def forward(self, x):
            x = F.relu(self.stem(x))
            x = x + self.b1.q(F.relu6(self.b1.e(x)))
            x = x + self.b2.q(F.relu6(self.b2.e(x)))
            return self.b2.z(x)
    gm, edges, adds = _chain(monkeypatch, M(), _x())
    assert [a[0] for a in adds] == ["b1.q", "b2.q"] and len(edges) == 5


class _PostIdentityIsAResidual(nn.Module):
    """t = bn(relu(a(x) + x)), an identity BN that ends the first add's post chain, is only the residual of b(s) + t.
    b_first: b is traced before the first block (as ResNet's downsample is traced after conv2)."""

    def __init__(self, b_first):
        super().__init__()
        self.stem = nn.Conv2d(3, 16, 3, 1, 1)
        self.a, self.b, self.z = nn.Conv2d(16, 16, 3, 1, 1), nn.Conv2d(16, 16, 1), nn.Conv2d(16, 8, 1)
        self.bn = _identity_bn(16)
        self.b_first = b_first

    def forward(self, x):
        x = F.relu(self.stem(x))
        if self.b_first:
            u = self.b(x)
            t = self.bn(F.relu(self.a(x) + x))
        else:
            t = self.bn(F.relu(self.a(x) + x))
            u = self.b(x)
        return self.z(u + t)


@pytest.mark.parametrize("b_first", [False, True], ids=["first_block_first", "second_producer_first"])
def test_identity_ending_a_post_chain_stays_the_residual_of_the_next_add(monkeypatch, b_first):
    """The identity BN belongs to the first fusion (it ends the clamps after its add) and is the second add's residual:
    the second fusion does not skip it, and takes the first producer's fp32 output as its residual, in either graph order."""
    gm, edges, adds = _chain(monkeypatch, _PostIdentityIsAResidual(b_first), _x(),
                             acts={"stem": 6.0, "a": 3.0, "b": 3.0, "z": 2.0})
    assert adds == [("a", "add", "relu", NONE, (0.0, INF)), ("b", "add_1", "bn", NONE, NONE)][::-1 if b_first else 1]
    assert ("b", "z", NONE) in edges and not _calls(gm, operator.add)
    nodes = {n.name: n for n in gm.graph.nodes}
    assert "bn" not in nodes and "relu_1" not in nodes
    b, a = next(n for n in gm.graph.nodes if n.target == "b"), next(n for n in gm.graph.nodes if n.target == "a")
    assert b.args[1].target is operator.getitem or b.args[1] is a
    assert (b.args[1].args[0] if b.args[1] is not a else a) is a
