"""dfq_b200.int8.chain_affine in the reference's evaluation state on the CPU: the functional-op observers that replace_op()
applies (utils/layer_transform.py's cursor protocol) replayed into the traced graph, the generated forward immune to the
patched ops, and the rules that fold the observers into the producers' epilogues - through the host twin of
dfq_i8_affine_conv_observed (tests/fakelib_int8_affine_observe.py), each chained model checked bit for bit against the
patched eager run of the per-layer model."""
import math
from collections import OrderedDict
from contextlib import contextmanager

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import fakelib_int8_affine_observe
import int8_affine_observe_oracle as AO
from test_int8_affine_chain_host import _qconv

f32 = np.float32
INF = math.inf


@contextmanager
def _state(model, records, ranges=None, bits=8):
    """replace_op() active with a CustomTensorOP of one QuantMeasure per operand of `records`, installed as
    model.custom_tensor_op; restored afterwards."""
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    n = sum(int(r[1].split("_")[-1]) for r in records)
    obs = [Q.QuantMeasure(num_bits=bits).eval() for _ in range(n)]
    for i, q in enumerate(obs):
        lo, hi = (ranges[i] if ranges else (-1.5 - 0.1 * i, 1.7 + 0.2 * i))
        q.running_min.fill_(float(f32(lo)))
        q.running_max.fill_(float(f32(hi)))
    ct = LT.CustomTensorOP(obs, [tuple(r) for r in records])
    model.add_module("custom_tensor_op", ct)
    prev = LT.module_tensor_op
    LT.module_tensor_op = ct
    LT.replace_op()
    try:
        yield ct
    finally:
        LT.restore_op()
        LT.module_tensor_op = prev


def _convert(model):
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (Q.QuantNConv2d, Q.QuantNLinear)))
    int8.convert_affine(model, graph, [Q.QuantNConv2d, Q.QuantNLinear])
    return model


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.detach().numpy().view(np.int32), b.detach().numpy().view(np.int32))


# ---- replay ---------------------------------------------------------------------------------------------------------------
def helper_outside_forward(a, b):
    return a + b, torch.cat([a, b], 1)


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.c1 = nn.Conv2d(3, 4, 3, padding=1)
        self.c2 = nn.Conv2d(3, 4, 3, padding=1)
        self.fail = False

    def forward(self, x):
        a = self.c1(x)
        b = self.c2(x)
        y = a + b
        z = torch.cat([y, a, b], 1)
        u = F.interpolate(z, scale_factor=2, mode='bilinear', align_corners=True)
        v = torch.mean(u, (2, 3))
        p = F.softmax(v, 1)
        t = a.add(b)
        s, c = helper_outside_forward(a, b)
        q = a + b
        y += q
        if self.fail:
            raise RuntimeError("forward failed")
        return p, y, t, s, c


_L0 = Net.forward.__code__.co_firstlineno
RECORD = [("add_1", "add_%d_2" % (_L0 + 3)), ("torch.cat_2", "torch_cat_%d_3" % (_L0 + 4)),
          ("F.interpolate_3", "F_interpolate_%d_1" % (_L0 + 5)), ("torch.mean_4", "torch_mean_%d_1" % (_L0 + 6)),
          ("F.softmax_5", "F_softmax_%d_1" % (_L0 + 7)), ("iadd_6", "iadd_%d_2" % (_L0 + 11))]
# the observed operands, in observer order: the add's two, the cat's three, then interpolate, mean, softmax, the iadd's two
OPERANDS = ["c1", "c2", "add", "c1", "c2", "cat", "interpolate", "mean", "add", "add_3"]


def test_replay_puts_the_observers_on_the_recorded_operands(monkeypatch):
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    fakelib_int8_affine_observe.install(monkeypatch)
    model = Net().eval()
    x = torch.randn(2, 3, 5, 6)
    with _state(model, RECORD) as ct:
        with torch.no_grad():
            ref = model(x)
        gm = int8.chain_affine(model)
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
        obs = [n for n in gm.graph.nodes if n.op == "call_module" and n.target.startswith("custom_tensor_op.")]
        assert [n.target for n in obs] == ["custom_tensor_op.%d" % i for i in range(10)]
        assert [n.args[0].name for n in obs] == OPERANDS
        assert all(len(n.users) == 1 for n in obs)
        assert not [n for n in gm.graph.nodes if n.target is operator_add()]
        with torch.no_grad():
            got = gm(x)
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
        assert torch.Tensor.__add__ is LT.___add__ and torch.cat is LT.torch_cat
    assert len(got) == len(ref) and all(_same(a, b) for a, b in zip(got, ref))
    assert gm.fused_observers == []


def operator_add():
    import operator
    return operator.add


def test_replay_restores_the_patched_ops_when_the_trace_fails(monkeypatch):
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    fakelib_int8_affine_observe.install(monkeypatch)
    model = Net().eval()
    model.fail = True
    with _state(model, RECORD):
        with pytest.raises(RuntimeError, match="forward failed"):
            int8.chain_affine(model)
        assert torch.Tensor.__add__ is LT.___add__ and torch.Tensor.__iadd__ is LT.___iadd__
        assert torch.cat is LT.torch_cat and torch.mean is LT.torch_mean
        assert F.interpolate is LT.F_interpolate and F.softmax is LT.F_softmax


def test_replay_refuses_unconsumed_records_and_moved_cursors(monkeypatch):
    from dfq_b200 import _lib, int8
    fakelib_int8_affine_observe.install(monkeypatch)
    model = Net().eval()
    with _state(model, RECORD + [("add_7", "add_99999_2")]):
        with pytest.raises(_lib.DfqError, match="add_99999_2"):
            int8.chain_affine(model)
    model = Net().eval()
    with _state(model, RECORD) as ct:
        ct.idx_name_tensor_op = 1
        with pytest.raises(_lib.DfqError, match="cursors"):
            int8.chain_affine(model)


def test_outside_the_evaluation_state_nothing_changes(monkeypatch):
    from dfq_b200 import int8
    fakelib_int8_affine_observe.install(monkeypatch)
    gm = int8.chain_affine(Net().eval())
    assert not [n for n in gm.graph.nodes if n.op == "call_module" and "custom_tensor_op" in n.target]
    assert sum(n.target is operator_add() for n in gm.graph.nodes) == 4


# ---- the rules ------------------------------------------------------------------------------------------------------------
class _MBBlock(nn.Module):
    """MobileNetV2's inverted residual, x + conv(x), between a stem and a head convolution."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(1)
        self.stem = _qconv(3, 16, 3, -2.5, 2.5)
        self.b = _qconv(16, 32, 1, 0.0, 4.0)
        self.c = _qconv(32, 32, 3, 0.0, 4.0, groups=32)
        self.d = _qconv(32, 16, 1, 0.0, 4.0)
        self.head = _qconv(16, 8, 1, -3.0, 5.0)
        self.relu = nn.ReLU()

    def forward(self, x):
        x = self.relu(self.stem(x))
        x = x + self.d(self.relu(self.c(self.relu(self.b(x)))))
        return self.head(x)


class _ResBlock(nn.Module):
    """ResNet's BasicBlock with a downsample: out += identity, then a ReLU."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(2)
        self.stem = _qconv(3, 16, 3, -2.5, 2.5)
        self.c1 = _qconv(16, 24, 3, 0.0, 3.0, stride=2)
        self.c2 = _qconv(24, 24, 3, 0.0, 3.0)
        self.ds = _qconv(16, 24, 1, 0.0, 3.0, padding=0, stride=2)
        self.head = _qconv(24, 8, 1, 0.0, 4.0)
        self.relu = nn.ReLU()

    def forward(self, x):
        x = self.relu(self.stem(x))
        out = self.c2(self.relu(self.c1(x)))
        identity = self.ds(x)
        out += identity
        return self.head(self.relu(out))


class _Mean(nn.Module):
    """The reference MobileNetV2's head: torch.mean(x.view(N, C, -1), -1) after the last convolution."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.a = _qconv(3, 16, 3, -2.5, 2.5)
        self.relu = nn.ReLU()

    def forward(self, x):
        x = self.relu(self.a(x))
        return torch.mean(x.view(x.size(0), x.size(1), -1), -1)


class _Cat(nn.Module):
    """Two producers concatenated in torch (DeepLab's ASPP), then a convolution."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(4)
        self.a = _qconv(3, 16, 3, -2.5, 2.5)
        self.b = _qconv(3, 8, 1, -2.5, 2.5, padding=0)
        self.c = _qconv(24, 8, 1, -1.0, 6.0, padding=0)
        self.relu = nn.ReLU()

    def forward(self, x):
        a = self.relu(self.a(x))
        b = self.b(x)
        return self.c(torch.cat([a, b], 1))


def _rec(cls, offset, name, n):
    return ("k", "%s_%d_%d" % (name, cls.forward.__code__.co_firstlineno + offset, n))


CASES = {
    "mobilenet": (_MBBlock, [_rec(_MBBlock, 2, "add", 2)], 1,
                  [("custom_tensor_op.1", "operand", "d"), ("custom_tensor_op.0", "residual", "d")]),
    "resnet": (_ResBlock, [_rec(_ResBlock, 4, "iadd", 2)], 1,
               [("custom_tensor_op.0", "operand", "c2"), ("custom_tensor_op.1", "residual", "c2")]),
    "mean": (_Mean, [_rec(_Mean, 2, "torch_mean", 1)], 0, [("custom_tensor_op.0", "output", "a")]),
    "cat": (_Cat, [_rec(_Cat, 3, "torch_cat", 2)], 0,
            [("custom_tensor_op.0", "output", "a"), ("custom_tensor_op.1", "output", "b")]),
}


def _chained(monkeypatch, cls, records, **state):
    from dfq_b200 import int8
    fake = fakelib_int8_affine_observe.install(monkeypatch)
    model = _convert(cls().eval())
    x = torch.randn(2, 3, 9, 9)
    ctx = _state(model, records, **state)
    ct = ctx.__enter__()
    try:
        gm = int8.chain_affine(model, residual=True)
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        with torch.no_grad():
            fake.calls.clear()
            got = gm(x)
            calls = list(fake.calls)
            ref = model(x)
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
    finally:
        ctx.__exit__(None, None, None)
    return gm, got, ref, calls


@pytest.mark.parametrize("case", list(CASES))
def test_observers_fold_into_the_producers(monkeypatch, case):
    cls, records, adds, folded = CASES[case]
    gm, got, ref, calls = _chained(monkeypatch, cls, records)
    assert _same(got, ref)
    assert sorted(gm.fused_observers) == sorted(folded)
    assert len(gm.fused_adds) == adds
    assert not [n for n in gm.graph.nodes if n.op == "call_module" and n.target.startswith("custom_tensor_op")]
    assert calls.count("dfq_i8_affine_conv_observed") == len({p for _, _, p in folded})


def test_generated_forward_is_immune_to_the_patched_ops(monkeypatch):
    """Records naming lines of the generated forward - its tensor adds, its cat and its mean - change nothing: the
    chained module calls no patched op, and its output equals, bit for bit, its output without those records."""
    from dfq_b200 import int8
    fakelib_int8_affine_observe.install(monkeypatch)
    model = Net().eval()
    x = torch.randn(2, 3, 5, 6)
    with _state(model, RECORD):
        gm = int8.chain_affine(model)                           # residual=False: the adds stay in the graph
        with torch.no_grad():
            ref = gm(x)
    code = gm.code.splitlines()

    def lines(word):
        found = [i + 1 for i, s in enumerate(code) if word in s]
        assert found, "the generated forward has no %r line:\n%s" % (word, gm.code)
        return found
    adds, cats, means = lines("torch.add("), lines("_raw_cat("), lines("_raw_mean(")
    assert not [s for s in code if any(w in s for w in ("torch.cat(", "torch.mean(", "functional.interpolate(",
                                                        "functional.softmax("))]
    for name, line in [("add_%d_2", adds[0]), ("iadd_%d_2", adds[-1]), ("torch_cat_%d_3", cats[0]),
                       ("torch_cat_%d_2", cats[-1]), ("torch_mean_%d_1", means[0])]:
        other = Net().eval()
        with _state(other, [("k", name % line)], ranges=[(0.0, 1e-3)] * 3) as ct:
            with torch.no_grad():
                got = gm(x)
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0, name % line
        assert len(got) == len(ref) and all(torch.equal(a, b) for a, b in zip(got, ref)), name % line


class _ShapeArith(nn.Module):
    """A residual add next to integer arithmetic on shape queries (x.size(1) * 0 + x.size(1)), traced as operator.add of
    a non-tensor node."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(5)
        self.a = _qconv(3, 16, 3, -2.5, 2.5)
        self.b = _qconv(16, 16, 3, 0.0, 4.0)
        self.relu = nn.ReLU()

    def forward(self, x):
        x = self.relu(self.a(x))
        y = x + self.b(x)
        return y.view(y.size(0), y.size(1) * 0 + y.size(1), -1)


@pytest.mark.parametrize("residual", [False, True])
def test_integer_arithmetic_on_shapes_stays_python(monkeypatch, residual):
    """An operator.add of integers stays operator.add (torch.add of two ints would raise) in the evaluation state."""
    import operator
    from dfq_b200 import int8
    fakelib_int8_affine_observe.install(monkeypatch)
    model = _convert(_ShapeArith().eval())
    x = torch.randn(2, 3, 9, 9)
    with _state(model, [_rec(_ShapeArith, 2, "add", 2)]) as ct:
        gm = int8.chain_affine(model, residual=residual)
        ints = [n for n in gm.graph.nodes if n.op == "call_function" and n.target is operator.add]
        assert len(ints) == 1 and ints[0].args[0].target is operator.mul
        assert sum(n.target is torch.add for n in gm.graph.nodes) == (0 if residual else 1)
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        with torch.no_grad():
            got = gm(x)
            ref = model(x)
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
    assert _same(got, ref)


@pytest.mark.parametrize("how", ["update_stat", "training", "bits", "range"])
def test_observers_that_stay_in_torch(monkeypatch, how):
    from dfq_b200 import int8
    fakelib_int8_affine_observe.install(monkeypatch)
    model = _convert(_Mean().eval())
    with _state(model, CASES["mean"][1], bits=16 if how == "bits" else 8,
                ranges=[(0.0, INF)] if how == "range" else None) as ct:
        q = ct._modules["0"]
        if how == "update_stat":
            q.update_stat = 8                                   # set_layer_bits' quirk: the bit width as update_stat
        if how == "training":
            q.train()
        gm = int8.chain_affine(model, residual=True)
    assert gm.fused_observers == []
    assert [n.target for n in gm.graph.nodes if n.op == "call_module" and "custom_tensor_op" in n.target] == \
        ["custom_tensor_op.0"]


# ---- the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 5, 8])
def test_oracle_equals_quantmeasure_composed_in_torch(monkeypatch, bits):
    """observed_value == clamp(QuantMeasure(clamp(y)) + QuantMeasure(r)) with QuantMeasure itself (host twin of its CUDA
    mode), NaN, +-inf, -0.0 and subnormals in both operands."""
    fakelib_int8_affine_observe.install(monkeypatch)
    rng = np.random.default_rng(bits)
    y = (rng.standard_normal((2, 19, 5, 4)) * 3).astype(f32)
    r = (rng.standard_normal(y.shape) * 3).astype(f32)
    y.reshape(-1)[:6] = r.reshape(-1)[-6:] = (np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-41)
    obs, res = (f32(-0.4), f32(3.9), bits), (f32(-2.2), f32(2.6), 9 - bits)
    for o, s, rr in ((obs, res, r), (obs, None, r), (None, res, r), (obs, None, None)):
        want = AO.torch_value(torch.from_numpy(y), None if rr is None else torch.from_numpy(rr), (0.0, 6.0), (-1.0, INF),
                              o, s).numpy()
        got = AO.observed_value(y, rr, (0.0, 6.0), (-1.0, INF), o, s, gpu_nan=False)
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(np.where(nan, 0, got).view(np.int32), np.where(nan, 0, want).view(np.int32))
