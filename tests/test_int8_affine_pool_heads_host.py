"""dfq_b200.int8.chain_affine(pools=True) and chain_affine(heads=True) on the CPU, through the host twins of
dfq_i8_affine_maxpool and dfq_i8_affine_conv_rows (tests/fakelib_int8_affine_pool_heads.py): the oracle against the
quantizer of torch's max_pool2d, the pool rule in codes and fp32 mode, the head rule with and without observers, what the
rules leave in torch, and each chained model checked bit for bit against the per-layer model (under replace_op()
where observers are recorded)."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_observed_state
import fakelib_int8_affine_pool_heads as fakelib_int8_affine_pool
import int8_affine_chain_oracle as AC
import int8_affine_oracle as A
import int8_affine_pool_heads_oracle as AP
from test_int8_affine_chain_host import _qconv
from test_int8_affine_layout_host import _graph, _same, _targ
from test_int8_affine_observe_host import _state


def _chain(monkeypatch, model, x, observed=False, **kw):
    """(chained GraphModule, fake, call): tests/test_int8_affine_layout_host.py's check - bit for bit against the per-layer
    model, which is left as it was - through the pool twin; call(**kw) chains the same converted model again."""
    from dfq_b200 import int8
    fake = fakelib_int8_affine_pool.install(monkeypatch)
    model = model.eval()
    records = affine_observed_state.record_ops(model, x) if observed else None

    def run():
        int8.convert_affine(model, _graph(model), _targ())
        layers = {n: (m, m.padding) for n, m in model.named_modules() if isinstance(m, int8._AffineInt8Layer)}
        gm = int8.chain_affine(model, residual=True, **kw)
        for n, m in model.named_modules():
            if isinstance(m, int8._AffineInt8Layer):
                assert layers[n] == (m, m.padding) and m.epilogue is None and m.out_slice is None, n
        assert not any(isinstance(m, int8.AffineInt8MaxPool2d) for m in model.modules())
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        with torch.no_grad():
            ref, got = model(x), gm(x)
        assert _same(ref, got)
        return gm
    if observed:
        with _state(model, records) as ct:
            gm = run()
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
    else:
        gm = run()
    return gm, fake, lambda **k: int8.chain_affine(model, residual=True, **k)


# ---- the oracle ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,s,p,d,ceil", [((2, 2), (2, 2), (0, 0), (1, 1), False), ((3, 3), (2, 2), (1, 1), (1, 1), True),
                                          ((3, 2), (1, 2), (1, 0), (2, 1), False), ((3, 3), (3, 3), (1, 1), (2, 2), True)])
@pytest.mark.parametrize("C,rng_", [(5, (-1.3, 2.2, 8)), (17, (0.4, 3.0, 4)), (33, (0.0, 1.0, 1))])
def test_codes_mode_is_the_code_of_torch_max_pool(k, s, p, d, ceil, C, rng_):
    """Without NaN, the max of the codes is the code of the max: pinned against dfq_i8_affine_quantize's oracle of the
    oracle of torch's max_pool2d, -inf, +inf, -0.0 and subnormals included, and so is S."""
    rng = np.random.default_rng(C)
    x = rng.normal(0.8, 1.5, (2, C, 7, 6)).astype(np.float32)
    x.reshape(-1)[:6] = [np.inf, -np.inf, -0.0, 1e-40, -1e-40, rng_[0]]
    q, _ = A.act_codes(x, *rng_)
    got, S = AP.maxpool_codes(AC.to_nhwc(q), C, k, s, p, d, ceil)
    y, want, want_S = AP.maxpool_fp32(x, k, s, p, d, ceil, rng_)
    assert np.array_equal(got, want) and np.array_equal(S, want_S)


def test_empty_window_and_nan_window():
    xq = np.zeros((1, 1, 1, 16), np.int8)
    xq[..., :3] = np.array([5, -128, 7], np.int8)
    q, S = AP.maxpool_codes(xq, 3, (2, 2), (1, 1), (1, 1), (2, 2), False)     # taps at -1 and 1: none inside
    assert q.shape == (1, 1, 1, 16) and (q[0, 0, 0, :3] == [-128, -128, -128]).all() and (q[0, 0, 0, 3:] == 0).all()
    assert S[0, 0, 0] == -3 * 128
    x = np.full((1, 1, 2, 2), 0.5, np.float32)
    x[0, 0, 0, 0] = np.nan                                       # the per-layer path: NaN wins, code -128
    y, qy, _ = AP.maxpool_fp32(x, (2, 2), (2, 2), (0, 0), (1, 1), False, (-1.0, 1.0, 8))
    assert np.isnan(y).all() and qy[0, 0, 0, 0] == -128
    qc, _ = AP.maxpool_codes(AC.to_nhwc(A.act_codes(x, -1.0, 1.0, 8)[0]), 1, (2, 2), (2, 2), (0, 0), (1, 1), False)
    half = A.act_codes(np.full((1, 1, 1, 1), 0.5, np.float32), -1.0, 1.0, 8)[0]
    assert qc[0, 0, 0, 0] == half.item() != -128                # the codes mode: the max of the other codes


# ---- the pool rule ------------------------------------------------------------------------------------------------------------
class PoolNet(nn.Module):
    """a -> relu -> max pool -> (b, and with two_keys d at another range); stem: b -> relu -> c + the pooled tensor, as
    ResNet's first block."""

    def __init__(self, consumer_groups=1, two_keys=False, stem=False, clamp_after=False, twice=False, k=3, ceil=False):
        super().__init__()
        torch.manual_seed(2)
        self.a = _qconv(3, 16, 3, -2.0, 2.0)
        self.b = _qconv(16, 16, 3, -0.5, 3.5, groups=consumer_groups)
        self.c = _qconv(16, 16, 3, -0.6, 3.0) if stem else None
        self.d = _qconv(16, 16, 3, -0.7, 3.5) if two_keys or stem else None
        self.two_keys, self.stem, self.clamp_after, self.twice, self.k, self.ceil = two_keys, stem, clamp_after, twice, k, \
            ceil

    def forward(self, x):
        t = F.max_pool2d(F.relu(self.a(x)), self.k, 2, 1, ceil_mode=self.ceil)
        if self.twice:
            t = F.max_pool2d(t, 2, 1)
        if self.clamp_after:
            t = F.relu6(t)
        if self.stem:
            return self.d(F.relu(self.c(F.relu(self.b(t))) + t))
        return (self.b(t), self.d(t)) if self.two_keys else self.b(t)


@pytest.mark.parametrize("kw,mode,sums", [
    (dict(), "codes", True), (dict(consumer_groups=16), "codes", False), (dict(k=2, ceil=True), "codes", True),
    (dict(two_keys=True), "fp32", True), (dict(stem=True), "fp32", True), (dict(twice=True), "codes", True),
    (dict(clamp_after=True), None, None)],
    ids=["dense", "depthwise_consumer", "ceil", "two_keys", "stem", "pool_pool", "clamp_after"])
def test_pool_rule(monkeypatch, kw, mode, sums):
    from dfq_b200 import int8
    x = torch.randn(2, 3, 11, 10)
    gm, fake, _ = _chain(monkeypatch, PoolNet(**kw), x, pools=True)
    pools = [m for m in gm.modules() if isinstance(m, int8.AffineInt8MaxPool2d)]
    if mode is None:                                            # a clamp after the pool ends the rule
        assert gm.fused_pools == [] and not pools
        assert "dfq_i8_affine_maxpool" not in fake.calls
        return
    assert [m for _, m, _ in gm.fused_pools] == [mode] * (2 if kw.get("twice") else 1)
    assert pools[-1].sums == sums and "dfq_i8_affine_maxpool" in fake.calls
    assert gm.fused_pools[0][2] == (("codes",) if mode == "codes" else ("fp32", "codes"))
    assert "b" in {q for _, q, _ in gm.requantized_edges}
    if kw.get("twice"):
        assert not pools[0].sums                                # its only consumer is the second pool


@pytest.mark.parametrize("observed", [False, True])
def test_stem_pool_is_a_residual(monkeypatch, observed):
    """ResNet's stem: the pool writes torch's fp32 output for the add (and its observer) and b's codes."""
    gm, _, _ = _chain(monkeypatch, PoolNet(stem=True), torch.randn(2, 3, 12, 12), observed=observed, pools=True)
    assert [m for _, m, _ in gm.fused_pools] == ["fp32"]
    assert len(gm.fused_adds) == 1
    assert sorted(w for _, w, _ in gm.fused_observers) == (["operand", "residual"] if observed else [])


class CatPoolNet(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.a = _qconv(3, 16, 3, -2.0, 2.0)
        self.b = _qconv(3, 8, 3, -2.0, 2.0)
        self.c = _qconv(24, 12, 3, -0.5, 3.5)

    def forward(self, x):
        t = torch.cat([F.relu(self.a(x)), F.relu6(self.b(x))], 1)
        return self.c(F.max_pool2d(t, 3, 2, ceil_mode=True))


@pytest.mark.parametrize("observed", [False, True])
def test_pool_after_a_fused_concatenation(monkeypatch, observed):
    gm, _, _ = _chain(monkeypatch, CatPoolNet(), torch.randn(2, 3, 9, 9), observed=observed, concat=True, pools=True)
    assert len(gm.fused_cats) == 1 and [m for _, m, _ in gm.fused_pools] == ["codes"]
    assert ("max_pool2d", "c") in {(p, q) for p, q, _ in gm.requantized_edges}
    writers = [m for m in gm.modules() if getattr(m, "out_slice", None) is not None]
    assert len(writers) == 2 and not any(w.sums for w in writers)   # the pool sums its own codes
    gm2, _, _ = _chain(monkeypatch, CatPoolNet(), torch.randn(2, 3, 9, 9), observed=observed, pools=True)
    assert gm2.fused_pools == [] and not hasattr(gm2, "fused_cats")   # without concat the cat's pool reads fp32


def test_flags_off_leave_the_pools(monkeypatch):
    """Without pools=True every pool stays in torch and the records are those of the call without the flag."""
    from dfq_b200 import int8
    x = torch.randn(2, 3, 11, 10)
    gm, _, call = _chain(monkeypatch, PoolNet(stem=True), x)
    assert not hasattr(gm, "fused_pools")
    assert not any(isinstance(m, int8.AffineInt8MaxPool2d) for m in gm.modules())
    off = call(pools=False)
    assert off.code == gm.code and off.requantized_edges == gm.requantized_edges and off.fused_adds == gm.fused_adds
    cat, _, call = _chain(monkeypatch, CatPoolNet(), torch.randn(2, 3, 9, 9), concat=True)
    assert cat.fused_pools == [] and call(concat=True, pools=False).code == cat.code


def test_pools_needs_residual():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="pools=True builds on residual"):
        int8.chain_affine(nn.Identity(), pools=True)


def test_pool_module_refuses_a_bad_output_range():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="max pool p: output"):
        int8.AffineInt8MaxPool2d(3, 2, 1, 1, False, 16, False, (0.0, np.inf, 8), name="p")
    with pytest.raises(_lib.DfqError, match="bits"):
        int8.AffineInt8MaxPool2d(3, 2, 1, 1, False, 16, False, (0.0, 1.0, 9), name="p")


# ---- torchvision networks -------------------------------------------------------------------------------------------------------
def fixed_range_model(net):
    """torchvision `net` (seeded; GoogLeNet without its auxiliary heads), or the module `net`, with BN folded, QuantNConv2d / QuantNLinear layers
    of 8-bit fake-quantized weights (the CPU recipe) and every input range [-2, 6]: a quantized model without the
    equalization that tests/affine_observed_state.py runs, which SqueezeNet (no BatchNorm) does not go through."""
    import torchvision
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    torch.manual_seed(0)
    model = net.eval() if isinstance(net, nn.Module) else getattr(torchvision.models, net)(num_classes=1000, **(
        dict(aux_logits=False, init_weights=True) if net == "googlenet" else {})).eval()
    graph, bottoms = trace_graph(model)
    LT.merge_batchnorm(model, graph, bottoms, [nn.Conv2d, nn.Linear])

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d:
                q = Q.QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation,
                                   ch.groups, ch.bias is not None)
            elif type(ch) is nn.Linear:
                q = Q.QuantNLinear(ch.in_features, ch.out_features, ch.bias is not None)
            else:
                swap(ch)
                continue
            q.load_state_dict(ch.state_dict(), strict=False)
            with torch.no_grad():
                q.weight.copy_(torch.from_numpy(A.fake_quant_weights(q.weight.detach().cpu().numpy(), 8)))
            q.quant.running_min.fill_(-2.0)
            q.quant.running_max.fill_(6.0)
            setattr(parent, name, q)
    swap(model)
    return model


@pytest.mark.parametrize("net,kw,carried,convs,cats,pools", [
    ("resnet18", dict(), 19, 20, 0, ["fp32"]),
    ("squeezenet1_1", dict(concat=True), 25, 26, 8, ["codes"] * 3),
    ("googlenet", dict(concat=True), 56, 57, 8, ["codes"] * 13)])
def test_networks_through_the_host_twins(monkeypatch, net, kw, carried, convs, cats, pools):
    """At 64x64 with the functional-op records of an eager run, BN folded, 8-bit weights and fixed ranges: chain_affine
    (residual=True, pools=True, ...) equals the patched per-layer run bit for bit and finds what the H100 run finds
    (tests/test_gpu_int8_affine_pool_heads.py): ResNet-18's stem pool in fp32 mode, every other pool in codes mode, and every
    functional-op observer fused."""
    from dfq_b200 import int8
    fakelib_int8_affine_pool.install(monkeypatch)               # the BN fold runs through the library too
    model = fixed_range_model(net)
    gm, _, _ = _chain(monkeypatch, model, torch.randn(1, 3, 64, 64).clamp_(-2.5, 2.5), observed=True, pools=True, **kw)
    n_convs = sum(isinstance(m, int8.AffineInt8Conv2d) for m in gm.modules())
    assert (len({q for _, q, _ in gm.requantized_edges}), n_convs) == (carried, convs)
    assert len(getattr(gm, "fused_cats", [])) == cats and [m for _, m, _ in gm.fused_pools] == pools
    n_obs = sum(int(r.split("_")[-1]) for _, r in affine_observed_state.record_ops(model, torch.zeros(1, 3, 64, 64)))
    assert len(gm.fused_observers) == n_obs


# ---- detection heads ----------------------------------------------------------------------------------------------------------
class HeadNet(nn.Module):
    """Two feature maps, a classification (k = 3) and a regression (k = 4) head on each, laid out as SSD's heads and
    concatenated along dim 1, the confidences through a softmax.  bad: the second regression head goes through a sigmoid
    before its permute, so its concatenation does not qualify."""

    def __init__(self, bad=False):
        super().__init__()
        torch.manual_seed(5)
        self.a = _qconv(3, 16, 3, -2.0, 2.0)
        self.b = _qconv(16, 16, 3, -0.5, 3.5, stride=2)
        self.ca, self.cb = _qconv(16, 2 * 3, 3, -0.4, 3.0), _qconv(16, 2 * 3, 1, -0.3, 3.2)
        self.la, self.lb = _qconv(16, 2 * 4, 3, -0.4, 3.0), _qconv(16, 2 * 4, 1, -0.3, 3.2, groups=1)
        self.bad = bad

    def forward(self, x):
        a = F.relu(self.a(x))
        b = F.relu6(self.b(a))
        c0, c1 = self.ca(a).permute(0, 2, 3, 1).contiguous(), self.cb(b).permute(0, 2, 3, 1).contiguous()
        l1 = self.lb(b)
        l0, l1 = self.la(a).permute(0, 2, 3, 1).contiguous(), (torch.sigmoid(l1) if self.bad else l1).permute(0, 2, 3, 1)
        confidences = torch.cat([c0.view(c0.size(0), -1, 3), c1.view(c1.size(0), -1, 3)], 1)
        locations = torch.cat([l0.view(l0.size(0), -1, 4), l1.reshape(l1.size(0), -1, 4)], 1)
        confidences = F.softmax(confidences, dim=2)
        return confidences, locations


@pytest.mark.parametrize("observed", [False, True])
@pytest.mark.parametrize("bad", [False, True])
def test_head_rule(monkeypatch, observed, bad):
    from dfq_b200 import int8
    gm, fake, _ = _chain(monkeypatch, HeadNet(bad), torch.randn(2, 3, 10, 9), observed=observed, heads=True)
    assert [(len(p), k) for _, p, k in gm.fused_heads] == ([(2, 3)] if bad else [(2, 3), (2, 4)])
    assert "dfq_i8_affine_conv_rows" in fake.calls
    heads = [m for m in gm.modules() if isinstance(m, int8.Int8HeadConcat)]
    assert len(heads) == len(gm.fused_heads) and all(h.rows for c in heads for h in c.heads)
    kinds = sorted(w for _, w, _ in gm.fused_observers)
    # the replay's observers: 2 + 2 cat operands and the softmax input; a cat left in torch keeps its operands' observers
    assert kinds == ((["head"] * (2 if bad else 4) + ["tail"] * 2) if observed else [])
    if observed:
        assert len({o for o, _, _ in gm.fused_observers}) == (3 if bad else 5)
    left = [n for n in gm.graph.nodes if n.op == "call_function" and "cat" in getattr(n.target, "__name__", "")]
    assert len(left) == (1 if bad else 0)


def test_heads_without_an_observer_on_the_cat_output(monkeypatch):
    """Without replace_op() the softmax reads the head concatenation directly: no tail."""
    gm, _, _ = _chain(monkeypatch, HeadNet(), torch.randn(3, 3, 9, 11), heads=True)
    assert len(gm.fused_heads) == 2 and gm.fused_observers == []


def test_heads_needs_residual_and_flags_off_leave_the_heads(monkeypatch):
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="heads=True builds on residual"):
        int8.chain_affine(nn.Identity(), heads=True)
    gm, _, _ = _chain(monkeypatch, HeadNet(), torch.randn(2, 3, 10, 9), observed=True)
    assert not hasattr(gm, "fused_heads") and not any(isinstance(m, int8.Int8HeadConcat) for m in gm.modules())


def test_rows_mode_refuses_codes_and_residuals():
    from dfq_b200 import _lib, int8
    layer = int8._AffineInt8Layer.__new__(int8.AffineInt8Conv2d)
    nn.Module.__init__(layer)
    for k in int8._AffineInt8Layer._copied:
        setattr(layer, k, None)
    layer.layer_name, layer.out_channels = "h", 8
    with pytest.raises(_lib.DfqError, match="rows exclude"):
        layer.chained(rows=True, epilogue=int8.Epilogue((-1.0, 1.0, 8)))
    with pytest.raises(_lib.DfqError, match="needs rows mode"):
        layer.chained(epilogue=int8.Epilogue(fp32=True)).observe(tail=(-1.0, 1.0, 8))


def test_ssd_lite_through_the_host_twins(monkeypatch):
    """SSD-Lite (tests/ssd_lite_like.py, is_test) at 64x64 with BN folded, 8-bit weights, ranges [-2, 6] and the records of
    an eager run: heads=True fuses both head concatenations (6 producers each, k = 21 and 4) and every observer the replay
    inserts - 10 adds x 2 operands, 12 head operands and the softmax input, 33 - bit-identical to the per-layer model."""
    from ssd_lite_like import SSDLiteLike
    fakelib_int8_affine_pool.install(monkeypatch)
    model = fixed_range_model(SSDLiteLike(21, is_test=True))
    gm, _, _ = _chain(monkeypatch, model, torch.randn(1, 3, 64, 64).clamp_(-2.5, 2.5), observed=True, concat=True,
                      fold_pads=True, heads=True)
    assert [(len(p), k) for _, p, k in gm.fused_heads] == [(6, 21), (6, 4)]
    n_obs = sum(int(r.split("_")[-1]) for _, r in affine_observed_state.record_ops(model, torch.zeros(1, 3, 64, 64)))
    assert n_obs == 33 and len({o for o, _, _ in gm.fused_observers}) == 33
    kinds = [w for _, w, _ in gm.fused_observers]
    assert (kinds.count("head"), kinds.count("tail")) == (12, 6)
