"""dfq_b200.int8.chain_affine(concat=True, fold_pads=True) on the CPU, through the host twins of dfq_i8_affine_conv_layout
and dfq_i8_affine_upsample_bilinear (tests/fakelib_int8_affine_layout.py): the oracle's pad-code identity, the pad and
concatenation rules and what each leaves in torch, each chained model checked bit for bit against the per-layer model
(under replace_op() where observers are recorded), and the padded DeepLab-v3+'s counts."""
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_observed_state
import fakelib_int8_affine_layout
import int8_affine_layout_oracle as AL
import int8_affine_oracle as A
from test_int8_affine_chain_host import _qconv
from test_int8_affine_observe_host import _state

f32 = np.float32


def _graph(model):
    from dfq_b200.utils import quantize as Q
    return OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (Q.QuantNConv2d, Q.QuantNLinear)))


def _targ():
    from dfq_b200.utils import quantize as Q
    return [Q.QuantNConv2d, Q.QuantNLinear]


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(u, v) for u, v in zip(a, b))
    return a.shape == b.shape and np.array_equal(a.detach().numpy().view(np.int32), b.detach().numpy().view(np.int32))


def _chain(monkeypatch, model, x, observed=False, **kw):
    """(chained GraphModule, fake): converts `model`, chains it with residual=True and `kw`, and checks it against the
    per-layer model bit for bit (under replace_op() with recorded observers when `observed`), and that the per-layer
    model is left as it was."""
    from dfq_b200 import int8
    fake = fakelib_int8_affine_layout.install(monkeypatch)
    model = model.eval()
    records = affine_observed_state.record_ops(model, x) if observed else None

    def run():
        int8.convert_affine(model, _graph(model), _targ())
        layers = {n: (m, m.padding) for n, m in model.named_modules() if isinstance(m, int8._AffineInt8Layer)}
        gm = int8.chain_affine(model, residual=True, **kw)
        for n, m in model.named_modules():
            if isinstance(m, int8._AffineInt8Layer):
                assert layers[n] == (m, m.padding) and m.pad_code is None and m.out_slice is None and m.epilogue is None, n
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
    return gm, fake


# ---- the oracle -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups,pad,stride,dil", [(1, (1, 1), (1, 1), (1, 1)), (1, (2, 1), (2, 1), (1, 2)),
                                                   (5, (1, 2), (1, 2), (2, 1))])
def test_pad_code_identity_against_a_direct_evaluation(groups, pad, stride, dil):
    rng = np.random.default_rng(sum(pad) + groups)
    C_, O_ = 5, 5 if groups > 1 else 7
    xq = rng.integers(-128, 128, (2, C_, 6, 5)).astype(np.int8)
    wq = rng.integers(-128, 128, (O_, C_ // groups, 3, 3)).astype(np.int8)
    z = -37
    want = AL.folded_terms_direct(xq, wq, pad, z, stride, dil, groups)
    got = A.terms(AL.pad_codes(xq, pad, z), wq, stride, (0, 0), dil, groups)
    for w, g in zip(want, got):
        assert np.array_equal(w, g)


def test_zero_code_follows_the_range():
    from dfq_b200 import int8
    for lo, hi, bits in ((-1.7, 2.9, 8), (0.0, 3.1, 8), (0.4, 3.3, 8), (-1.0, 1.0, 1), (-0.3, 5.0, 4)):
        assert int8.affine_code_of(0.0, lo, hi, bits) == AL.zero_code(lo, hi, bits)
    assert int8.affine_code_of(0.0, 0.4, 3.3, 8) == -128


# ---- pads -------------------------------------------------------------------------------------------------------------------
class PadNet(nn.Module):
    def __init__(self, pad=(1, 1, 1, 1), mode="constant", value=0.0, conv_pad=0, second_user=False):
        super().__init__()
        torch.manual_seed(0)
        self.c0 = _qconv(3, 16, 3, -2.0, 2.0)
        self.c1 = _qconv(16, 16, 3, -0.5, 3.0, padding=conv_pad)
        self.dw = _qconv(16, 16, 3, 0.0, 4.0, groups=16, padding=0)
        self.c2 = _qconv(16, 8, 1, -1.0, 5.0)
        self.pad, self.mode, self.value, self.second_user = pad, mode, value, second_user

    def forward(self, x):
        y = F.relu(self.c0(x))
        p = F.pad(y, self.pad, self.mode, self.value) if self.mode == "constant" else F.pad(y, self.pad, self.mode)
        z = F.relu6(self.c1(p))
        out = self.c2(F.relu(self.dw(F.pad(z, (1, 1, 1, 1)))))
        return (out, p.sum()) if self.second_user else out


@pytest.mark.parametrize("kw,folded", [
    (dict(), 2), (dict(pad=(2, 2, 1, 1)), 2), (dict(pad=(1, 2, 1, 1)), 1), (dict(value=0.5), 1),
    (dict(mode="reflect"), 1), (dict(second_user=True), 1), (dict(conv_pad=1), 1)],
    ids=["symmetric", "t_ne_l", "asymmetric", "non_zero", "reflect", "two_users", "conv_padding"])
def test_pad_rule_and_its_refusals(monkeypatch, kw, folded):
    x = torch.randn(2, 3, 9, 8)
    gm, fake = _chain(monkeypatch, PadNet(**kw), x, fold_pads=True)
    assert len(gm.folded_pads) == folded
    assert gm.folded_pads[-1][1] == "dw" and gm.folded_pads[-1][2] == (1, 1)
    assert "dfq_i8_affine_conv_layout" in fake.calls
    left = [n for n in gm.graph.nodes if n.op == "call_function" and n.target in (F.pad, torch._C._nn.pad)]
    assert len(left) == 2 - folded
    gm2, _ = _chain(monkeypatch, PadNet(**kw), x)                # without the flag every pad stays
    assert not hasattr(gm2, "folded_pads")


# ---- concatenations -----------------------------------------------------------------------------------------------------------
class CatNet(nn.Module):
    def __init__(self, widths=(16, 8), consumer_groups=1, upsample=None, two_keys=False):
        super().__init__()
        torch.manual_seed(1)
        self.a = _qconv(3, widths[0], 3, -2.0, 2.0)
        self.b = _qconv(3, widths[1], 3, -2.0, 2.0, stride=2 if upsample else 1)
        n = sum(widths)
        self.c = _qconv(n, n if consumer_groups > 1 else 12, 3, -0.5, 3.5, groups=consumer_groups)
        self.d = _qconv(n, 5, 1, -0.7 if two_keys else -0.5, 3.5) if two_keys else None
        self.upsample, self.two_keys = upsample, two_keys

    def forward(self, x):
        a = F.relu(self.a(x))
        b = F.relu6(self.b(x))
        if self.upsample == "size":
            b = F.interpolate(b, size=a.size()[2:], mode="bilinear", align_corners=True)
        elif self.upsample == "scale":
            b = F.interpolate(b, scale_factor=2, mode="bilinear", align_corners=False)
        t = torch.cat([a, b], dim=1)
        return (self.c(t), self.d(t)) if self.two_keys else self.c(t)


@pytest.mark.parametrize("observed", [False, True])
@pytest.mark.parametrize("kw,cats,ups,sums", [
    (dict(), 1, 0, True), (dict(consumer_groups=24), 1, 0, False), (dict(widths=(17, 8)), 0, 0, None),
    (dict(upsample="size"), 1, 1, True), (dict(upsample="scale"), 0, 0, None), (dict(two_keys=True), 0, 0, None)],
    ids=["dense", "depthwise_consumer", "unaligned", "upsample", "scale_factor", "two_keys"])
def test_concatenation_rule(monkeypatch, observed, kw, cats, ups, sums):
    from dfq_b200 import int8
    x = torch.randn(2, 3, 8, 8)
    gm, fake = _chain(monkeypatch, CatNet(**kw), x, observed=observed, concat=True)
    assert (len(gm.fused_cats), len(gm.fused_upsamples)) == (cats, ups)
    assert gm.fused_pools == []
    if cats:
        writers = [m for m in gm.modules() if getattr(m, "out_slice", None) is not None]
        assert len(writers) == 2 and all(w.sums == sums for w in writers)
        assert "dfq_i8_affine_conv_layout" in fake.calls
        assert gm.fused_cats[0][2] == [0, 16]
        kinds = sorted(w for _, w, _ in gm.fused_observers)
        assert kinds == ((["cat", "cat"] + (["output"] if ups else [])) if observed else [])
    if ups:
        assert any(isinstance(m, int8.AffineInt8UpsampleBilinear) for m in gm.modules())
        assert "dfq_i8_affine_upsample_bilinear" in fake.calls
    if not cats:
        assert any(n.op == "call_function" and "cat" in getattr(n.target, "__name__", "") for n in gm.graph.nodes)


def test_concat_needs_residual():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="builds on residual"):
        int8.chain_affine(nn.Identity(), concat=True)


# ---- the padded DeepLab-v3+ -----------------------------------------------------------------------------------------------
def test_deeplab_counts_through_the_host_twins(monkeypatch):
    """At 33x33 with the functional-op records of an eager run: chain_affine(residual=True, concat=True, fold_pads=True)
    equals the patched per-layer run bit for bit and finds what the H100 run finds (tests/test_gpu_int8_affine_layout.py):
    17 pads, 2 concatenations, 2 upsamples, 30 of 30 observers, 59 of 61 convolution inputs carried."""
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    fakelib_int8_affine_layout.install(monkeypatch)
    torch.manual_seed(0)
    model = affine_observed_state.build("deeplab").eval()
    graph, bottoms = trace_graph(model)
    LT.merge_batchnorm(model, graph, bottoms, [nn.Conv2d, nn.Linear])

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is not nn.Conv2d:
                swap(ch)
                continue
            q = Q.QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation,
                               ch.groups, ch.bias is not None)
            q.load_state_dict(ch.state_dict(), strict=False)
            with torch.no_grad():
                q.weight.copy_(torch.from_numpy(A.fake_quant_weights(q.weight.numpy(), 8)))
            q.quant.running_min.fill_(-2.0)
            q.quant.running_max.fill_(6.0)
            setattr(parent, name, q)
    swap(model)
    gm, fake = _chain(monkeypatch, model, torch.randn(1, 3, 33, 33).clamp_(-2.5, 2.5), observed=True, concat=True,
                      fold_pads=True)
    convs = [n for n, m in gm.named_modules() if isinstance(m, int8.AffineInt8Conv2d)]
    carried = {q for _, q, _ in gm.requantized_edges}
    assert (len(gm.folded_pads), len(gm.fused_cats), len(gm.fused_upsamples), len(gm.fused_observers)) == (17, 2, 2, 30)
    assert (len(carried), len(convs)) == (59, 61)
    assert sorted(set(convs) - carried) == ["aspp.image_pool.1", "backbone.features.0.0"]
