"""Host side of convert_affine on the layers that quantize their own weights on every forward (QConv2d / QLinear of
--distill_range, QuantConv2d / QuantLinear of --trainable), through the oracle-backed fake library: the weights go through
the per-forward quantizer and the bias through the implicit-range prologue, the layer's bits must be bits_weight, learned
scales are refused, refusals leave the model as it was, and QuantN* layers convert as before."""
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

import fakelib_int8_affine
import int8_affine_oracle as A
from oracle import dfq_oracle as O

f32 = np.float32
FAMILIES = {"distill_range": ("QConv2d", "QLinear"), "trainable": ("QuantConv2d", "QuantLinear")}


def _targ(family):
    from dfq_b200.utils import quantize as Q
    return [getattr(Q, n) for n in FAMILIES[family]]


def _graph(model, targ):
    return OrderedDict((id(m), m) for m in model.modules() if type(m) in targ)


def _model(family, seed=0, bias_bits=16):
    """Conv, depthwise conv, 1x1 conv and a Linear of the family, unquantized fp32 weights, frozen input ranges."""
    Conv, Lin = _targ(family)
    torch.manual_seed(seed)
    model = nn.Sequential(Conv(3, 16, 3, padding=1), nn.ReLU(), Conv(16, 16, 3, padding=1, groups=16), nn.ReLU(),
                          Conv(16, 24, 1, bias=False), nn.Flatten(1), Lin(24 * 36, 10)).eval()
    with torch.no_grad():
        for m, (lo, hi) in zip([m for m in model if hasattr(m, "quant")], ((-2.5, 2.5), (0., 4.), (0., 3.), (0., 5.))):
            m.num_bits_bias = bias_bits
            if m.bias is not None:
                m.bias.normal_(0, 0.3)
            m.quant.running_min.fill_(lo)
            m.quant.running_max.fill_(hi)
    return model


def _params(model):
    return [(p.detach().clone(), p) for p in model.parameters()]


def _unchanged(saved):
    return all(torch.equal(a.view(torch.int32), b.detach().view(torch.int32)) for a, b in saved)


@pytest.mark.parametrize("bias_bits", [16, 32])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_per_forward_layers_convert_from_the_forwards_own_quantized_tensors(monkeypatch, family, bias_bits):
    """Every layer is replaced; its codes dequantize to _quant_param_per_forward's output and its bias is quantize(bias)'s
    implicit-range output (prologue 1 on host tensors), both checked against the oracle too; the originals are untouched."""
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    fake = fakelib_int8_affine.install(monkeypatch)
    model = _model(family, bias_bits=bias_bits)
    targ = _targ(family)
    originals = [m for m in model if type(m) in targ]
    saved = _params(model)
    names = int8.convert_affine(model, _graph(model, targ), targ)
    assert names == ["0", "2", "4", "6"]
    assert [type(model[i]).__name__ for i in (0, 2, 4, 6)] == ["AffineInt8Conv2d"] * 3 + ["AffineInt8Linear"]
    # one per-forward quantization per weight and per bias (layer 4 has none), then one pack per layer
    assert fake.calls.count("dfq_observe_quant") == 4 + 3 and fake.calls.count("dfq_i8_affine_pack") == 4
    assert fake.calls.index("dfq_i8_affine_pack") > max(i for i, c in enumerate(fake.calls) if c == "dfq_observe_quant")
    assert _unchanged(saved)
    for i, orig in zip((0, 2, 4, 6), originals):
        mod = model[i]
        w = orig.weight.detach()
        want = Q._quant_param_per_forward(w.clone(), 8).numpy()
        assert np.array_equal(want.view(np.int32), O.quantize(w.numpy(), 8, float(w.min()), float(w.max())).view(np.int32))
        assert not np.array_equal(want, w.numpy())
        want = want.reshape(want.shape + (1, 1)) if want.ndim == 2 else want
        q, bad = A.weight_codes(want, mod.w_min, mod.w_scale, 8)
        assert bad == 0 and mod.w_min == float(want.min()) and mod.w_bits == 8
        back = ((q.astype(f32) + f32(128)) * f32(mod.w_scale)).astype(f32) + f32(mod.w_min)
        assert np.array_equal(back.view(np.int32), want.view(np.int32))
        if orig.bias is None:
            assert not mod.bias.any()
            continue
        b = orig.bias.detach()
        want_b = Q.quantize(b.clone(), num_bits=bias_bits).numpy()
        assert np.array_equal(mod.bias.numpy().view(np.int32), want_b.view(np.int32))
        assert np.array_equal(want_b.view(np.int32), O.quantize_tensor_range(b.numpy(), bias_bits, float(b.min()),
                                                                              float(b.max()), False, 1).view(np.int32))


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bits_rule_and_learned_scales_refused_leaving_the_model_as_it_was(monkeypatch, family):
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8_affine.install(monkeypatch)
    targ = _targ(family)

    def refused(model, match, **kw):
        before, saved = [type(m) for m in model], _params(model)
        with pytest.raises(_lib.DfqError, match=match):
            int8.convert_affine(model, _graph(model, targ), targ, **kw)
        assert [type(m) for m in model] == before and _unchanged(saved)

    # set_layer_bits writes bits_weight into every layer's num_bits: converting at another width is refused by name
    model = _model(family)
    Q.set_layer_bits(_graph(model, targ), 4, 8, 16, targ)
    for m in model:
        if hasattr(m, "quant"):
            m.quant.running_min.fill_(-1.0); m.quant.running_max.fill_(3.0)
    refused(model, r"layer 0 quantizes its weights to 4 bits on every forward, not bits_weight = 8")
    names = int8.convert_affine(model, _graph(model, targ), targ, bits_weight=4)
    assert names == ["0", "2", "4", "6"] and all(model[i].w_bits == 4 for i in (0, 2, 4, 6))
    model = _model(family)
    model[4].num_bits = 6
    refused(model, r"layer 4 quantizes its weights to 6 bits")
    model = _model(family)
    model[2].num_bits = 16
    refused(model, r"layer 2 quantizes its weights to 16 bits", bits_weight=8)
    refused(_model(family), r"layer 0: weight codes of 16 bits", bits_weight=16)
    if family == "distill_range":
        model = _model(family)
        model[2].set_scale(scale=torch.full((16,), 1.5))
        refused(model, r"layer 2 carries learned scales .*merge_scale_to_weight")
        model = _model(family)
        model[6].set_scale(scale_prev=torch.full((24 * 36,), 0.5))
        refused(model, r"layer 6 carries learned scales")
        model[6].merge_scale_to_weight()                 # merged: scale_prev is None again and the layer converts
        assert int8.convert_affine(model, _graph(model, targ), targ) == ["0", "2", "4", "6"]


def test_quantn_layers_convert_as_before(monkeypatch):
    """QuantNConv2d / QuantNLinear: packed from their own (offline fake-quantized) weights and biases as from_conv /
    from_linear pack them, without a per-forward quantization."""
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    fake = fakelib_int8_affine.install(monkeypatch)
    torch.manual_seed(3)
    model = nn.Sequential(Q.QuantNConv2d(3, 16, 3, padding=1), nn.ReLU(), Q.QuantNConv2d(16, 16, 3, groups=16), nn.Flatten(1),
                          Q.QuantNLinear(16 * 16, 5)).eval()
    with torch.no_grad():
        for m in (model[0], model[2], model[4]):
            m.weight.copy_(torch.from_numpy(A.fake_quant_weights(m.weight.numpy(), 8)))
            m.quant.running_min.fill_(-1.0); m.quant.running_max.fill_(2.0)
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    want = [int8.AffineInt8Conv2d.from_conv(model[0], -1.0, 2.0, name="0"),
            int8.AffineInt8Conv2d.from_conv(model[2], -1.0, 2.0, name="2"),
            int8.AffineInt8Linear.from_linear(model[4], -1.0, 2.0, name="4")]
    fake.calls.clear()
    assert int8.convert_affine(model, _graph(model, targ), targ) == ["0", "2", "4"]
    assert "dfq_observe_quant" not in fake.calls
    for i, w in zip((0, 2, 4), want):
        got = model[i]
        assert type(got) is type(w) and (got.w_min, got.w_scale, got.w_bits) == (w.w_min, w.w_scale, w.w_bits)
        assert tuple(got.constants[0]) == tuple(w.constants[0])
        for buf in ("weight_codes", "tap_table", "bias"):
            assert torch.equal(getattr(got, buf), getattr(w, buf)), (i, buf)
