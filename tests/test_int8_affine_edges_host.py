"""The affine int8 path off its 8-bit defaults on the CPU: weight-grid recovery over the reference's CPU recipe at 1-8 bits,
convert_affine at every weight width and its refusals at K = 2^17 and on a weight grid narrower than the weights', and
SSD-Lite chained through the host twins of the affine entries (tests/fakelib_int8_affine_observe.py) against the patched
per-layer run.  The -m gpu twin is tests/test_gpu_int8_affine_edges.py."""
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

import affine_observed_state
import fakelib_int8_affine
import fakelib_int8_affine_observe
import int8_affine_oracle as A
from oracle import dfq_oracle as D
from test_int8_affine_observe_host import _same, _state

f32 = np.float32


def _tensors(rng):
    """Weights as the reference's models hold them: conv, linear and depthwise shapes at scales 1e-4 to 10, all-positive
    tensors whose minimum is far from 0, a constant tensor and a tensor with one constant channel."""
    out = []
    for i in range(40):
        shape = [(64, 32, 3, 3), (1000, 64), (96, 1, 3, 3), (7, 5), (128, 256, 1, 1)][i % 5]
        scale = 10 ** rng.uniform(-4, 1)
        w = (rng.standard_normal(shape) * scale).astype(f32)
        if i % 7 == 0:
            w = (np.abs(w) + f32(scale)).astype(f32)
        out.append(w)
    out.append(np.full((8, 4, 3, 3), f32(-0.0371), f32))
    w = (rng.standard_normal((6, 5, 3, 3)) * 0.2).astype(f32)
    w[2] = f32(0.125)
    out.append(w)
    return out


@pytest.mark.parametrize("bits", range(1, 9))
def test_weight_grid_recovery_over_the_cpu_recipe(bits):
    """quantize_targ_layer on CPU parameters divides by the scale (dfq_oracle.quantize div_mode "div"); some candidate of
    weight_grid_candidates reproduces every weight it produced, the codes span [-128, 2^bits - 129] and dequantize back
    bit for bit."""
    from dfq_b200 import int8
    rng = np.random.default_rng(100 + bits)
    for w in _tensors(rng):
        w_hat = D.quantize(w, bits, div_mode="div")
        mn = w_hat.min()
        cands = int8.weight_grid_candidates(mn, w_hat.max(), bits)
        fw = next((c for c in cands if A.weight_codes(w_hat, mn, c, bits)[1] == 0), None)
        assert fw is not None, (w.shape, float(np.abs(w).max()))
        q, _ = A.weight_codes(w_hat, mn, fw, bits)
        assert q.min() == -128 and q.max() <= 2 ** bits - 129
        assert q.max() == 2 ** bits - 129 or w_hat.max() == mn
        back = ((q.astype(f32) + f32(128)) * fw).astype(f32) + f32(mn)
        assert np.array_equal(back.view(np.int32), w_hat.view(np.int32))


def _model(bits, div_mode="div", wide=None):
    """conv -> depthwise -> 1x1 -> Linear with bits-bit weights from the CPU recipe; `wide` appends one more target layer."""
    from dfq_b200.utils import quantize as Q
    torch.manual_seed(bits)
    layers = [Q.QuantNConv2d(3, 16, 3, padding=1), Q.QuantNConv2d(16, 16, 3, padding=1, groups=16), Q.QuantNConv2d(16, 24, 1),
              nn.Flatten(1), Q.QuantNLinear(24 * 36, 10)]
    model = nn.Sequential(*layers + ([wide] if wide is not None else [])).eval()
    with torch.no_grad():
        for m in model:
            if hasattr(m, "quant"):
                m.weight.copy_(torch.from_numpy(D.quantize(m.weight.numpy(), bits, div_mode=div_mode)))
                m.quant.running_min.fill_(-1.5)
                m.quant.running_max.fill_(2.5)
    return model


def _graph(model):
    from dfq_b200.utils import quantize as Q
    return OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (Q.QuantNConv2d, Q.QuantNLinear)))


def _targ():
    from dfq_b200.utils import quantize as Q
    return [Q.QuantNConv2d, Q.QuantNLinear]


@pytest.mark.parametrize("bits", range(1, 9))
def test_convert_affine_packs_every_weight_width(monkeypatch, bits):
    """convert_affine(bits_weight=b) on weights of b bits: every layer packs at b bits, its codes and tap table are the
    oracle's, and the codes reach both ends of the b-bit range."""
    from dfq_b200 import int8
    fakelib_int8_affine.install(monkeypatch)
    model = _model(bits)
    w = {i: model[i].weight.detach().numpy().copy() for i in (0, 1, 2, 4)}
    names = int8.convert_affine(model, _graph(model), _targ(), bits_weight=bits)
    assert names == ["0", "1", "2", "4"]
    for i, wt in w.items():
        mod = model[i]
        assert mod.w_bits == bits and mod.w_min == float(wt.min())
        wt = wt.reshape(wt.shape + (1, 1)) if wt.ndim == 2 else wt
        q, bad = A.weight_codes(wt, mod.w_min, mod.w_scale, bits)
        assert bad == 0 and q.min() == -128 and q.max() == 2 ** bits - 129
        kh, kw = mod.kernel_size
        if mod.groups == 1:
            codes = mod.weight_codes.numpy().reshape(mod.out_channels, kh, kw, mod.cpad)
            assert np.array_equal(codes[..., :mod.in_channels], q.transpose(0, 2, 3, 1))
            assert np.array_equal(mod.tap_table.numpy().reshape(-1, kh + 1, kw + 1), A.tap_table(q))
        else:
            codes = mod.weight_codes.numpy().reshape(kh * kw, mod.cpad)
            assert np.array_equal(codes[:, :mod.in_channels], q.reshape(mod.in_channels, kh * kw).T)
        assert not codes[..., mod.in_channels:].any()


def test_weights_on_a_wider_grid_are_refused(monkeypatch):
    """8-bit weights converted with bits_weight=4 lie on no 4-bit grid: DfqError naming the first layer, nothing replaced."""
    from dfq_b200 import _lib, int8
    fakelib_int8_affine.install(monkeypatch)
    model = _model(8)
    before = [type(m) for m in model]
    with pytest.raises(_lib.DfqError, match=r"layer 0: its weights are not on a 4-bit min / max grid"):
        int8.convert_affine(model, _graph(model), _targ(), bits_weight=4)
    assert [type(m) for m in model] == before
    model = _model(4)
    assert int8.convert_affine(model, _graph(model), _targ(), bits_weight=4) == ["0", "1", "2", "4"]


def test_k_limit_through_the_fake_library(monkeypatch):
    """K = kh * kw * C / groups = 131072 is refused by name before anything is replaced (a 1x1 Conv2d of 131072 inputs, a
    2x4 kernel on 16384, a Linear of 131072 features); K = 131071 and 131056, the largest accepted, convert."""
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8_affine.install(monkeypatch)
    for wide in (Q.QuantNConv2d(131072, 2, 1), Q.QuantNConv2d(16384, 2, (2, 4)), Q.QuantNLinear(131072, 3)):
        model = _model(8, wide=wide)
        before = [type(m) for m in model]
        with pytest.raises(_lib.DfqError, match=r"layer 5: K = kh \* kw \* C / groups = 131072 reaches 131072"):
            int8.convert_affine(model, _graph(model), _targ())
        assert [type(m) for m in model] == before
        with pytest.raises(_lib.DfqError, match="131072 reaches 131072"):
            int8.AffineInt8Conv2d.from_conv(wide, -1.0, 1.0) if isinstance(wide, nn.Conv2d) else \
                int8.AffineInt8Linear.from_linear(wide, -1.0, 1.0)
    for C in (131071, 131056):
        wide = Q.QuantNConv2d(C, 2, 1)
        with torch.no_grad():
            wide.weight.copy_(torch.from_numpy(D.quantize(wide.weight.numpy(), 8, div_mode="div")))
        wide.quant.running_min.fill_(-1.0)
        wide.quant.running_max.fill_(1.0)
        model = nn.Sequential(wide)
        assert int8.convert_affine(model, _graph(model), _targ()) == ["0"]
        assert model[0].cpad == {131071: 131072, 131056: 131056}[C]


# ---- SSD-Lite through the host twins ----------------------------------------------------------------------------------
def _ssd_lite(size):
    """SSD-Lite (is_test) with BN folded, 8-bit weights, one input range per layer and its records (10 adds, two 6-way
    cats, a softmax) from an eager run at size x size."""
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    torch.manual_seed(0)
    model = affine_observed_state.build("ssd").eval()
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    graph, bottoms = trace_graph(model)
    LT.merge_batchnorm(model, graph, bottoms, [nn.Conv2d, nn.Linear])

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d:
                q = Q.QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation,
                                   ch.groups, ch.bias is not None)
            else:
                swap(ch)
                continue
            q.load_state_dict(ch.state_dict(), strict=False)
            with torch.no_grad():
                q.weight.copy_(torch.from_numpy(A.fake_quant_weights(q.weight.numpy(), 8)))
            q.quant.running_min.fill_(-2.0)
            q.quant.running_max.fill_(6.0)
            setattr(parent, name, q)
    swap(model)
    x = torch.randn(2, 3, size, size).clamp_(-2.5, 2.5)
    return model, x, affine_observed_state.record_ops(model, x)


def test_ssd_lite_chained_equals_the_patched_per_layer_run(monkeypatch):
    """At 64x64 (1x1 and 2x2 tail maps from the third extra block on): both outputs of chain_affine, with and without residual
    fusion, equal the per-layer affine model's under replace_op() bit for bit.  Without residual fusion 53 edges carry codes;
    with it 85, through the 10 adds, and the 20 observers on their operands fold into the producers' epilogues.  The 12
    cat-operand observers stay in torch: every head permutes before the cat."""
    from dfq_b200 import int8
    fake = fakelib_int8_affine_observe.install(monkeypatch)
    model, x, records = _ssd_lite(64)
    names = [name.rsplit("_", 2)[0] + "/" + name.rsplit("_", 1)[1] for _, name in records]
    assert sorted(set(names)) == ["F_softmax/1", "add/2", "torch_cat/6"]
    assert (names.count("add/2"), names.count("torch_cat/6"), names.count("F_softmax/1")) == (10, 2, 1)
    ranges = [(-3.0 - 0.1 * i, 4.0 + 0.1 * i) for i in range(10 * 2 + 2 * 6 + 1)]
    with _state(model, records, ranges=ranges) as ct:
        assert len(int8.convert_affine(model, _graph(model), _targ())) == 86
        gms = {res: int8.chain_affine(model, residual=res) for res in (False, True)}
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        with torch.no_grad():
            ref = model(x)
            got = {res: gm(x) for res, gm in gms.items()}
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
    assert "dfq_i8_affine_conv_observed" in fake.calls
    assert [r.shape for r in ref] == [(2, 144, 21), (2, 144, 4)]
    for res, out in got.items():
        assert len(out) == 2 and all(_same(a, b) for a, b in zip(out, ref)), res
    assert len(gms[False].requantized_edges) == 53 and gms[False].fused_observers == []
    gm = gms[True]
    assert (len(gm.requantized_edges), len(gm.fused_adds), len(gm.fused_observers)) == (85, 10, 20)
    assert sorted({w for _, w, _ in gm.fused_observers}) == ["operand", "residual"]
    left = [n for n in gm.graph.nodes if n.op == "call_module" and n.target.startswith("custom_tensor_op")]
    assert len(left) == 13                                      # 12 cat operands and the softmax's
