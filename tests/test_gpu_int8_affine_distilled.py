"""convert_affine and chain_affine on the H100 in the reference's --distill_range and --trainable states
(tests/affine_distilled_state.py): layers that quantize their weights and bias on every forward.  Per layer, the packed
codes dequantize to _quant_param_per_forward's weights and the bias equals the forward's quantized bias bit for bit, and
the output stays within the bounds of test_gpu_int8_affine_edges.py of the fake-quantized layer's; the whole converted
model stays near the fake-quantized one, and chain_affine equals the per-layer model bit for bit with the fused counts of
the default (QuantN*) state.  Then the bits rule, learned scales and low-bit weights.

Measured on an H100 (distilled-range state, 8-bit weights): worst |int - fake quant| 11.75 / 7.5 / 230.5 / 25.0 ulp of the
bound on MobileNetV2 / ResNet-18 / DeepLab / SSD-Lite, 0.2 / 0.13 / 0.17 / 0.2 of the combined bound (16 ulp of the bound
plus 4 ulp of the offset bound, asserted <= 1: DeepLab's 1x1 expansions cancel far below their offsets' rounding, see
test_gpu_int8_affine_edges.py), |int - double| at most 1.14 ulp; relative error against the fake-quantized model 3.2e-3 /
7.5e-3 (asserted below 1e-2, the classifiers' bound in test_gpu_int8_affine.py) / 5.1e-3 / 8.5e-3.  The trainable state
gives the same numbers: without learned scales both forwards quantize the same tensors."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import affine_distilled_state as D

pytestmark = pytest.mark.gpu

# chain_affine flags and fused counts per network, the same as in the default evaluation state
# (test_gpu_int8_affine_observe.py, test_gpu_int8_affine_layout.py, test_gpu_int8_affine_pool_heads.py)
CHAIN = {
    "mobilenet_v2": dict(size=224, flags=dict(residual=True), counts=dict(observers=21, fused_observers=21, adds=10)),
    "resnet18": dict(size=224, flags=dict(residual=True), counts=dict(observers=16, fused_observers=16, adds=8)),
    "deeplab": dict(size=129, flags=dict(residual=True, concat=True, fold_pads=True),
                    counts=dict(observers=30, fused_observers=30, pads=17, cats=2, upsamples=2)),
    "ssd": dict(size=300, flags=dict(residual=True, concat=True, fold_pads=True, pools=True, heads=True),
                counts=dict(observers=33, distinct_fused_observers=33, heads=[(6, 21), (6, 4)])),
}


@pytest.fixture
def no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_equal(u, v) for u, v in zip(a, b))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _effective(twin):
    """The weight and bias the per-forward layer's forward uses, on the GPU."""
    from dfq_b200.utils import quantize as Q
    with torch.no_grad():
        w = Q._quant_param_per_forward(twin.weight.detach().clone(), twin.num_bits)
        b = None if twin.bias is None else Q.quantize(twin.bias.detach().clone(), num_bits=twin.num_bits_bias)
    return w, b


def _dequantized_codes(lay):
    """fp32(fp32((q + 128) fw) + mw) of the packed codes, in the layer's weight shape [O, C / groups, kh, kw]."""
    kh, kw = lay.kernel_size
    q = lay.weight_codes
    if lay.groups == 1:
        q = q.view(lay.out_channels, kh, kw, lay.cpad)[..., :lay.in_channels].permute(0, 3, 1, 2)
    else:
        q = q.view(kh, kw, lay.cpad)[..., :lay.in_channels].permute(2, 0, 1).unsqueeze(1)
    t = (q.float() + 128.0) * torch.tensor(lay.w_scale, dtype=torch.float32, device=q.device)
    return t + torch.tensor(lay.w_min, dtype=torch.float32, device=q.device)


def _check_layers(names, twins, converted, seen):
    """Per layer: the codes and bias bit for bit, and (worst |int - fake quant| in ulp of sum |x^| |w^| + |b|, worst
    |int - double| in ulp of the offset bound sum (|x^| + |ma|)(|w^| + |mw|) + |b|, worst |int - fake quant| / (16 ulp of
    the bound + 4 ulp of the offset bound)) - test_gpu_int8_affine_edges.py's bounds, with x^ the observer's output and w^,
    b the forward's quantized weight and bias."""
    worst, worst64, within = 0.0, 0.0, 0.0
    for n in names:
        lay, twin = converted[n], twins[n]
        w, b = _effective(twin)
        assert lay.w_bits == twin.num_bits, n
        assert _same_bits(_dequantized_codes(lay), w.reshape(lay.out_channels, -1, *lay.kernel_size)), n
        assert _same_bits(lay.bias, torch.zeros_like(lay.bias) if b is None else b), n
        xin, yfq = seen[n]
        xh = twin.quant(xin)
        y = lay(xin)
        if isinstance(twin, nn.Conv2d):
            conv = lambda a, c: F.conv2d(a, c, None, twin.stride, twin.padding, twin.dilation, twin.groups)
        else:
            conv = lambda a, c: F.linear(a, c)
        bb = (torch.zeros(lay.out_channels, device=y.device) if b is None else b).double().reshape((-1,) + (1,) * (y.dim() - 2))
        bound = conv(xh.abs().double(), w.abs().double()) + bb.abs()
        y64 = conv(xh.double(), w.double()) + bb
        ma, mw = abs(float(twin.quant.running_min)), abs(float(w.min()))
        bound64 = conv(xh.abs().double() + ma, w.abs().double() + mw) + bb.abs()
        ulp = torch.from_numpy(np.spacing(bound.float().cpu().numpy())).cuda().double()
        ulp64 = torch.from_numpy(np.spacing(bound64.float().cpu().numpy())).cuda().double()
        diff = (y.double() - yfq.double()).abs()
        worst = max(worst, float((diff / ulp).max()))
        worst64 = max(worst64, float(((y.double() - y64).abs() / ulp64).max()))
        within = max(within, float((diff / (16 * ulp + 4 * ulp64)).max()))
    return worst, worst64, within


def _record(model, names):
    seen, mods = {}, dict(model.named_modules())
    hooks = [mods[n].register_forward_hook(lambda m, i, o, n=n: seen.__setitem__(n, (i[0].detach(), o.detach())))
             for n in names]
    return seen, hooks


def _params(model):
    return {n: p.detach().clone() for n, p in model.named_parameters()}


def _convert_and_chain(net, kind, bits_weight=8):
    """Build the state, convert it per layer and chain it: the per-layer checks, the whole-model error, chain_affine's
    equality and counts."""
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    spec = CHAIN[net]
    size = spec["size"]
    with D.distilled_state(net, kind, size=size, batch=4, bits_weight=bits_weight) as (model, qgraph, qtarg):
        ct = LT.module_tensor_op
        twins = {n: m for n, m in model.named_modules() if type(m) in qtarg}
        before = {n: _params(m) for n, m in twins.items()}
        g = torch.Generator(device="cuda").manual_seed(2)
        x = D.inputs(net, 4, size, g)
        seen, hooks = _record(model, list(twins))
        with torch.no_grad():
            ref = model(x)
        for h in hooks:
            h.remove()
        names = int8.convert_affine(model, qgraph, qtarg, bits_weight=bits_weight)
        mods = dict(model.named_modules())
        assert sorted(names) == sorted(twins) and all(isinstance(mods[n], int8._AffineInt8Layer) for n in names)
        assert all(_equal(before[n][k], v) for n, m in twins.items() for k, v in _params(m).items())
        with torch.no_grad():
            worst, worst64, within = _check_layers(names, twins, mods, seen)
            got = model(x)
            gm = int8.chain_affine(model, **spec["flags"])
            chained = gm(x)
        assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
        err = max(float((a - r).norm() / r.norm()) for a, r in zip(got if isinstance(got, tuple) else (got,),
                                                                      ref if isinstance(ref, tuple) else (ref,)))
        kinds = [w for _, w, _ in gm.fused_observers]
        print("%s (%s, %d-bit weights): %d layers, worst |int - fake quant| %.2f ulp (%.3g of 16 ulp + 4 offset ulp), "
              "|int - double| %.2f ulp, relative error against the fake-quantized model %.3g; chained: observers %d, fused "
              "%d %s, adds %d, pads %d, cats %d, upsamples %d, heads %s" % (
                  net, kind, bits_weight, len(names), worst, within, worst64, err, ct.len, len(gm.fused_observers),
                  {k: kinds.count(k) for k in set(kinds)}, len(getattr(gm, "fused_adds", [])),
                  len(getattr(gm, "folded_pads", [])), len(getattr(gm, "fused_cats", [])),
                  len(getattr(gm, "fused_upsamples", [])), [(len(p), k) for _, p, k in getattr(gm, "fused_heads", [])]))
        assert worst64 <= 4 and within <= 1, (worst64, within)
        if net in ("mobilenet_v2", "resnet18"):
            assert err < 1e-2, err
        assert _equal(got, chained)
        c = spec["counts"]
        assert ct.len == c["observers"]
        if "fused_observers" in c:
            assert len(gm.fused_observers) == c["fused_observers"]
        if "adds" in c:
            assert len(gm.fused_adds) == c["adds"]
        if "pads" in c:
            assert (len(gm.folded_pads), len(gm.fused_cats), len(gm.fused_upsamples)) == (c["pads"], c["cats"],
                                                                                          c["upsamples"])
        if "heads" in c:
            assert [(len(p), k) for _, p, k in gm.fused_heads] == c["heads"]
            assert len({o for o, _, _ in gm.fused_observers}) == c["distinct_fused_observers"]


@pytest.mark.parametrize("net", list(CHAIN))
def test_distill_range_state_per_layer_whole_model_and_chained(net, no_tf32):
    _convert_and_chain(net, "distill_range")


@pytest.mark.parametrize("net", ["mobilenet_v2", "resnet18"])
def test_trainable_state_per_layer_whole_model_and_chained(net, no_tf32):
    _convert_and_chain(net, "trainable")


def test_low_bit_weights_convert_at_their_width_and_are_refused_at_another(no_tf32):
    """set_layer_bits(bits_weight=4): bits_weight=8 is refused naming the first layer and leaves the model as it was;
    bits_weight=4 converts every layer from 4-bit codes and chains bit for bit."""
    from dfq_b200 import _lib, int8
    with D.distilled_state("resnet18", size=224, batch=4, bits_weight=4) as (model, qgraph, qtarg):
        mods, params = [type(m) for m in model.modules()], _params(model)
        with pytest.raises(_lib.DfqError, match=r"layer conv1 quantizes its weights to 4 bits on every forward, "
                                                r"not bits_weight = 8"):
            int8.convert_affine(model, qgraph, qtarg)
        assert [type(m) for m in model.modules()] == mods
        assert all(_equal(v, params[k]) for k, v in _params(model).items())
    _convert_and_chain("resnet18", "distill_range", bits_weight=4)


def test_learned_scales_and_bits_mismatch_refused_leaving_the_model_unchanged():
    from dfq_b200 import _lib, int8
    with D.distilled_state("mobilenet_v2", size=96, batch=2, batches=1) as (model, qgraph, qtarg):
        layers = [m for m in qgraph.values()]
        mods = [type(m) for m in model.modules()]

        def refused(match):
            params = _params(model)
            with pytest.raises(_lib.DfqError, match=match):
                int8.convert_affine(model, qgraph, qtarg)
            assert [type(m) for m in model.modules()] == mods
            assert all(_equal(v, params[k]) for k, v in _params(model).items())

        names = {id(m): n for n, m in model.named_modules()}
        conv = next(m for m in layers if isinstance(m, nn.Conv2d) and m.groups == 1 and m.kernel_size == (1, 1))
        conv.set_scale(scale=torch.full((conv.out_channels,), 1.25, device="cuda"))
        refused(r"layer %s carries learned scales .*merge_scale_to_weight" % names[id(conv)])
        conv.scale = None
        lin = layers[-1]
        lin.set_scale(scale_prev=torch.full((lin.in_features,), 0.5, device="cuda"))
        refused(r"layer %s carries learned scales" % names[id(lin)])
        lin.scale_prev = None
        layers[3].num_bits = 6
        refused(r"layer %s quantizes its weights to 6 bits" % names[id(layers[3])])
        layers[3].num_bits = 8
        assert len(int8.convert_affine(model, qgraph, qtarg)) == len(layers)
