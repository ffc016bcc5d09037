"""Host side of the affine int8 scheme (dfq_b200.int8.convert_affine, tests/int8_affine_oracle.py): the oracle's
decomposition against exact rational arithmetic, its codes against the fake quantization, the weight-grid recovery and the
converter's plan and refusals through an oracle-backed fake library."""
import math
from collections import OrderedDict
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn as nn

import fakelib_int8_affine
import int8_affine_oracle as A

f32 = np.float32


def _graph(model):
    return OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))


def _ulp(v):
    return float(np.spacing(f32(abs(v)))) if v != 0 else float(np.spacing(f32(0)))


GEOMETRIES = [  # (N, C, H, W, O, k, stride, pad, dil, groups): borders of stride / padding / dilation
    (1, 3, 5, 5, 2, (3, 3), (1, 1), (1, 1), (1, 1), 1),
    (1, 5, 6, 4, 3, (3, 2), (2, 1), (2, 1), (1, 2), 1),
    (2, 2, 4, 5, 2, (3, 3), (1, 2), (3, 2), (2, 1), 1),        # padding past the dilated kernel: empty windows
    (1, 4, 5, 6, 4, (3, 3), (2, 2), (1, 1), (1, 1), 4),        # depthwise
    (1, 3, 6, 5, 3, (2, 3), (1, 1), (2, 0), (2, 2), 3),
]


@pytest.mark.parametrize("case", GEOMETRIES, ids=lambda c: "x".join(map(str, c[:5])) + "-g%d" % c[-1])
def test_oracle_decomposition_equals_exact_rational_arithmetic(case):
    """sum over the in-image taps of (qa fa + ma)(qw fw + mw), in Fractions, equals kP P + kA A + kW Wv + kN Nv with the
    constants taken exactly; the double epilogue lands within its rounding of that value."""
    N, Cn, H, W, O_, k, s, p, d, g = case
    rng = np.random.default_rng(sum(map(int, case[:5])))
    x = rng.standard_normal((N, Cn, H, W)).astype(f32) * 2
    w_hat = A.fake_quant_weights(rng.standard_normal((O_, Cn // g) + k).astype(f32), 8)
    rmin, rmax = f32(-1.7), f32(2.9)
    xq, _ = A.act_codes(x, rmin, rmax, 8)
    mw = f32(w_hat.min())
    fw = f32((float(w_hat.max()) - float(mw)) / 255.)
    wq, bad = A.weight_codes(w_hat, mw, fw, 8)
    assert bad == 0
    _, ma, fa, _, _ = A.act_scalars(rmin, rmax, 8)
    P, Ax, Wv, Nv = A.terms(xq, wq, s, p, d, g)
    y = A.epilogue(P, Ax, Wv, Nv, A.constants(ma, fa, mw, fw))
    Fa, Fma, Fw, Fmw = Fraction(float(fa)), Fraction(float(ma)), Fraction(float(fw)), Fraction(float(mw))
    Fma2, Fmw2 = Fma + 128 * Fa, Fmw + 128 * Fw
    kx = (Fa * Fw, Fa * Fmw2, Fma2 * Fw, Fma2 * Fmw2)
    OH, OW = y.shape[2:]
    Cg = Cn // g
    for n in range(N):
        for o in range(O_):
            for oh in range(OH):
                for ow in range(OW):
                    exact, mag = Fraction(0), 0.
                    for c in range(Cg):
                        ci = o if g > 1 else c
                        for r in range(k[0]):
                            ih = oh * s[0] - p[0] + r * d[0]
                            for t in range(k[1]):
                                iw = ow * s[1] - p[1] + t * d[1]
                                if 0 <= ih < H and 0 <= iw < W:
                                    a = (int(xq[n, ci, ih, iw]) + 128) * Fa + Fma
                                    b = (int(wq[o, c, r, t]) + 128) * Fw + Fmw
                                    exact += a * b
                                    mag += abs(float(a) * float(b))
                    terms = [int(v[n, o, oh, ow]) for v in (P, Ax, Wv, Nv)]
                    assert sum(kk * tt for kk, tt in zip(kx, terms)) == exact
                    dbl = sum(abs(float(kk) * tt) for kk, tt in zip(kx, terms)) + mag
                    err = abs(Fraction(float(y[n, o, oh, ow])) - exact)
                    assert err <= Fraction(_ulp(float(exact))) / 2 + Fraction(8 * 2. ** -53 * dbl), (n, o, oh, ow)


@pytest.mark.parametrize("bits", [2, 3, 4, 5, 6, 7, 8])
def test_codes_dequantize_to_the_fake_quantization_bit_for_bit(bits):
    """At rounding boundaries (each code's half point and its fp32 neighbours), the range's ends, beyond them, +-inf, -0.0."""
    rng = np.random.default_rng(bits)
    for rmin, rmax in ((f32(-1.3), f32(2.7)), (f32(0.0), f32(6.0)), (f32(-0.25), f32(-0.25)), (f32(3e-9), f32(5e-9))):
        _, ma, fa, _, qmax = A.act_scalars(rmin, rmax, bits)
        half = ((np.arange(int(qmax) + 1) + 0.5) * float(fa) + float(ma)).astype(f32)
        x = np.concatenate([half, np.nextafter(half, f32(np.inf)), np.nextafter(half, f32(-np.inf)),
                            np.array([rmin, rmax, np.inf, -np.inf, -0.0, 0.0, 1e30, -1e30], f32),
                            (rng.standard_normal(997) * 3).astype(f32)])
        q, S = A.act_codes(x.reshape(1, -1, 1, 1), rmin, rmax, bits)
        assert q.min() >= -128 and q.max() <= qmax - 128
        got = A.act_dequant(q, rmin, rmax, bits).reshape(-1)
        ref = A.fake_quant(x, rmin, rmax, bits)
        assert np.array_equal(got.view(np.int32), ref.view(np.int32)), (rmin, rmax)
        assert S.reshape(-1)[0] == int(q.astype(np.int64).sum())
    # the 1e-8 floor: an empty range quantizes at scale fp32(1e-8)
    assert A.act_scalars(f32(0.5), f32(0.5), 8)[2] == f32(1e-8)
    # NaN has no code in the fake quantization (its output is NaN); the affine quantizer gives it code 0 (stored -128)
    q, _ = A.act_codes(np.array([np.nan], f32).reshape(1, 1, 1, 1), f32(-1), f32(1), 8)
    assert q.reshape(-1)[0] == -128 and np.isnan(A.fake_quant(np.array([np.nan], f32), f32(-1), f32(1), 8)[0])


@pytest.mark.parametrize("bits", [2, 4, 6, 8])
def test_weight_grid_recovery_reproduces_every_weight(bits):
    from dfq_b200 import int8
    rng = np.random.default_rng(10 + bits)
    for w in (rng.standard_normal((16, 8, 3, 3)).astype(f32) * 0.3, rng.uniform(0.1, 0.2, (7, 5)).astype(f32),
              np.full((4, 4), f32(-0.75))):
        w_hat = A.fake_quant_weights(w, bits)
        cands = int8.weight_grid_candidates(w_hat.min(), w_hat.max(), bits)
        fw = next(c for c in cands if A.weight_codes(w_hat, w_hat.min(), c, bits)[1] == 0)
        q, _ = A.weight_codes(w_hat, w_hat.min(), fw, bits)
        assert q.min() >= -128 and q.max() <= 2 ** bits - 1 - 128
        back = ((q.astype(f32) + f32(128)) * fw).astype(f32) + f32(w_hat.min())
        assert np.array_equal(back.view(np.int32), w_hat.view(np.int32))
    # weights that were never fake-quantized are on no candidate's grid
    w = rng.standard_normal((32, 16)).astype(f32)
    assert all(A.weight_codes(w, w.min(), c, bits)[1] > 0 for c in int8.weight_grid_candidates(w.min(), w.max(), bits))
    assert int8.weight_grid_candidates(f32(0), f32(np.inf), bits) == []


def _affine_model(seed=0):
    from dfq_b200.utils import quantize as Q
    torch.manual_seed(seed)
    model = nn.Sequential(Q.QuantNConv2d(3, 16, 3, padding=1), nn.ReLU(), Q.QuantNConv2d(16, 16, 3, padding=1, groups=16),
                          nn.ReLU(), Q.QuantNConv2d(16, 24, 1), nn.Flatten(1), Q.QuantNLinear(24 * 36, 10)).eval()
    with torch.no_grad():
        for m, (lo, hi) in zip([m for m in model if hasattr(m, "quant")], ((-2.5, 2.5), (0., 4.), (0., 3.), (0., 5.))):
            m.weight.copy_(torch.from_numpy(A.fake_quant_weights(m.weight.numpy(), 8)))
            m.quant.running_min.fill_(lo)
            m.quant.running_max.fill_(hi)
    return model


def test_convert_affine_plans_packs_and_swaps_through_the_fake_library(monkeypatch):
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    fake = fakelib_int8_affine.install(monkeypatch)
    model = _affine_model()
    w = [m.weight.detach().clone() for m in model if hasattr(m, "quant")]
    names = int8.convert_affine(model, _graph(model), [Q.QuantNConv2d, Q.QuantNLinear])
    assert names == ["0", "2", "4", "6"]
    assert [type(model[i]).__name__ for i in (0, 2, 4, 6)] == ["AffineInt8Conv2d"] * 3 + ["AffineInt8Linear"]
    assert fake.calls.count("dfq_i8_affine_pack") == 4
    for i, wt in zip((0, 2, 4, 6), w):
        mod, wn = model[i], wt.numpy()
        wn = wn.reshape(wn.shape + (1, 1)) if wn.ndim == 2 else wn
        q, bad = A.weight_codes(wn, mod.w_min, mod.w_scale, 8)
        assert bad == 0 and mod.w_min == float(wn.min())
        kh, kw = mod.kernel_size
        if mod.groups == 1:
            codes = mod.weight_codes.numpy().reshape(mod.out_channels, kh, kw, mod.cpad)
            assert np.array_equal(codes[..., :mod.in_channels], q.transpose(0, 2, 3, 1))
            assert not codes[..., mod.in_channels:].any()
            assert np.array_equal(mod.tap_table.numpy().reshape(-1, kh + 1, kw + 1), A.tap_table(q))
        else:
            codes = mod.weight_codes.numpy().reshape(kh * kw, mod.cpad)
            assert np.array_equal(codes, q.reshape(16, 9).T) and mod.tap_table.numel() == 0
        _, ma, fa, _, _ = A.act_scalars(mod.act_min, mod.act_max, 8)
        assert tuple(mod.constants[0]) == A.constants(ma, fa, mod.w_min, mod.w_scale)
    with pytest.raises(_lib.DfqError, match="GPU"):
        model(torch.randn(1, 3, 6, 6))


def test_chain_int8_keeps_affine_layers_as_opaque_leaves(monkeypatch):
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8_affine.install(monkeypatch)
    model = _affine_model(1)
    int8.convert_affine(model, _graph(model), [Q.QuantNConv2d, Q.QuantNLinear])
    for kw in (dict(), dict(residual=True, pool_cat=True, upsample=True, layout=True)):
        gm = int8.chain_int8(model, **kw)
        mods = [n.target for n in gm.graph.nodes if n.op == "call_module"]
        assert mods == ["0", "1", "2", "3", "4", "5", "6"]
        assert gm.requantized_edges == [] and all(type(getattr(gm, t)) is type(model[int(t)]) for t in ("0", "2", "4", "6"))
        assert all(getattr(gm, t) is model[int(t)] for t in ("0", "2", "4", "6"))


def test_convert_affine_refuses_before_replacing_anything(monkeypatch):
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q
    fakelib_int8_affine.install(monkeypatch)
    targ = [Q.QuantNConv2d, Q.QuantNLinear]

    def refused(model, match, **kw):
        before = [type(m) for m in model]
        with pytest.raises(_lib.DfqError, match=match):
            int8.convert_affine(model, _graph(model), targ, **kw)
        assert [type(m) for m in model] == before

    model = _affine_model()
    with torch.no_grad():
        model[4].weight.add_(1e-3 * torch.randn_like(model[4].weight))        # no longer on a grid
    refused(model, r"layer 4: its weights are not on a 8-bit min / max grid .*run quantize_targ_layer first")
    refused(_affine_model(), r"layer 0: weight codes of 9 bits", bits_weight=9)
    model = _affine_model()
    model[2].quant.num_bits = 16
    refused(model, r"layer 2: activation codes of 16 bits")
    model = _affine_model()
    model[4].quant.running_max.fill_(float("nan"))
    refused(model, r"layer 4: activation range")
    grouped = nn.Sequential(Q.QuantNConv2d(8, 16, 3), Q.QuantNConv2d(16, 16, 1, groups=2))
    refused(grouped, r"layer 1 cannot run in int8: needs groups == 1 or depthwise")
    wide = nn.Sequential(Q.QuantNConv2d(16384, 2, 3))                       # K = 9 * 16384 = 147456
    refused(wide, r"layer 0: K = kh \* kw \* C / groups = 147456 reaches 131072")
    plain = nn.Sequential(nn.Conv2d(4, 4, 1))
    with pytest.raises(_lib.DfqError, match="no `quant` observer"):
        int8.convert_affine(plain, _graph(plain), [nn.Conv2d])
    reflect = nn.Sequential(Q.QuantNConv2d(4, 4, 3, padding=1))
    reflect[0].padding_mode = "reflect"
    refused(reflect, "zero padding only")


def test_fake_library_refuses_what_the_kernels_refuse(monkeypatch):
    """The ABI's refusals as the fake states them: bits > 8 and K >= 131072 unsupported, non-finite constants an argument
    error (the -m gpu tests check the library itself)."""
    import ctypes as C
    from dfq_b200 import _lib, int8
    fake = fakelib_int8_affine.install(monkeypatch)
    layer = int8.AffineInt8Conv2d.from_conv(_affine_model()[0], -1.0, 1.0)
    g = layer._geometry(1, 4, 4)
    x = torch.zeros(1, 3, 4, 4)
    q, S = torch.zeros(16 * 16, dtype=torch.int8), torch.zeros(16, dtype=torch.int32)
    assert fake.dfq_i8_affine_quantize(C.c_void_p(x.data_ptr()), C.c_void_p(q.data_ptr()), C.c_void_p(S.data_ptr()),
                                       1, 3, 4, 4, 16, C.c_float(-1), C.c_float(1), 9, None) == -2
    k = np.zeros(1, _lib.I8_AFFINE_DT)
    k[0] = (1.0, math.inf, 0.0, 0.0)
    y = torch.zeros(1, 16, 4, 4)
    assert fake.dfq_i8_affine_conv(q.data_ptr(), S.data_ptr(), layer.weight_codes.data_ptr(), layer.tap_table.data_ptr(),
                                   k.ctypes.data, None, y.data_ptr(), None, g.ctypes.data, None) == -1
