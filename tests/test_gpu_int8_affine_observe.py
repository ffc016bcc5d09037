"""The observed affine epilogue on the H100 (dfq_i8_affine_conv_observed, dfq_b200.int8.chain_affine in the reference's
evaluation state): y, codes and S against tests/int8_affine_observe_oracle.py bit for bit, the fake quantization against
QuantMeasure itself, the entry's refusals, and three models in the evaluation state chained against their per-layer
affine model."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import affine_observed_state
import int8_affine_chain_oracle as AC
import int8_affine_observe_oracle as AO
import int8_affine_oracle as A
from test_gpu_int8_affine import _fake_quantized_conv, _same_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-40, -1e-41], f32)
OFF = (0.0, 0.0, 0)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _launch(layer, xq, S, g, r=None, y=None, yq=None, S_out=None, out=(0.0, 0.0, 0), pre=NONE, post=NONE, obs=OFF,
            res=OFF):
    from dfq_b200 import _lib
    d = np.zeros(1, _lib.I8_AFFINE_EPILOGUE_DT)
    d[0] = tuple(0 if t is None else t.data_ptr() for t in (r, y, yq, S_out)) + tuple(out) + tuple(pre) + tuple(post)
    o = np.zeros(1, _lib.I8_AFFINE_OBSERVE_DT)
    o[0] = tuple(obs) + tuple(res)
    return _lib.load().dfq_i8_affine_conv_observed(_p(xq), _p(S), _p(layer.weight_codes),
                                                   _p(layer.tap_table) if layer.tap_table.numel() else None,
                                                   _lib.table_ptr(layer.constants), _p(layer.bias), _lib.table_ptr(d),
                                                   _lib.table_ptr(o), _lib.table_ptr(g), _lib.stream_ptr())


def _case(N, Cin, H, W, O, k, s, p, d, g=1, bits=8, obs_bits=8, res_bits=8, outputs="both", residual=True, seed=0,
          pre=(0.0, 6.0), post=NONE, oracle=True):
    from dfq_b200 import _lib, int8
    torch.manual_seed(seed)
    conv = _fake_quantized_conv(nn.Conv2d(Cin, O, k, s, p, d, g).cuda())
    bias = conv.bias.detach().cpu().numpy().copy()
    bias[:min(O, SPECIAL.size)] = SPECIAL[:min(O, SPECIAL.size)]
    with torch.no_grad():
        conv.bias.copy_(torch.from_numpy(bias))
    x = torch.randn(N, Cin, H, W, device="cuda") * 2
    layer = int8.AffineInt8Conv2d.from_conv(conv, f32(float(x.min()) * 0.8), f32(float(x.max()) * 0.8))
    xq, S, *_ = layer._input(x)
    geo = layer._geometry(N, H, W)
    OH, OW = int(geo[0]["OH"]), int(geo[0]["OW"])
    cpad = (O + 15) // 16 * 16
    y_pl, _ = layer.run(x)
    r = None
    if residual:
        rng = np.random.default_rng(seed + 1)
        rn = (rng.standard_normal((N, O, OH, OW)) * 3).astype(f32)
        rn.reshape(-1)[::97][:SPECIAL.size] = SPECIAL[:rn.reshape(-1)[::97].size]
        r = torch.from_numpy(rn).cuda()
    obs = (f32(-0.3), f32(4.1), obs_bits) if obs_bits else OFF
    res = (f32(-2.7), f32(3.3), res_bits) if res_bits else OFF
    out = (f32(-1.1), f32(5.5), bits)
    want_y, want_q = outputs in ("both", "y"), outputs in ("both", "codes", "codes_noS")
    y = torch.full((N, O, OH, OW), 7.25, device="cuda") if want_y else None
    yq = torch.full((N * OH * OW * cpad + 64,), 99, dtype=torch.int8, device="cuda") if want_q else None
    S_out = torch.full((N * OH * OW + 16,), -2 ** 31, dtype=torch.int32, device="cuda") if outputs in ("both", "codes") \
        else None
    _lib.check(_launch(layer, xq, S, geo, r, y, yq, S_out, out, pre, post, obs, res), "dfq_i8_affine_conv_observed")
    torch.cuda.synchronize()
    # the per-layer path in torch: clamp, QuantMeasure on both operands, the add, clamp, then the quantizer
    v_pl = AO.torch_value(y_pl, r, pre, post, obs if obs_bits else None, res if res_bits else None)
    q_pl, S_pl = A.act_codes(v_pl.cpu().numpy(), *out)
    if oracle:
        xo, _ = A.act_codes(x.cpu().numpy(), layer.act_min, layer.act_max, 8)
        wo, _ = A.weight_codes(conv.weight.detach().cpu().numpy(), layer.w_min, layer.w_scale, 8)
        terms = A.terms(xo, wo, conv.stride, conv.padding, conv.dilation, conv.groups)
        v_o, q_o, S_o = AO.observed(*terms, tuple(layer.constants[0]), bias, None if r is None else r.cpu().numpy(), pre,
                                    post, out, obs if obs_bits else None, res if res_bits else None)
    v_pl = v_pl.cpu().numpy()
    if want_y:
        got = y.cpu().numpy()
        nan = np.isnan(v_pl)
        assert np.array_equal(np.isnan(got), nan) and _same_bits(np.where(nan, 0, got), np.where(nan, 0, v_pl)), \
            "y vs QuantMeasure in torch"
        if oracle:
            assert _same_bits(got, v_o), "y vs oracle"
    if want_q:
        codes = yq.cpu().numpy()
        assert (codes[N * OH * OW * cpad:] == 99).all(), "past the codes"
        codes = codes[:N * OH * OW * cpad].reshape(N, OH, OW, cpad)
        assert np.array_equal(codes, AC.to_nhwc(q_pl)), "codes vs the quantizer of the per-layer value"
        if oracle:
            assert np.array_equal(codes, AC.to_nhwc(q_o)), "codes vs oracle"
    if S_out is not None:
        s = S_out.cpu().numpy()
        assert (s[N * OH * OW:] == -2 ** 31).all()
        assert np.array_equal(s[:N * OH * OW].reshape(N, OH, OW), S_pl)
        if oracle:
            assert np.array_equal(s[:N * OH * OW].reshape(N, OH, OW), S_o)


DENSE = [  # (N, Cin, H, W, O, k, s, p, d), obs bits, res bits
    ((2, 19, 9, 7, 1, 3, 1, 1, 1), 8, 8),
    ((2, 19, 9, 7, 15, 3, 1, 1, 1), 7, 0),
    ((1, 32, 15, 15, 16, 3, 2, 1, 1), 0, 6),
    ((3, 16, 7, 7, 17, 1, 1, 0, 1), 5, 4),
    ((2, 24, 10, 11, 63, 3, 1, 2, 2), 4, 0),
    ((2, 40, 8, 8, 64, 3, 1, 1, 1), 0, 3),
    ((1, 16, 12, 13, 65, 3, 2, 1, 1), 2, 2),
    ((2, 33, 9, 9, 130, 3, 1, 1, 1), 1, 8),
]


@pytest.mark.parametrize("case,ob,rb", DENSE, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_dense_observed_epilogue_bit_exact(case, ob, rb):
    _case(*case, obs_bits=ob, res_bits=rb, seed=sum(case))


DW = [  # (N, C, H, W, k, s, p, d), obs bits, res bits
    ((2, 15, 9, 7, 3, 1, 1, 1), 8, 8),
    ((2, 16, 8, 8, 3, 2, 1, 1), 3, 0),
    ((1, 17, 11, 9, 5, 1, 2, 1), 0, 5),
    ((2, 65, 7, 7, 3, 1, 2, 2), 6, 1),
    ((1, 130, 10, 10, 3, 2, 1, 1), 8, 7),
]


@pytest.mark.parametrize("case,ob,rb", DW, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_depthwise_observed_epilogue_bit_exact(case, ob, rb):
    N, Cn, H, W, k, s, p, d = case
    _case(N, Cn, H, W, Cn, k, s, p, d, g=Cn, obs_bits=ob, res_bits=rb, seed=sum(case))


@pytest.mark.parametrize("which", ["obs", "res", "both"])
@pytest.mark.parametrize("outputs", ["y", "codes", "codes_noS", "both"])
@pytest.mark.parametrize("depthwise", [False, True])
def test_observer_and_output_selection(which, outputs, depthwise):
    ob, rb = (8 if which != "res" else 0), (8 if which != "obs" else 0)
    if depthwise:
        _case(2, 40, 9, 9, 40, 3, 1, 1, 1, g=40, obs_bits=ob, res_bits=rb, outputs=outputs, seed=11)
    else:
        _case(2, 24, 9, 9, 80, 3, 1, 1, 1, obs_bits=ob, res_bits=rb, outputs=outputs, seed=12)


@pytest.mark.parametrize("bits", range(1, 9))
def test_every_observer_bit_width(bits):
    _case(1, 16, 6, 6, 20, 3, 1, 1, 1, bits=8, obs_bits=bits, res_bits=9 - bits, seed=bits, pre=NONE, post=(-1.0, 2.0))


def test_observer_without_residual():
    _case(2, 16, 7, 7, 24, 3, 1, 1, 1, obs_bits=8, res_bits=0, residual=False, seed=5)


def test_depthwise_grid_stride_loop():
    _case(16, 96, 112, 112, 96, 3, 1, 1, 1, g=96, obs_bits=8, res_bits=8, seed=13, oracle=False)


def test_fake_quantization_equals_quantmeasure():
    """The oracle's fq (the epilogue's) against QuantMeasure's own CUDA output on the same values, special values included."""
    from dfq_b200.utils.quantize import QuantMeasure
    rng = np.random.default_rng(3)
    v = np.concatenate([(rng.standard_normal(50000) * 4).astype(f32), SPECIAL, np.array([3e38, -3e38, 1e-45], f32)])
    for lo, hi, bits in ((-0.3, 4.1, 8), (-2.7, 3.3, 1), (0.0, 6.0, 5), (1e-3, 1e-3, 8)):
        q = QuantMeasure(num_bits=bits).cuda().eval()
        q.running_min.fill_(float(f32(lo))); q.running_max.fill_(float(f32(hi)))
        with torch.no_grad():
            got = q(torch.from_numpy(v).cuda()).cpu().numpy()
        want = AO.fq(v, (f32(lo), f32(hi), bits))
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan) and _same_bits(np.where(nan, 0, got), np.where(nan, 0, want))


def test_abi_refusals_leave_the_buffers_untouched():
    from dfq_b200 import int8
    conv = _fake_quantized_conv(nn.Conv2d(16, 8, 3, padding=1).cuda())
    layer = int8.AffineInt8Conv2d.from_conv(conv, -1.0, 1.0)
    g = layer._geometry(1, 4, 4)
    xq, S, *_ = layer._input(torch.randn(1, 16, 4, 4, device="cuda"))
    y, r = torch.full((128,), 3.5, device="cuda"), torch.zeros(128, device="cuda")
    yq, S_out = torch.full((256 + 16,), 99, dtype=torch.int8, device="cuda"), torch.full((16,), -7, dtype=torch.int32,
                                                                                            device="cuda")
    base = dict(r=r, y=y, yq=yq[:256], S_out=S_out, out=(-1.0, 1.0, 8), pre=NONE, post=NONE, obs=(-1.0, 1.0, 8),
                res=(-1.0, 1.0, 8))

    def call(**kw):
        a = dict(base)
        a.update(kw)
        return _launch(layer, xq, S, g, **a)

    refused = [
        (dict(y=None, yq=None, S_out=None), -1), (dict(yq=None), -1), (dict(pre=(1.0, 0.0)), -1),
        (dict(out=(-1.0, 1.0, 9)), -2), (dict(r=y), -1),
        (dict(obs=(0.0, 0.0, 0), res=(0.0, 0.0, 0)), -1), (dict(obs=(-1.0, 1.0, -1)), -1),
        (dict(res=(-1.0, 1.0, -3)), -1), (dict(obs=(-1.0, 1.0, 9)), -2), (dict(res=(-1.0, 1.0, 16)), -2),
        (dict(obs=(-1.0, math.inf, 8)), -1), (dict(res=(math.nan, 1.0, 8)), -1), (dict(obs=(-3e38, 3e38, 1)), -1),
        (dict(r=None), -1),
    ]
    for kw, rc in refused:
        assert call(**kw) == rc, kw
        torch.cuda.synchronize()
        assert (y == 3.5).all() and (yq == 99).all() and (S_out == -7).all(), kw
    assert call() == 0
    torch.cuda.synchronize()
    assert (yq[256:] == 99).all() and not (S_out == -7).any()


# ---- models in the reference's evaluation state ---------------------------------------------------------------------------
# (net, input size, functional-op observers, chain_affine(residual=True): fused adds, fused observers), as measured on an
# H100.
NETS = [("mobilenet_v2", 224, 21, 10, 21), ("resnet18", 224, 16, 8, 16), ("deeplab", 129, 30, 10, 28)]


@pytest.mark.parametrize("net,size,n_obs,adds,fused_obs", NETS, ids=[n[0] for n in NETS])
def test_evaluation_state_chained_equals_per_layer(net, size, n_obs, adds, fused_obs):
    from dfq_b200 import int8
    from dfq_b200.utils import layer_transform as LT
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state(net, size=size) as (model, qgraph, qtarg):
            ct = LT.module_tensor_op
            int8.convert_affine(model, qgraph, qtarg)
            chained, gm = int8.chain_affine(model), int8.chain_affine(model, residual=True)
            x = torch.randn(4, 3, size, size, device="cuda",
                            generator=torch.Generator(device="cuda").manual_seed(2)).clamp_(-2.5, 2.5)
            with torch.no_grad():
                ref = model(x)
                got = {"chained": chained(x), "residual": gm(x)}
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
            n_nodes = sum(1 for n in chained.graph.nodes if n.op == "call_module" and n.target.startswith("custom_tensor_op"))
            print("%s: observers %d, records %d, adds %d, fused observers %d %s" % (
                net, n_nodes, ct.num_op, len(gm.fused_adds), len(gm.fused_observers),
                sorted({w for _, w, _ in gm.fused_observers})))
            for k, v in got.items():
                assert torch.equal(ref.view(torch.int32), v.view(torch.int32)), k
            assert n_nodes == ct.len
            if n_obs is not None:
                assert (n_nodes, len(gm.fused_adds), len(gm.fused_observers)) == (n_obs, adds, fused_obs)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
