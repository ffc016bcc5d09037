"""-m gpu: the drop-in entry points (merge_batchnorm -> create_relation -> cross_layer_equalization -> bias_correction
-> quantize_targ_layer) on seeded models of the reference's architectures, real CUDA library vs

  (1) the same host code executed with the numpy oracle (tests/fakelib.py): bit-exact for BN fold, equalization
      (weights, biases, fake_weight/fake_bias, S, sweep count) and the 8-bit weight codes; 1e-5 normwise for bias
      correction;
  (2) the committed fixtures produced by the reference itself (tests/golden/ref_*.npz): 1e-5 normwise up to the
      equalization, relaxed downstream (the reference's host sqrt is not correctly rounded and bias correction is
      ill-conditioned in the last bit of the weights, DESIGN.md section 6).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import fakelib
from dfq_b200 import workload

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TARG = [nn.Conv2d, nn.Linear]


def _nw(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def _pipeline(name, seed, stages, signed=False):
    from dfq_b200 import dfq
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph, bottoms, _ = workload.build_graph(topo, seed=seed)
    snaps = {}

    def snap(tag):
        d = {}
        for i, k in enumerate(graph):
            m = graph[k]
            if type(m) in TARG:
                d["w%d" % i] = m.weight.detach().cpu().numpy().copy()
                if m.bias is not None:
                    d["b%d" % i] = m.bias.detach().cpu().numpy().copy()
            if hasattr(m, "fake_bias") and not isinstance(m, str):
                d["fb%d" % i] = m.fake_bias.cpu().numpy().copy(); d["fw%d" % i] = m.fake_weight.cpu().numpy().copy()
        snaps[tag] = d

    LT.merge_batchnorm(None, graph, bottoms, TARG); snap("fold")
    rels = create_relation(graph, bottoms, TARG, delete_single=(name == "ssd"))
    dfq.cross_layer_equalization(graph, rels, TARG, converge_thres=2e-7, signed=signed); snap("cle")
    snaps["n_sweeps"] = dfq.cross_layer_equalization.last_result.n_sweeps
    snaps["S"] = [r.S.cpu().numpy().copy() for r in rels]
    if "bc" in stages:
        dfq.bias_correction(graph, bottoms, TARG, signed=signed); snap("bc")
    if "q" in stages:
        LT.quantize_targ_layer(graph, 8, 16, TARG); snap("q")
    return snaps, graph, rels


@pytest.mark.parametrize("name,seed", [("resnet18", 3), ("mobilenetv2", 0), ("deeplab", 5), ("ssd", 7)])
def test_pipeline_cuda_vs_oracle_executor(name, seed, monkeypatch):
    stages = ("bc", "q")
    real, _, _ = _pipeline(name, seed, stages)
    with monkeypatch.context() as mp:
        fakelib.install(mp)
        ref, _, _ = _pipeline(name, seed, stages)
    assert real["n_sweeps"] == ref["n_sweeps"]
    for tag in ("fold", "cle"):
        for k, v in ref[tag].items():
            assert np.array_equal(real[tag][k], v), "%s %s %s: normwise %g" % (name, tag, k, _nw(real[tag][k], v))
    for a, b in zip(real["S"], ref["S"]):
        assert np.array_equal(a, b)
    for k, v in ref["bc"].items():
        assert _nw(real["bc"][k], v) < 1e-5, (name, "bc", k, _nw(real["bc"][k], v))
    for k, v in ref["q"].items():
        if k.startswith("w"):
            assert np.array_equal(real["q"][k], v), (name, "q", k)        # weights untouched by BC: codes bit-exact
        else:
            assert _nw(real["q"][k], v) < 1e-4, (name, "q", k)


@pytest.mark.parametrize("name,seed,signed", [("resnet18", 3, False), ("mobilenetv2", 0, False), ("mobilenetv2", 0, True),
                                              ("deeplab", 5, False), ("ssd", 7, False)])
def test_pipeline_cuda_vs_reference_fixture(name, seed, signed):
    """Every committed reference pipeline fixture (tools/make_golden.py ran dfq.py on the seeded model): unsigned and
    signed MobileNetV2, ResNet-18, DeepLab-v3+ (cat / interpolate topology) and SSD-lite (delete_single=True chains)."""
    gold = np.load(os.path.join(GOLD, "ref_%s%s.npz" % (name, "_signed" if signed else "")))
    real, graph, rels = _pipeline(name, seed, ("bc",), signed=signed)
    keys = list(graph.keys())
    # the fixture's host computed sqrt with MKL VML (faithful, not correctly rounded); the last sweeps of the reference
    # straddle its 2e-7 threshold by ~1 % (SURVEY H2), so the count may differ by one - the weights do not (1e-5)
    assert abs(real["n_sweeps"] - int(gold["n_sweeps"])) <= 1
    assert np.array_equal(np.array([[keys.index(a), keys.index(b), keys.index(c)] for a, b, c in (r.get_idxs() for r in rels)]),
                          gold["relations"])
    for i, S in enumerate(real["S"]):
        assert _nw(S, gold["S_%d" % i]) < 1e-5
    tl = [i for i, k in enumerate(keys) if type(graph[k]) in TARG]
    for tag in ("fold", "cle"):
        for j, i in enumerate(tl):
            w = real[tag]["w%d" % i]
            assert abs(np.abs(w).max() - gold[tag + "_w_absmax"][j]) <= 1e-5 * gold[tag + "_w_absmax"][j]
            # ... and the fp64 sum of the whole tensor (the fixtures hold max|w|, the sum and a sha256 per tensor, not the
            # tensors): 1e-5 of sum|w|, i.e. a systematic error of 1e-5 in any row or column would show
            assert abs(w.astype(np.float64).sum() - gold[tag + "_w_sum"][j]) <= 1e-5 * np.abs(w).astype(np.float64).sum(), (tag, j)
            if "%s_bias_%d" % (tag, i) in gold.files:
                assert _nw(real[tag]["b%d" % i], gold["%s_bias_%d" % (tag, i)]) < 1e-5
        for k in real[tag]:
            if k.startswith("fb"):
                assert _nw(real[tag][k], gold["%s_fb_%s" % (tag, k[2:])]) < 1e-5
                assert _nw(real[tag]["fw" + k[2:]], gold["%s_fw_%s" % (tag, k[2:])]) < 1e-5
    for j, i in enumerate(tl):
        if "bc_bias_%d" % i in gold.files:
            assert _nw(real["bc"]["b%d" % i], gold["bc_bias_%d" % i]) < 5e-2


def test_quant_modules_forward_on_gpu_matches_torch_eager_reference_chain():
    """Activations: the reference runs quantize.py:70-74 on CUDA tensors, where PyTorch's div_(python_float) is a
    multiply by the fp32 reciprocal.  The kernel must match that op chain executed by PyTorch CUDA eager bit for bit."""
    from dfq_b200.utils import quantize as Q
    torch.manual_seed(0)
    x = torch.randn(64, 32, 28, 28, device="cuda") * 2
    for bits, mn, mx in ((8, -2.11790393, 2.64), (8, 0.0, 5.3), (4, -1.0, 1.0), (16, -3.3, 7.7)):
        qmax = 2. ** bits - 1.
        scale = max((mx - mn) / qmax, 1e-8)
        ref = x.clone().add_(-mn).div_(scale).clamp_(0., qmax).round_().mul_(scale).add_(mn)
        got = Q.quantize(x, bits, mn, mx)
        assert torch.equal(got, ref), (bits, mn, mx, (got != ref).sum().item())
    # observer in eval mode with set ranges; no host sync is needed but the result is the same
    qm = Q.QuantMeasure().cuda().eval()
    qm.running_min.fill_(-2.11790393); qm.running_max.fill_(2.64)
    mn, mx = float(qm.running_min), float(qm.running_max)
    scale = max((mx - mn) / 255., 1e-8)
    ref = x.clone().add_(-mn).div_(scale).clamp_(0., 255.).round_().mul_(scale).add_(mn)
    assert torch.equal(qm(x), ref)
    # update_stat: running range follows the per-sample extrema (quantize.py:103-107)
    qm2 = Q.QuantMeasure(True).cuda().eval()
    _ = qm2(x)
    want_max = x.view(64, -1).max(-1)[0].mean(); want_min = x.view(64, -1).min(-1)[0].mean()
    assert abs(float(qm2.running_max) - float(want_max)) <= 1e-6 * abs(float(want_max))
    assert abs(float(qm2.running_min) - float(want_min)) <= 1e-6 * abs(float(want_min))
    # Quant layers run and agree with the eager chain built from their own quantized operands
    conv = Q.QuantConv2d(32, 16, 3, padding=1).cuda().eval()
    conv.quant.running_min.fill_(-6.); conv.quant.running_max.fill_(6.)
    y = conv(x[:4])
    w = conv.weight.detach()
    wmn, wmx = float(w.min()), float(w.max()); ws = max((wmx - wmn) / 255., 1e-8)
    qw = w.clone().add_(-wmn).div_(ws).clamp_(0., 255.).round_().mul_(ws).add_(wmn)
    xs = max(12. / 255., 1e-8)
    qx = x[:4].clone().add_(6.).div_(xs).clamp_(0., 255.).round_().mul_(xs).add_(-6.)
    b = conv.bias.detach()
    bmn, bmx = b.min(), b.max()
    bs = (bmx - bmn) / 65535.
    qb = b.clone().add_(-bmn).div_(bs).clamp_(0., 65535.).round_().mul_(bs).add_(bmn)
    ref = torch.nn.functional.conv2d(qx, qw, qb, 1, 1)
    assert torch.allclose(y, ref, rtol=1e-5, atol=1e-5)


def test_graph_calibration_matches_separate_calls_on_gpu():
    from dfq_b200 import dfq
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    topo = workload.load_topology(os.path.join(GOLD, "topology_mobilenetv2.json"))
    ga, ba, _ = workload.build_graph(topo, seed=21)
    gb, bb, _ = workload.build_graph(topo, seed=21)
    LT.merge_batchnorm(None, ga, ba, TARG)
    rels = create_relation(ga, ba, TARG)
    dfq.cross_layer_equalization(ga, rels, TARG)
    dfq.bias_correction(ga, ba, TARG)
    LT.quantize_targ_layer(ga, 8, 16, TARG)
    cal = GraphCalibration(gb, bb, TARG)
    res = cal.run(equalize=True, correction=True, quantize_bits=(8, 16))
    assert res.n_sweeps == dfq.cross_layer_equalization.last_result.n_sweeps
    for ra, rb in zip(rels, cal.relations):
        assert np.array_equal(ra.S.numpy(), rb.S.numpy())
    for ma, mb in zip(ga.values(), gb.values()):
        if type(ma) in TARG:
            assert np.array_equal(ma.weight.detach().numpy(), mb.weight.detach().numpy())
            assert np.array_equal(ma.bias.detach().numpy(), mb.bias.detach().numpy())


def test_native_host_staging_equals_the_tensor_library_path(monkeypatch):
    """Session.upload()/download() gather and scatter the model with dfq_host_copy_segments (pipelined in parts with the
    H2D copy): same arena image and same results as the per-tensor torch path, also when a parameter's .data was re-pointed
    or made non-contiguous between two runs (the addresses are read per call; a non-contiguous tensor falls back)."""
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200 import engine as engine_mod
    from dfq_b200.engine import Session
    topo = workload.load_topology(os.path.join(GOLD, "topology_mobilenetv2.json"))
    ga, ba, _ = workload.build_graph(topo, seed=33)
    gb, bb, _ = workload.build_graph(topo, seed=33)
    cal_a = GraphCalibration(ga, ba, TARG)
    calls = []
    orig = Session._host_copy

    def spy(self, x, which, direction, i0=0, i1=None):
        ok = orig(self, x, which, direction, i0, i1)
        calls.append((which, ok))
        return ok
    monkeypatch.setattr(Session, "_host_copy", spy)
    monkeypatch.setattr(engine_mod, "_UPLOAD_PARTS", 3)                      # staged in parts, each followed by its H2D copy
    cal_a.upload()
    assert calls and all(ok for _, ok in calls) and 2 <= len(calls) <= 3
    image_native = cal_a.sess.arena.clone()
    cal_a.run_device(equalize=True, correction=True)
    cal_a.download()
    assert ("d2h", True) in calls
    monkeypatch.setattr(Session, "_host_copy", lambda self, *a, **k: False)  # the tensor-library path
    cal_b = GraphCalibration(gb, bb, TARG)
    cal_b.upload()
    xa, xb = cal_a.sess._transfer_lists(), cal_b.sess._transfer_lists()
    for (a, e) in xa["h2d_runs"]:
        assert torch.equal(image_native[a:e], cal_b.sess.arena[a:e])
    cal_b.run_device(equalize=True, correction=True)
    cal_b.download()
    for ma, mb in zip(ga.values(), gb.values()):
        if type(ma) in TARG:
            assert torch.equal(ma.weight, mb.weight) and torch.equal(ma.bias, mb.bias)
        if hasattr(ma, "fake_bias") and not isinstance(ma, str):
            assert torch.equal(ma.fake_bias, mb.fake_bias) and torch.equal(ma.fake_weight, mb.fake_weight)
    for ra, rb in zip(cal_a.relations, cal_b.relations):
        assert torch.equal(ra.S, rb.S)
    # second residency of the SAME plan after the caller re-pointed one weight and made another one non-contiguous
    monkeypatch.setattr(Session, "_host_copy", spy)
    convs = [m for m in ga.values() if type(m) == nn.Conv2d and m.weight.dim() == 4 and m.weight.size(1) > 1]
    convs[0].weight.data = convs[0].weight.data.clone()
    w = convs[1].weight.data
    convs[1].weight.data = w.permute(1, 0, 2, 3).contiguous().permute(1, 0, 2, 3)   # same values, non-contiguous
    assert not convs[1].weight.is_contiguous()
    expect_w0, expect_w1 = convs[0].weight.detach().clone(), convs[1].weight.detach().clone()
    del calls[:]
    cal_a.upload()
    assert any(not ok for _, ok in calls)                                    # fell back for the non-contiguous part
    la, lb = cal_a._layer[[k for k in ga if ga[k] is convs[0]][0]], cal_a._layer[[k for k in ga if ga[k] is convs[1]][0]]
    for li, ew in ((la, expect_w0), (lb, expect_w1)):
        l = cal_a.sess.layer(li)
        n = l["rows"] * l["cols"] * l["kk"]
        assert torch.equal(cal_a.sess.arena[l["w_off"]: l["w_off"] + n].cpu(), ew.contiguous().reshape(-1))


def test_relations_in_arbitrary_order_use_the_per_relation_path():
    """A hand-written relation list that is NOT in forward chain order must still follow dfq.py's Gauss-Seidel order."""
    from dfq_b200 import dfq
    from dfq_b200.utils.relation import Relation
    from oracle import dfq_oracle as O
    torch.manual_seed(3)
    convs = [nn.Conv2d(8, 16, 3, bias=True), nn.Conv2d(16, 12, 3, bias=True), nn.Conv2d(12, 10, 3, bias=False)]
    bns = [nn.BatchNorm2d(16), nn.BatchNorm2d(12)]
    for bn in bns:
        bn.register_buffer("fake_weight", torch.rand(bn.num_features) + 0.5)
        bn.register_buffer("fake_bias", torch.randn(bn.num_features))
    graph = {0: convs[0], 1: bns[0], 2: convs[1], 3: bns[1], 4: convs[2]}
    rels = [Relation(2, 4, 3), Relation(0, 2, 1)]          # backward order
    layers = [O.OLayer(c.weight.detach().numpy().copy(), None if c.bias is None else c.bias.detach().numpy().copy()) for c in convs]
    obns = [(b.fake_weight.numpy().copy(), b.fake_bias.numpy().copy()) for b in bns]
    n_ref, _ = O.cross_layer_equalization(layers, obns, [O.ORelation(1, 2, 1), O.ORelation(0, 1, 0)])
    dfq.cross_layer_equalization(graph, rels, [nn.Conv2d])
    assert dfq.cross_layer_equalization.last_result.n_sweeps == n_ref
    for c, l in zip(convs, layers):
        assert np.array_equal(c.weight.detach().numpy(), l.w)
        if l.b is not None:
            assert np.array_equal(c.bias.detach().numpy(), l.b)


def test_traced_torchvision_resnet18_calibrates_end_to_end():
    """No reference tracer in the loop: torch.fx graph (dfq_b200.trace) of a torchvision ResNet-18 -> one-residency
    calibration; equal to the drop-in calls run one after the other on an identical copy, and the model still runs."""
    tv = pytest.importorskip("torchvision")
    import copy
    from dfq_b200 import dfq
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    torch.manual_seed(0)
    ma = tv.models.resnet18().eval()
    for m in ma.modules():                      # non-trivial BN statistics
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.data.uniform_(0.5, 1.5); m.bias.data.normal_(0, 0.2)
    mb = copy.deepcopy(ma)
    x = torch.randn(2, 3, 64, 64)
    y0 = ma(x)
    ga, ba = trace_graph(ma)
    LT.merge_batchnorm(ma, ga, ba, TARG)
    rels = create_relation(ga, ba, TARG)
    dfq.cross_layer_equalization(ga, rels, TARG)
    dfq.bias_correction(ga, ba, TARG)
    gb, bb = trace_graph(mb)
    cal = GraphCalibration(gb, bb, TARG)
    res = cal.run(equalize=True, correction=False)
    assert res.n_sweeps == dfq.cross_layer_equalization.last_result.n_sweeps and len(cal.relations) == len(rels) == 8
    # equalization alone leaves the function unchanged (scaling is absorbed by ReLU's positive homogeneity)
    assert torch.allclose(mb(x), y0, rtol=1e-3, atol=1e-3)
    for ra, rb in zip(rels, cal.relations):
        assert np.array_equal(ra.S.numpy(), rb.S.numpy())


def test_resnet18_activation_ranges_over_64_images():
    """BASELINE configs[2]: ResNet-18 with QuantN* layers, observers driven in update_stat mode over 64 synthetic images
    (4 batches of 16, clamp(N(0,1)) like the reference's fallback data).  Every observer's running_min/max must equal the
    statistic of quantize.py:103-107 (per-sample max -> batch mean -> running max) computed by plain torch on the very tensors
    the observers saw, and the device-resident path must never have synchronised to do so."""
    tv = pytest.importorskip("torchvision")
    from dfq_b200.improve_dfq import set_update_stat
    from dfq_b200.utils.quantize import QuantMeasure, QuantNConv2d, QuantNLinear
    torch.manual_seed(0)
    model = tv.models.resnet18().eval()

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d:
                q = QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation, ch.groups,
                                 ch.bias is not None)
                q.weight.data.copy_(ch.weight.data)
                if ch.bias is not None:
                    q.bias.data.copy_(ch.bias.data)
                setattr(parent, name, q)
            elif type(ch) is nn.Linear:
                q = QuantNLinear(ch.in_features, ch.out_features, ch.bias is not None)
                q.weight.data.copy_(ch.weight.data); q.bias.data.copy_(ch.bias.data)
                setattr(parent, name, q)
            else:
                swap(ch)
    swap(model)
    model = model.cuda().eval()
    layers = [m for m in model.modules() if isinstance(m, (QuantNConv2d, QuantNLinear))]
    assert len(layers) == 21
    set_update_stat(model, [QuantMeasure], True)
    ref = {id(l): [torch.zeros((), device="cuda"), torch.zeros((), device="cuda")] for l in layers}

    def pre_hook(mod, args):
        x = args[0].detach()
        b = x.size(0)
        mx = x.reshape(b, -1).max(-1)[0].mean(); mn = x.reshape(b, -1).min(-1)[0].mean()
        ref[id(mod)][0] = torch.minimum(ref[id(mod)][0], mn); ref[id(mod)][1] = torch.maximum(ref[id(mod)][1], mx)
    hooks = [l.register_forward_pre_hook(pre_hook) for l in layers]
    g = torch.Generator(device="cuda").manual_seed(1)
    with torch.no_grad():
        for _ in range(4):
            model(torch.randn(16, 3, 64, 64, device="cuda", generator=g).clamp_(-2.5, 2.5))
    for h in hooks:
        h.remove()
    for l in layers:
        mn, mx = float(l.quant.running_min), float(l.quant.running_max)
        rmn, rmx = float(ref[id(l)][0]), float(ref[id(l)][1])
        assert abs(mn - rmn) <= 1e-6 * max(1.0, abs(rmn)) and abs(mx - rmx) <= 1e-6 * max(1.0, abs(rmx)), (mn, rmn, mx, rmx)
    assert sum(1 for l in layers if float(l.quant.running_max) > 0) == len(layers)


def test_golden_ncnn_table_through_the_cuda_library(monkeypatch):
    """The reference's golden artefact through libdfq_sm90.so: BN fold (dfq_bn_fold), signed equalization to convergence
    (dfq_cle_run) and the per-tensor extrema of the export (dfq_minmax) run on the GPU on the bundled checkpoint; the 53
    weight-scale rows and 53 activation-scale rows of model_quant_relu_equal.table must come out to 1e-5 (the table was
    written by a host whose sqrt differs from IEEE in the last bit: S is only determined to ~1e-6, DESIGN.md section 4)."""
    import ncnn_table_case as case
    if case.checkpoint_path() is None:
        pytest.skip("checkpoint not staged: run __graft_entry__.build() with a readable reference checkout")
    got_w, gold_w, got_a, gold_a = case.run(monkeypatch)
    assert got_w.shape == gold_w.shape == (53,) and got_a.shape == gold_a.shape == (53,)
    ew, ea = np.abs(got_w / gold_w - 1).max(), np.abs(got_a / gold_a - 1).max()
    print("golden table through CUDA: weight rows %.3g, activation rows %.3g (max relative error)" % (ew, ea))
    assert ew < 1e-5 and ea < 1e-5, (ew, ea)


def export_round_trip(tmp_path, monkeypatch=None):
    """Shared with the CPU twin (tests/test_host_logic.py): calibrate a ResNet-18-shaped graph of QuantN layers, write the
    ncnn calibration table and the calibration state (export.py, SURVEY 8(f) rank 4), read both back."""
    from dfq_b200 import dfq, export
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
    topo = workload.load_topology(os.path.join(GOLD, "topology_resnet18.json"))
    graph, bottoms, _ = workload.build_graph(topo, seed=9, conv_cls=Q.QuantNConv2d, linear_cls=Q.QuantNLinear)
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    LT.merge_batchnorm(None, graph, bottoms, targ)
    rels = create_relation(graph, bottoms, targ)
    dfq.cross_layer_equalization(graph, rels, targ)
    dfq.bias_correction(graph, bottoms, targ)
    g = torch.Generator().manual_seed(1)
    layers = [m for m in graph.values() if type(m) in targ]
    for m in layers:                                       # observer ranges as set_quant_minmax / update_quant_range leave them
        m.quant.running_min.fill_(-float(torch.rand(1, generator=g)) - 0.1); m.quant.running_max.fill_(float(torch.rand(1, generator=g)) + 0.1)
    table = str(tmp_path / "model.table")
    names = ["conv_%d" % i for i in range(len(layers))]
    rows = export.write_ncnn_table(graph, table, targ, names)
    lines = [l.split() for l in open(table).read().strip().splitlines()]
    assert len(lines) == 2 * len(layers)
    for i, m in enumerate(layers):
        w = m.weight.detach()
        want_w = 128. / float(w.abs().max())
        assert lines[i][0] == names[i] + "_param_0" and len(lines[i]) == 1 + w.shape[0]          # one value per output channel
        assert all(abs(float(v) / want_w - 1) < 1e-6 for v in lines[i][1:]) and abs(rows[i][0] / want_w - 1) < 1e-6
        want_a = 128. / max(abs(float(m.quant.running_min)), abs(float(m.quant.running_max)))
        assert lines[len(layers) + i][0] == names[i] and abs(float(lines[len(layers) + i][1]) / want_a - 1) < 1e-6
    state_path = str(tmp_path / "calibration.pt")
    export.save_calibration(graph, rels, state_path)
    state = torch.load(state_path)
    keys = list(graph.keys())
    assert len(state["S"]) == len(rels) and all(torch.equal(a, r.S.cpu()) for a, r in zip(state["S"], rels))
    n_l = n_b = 0
    for i, k in enumerate(keys):
        m = graph[k]
        if type(m) in targ:
            assert torch.equal(state["layers"][i]["weight"], m.weight.detach().cpu()) and torch.equal(state["layers"][i]["bias"], m.bias.detach().cpu())
            n_l += 1
        elif hasattr(m, "fake_bias") and not isinstance(m, str):
            assert torch.equal(state["bn"][i]["fake_bias"], m.fake_bias.cpu()) and torch.equal(state["bn"][i]["fake_weight"], m.fake_weight.cpu())
            n_b += 1
    assert n_l == len(layers) == 21 and n_b == 20
    return len(lines)


def test_export_round_trip_on_cuda_results(tmp_path):
    """write_ncnn_table / save_calibration on a model calibrated by libdfq_sm90.so (convert_ncnn.py:178-201 format)."""
    assert export_round_trip(tmp_path) == 42
