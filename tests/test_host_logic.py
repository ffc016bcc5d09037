"""Host logic of the drop-in modules, end to end on the CPU: the product's graph walks, arena planning, descriptor
tables and write-back are executed with `tests/fakelib.py` (the numpy oracle behind the C-ABI signatures) and compared
with fixtures produced by running the REFERENCE on the same seeded models (tests/golden/ref_*.npz).

What this pins without a GPU: create_relation, merge_batchnorm pairing, relation/step/col_mode planning, the bias
correction recipe (find_prev_bn, cat/add merging, -delta forwarding, dependency levels), quantize_targ_layer task lists,
in-place write-back into the module parameters.  The -m gpu suite runs the same checks against the real library."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import fakelib
from dfq_b200 import workload

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _nw(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def run_pipeline_and_compare(name, seed, gold, tol=1e-5, quantize=True):
    from dfq_b200 import dfq
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph, bottoms, _ = workload.build_graph(topo, seed=seed)
    targ = [nn.Conv2d, nn.Linear]
    keys = list(graph.keys())
    pos = {k: i for i, k in enumerate(keys)}
    tl = [k for k in keys if type(graph[k]) in targ]
    assert np.array_equal(np.array([pos[k] for k in tl]), gold["targets"])

    import hashlib
    state = {"exact": True}

    def check(tag, tol_w):
        # Bias correction is ill-conditioned with respect to 1-ulp changes of the weights (DESIGN.md section 6): a
        # shifted zero level of the 8-bit grid moves every element's error by the same amount and the mat-vec sums it
        # over thousands of inputs.  The reference's own sqrt (MKL VML) is not correctly rounded, so downstream of the
        # equalization the strict 1e-5 check only applies when the equalized weights equal the fixture's bit for bit
        # (always the case on the machine that produced the fixture); otherwise 5e-2.
        tol = 1e-5 if (state["exact"] or tag in ("fold", "cle")) else 5e-2
        for j, k in enumerate(tl):
            w = graph[k].weight.detach().cpu().numpy()
            if tag == "cle" and hashlib.sha256(np.ascontiguousarray(w).tobytes()).hexdigest() != str(gold["cle_w_sha"][j]):
                state["exact"] = False
            assert abs(np.abs(w).max() - gold[tag + "_w_absmax"][j]) <= tol_w * gold[tag + "_w_absmax"][j], (tag, j)
            assert abs(w.astype(np.float64).sum() - gold[tag + "_w_sum"][j]) <= 10 * tol_w * np.abs(w).astype(np.float64).sum(), (tag, j)
            name_b = "%s_bias_%d" % (tag, pos[k])
            if name_b in gold.files:
                assert graph[k].bias is not None
                # stage "q": the biases sit on a 16-bit grid of their own range; a bias that was 1e-7 away (the bias
                # correction's tolerance) from a rounding boundary lands one step (range/65535) away from the fixture's
                tol_b = tol + (4.0 / 65535 if tag == "q" else 0.0)
                assert _nw(graph[k].bias.detach().cpu().numpy(), gold[name_b]) < tol_b, name_b
        for k in keys:
            if hasattr(graph[k], "fake_bias") and not isinstance(graph[k], str):
                assert _nw(graph[k].fake_bias.cpu().numpy(), gold["%s_fb_%d" % (tag, pos[k])]) < tol
                assert _nw(graph[k].fake_weight.cpu().numpy(), gold["%s_fw_%d" % (tag, pos[k])]) < tol

    LT.merge_batchnorm(None, graph, bottoms, targ)
    check("fold", 1e-6)
    rels = create_relation(graph, bottoms, targ)
    got = np.array([[pos[a], pos[b], pos[c]] for a, b, c in (r.get_idxs() for r in rels)], np.int64)
    assert np.array_equal(got, gold["relations"])
    dfq.cross_layer_equalization(graph, rels, targ, converge_thres=2e-7)
    assert dfq.cross_layer_equalization.last_result.n_sweeps == int(gold["n_sweeps"])
    for i, r in enumerate(rels):
        assert _nw(r.S.cpu().numpy(), gold["S_%d" % i]) < tol, "S_%d" % i
    check("cle", 1e-5)
    dfq.bias_correction(graph, bottoms, targ)
    check("bc", 1e-5)
    if quantize:
        LT.quantize_targ_layer(graph, 8, 16, targ)
        check("q", 2e-2)      # a 1-ulp difference before quantization may move a value by one 8-bit step
    return graph, bottoms, rels


def test_resnet18_pipeline_matches_reference_fixture(monkeypatch):
    fake = fakelib.install(monkeypatch, fakelib.torch_sqrt)
    gold = np.load(os.path.join(GOLD, "ref_resnet18.npz"))
    run_pipeline_and_compare("resnet18", 3, gold)
    assert fake.calls == ["dfq_bn_fold", "dfq_cle_run", "dfq_bias_correct", "dfq_quantize_tensors"]


@pytest.mark.timeout(900)
def test_mobilenetv2_pipeline_matches_reference_fixture(monkeypatch):
    fakelib.install(monkeypatch, fakelib.torch_sqrt)
    gold = np.load(os.path.join(GOLD, "ref_mobilenetv2.npz"))
    graph, bottoms, rels = run_pipeline_and_compare("mobilenetv2", 0, gold)
    assert len(rels) == 37


def test_relation_chains_and_delete_single():
    from dfq_b200.utils.relation import create_relation
    for name, n_rel, n_rel_ds in (("mobilenetv2", 37, None), ("resnet18", 8, 0), ("deeplab", 35, None), ("ssd", None, 42)):
        topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
        graph, bottoms, _ = workload.build_graph(topo, seed=1)
        targ = [nn.Conv2d, nn.Linear]
        rels = create_relation(graph, bottoms, targ)
        if n_rel is not None:
            assert len(rels) == n_rel, (name, len(rels))
        if n_rel_ds is not None:
            assert len(create_relation(graph, bottoms, targ, delete_single=True)) == n_rel_ds, name
        # forward chain order: the relation whose second is X precedes the relation whose first is X
        first_at = {r.get_idxs()[0]: i for i, r in enumerate(rels)}
        for i, r in enumerate(rels):
            if r.get_idxs()[1] in first_at:
                assert first_at[r.get_idxs()[1]] > i


def test_layer_equalization_entry_point_in_place(monkeypatch):
    fakelib.install(monkeypatch)
    from dfq_b200 import dfq
    from oracle import dfq_oracle as O
    torch.manual_seed(0)
    w1, w2, b1 = torch.randn(32, 16, 3, 3), torch.randn(24, 32, 3, 3), torch.randn(32)
    bw, bb = torch.rand(32) + 0.5, torch.randn(32)
    n = [t.clone().numpy() for t in (w1, w2, b1, bw, bb)]
    S_ref = O.layer_equalization(*n, signed=True)
    p1 = w1.data_ptr()
    r = dfq._layer_equalization(w1, w2, b1, bw, bb, signed=True)
    assert r[0] is w1 and r[1] is w2 and r[2] is b1 and w1.data_ptr() == p1
    for got, want in zip((w1, w2, b1, bw, bb, r[3]), n + [S_ref]):
        assert np.array_equal(got.numpy(), want)


def test_cross_layer_equalization_creates_bias_only_for_first_layers(monkeypatch):
    fakelib.install(monkeypatch)
    from dfq_b200 import dfq
    from dfq_b200.utils.relation import Relation
    c1, c2 = nn.Conv2d(4, 8, 3, bias=False), nn.Conv2d(8, 6, 3, bias=False)
    bn = nn.BatchNorm2d(8)
    bn.register_buffer("fake_weight", torch.rand(8) + 0.5); bn.register_buffer("fake_bias", torch.randn(8))
    graph = {1: c1, 2: bn, 3: c2}
    w1_param = c1.weight
    dfq.cross_layer_equalization(graph, [Relation(1, 3, 2)], [nn.Conv2d])
    assert c1.bias is not None and c1.bias.requires_grad is False and c2.bias is None   # dfq.py:91-92
    assert c1.weight is w1_param


def test_bias_absorption_and_clip(monkeypatch):
    fakelib.install(monkeypatch)
    from dfq_b200 import dfq
    from dfq_b200.utils.relation import Relation
    from oracle import dfq_oracle as O
    torch.manual_seed(2)
    c1, relu, c2 = nn.Conv2d(4, 8, 3, bias=True), nn.ReLU(), nn.Conv2d(8, 6, 3, bias=False)
    bn = nn.BatchNorm2d(8)
    bn.register_buffer("fake_weight", torch.rand(8) * 0.2); bn.register_buffer("fake_bias", torch.randn(8) + 0.5)
    graph = {1: c1, 2: bn, 3: relu, 4: c2}
    bottoms = {1: ["Data"], 2: [1], 3: [2], 4: [3]}
    c = O.bias_absorb_c(bn.fake_weight.numpy(), bn.fake_bias.numpy(), 3)
    wc = O.bias_absorb_wc(c2.weight.detach().numpy(), c, 8)
    b1 = c1.bias.detach().numpy().copy(); fb = bn.fake_bias.numpy().copy()
    dfq.bias_absorption(graph, [Relation(1, 4, 2)], bottoms, 3)
    assert np.allclose(c1.bias.detach().numpy(), b1 - c) and np.allclose(bn.fake_bias.numpy(), fb - c)
    assert np.allclose(c2.bias.detach().numpy(), wc, rtol=1e-5, atol=1e-6)
    with torch.no_grad():
        c2.weight.mul_(100)
    dfq.clip_weight(graph, range_clip=[-15, 15], targ_type=[nn.Conv2d])
    assert float(c2.weight.max()) <= 15 and float(c2.weight.min()) >= -15


def test_quantize_function_and_observer_follow_reference_fixture(monkeypatch):
    fakelib.install(monkeypatch)
    from dfq_b200.utils import quantize as Q
    ops = np.load(os.path.join(GOLD, "ref_ops.npz"))
    for bits in (8, 4, 16):
        for sym in (0, 1):
            x = torch.from_numpy(ops["q_%d_%d_in" % (bits, sym)].copy())
            y = Q.quantize(x, bits, float(x.min()), float(x.max()), symmetric=bool(sym))
            assert np.array_equal(y.numpy(), ops["q_%d_%d_out" % (bits, sym)])
    b = torch.from_numpy(ops["qimp_in"].copy())
    assert np.array_equal(Q.quantize(b, num_bits=16).numpy(), ops["qimp_out16"])
    assert np.array_equal(Q.quantize(b, num_bits=8).numpy(), ops["qimp_out8"])
    # in-place flavour
    x = torch.from_numpy(ops["q_8_0_in"].copy())
    y = Q.quantize(x, 8, float(x.min()), float(x.max()), inplace=True)
    assert np.array_equal(x.numpy(), ops["q_8_0_out"])
    # set_layer_bits quirk Q1: the activation bit width lands in update_stat, num_bits stays 8
    conv = Q.QuantNConv2d(3, 4, 3)
    Q.set_layer_bits({1: conv}, 6, 6, 16, [Q.QuantNConv2d])
    assert conv.quant.update_stat == 6 and conv.quant.num_bits == 8


def test_graph_calibration_equals_the_four_separate_calls(monkeypatch):
    """dfq_b200.calibrate.GraphCalibration (one staging, fused plan) == merge_batchnorm + create_relation +
    cross_layer_equalization + bias_correction + quantize_targ_layer called one after the other."""
    fake = fakelib.install(monkeypatch)
    from dfq_b200 import dfq
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    topo = workload.load_topology(os.path.join(GOLD, "topology_resnet18.json"))
    targ = [nn.Conv2d, nn.Linear]
    ga, ba, _ = workload.build_graph(topo, seed=11)
    gb, bb, _ = workload.build_graph(topo, seed=11)
    LT.merge_batchnorm(None, ga, ba, targ)
    rels = create_relation(ga, ba, targ)
    dfq.cross_layer_equalization(ga, rels, targ)
    dfq.bias_correction(ga, ba, targ)
    LT.quantize_targ_layer(ga, 8, 16, targ)
    cal = GraphCalibration(gb, bb, targ)
    fake.stats.clear()
    res = cal.run(equalize=True, correction=True, quantize_bits=(8, 16))
    # the fused plan's shortcuts were taken (and verified inside the fake): the fold pre-scanned every `second` layer, and the
    # correction took those layers' ranges from the column extrema the equalization left behind
    assert fake.stats.get("cols_ready", 0) == len(cal.relations) and fake.stats.get("hinted", 0) > 0
    assert res.n_sweeps == dfq.cross_layer_equalization.last_result.n_sweeps
    assert len(cal.relations) == len(rels)
    for ra, rb in zip(rels, cal.relations):
        assert np.array_equal(ra.S.numpy(), rb.S.numpy())
    for (ka, ma), (kb, mb) in zip(ga.items(), gb.items()):
        if type(ma) in targ:
            assert np.array_equal(ma.weight.detach().numpy(), mb.weight.detach().numpy())
            assert np.array_equal(ma.bias.detach().numpy(), mb.bias.detach().numpy())
        if isinstance(ma, nn.BatchNorm2d) and hasattr(ma, "fake_bias"):
            assert np.array_equal(ma.fake_bias.numpy(), mb.fake_bias.numpy())
            assert np.array_equal(ma.fake_weight.numpy(), mb.fake_weight.numpy())
            assert float(mb.weight.min()) == 1.0 and float(mb.running_var.max()) == 1.0 and mb.eps in (0, 1e-12)


@pytest.mark.parametrize("name,seed", [("resnet18", 3), ("mobilenetv2", 0)])
def test_set_quant_minmax_matches_reference_fixture(monkeypatch, name, seed):
    """Data-free activation ranges (layer_transform.py:347-609) on the full graphs: every layer observer and every
    functional-op observer (residual adds, the pooling mean) must get the reference's running_min / running_max."""
    fakelib.install(monkeypatch, fakelib.torch_sqrt)
    from dfq_b200 import dfq
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
    gold = np.load(os.path.join(GOLD, "ref_minmax_%s.npz" % name))
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph, bottoms, _ = workload.build_graph(topo, seed=seed, conv_cls=Q.QuantNConv2d, linear_cls=Q.QuantNLinear)
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    record = [tuple(x) for x in topo["tensor_ops"]]
    ops = []
    for _, op_name in record:
        ops.extend(Q.QuantMeasure(num_bits=8, momentum=0.1) for _ in range(int(op_name.split('_')[-1])))
    monkeypatch.setattr(LT, "module_tensor_op", LT.CustomTensorOP(ops, record))
    LT.merge_batchnorm(None, graph, bottoms, targ)
    rels = create_relation(graph, bottoms, targ)
    dfq.cross_layer_equalization(graph, rels, targ, converge_thres=2e-7)
    dfq.bias_correction(graph, bottoms, targ)
    LT.set_quant_minmax(graph, bottoms, verbose=False)
    n = 0
    for i, k in enumerate(graph):
        m = graph[k]
        if hasattr(m, "quant") and not isinstance(m, str):
            want = gold["layer_%d" % i]
            got = np.array([float(m.quant.running_min), float(m.quant.running_max)])
            assert np.allclose(got, want, rtol=3e-4, atol=1e-5, equal_nan=True), (i, got, want)   # downstream of the fp32-BLAS bias correction
            n += 1
    for j, qm in enumerate(ops):
        want = gold["op_%d" % j]
        got = np.array([float(qm.running_min), float(qm.running_max)])
        assert np.allclose(got, want, rtol=3e-4, atol=1e-5, equal_nan=True), ("op", j, got, want)
    assert n + len(ops) == len(gold.files)


def test_live_ncnn_table_through_the_product_host_path(monkeypatch):
    """The reference's checked-in calibration table reproduced by THIS package's entry points end to end (53 weight-scale
    rows and 53 activation-scale rows; tests/ncnn_table_case.py).  Arithmetic by the oracle-backed executor; the -m gpu twin
    in tests/test_gpu_pipeline.py runs the same case on libdfq_sm90.so."""
    import ncnn_table_case as case
    if case.checkpoint_path() is None:
        pytest.skip("MobileNetV2 checkpoint not staged in oracle/_ref")
    fakelib.install(monkeypatch, fakelib.torch_sqrt)
    got_w, gold_w, got_a, gold_a = case.run(monkeypatch)
    assert got_w.shape == gold_w.shape == (53,) and got_a.shape == gold_a.shape == (53,)
    assert np.abs(got_w / gold_w - 1).max() < 2e-6, np.abs(got_w / gold_w - 1).max()
    assert np.abs(got_a / gold_a - 1).max() < 5e-6, np.abs(got_a / gold_a - 1).max()


@pytest.mark.parametrize("name", ["resnet18", "mobilenetv2"])
def test_bias_correction_alone_against_reference_produced_numbers_cpu(name, monkeypatch):
    """CPU twin of tests/test_gpu_entrypoints.py::test_bias_correction_alone_against_reference_produced_numbers: the
    product's recipe/levels/write-back with the oracle-backed executor vs what the reference's bias_correction produced."""
    import test_gpu_entrypoints as T
    fakelib.install(monkeypatch)
    worst = T.run_bias_correction_against_reference_fixture(name)
    assert worst < 1e-5


def test_export_round_trip_cpu(tmp_path, monkeypatch):
    """CPU twin of tests/test_gpu_pipeline.py::test_export_round_trip_on_cuda_results (oracle-backed executor)."""
    import test_gpu_pipeline as T
    fakelib.install(monkeypatch)
    assert T.export_round_trip(tmp_path) == 42


def test_native_host_staging_through_a_cpu_session(monkeypatch):
    """Session.upload()/download() with the REAL dfq_host_copy_segments (the library loads without a GPU) attached to the
    oracle-backed fake: parts planning, the gather per part, the split download and the scatter give the same calibrated model
    as the per-tensor torch path - the CPU twin of test_gpu_pipeline.py::test_native_host_staging_equals_the_tensor_library_path."""
    import ctypes as C
    from dfq_b200 import _build, _lib, engine
    from dfq_b200.calibrate import GraphCalibration
    _build.build()
    real = C.CDLL(_lib.LIB_PATH)
    fn = real.dfq_host_copy_segments
    fn.argtypes = _lib.SIGNATURES["dfq_host_copy_segments"]
    fn.restype = C.c_int
    topo = workload.load_topology(os.path.join(GOLD, "topology_mobilenetv2.json"))
    targ = [nn.Conv2d, nn.Linear]
    ga, ba, _ = workload.build_graph(topo, seed=4)
    gb, bb, _ = workload.build_graph(topo, seed=4)
    fake = fakelib.install(monkeypatch)
    cal_b = GraphCalibration(gb, bb, targ)                 # tensor-library path (the fake has no host-copy entry)
    cal_b.run(equalize=True, correction=True)
    calls = []

    def spy(*a):
        calls.append(int(a[5]))                            # direction
        return fn(*a)
    fake.dfq_host_copy_segments = spy
    monkeypatch.setattr(engine, "_UPLOAD_PARTS", 3)
    cal_a = GraphCalibration(ga, ba, targ)
    parts = cal_a.sess._upload_parts(cal_a.sess._transfer_lists())
    up = cal_a.sess._transfer_lists()["h2d_bounds"]
    assert 2 <= len(parts) <= 3 and parts[0][0] == 0 and parts[-1][1] == len(up)
    assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))                       # contiguous, nothing skipped
    for i0, i1, runs in parts:                                                         # every mirror lies inside a run of its part
        for b in up[i0:i1]:
            assert any(a <= b.off and b.off + b.n <= e for a, e in runs)
    cal_a.run(equalize=True, correction=True)
    assert calls.count(0) == len(parts) and calls.count(1) == 1
    for ma, mb in zip(ga.values(), gb.values()):
        if type(ma) in targ:
            assert torch.equal(ma.weight, mb.weight) and torch.equal(ma.bias, mb.bias)
        if isinstance(ma, nn.BatchNorm2d) and hasattr(ma, "fake_bias"):
            assert torch.equal(ma.fake_bias, mb.fake_bias) and torch.equal(ma.fake_weight, mb.fake_weight)
            assert float(ma.weight.detach().min()) == 1.0 and float(ma.running_mean.abs().max()) == 0.0
    for ra, rb in zip(cal_a.relations, cal_b.relations):
        assert torch.equal(ra.S, rb.S)
