"""GraphCalibration with bias absorption and weight clipping (the mains' --absorption and --clip_weight) against the
separate dfq_b200 calls in the mains' order (main_cls.py:149-181): merge_batchnorm -> cross_layer_equalization ->
bias_absorption -> clip_weight -> bias_correction -> quantize_targ_layer.  Bit for bit, on both bias-correction kernels."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from absorb_clip_case import edge_topology
from dfq_b200 import workload

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TARG = [nn.Conv2d, nn.Linear]


def _topology(name):
    if name == "edges":
        return edge_topology()
    if name == "stack":
        return workload.stack_topology(3, channels=64)
    return workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))


def _separate(g, b, equalize, absorption, n, clip, correction, qbits, signed):
    from dfq_b200 import dfq
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    LT.merge_batchnorm(None, g, b, TARG)
    rels = create_relation(g, b, TARG)
    if equalize:
        dfq.cross_layer_equalization(g, rels, TARG, signed=signed)
    if absorption:
        dfq.bias_absorption(g, rels, b, n)
    if clip is not None:
        dfq.clip_weight(g, list(clip), TARG)
    if correction:
        dfq.bias_correction(g, b, TARG, signed=signed)
    if qbits is not None:
        LT.quantize_targ_layer(g, qbits[0], qbits[1], TARG)
    return rels


def _assert_same(ga, gb, rels_a, rels_b, check_s=True):
    for ra, rb in zip(rels_a, rels_b):
        if check_s:
            assert np.array_equal(ra.S.numpy(), rb.S.numpy())
    for ka, ma, mb in zip(ga, ga.values(), gb.values()):
        if type(ma) in TARG:
            assert np.array_equal(ma.weight.detach().numpy(), mb.weight.detach().numpy()), ("weight", ka)
            assert np.array_equal(ma.bias.detach().numpy(), mb.bias.detach().numpy()), ("bias", ka)
        if isinstance(ma, nn.BatchNorm2d) and hasattr(ma, "fake_bias"):
            assert np.array_equal(ma.fake_weight.numpy(), mb.fake_weight.numpy()), ("fake_weight", ka)
            assert np.array_equal(ma.fake_bias.numpy(), mb.fake_bias.numpy()), ("fake_bias", ka)


def _compare(topo, seed, **kw):
    from dfq_b200.calibrate import GraphCalibration
    ga, ba, _ = workload.build_graph(topo, seed=seed)
    gb, bb, _ = workload.build_graph(topo, seed=seed)
    equalize, correction = kw.get("equalize", True), kw.get("correction", True)
    absorption, n, clip = kw.get("absorption", False), kw.get("absorption_n", 3), kw.get("clip_weight")
    qbits, signed = kw.get("quantize_bits"), kw.get("signed", False)
    rels = _separate(ga, ba, equalize, absorption, n, clip, correction, qbits, signed)
    cal = GraphCalibration(gb, bb, TARG)
    cal.run(**kw)
    _assert_same(ga, gb, rels, cal.relations, check_s=equalize)
    return cal


# The seeded BNs have beta ~ N(0, 0.2) and gamma in [0.5, 1.5]: with the reference's N = 3, c = clamp(beta - 3 gamma, 0) is
# zero everywhere, so the tests also take N <= 0, where c is positive on about half of the channels or more.
FLAGS = [dict(absorption=True, absorption_n=0.0), dict(clip_weight=(-0.05, 0.05)),
         dict(absorption=True, absorption_n=-0.25, clip_weight=(-0.05, 0.05)), dict(absorption=True)]


@pytest.mark.parametrize("variant", ["engine", "stream"])
@pytest.mark.parametrize("name", ["mobilenetv2", "resnet18", "deeplab", "ssd", "stack", "edges"])
def test_flags_match_separate_calls(name, variant, monkeypatch):
    monkeypatch.setenv("DFQ_BC_STREAM", "1" if variant == "stream" else "0")
    topo = _topology(name)
    for i, flags in enumerate(FLAGS):
        for qbits in (None, (8, 16)):
            _compare(topo, 50 + i, quantize_bits=qbits, **flags)
    _compare(topo, 60, signed=True, absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05), quantize_bits=(8, 16))


@pytest.mark.parametrize("clip", [(-0.05, 0.05), (0.01, 0.01), (-15.0, 15.0), (-1e30, 1e30)])
def test_clip_ranges(clip):
    """A range that bites on most weights, lo == hi, the mains' range and one that clips nothing."""
    _compare(_topology("edges"), 7, absorption=True, absorption_n=0.0, clip_weight=clip, quantize_bits=(8, 16))
    _compare(_topology("resnet18"), 8, clip_weight=clip)


def test_absorption_rules_on_edges():
    """Exactly the relations with a torch.nn.ReLU between the layers absorb (not those without an activation): their
    `first` bias and BN fake_bias lose c, and only they.  (A ReLU6 is refused by the walk itself: see
    tests/test_calibrate_absorb_clip_host.py.)"""
    from dfq_b200.calibrate import GraphCalibration
    topo = _topology("edges")
    ga, ba, _ = workload.build_graph(topo, seed=3)
    gb, bb, _ = workload.build_graph(topo, seed=3)
    ca, cb = GraphCalibration(ga, ba, TARG), GraphCalibration(gb, bb, TARG)
    ca.run(correction=False)
    cb.run(correction=False, absorption=True, absorption_n=0.0)
    name = {id(m): k["key"] for k, m in zip(topo["nodes"], ga.values()) if not isinstance(m, str)}
    pairs, absorbed = [], []
    for rr, rb in zip(ca.relations, cb.relations):
        first, second, bn = rr.get_idxs()
        bn2 = rb.get_idxs()[2]
        pairs.append((name[first], name[second]))
        if not np.array_equal(ga[bn].fake_bias.numpy(), gb[bn2].fake_bias.numpy()):
            absorbed.append((name[first], name[second]))
            assert not np.array_equal(ga[first].bias.numpy(), gb[rb.get_idxs()[0]].bias.numpy())
    assert ("c3", "c4") in pairs
    assert absorbed == [("c0", "c1"), ("c1", "c2"), ("c2", "c3")]


def test_absorption_without_equalization():
    _compare(_topology("stack"), 4, equalize=False, absorption=True, absorption_n=0.0)
    _compare(_topology("edges"), 5, equalize=False, absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05),
             quantize_bits=(8, 16))
    _compare(_topology("resnet18"), 6, equalize=False, correction=False, absorption=True, absorption_n=0.0,
             clip_weight=(-0.05, 0.05))


def test_one_copy_each_way_and_no_host_sync(monkeypatch):
    """One H2D and one D2H per run(), and run_device itself never waits for the device."""
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200.engine import Session
    g, b, _ = workload.build_graph(_topology("resnet18"), seed=9)
    cal = GraphCalibration(g, b, TARG)
    calls = []
    orig = Session._host_copy

    def spy(self, x, which, direction):
        ok = orig(self, x, which, direction)
        calls.append((which, ok))
        return ok
    monkeypatch.setattr(Session, "_host_copy", spy)
    kw = dict(absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05), quantize_bits=(8, 16))
    cal.plan_absorption()
    cal.upload()
    torch.cuda.synchronize()
    syncs = []
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: syncs.append("device"))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", lambda self: syncs.append("stream"))
    torch.cuda.set_sync_debug_mode("error")        # any synchronising tensor-library call raises
    try:
        cal.run_device(**kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert syncs == []
    monkeypatch.undo()
    monkeypatch.setattr(Session, "_host_copy", spy)
    cal.download()
    arena = cal.sess.arena
    assert calls == [("h2d", True), ("d2h", True)]
    h2d0, d2h0 = cal.sess.h2d_bytes, cal.sess.d2h_bytes
    calls.clear()
    cal.run(**kw)
    assert calls == [("h2d", True), ("d2h", True)]
    assert cal.sess.arena is arena              # a second run plans nothing: the arena is not regrown on the device
    assert cal.sess.h2d_bytes == 2 * h2d0 and cal.sess.d2h_bytes == 2 * d2h0


@pytest.mark.parametrize("kw", [dict(absorption=True, absorption_n=float("nan")), dict(absorption=True, absorption_n=float("inf")),
                                dict(clip_weight=(1.0, -1.0)), dict(clip_weight=(float("nan"), 1.0)),
                                dict(clip_weight=(-1.0, float("inf"))), dict(clip_weight=(1.0,)), dict(clip_weight="ab")])
def test_refusals_before_any_launch(kw):
    from dfq_b200._lib import DfqError
    from dfq_b200.calibrate import GraphCalibration
    g, b, _ = workload.build_graph(_topology("edges"), seed=1)
    w0 = {k: m.weight.detach().clone() for k, m in g.items() if type(m) in TARG}
    cal = GraphCalibration(g, b, TARG)
    with pytest.raises(DfqError):
        cal.run(**kw)
    assert cal.sess.arena is None
    for k, w in w0.items():
        assert torch.equal(g[k].weight, w)


def test_matches_the_reference_fixture():
    """GraphCalibration with both flags against the reference's own merge_batchnorm -> cross_layer_equalization ->
    bias_absorption -> clip_weight -> bias_correction (tests/golden/ref_absorb_clip.npz, tools/make_golden.py
    absorb_clip): weights bit for bit, biases and BN vectors within the correction's 1e-5."""
    from absorb_clip_case import FIXTURE_CASES, topology
    from dfq_b200.calibrate import GraphCalibration
    gold = np.load(os.path.join(GOLD, "ref_absorb_clip.npz"))
    ulps = lambda a, b: int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max())
    for name, seed, n, clip in FIXTURE_CASES:
        # the equalization alone against the reference's: the clip may not add any difference to what it leaves
        g, b, _ = workload.build_graph(topology(name), seed=seed)
        GraphCalibration(g, b, TARG).run(correction=False)
        cle_ulps = {p: ulps(m.weight.detach().numpy(), gold["%s_cle_w_%d" % (name, p)])
                    for p, m in enumerate(g.values()) if type(m) in TARG}
        g, b, _ = workload.build_graph(topology(name), seed=seed)
        GraphCalibration(g, b, TARG).run(absorption=True, absorption_n=n, clip_weight=clip)
        for p, m in enumerate(g.values()):
            if type(m) in TARG:
                got = ulps(m.weight.detach().numpy(), gold["%s_clip_w_%d" % (name, p)])
                assert got <= cle_ulps[p], (name, p, got, cle_ulps)
                np.testing.assert_allclose(m.bias.detach().numpy(), gold["%s_bc_b_%d" % (name, p)], rtol=1e-5, atol=1e-5)
            elif isinstance(m, nn.BatchNorm2d) and hasattr(m, "fake_bias"):
                np.testing.assert_allclose(m.fake_weight.numpy(), gold["%s_bc_fw_%d" % (name, p)], rtol=1e-5, atol=1e-5)
                np.testing.assert_allclose(m.fake_bias.numpy(), gold["%s_bc_fb_%d" % (name, p)], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("variant", ["engine", "stream"])
def test_both_kernels_on_mixed_tile_kinds(variant, monkeypatch):
    """dfq_bias_correct_absorb_clip against the separate steps (raw-sum absorption, c subtracted, clamp, correction) in one
    session each, on the tile kinds of test_gpu_engine.py's correction grid: 3x3 dense rows, depthwise, > 512 columns,
    27-float rows, rows longer than a stage (TK_DIRECT), a Linear with 2048 columns and a 2-group layer."""
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_BC_STREAM", "1" if variant == "stream" else "0")
    g = torch.Generator().manual_seed(17)
    R = lambda *s: torch.randn(*s, generator=g)
    seconds = [R(48, 64, 3, 3) * 0.1, R(64, 1, 3, 3) * 0.3, R(36, 640, 1, 1) * 0.05, R(16, 3, 3, 3) * 0.4,
               R(6, 1200, 2, 2) * 0.02, R(8, 1153, 2, 2) * 0.05, R(16, 2048) * 0.02, R(12, 32, 3, 3) * 0.1]
    groups = [1, 64, 1, 1, 1, 1, 1, 2]
    lo, hi = -0.04, 0.04
    cases = []
    for w2, G in zip(seconds, groups):
        n = G * w2.shape[1]
        cases.append(dict(w1=R(n, 8), b1=R(n), w2=w2, b2=R(w2.shape[0]), fw=torch.rand(n, generator=g) + 0.4, fb=R(n) * 0.5))

    def build():
        sess = Session()
        L = []
        for c in cases:
            l1 = sess.add_layer(c["w1"].clone(), c["b1"].clone())
            l2 = sess.add_layer(c["w2"].clone(), c["b2"].clone())
            L.append((l1, l2, sess.bind(c["fw"].clone()), sess.bind(c["fb"].clone()), c["fw"].numel()))
        items = [dict(layer=l2, signed=False, level=0, next_bn_b_off=-1,
                      terms=[dict(bn_w_off=ow, bn_b_off=ob, n=n, relu=True, op="set")]) for _, l2, ow, ob, n in L]
        return sess, L, items
    # fused
    sa, La, items = build()
    at = sa.plan_absorb([(l1, l2, ow, ob) for l1, l2, ow, ob, _ in La])
    plan = sa.plan_bias_correct(items)
    sa.upload()
    sa.run_bias_correct_absorb_clip(plan, 8, absorb=at, absorb_n=0.0, clip=(lo, hi))
    # separate
    sb, Lb, items = build()
    cs = [sb.bind(torch.zeros(n)) for *_, n in Lb]
    raw = [dict(layer=l2, signed=False, level=0, next_bn_b_off=-1, raw_sum=True, add=True,
                terms=[dict(bn_w_off=co, bn_b_off=co, n=n, relu=False, op="set")]) for (_, l2, _, _, n), co in zip(Lb, cs)]
    plan_raw, plan_b = sb.plan_bias_correct(raw), sb.plan_bias_correct(items)
    sb.upload()
    for (l1, l2, ow, ob, n), co in zip(Lb, cs):
        c = (sb.view(ob, n) - 0.0 * sb.view(ow, n)).clamp(min=0)
        sb.view(co, n).copy_(c)
    sb.run_bias_correct_plan(plan_raw, 8)
    for (l1, l2, ow, ob, n), co in zip(Lb, cs):
        sb.view(sb.layer(l1)["bias_off"], n).sub_(sb.view(co, n))
        sb.view(ob, n).sub_(sb.view(co, n))
    for l in range(len(sb._layers)):
        x = sb.layer(l)
        sb.view(x["w_off"], x["rows"] * x["cols"] * x["kk"]).clamp_(lo, hi)
    sb.run_bias_correct_plan(plan_b, 8)
    for (a1, a2, aw, ab, n), (b1, b2, bw, bb, _) in zip(La, Lb):
        for la, lb in ((a1, b1), (a2, b2)):
            xa, xb = sa.layer(la), sb.layer(lb)
            size = xa["rows"] * xa["cols"] * xa["kk"]
            assert torch.equal(sa.view(xa["w_off"], size), sb.view(xb["w_off"], size))
            assert torch.equal(sa.view(xa["bias_off"], xa["rows"]), sb.view(xb["bias_off"], xb["rows"])), (variant, la)
        assert torch.equal(sa.view(ab, n), sb.view(bb, n))
