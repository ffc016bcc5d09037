"""GraphCalibration's absorption and clip flags without a GPU: the refusals, which relations absorb, and the ABI of
dfq_bias_correct_absorb_clip's relation table."""
import numpy as np
import pytest
import torch.nn as nn

from dfq_b200 import _lib, workload
from dfq_b200._lib import DfqError
from dfq_b200.calibrate import GraphCalibration
from dfq_b200.graphwalk import relu_between
from dfq_b200.utils.relation import create_relation
from absorb_clip_case import edge_topology

TARG = [nn.Conv2d, nn.Linear]


@pytest.mark.parametrize("n, clip", [(float("nan"), None), (float("inf"), None), (-float("inf"), None), (3, (1.0, -1.0)),
                                     (3, (float("nan"), 1.0)), (3, (-1.0, float("inf"))), (3, (-1e39, 1.0)), (3, (1.0,)),
                                     (3, "ab"), (3, 5.0)])
def test_refusals(n, clip):
    with pytest.raises(DfqError):
        GraphCalibration._check_flags(n, clip)


@pytest.mark.parametrize("n, clip", [(3, None), (0.0, (-15, 15)), (-2.5, (0.01, 0.01)), (3, [-0.05, 0.05])])
def test_accepted(n, clip):
    GraphCalibration._check_flags(n, clip)


def test_which_relations_absorb():
    """A torch.nn.ReLU on the walk from `second` back to `first` absorbs; no activation does not."""
    topo = edge_topology()
    g, b, _ = workload.build_graph(topo, seed=0)
    name = {id(m): k["key"] for k, m in zip(topo["nodes"], g.values()) if not isinstance(m, str)}
    got = [(name[r.get_idxs()[0]], name[r.get_idxs()[1]], relu_between(g, b, r.get_idxs()[1], r.get_idxs()[0]))
           for r in create_relation(g, b, TARG)]
    assert got == [("c0", "c1", True), ("c1", "c2", True), ("c2", "c3", True), ("c3", "c4", False)]
    keys = list(g)
    relu6 = next(k for k in keys if type(g[k]) == nn.ReLU6)
    second = next(k for k in keys if b[k] == [relu6])
    first = next(k for k in keys if name.get(k) == "c4")
    assert relu_between(g, b, second, first) is False          # ReLU6 does not count


def test_absorb_table_abi():
    assert _lib.ABSORB_DT.itemsize == _lib.ABSORB_SIZES[28][1] == 40
    lib = _lib.load(build_if_missing=False)
    assert lib.dfq_struct_size(28) == 40
    assert "dfq_bias_correct_absorb_clip" in _lib.SIGNATURES


def test_float_products_are_exact_in_double():
    """Why the correction kernels may accumulate `acc += (double)a * (double)b` or `fma(a, b, acc)` alike: the double
    product of two floats never rounds (24 + 24 significant bits), at any exponent two finite floats can have."""
    from fractions import Fraction
    rng = np.random.default_rng(5)
    a = np.concatenate([rng.standard_normal(4000).astype(np.float32),
                        np.array([3.4028235e38, 1.1754944e-38, 1e-45, -1e-45, 16777215.0, 0.1, -0.3], np.float32)])
    b = np.concatenate([rng.standard_normal(4000).astype(np.float32) * np.float32(1e-3),
                        np.array([3.4028235e38, 1e-45, 1e-45, 3.4028235e38, 16777213.0, 0.7, 1.1], np.float32)])
    for x, y in zip(a.tolist(), b.tolist()):
        assert Fraction(float(np.float64(x) * np.float64(y))) == Fraction(x) * Fraction(y)


def _separate(g, b, equalize, absorption, n, clip, correction, qbits):
    from dfq_b200 import dfq
    from dfq_b200.utils import layer_transform as LT
    LT.merge_batchnorm(None, g, b, TARG)
    rels = create_relation(g, b, TARG)
    if equalize:
        dfq.cross_layer_equalization(g, rels, TARG)
    if absorption:
        dfq.bias_absorption(g, rels, b, n)
    if clip is not None:
        dfq.clip_weight(g, list(clip), TARG)
    if correction:
        dfq.bias_correction(g, b, TARG)
    if qbits is not None:
        LT.quantize_targ_layer(g, qbits[0], qbits[1], TARG)


@pytest.mark.parametrize("name", ["edges", "stack"])
@pytest.mark.parametrize("kw", [dict(absorption=True, absorption_n=0.0), dict(clip_weight=(-0.05, 0.05)),
                                dict(absorption=True, absorption_n=-0.25, clip_weight=(-0.05, 0.05), quantize_bits=(8, 16)),
                                dict(absorption=True, absorption_n=0.0, clip_weight=(0.01, 0.01), correction=False),
                                dict(absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05), equalize=False)])
def test_plan_matches_separate_calls_on_the_host_twin(name, kw, monkeypatch):
    """GraphCalibration's plan on the oracle-backed twin of dfq_bias_correct_absorb_clip against the separate drop-in calls on
    the same stand-in: which relations absorb, the group slices of the dots (depthwise and 2-group seconds), the order in which
    the bias updates round (a middle layer is `second` of one absorbing relation and `first` of the next), that every
    layer is clipped (Data-fed first conv, Linear head) and that the correction sees the absorbed and clipped model."""
    import fakelib_absorb_clip
    from absorb_clip_case import topology
    fake = fakelib_absorb_clip.install(monkeypatch)
    topo = topology(name)
    ga, ba, _ = workload.build_graph(topo, seed=21)
    gb, bb, _ = workload.build_graph(topo, seed=21)
    _separate(ga, ba, kw.get("equalize", True), kw.get("absorption", False), kw.get("absorption_n", 3), kw.get("clip_weight"),
              kw.get("correction", True), kw.get("quantize_bits"))
    cal = GraphCalibration(gb, bb, TARG)
    cal.run(**kw)
    n_abs, clip_only, n_bc = fake.absorb_clip[-1]
    if kw.get("absorption"):
        want = sum(relu_between(gb, bb, r.get_idxs()[1], r.get_idxs()[0]) for r in cal.relations)
        assert n_abs == want > 0
    if kw.get("clip_weight") is not None:
        assert len(clip_only) + n_bc == sum(type(m) in TARG for m in gb.values()) and len(clip_only) > 0
    for ka, ma, mb in zip(ga, ga.values(), gb.values()):
        if type(ma) in TARG:
            assert np.array_equal(ma.weight.detach().numpy(), mb.weight.detach().numpy()), ("weight", ka)
            assert np.array_equal(ma.bias.detach().numpy(), mb.bias.detach().numpy()), ("bias", ka)
        if isinstance(ma, nn.BatchNorm2d) and hasattr(ma, "fake_bias"):
            assert np.array_equal(ma.fake_bias.numpy(), mb.fake_bias.numpy()), ("fake_bias", ka)


@pytest.mark.parametrize("kw", [dict(absorption=True, absorption_n=float("nan")), dict(absorption=True, absorption_n=1e39),
                                dict(absorption=True, absorption_n="three"), dict(clip_weight=(1.0, -1.0)),
                                dict(clip_weight=(float("nan"), 1.0)), dict(clip_weight=(-1e39, 1.0)), dict(clip_weight=(1.0,))])
def test_refusals_launch_nothing_on_the_host_twin(kw, monkeypatch):
    import fakelib_absorb_clip
    from absorb_clip_case import topology
    fake = fakelib_absorb_clip.install(monkeypatch)
    g, b, _ = workload.build_graph(topology("edges"), seed=2)
    cal = GraphCalibration(g, b, TARG)
    planned = list(fake.calls)                  # the constructor's planning queries
    with pytest.raises(DfqError):
        cal.run(**kw)
    assert fake.calls == planned and cal.sess.arena is None


def test_oracle_matches_the_reference_fixture():
    """The oracle's bias_absorb_c / bias_absorb_wc / clip_weight against the reference's bias_absorption and clip_weight
    (tests/golden/ref_absorb_clip.npz, tools/make_golden.py absorb_clip), relation by relation in the reference's order."""
    import os
    from absorb_clip_case import FIXTURE_CASES, topology
    from oracle import dfq_oracle as O
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_absorb_clip.npz"))
    for name, seed, n, (lo, hi) in FIXTURE_CASES:
        g, b, _ = workload.build_graph(topology(name), seed=seed)
        keys = list(g)
        G = lambda tag, kind, p: gold["%s_%s_%s_%d" % (name, tag, kind, p)]
        bias = {int(k[len(name) + 7:]): G("cle", "b", int(k[len(name) + 7:])).copy() for k in gold.files
                if k.startswith(name + "_cle_b_")}
        n_absorbing = 0
        for first, second, bn in gold[name + "_relations"]:
            fw, fb = G("cle", "fw", bn), G("cle", "fb", bn)
            if not relu_between(g, b, keys[second], keys[first]):
                assert np.array_equal(G("absorb", "fb", bn), fb)
                continue
            c = O.bias_absorb_c(fw, fb, n)
            n_absorbing += int(c.any())
            assert np.array_equal(G("absorb", "fb", bn), fb - c)
            bias[first] = bias[first] - c
            bias[second] = bias[second] + O.bias_absorb_wc(G("cle", "w", second), c, fw.size)
        assert n_absorbing > 0
        for p, v in bias.items():
            np.testing.assert_allclose(G("absorb", "b", p), v, rtol=1e-6, atol=1e-6)
        bites = 0
        for k in gold.files:
            if k.startswith(name + "_cle_w_"):
                p = int(k[len(name) + 7:])
                clipped = O.clip_weight(gold[k], lo, hi)
                assert np.array_equal(G("clip", "w", p), clipped)
                bites += int(not np.array_equal(clipped, gold[k]))
        assert bites > 1
