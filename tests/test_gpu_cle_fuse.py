"""-m gpu: k_cle_stack's first two sweeps in one pass (DFQ_LAYER_ROWS_READY) against its per-sweep path on identical input
bits, on both sides of its guard.  Each problem runs twice: with the deferred fold's row scan (the kernel fuses where the
guard accepts) and with a fold plan stripped of it (never fuses).  Weights, biases, BN vectors, S, the column extrema left
for the bias correction, sweeps per group and the exit state are bit-identical; the metric sums agree to rounding.  Which
problems fuse is predicted on the CPU by tests/fakelib_fuse.py's fuse_guard from the oracle's folded weights."""
import numpy as np
import pytest
import torch

import fakelib_fuse
import stack_cases as SC
from oracle import dfq_oracle as O
from test_gpu_engine import _bind_chains

pytestmark = pytest.mark.gpu


def _run(lay, one_group, params, scan_rows, monkeypatch):
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_CLE_STACK", "1")
    p = dict(SC.DEFAULT_PARAMS, **params)
    sess = Session()
    rels, groups, folds, _ = _bind_chains(sess, lay, one_group, p["signed"])
    cle = sess.plan_cle(rels, groups=groups)
    fold = sess.plan_bn_fold(folds, cle_plan=cle)
    assert fold["deferred"] and len(fold["rows_scanned"]) == len(lay)
    if not scan_rows:
        fold["ft"]["scan_rows"][:] = 0
        fold["rows_scanned"] = []
    sess.upload()
    sess.run_bn_fold(fold)
    res = sess.run_cle_plan(cle, s_range=p["s_range"], converge_thres=p["converge_thres"], converge_count=p["converge_count"],
                            signed=p["signed"], eps=p["eps"], max_sweeps=p["max_sweeps"], cols_ready=fold["scanned"])
    view = lambda off, n: sess.view(int(off), int(n)).cpu().numpy().copy()
    h = sess.cle_col_hints(cle, res)
    out = [view(o, sess.layer(r[0])["rows"]) for o, r in zip(cle["s_offs"], rels)]
    out += [view(a, n) for a, n in zip(h["colmin_off"], h["n_col"])] + [view(a, n) for a, n in zip(h["colmax_off"], h["n_col"])]
    out += [view(d[k], d["w"].shape[0]) for cl in lay for d in cl for k in ("fake_w_off", "fake_b_off")]
    sess.download()
    out += [d[k].numpy().copy() for cl in lay for d in cl for k in ("w", "bias")]
    return res, out


def _predict(lay_np, one_group, params):
    """fuse_guard on the oracle's fold of the input bits"""
    p = dict(SC.DEFAULT_PARAMS, **params)
    blocks = []
    for ci, cl in enumerate(lay_np):
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            w = [O.bn_fold(d["w"], d["bias"], d["gamma"], d["beta"], d["mean"], d["var"], d["bn_eps"])[0] for d in cl]
        blocks.append((0 if one_group else ci, w[0], w[1].reshape(w[1].shape[0], w[1].shape[1], -1)))
    return fakelib_fuse.fuse_guard(blocks, s_range=p["s_range"], eps=p["eps"], signed=p["signed"],
                                    converge_thres=p["converge_thres"], converge_count=p["converge_count"],
                                    max_sweeps=p["max_sweeps"])


def _compare(make, one_group, params, monkeypatch, nan=False):
    """make(): fresh chain layer dicts (identical bits on every call).  Returns the fused run's result."""
    lay_np = [[dict(((n, d[n].numpy().copy()) for n in SC.VECTORS), bn_eps=d["bn_eps"]) for d in cl] for cl in make()]
    fu, a = _run(make(), one_group, params, True, monkeypatch)
    ps, b = _run(make(), one_group, params, False, monkeypatch)
    assert ps.fused_sweeps == 0
    assert fu.fused_sweeps == (2 if _predict(lay_np, one_group, params) else 0)
    assert (fu.n_sweeps, fu.converged) == (ps.n_sweeps, ps.converged)
    assert np.array_equal(fu.group_sweeps, ps.group_sweeps), (fu.group_sweeps, ps.group_sweeps)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y, equal_nan=nan), i
    np.testing.assert_allclose(fu.diffs, ps.diffs, rtol=1e-12, atol=0)
    np.testing.assert_allclose(fu.last_diff, ps.last_diff, rtol=1e-12, atol=0)
    return fu


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_stack_cases_fused_equals_per_sweep(case, monkeypatch):
    """Every edge case of tests/stack_cases.py (9 to 93 sweeps, the count branch, max_sweeps, signed, clamps, eps, degenerate
    rows, BN edge cases): the fused run is the per-sweep run, and it fuses exactly where the guard predicts."""
    res = _compare(lambda: SC.chain_layers(case["chains"], case["seed"], case["edit"]), case["one_group"], case["params"],
                   monkeypatch, nan=case["nonfinite"])
    print(case["name"], "fused" if res.fused_sweeps else "per-sweep", list(res.group_sweeps))


def _recalibrated(blocks):
    """STACK_BLOCKS where the blocks in `blocks` carry the weights and biases one calibration left, behind an identity BN
    (gamma 1, beta 0, mean 0, var 1, eps 0: fold factor exactly 1, bias unchanged); the other blocks are fresh."""
    def make():
        lay = SC.chain_layers(SC.STACK_BLOCKS)
        layers, _, _, _, _ = SC.oracle_chains(
            [[dict(((n, d[n].numpy().copy()) for n in SC.VECTORS), bn_eps=d["bn_eps"]) for d in cl] for cl in lay], False)
        for b in blocks:
            for k, d in enumerate(lay[b]):
                ol = layers[2 * b + k]
                d["w"] = torch.from_numpy(ol.w.reshape(d["w"].shape).copy())
                d["bias"] = torch.from_numpy(ol.b.copy())
                n = d["w"].shape[0]
                d["gamma"], d["beta"], d["mean"], d["var"] = torch.ones(n), torch.zeros(n), torch.zeros(n), torch.ones(n)
                d["bn_eps"] = 0.0
        return lay
    return make


FRESH = lambda: SC.chain_layers(SC.STACK_BLOCKS)


@pytest.mark.parametrize("name,make,params,fused,sweeps", [
    ("default", FRESH, {}, True, None),
    ("recalibrated", _recalibrated(range(len(SC.STACK_BLOCKS))), {}, False, 1),
    ("one_recalibrated_among_fresh", _recalibrated([2]), {}, False, None),
    ("threshold_stops_after_sweep_1", FRESH, dict(converge_thres=1.0), False, 1),
    ("converge_count_1", FRESH, dict(converge_count=1), False, None),
    ("max_sweeps_1", FRESH, dict(max_sweeps=1), False, 1),
    ("max_sweeps_3", FRESH, dict(converge_thres=0.0, converge_count=3, max_sweeps=3), True, 3),
], ids=lambda v: v if isinstance(v, str) else None)
def test_guard_both_sides(name, make, params, fused, sweeps, monkeypatch):
    res = _compare(make, False, params, monkeypatch)
    assert res.fused_sweeps == (2 if fused else 0), name
    if sweeps is not None:
        assert set(res.group_sweeps.tolist()) == {sweeps}, (name, res.group_sweeps)
    if name == "one_recalibrated_among_fresh":
        assert res.group_sweeps[2] == 1 and min(np.delete(res.group_sweeps, 2)) >= 2, res.group_sweeps
