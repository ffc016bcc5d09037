"""-m gpu: the deferred fold's row scan of a PREFIX of every first conv (DfqFold.row_prefix, DfqLayer.rext_rows) and
k_cle_stack's guard from that prefix, against a full row scan (DFQ_ROW_PREFIX=0) and against the per-sweep path (no row scan),
on identical input bits.  Weights, biases, both layers' fake_weight / fake_bias, S, the column extrema left for the bias
correction, the correction's delta / E[x] / range, the row extrema scratch after the call, sweeps per group and the exit state
are bit-identical; fused_sweeps and bc_prepared agree.  DfqCleResult.rows_streamed shows which way the kernel went:
the prefix decided (rows streamed in the fused pass), the prefix left a group undecided (the kernel scanned the rest and the
full guard decided), or the host did not let the guard use the prefix."""
import numpy as np
import pytest
import torch

import stack_cases as SC
from test_gpu_cle_fuse import FRESH, _recalibrated
from test_gpu_engine import _bind_chains

pytestmark = pytest.mark.gpu

STREAMED, UNDECIDED, HOST_FULL, FULL = 1, 2, 3, 0     # dfq_b200._lib.ROWS_*


def _run(make, one_group, params, mode, monkeypatch, prefix=16, correct=True):
    """mode: "prefix" (DFQ_ROW_PREFIX=prefix), "full" (DFQ_ROW_PREFIX=0) or "per_sweep" (the fold plan stripped of its row scan)."""
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_CLE_STACK", "1")
    monkeypatch.setenv("DFQ_BC_STREAM", "1")
    monkeypatch.setenv("DFQ_ROW_PREFIX", str(prefix if mode == "prefix" else 0))
    p = dict(SC.DEFAULT_PARAMS, **params)
    lay = make()
    sess = Session()
    rels, groups, folds, items = _bind_chains(sess, lay, one_group, p["signed"])
    cle = sess.plan_cle(rels, groups=groups)
    fold = sess.plan_bn_fold(folds, cle_plan=cle)
    assert fold["deferred"] and len(fold["rows_scanned"]) == len(lay)
    assert fold["row_prefix"] == (prefix if mode == "prefix" else 0)
    if mode == "per_sweep":
        fold["ft"]["scan_rows"][:] = 0
        fold["rows_scanned"] = []
    rows_scanned = list(fold["rows_scanned"])
    bc = sess.plan_bias_correct(items, cle_plan=cle) if correct else None
    sess.upload()
    sess.run_bn_fold(fold)
    res = sess.run_cle_plan(cle, s_range=p["s_range"], converge_thres=p["converge_thres"], converge_count=p["converge_count"],
                            signed=p["signed"], eps=p["eps"], max_sweeps=p["max_sweeps"], cols_ready=fold["scanned"])
    if correct:
        sess.run_bias_correct_plan(bc, 8, col_hints=sess.cle_col_hints(cle, res))
    view = lambda off, n: sess.view(int(off), int(n)).cpu().numpy().copy()
    h = sess.cle_col_hints(cle, res)
    out = [view(o, sess.layer(r[0])["rows"]) for o, r in zip(cle["s_offs"], rels)]
    out += [view(a, n) for a, n in zip(h["colmin_off"], h["n_col"])] + [view(a, n) for a, n in zip(h["colmax_off"], h["n_col"])]
    out += [view(d[k], d["w"].shape[0]) for cl in lay for d in cl for k in ("fake_w_off", "fake_b_off")]
    if correct:
        bt = bc["bt"]
        out += [view(b["delta_off"], sess.layer(int(b["layer"]))["rows"]) for b in bt]
        out += [view(b["expect_off"], b["expect_len"]) for b in bt] + [view(b["minmax_off"], 2) for b in bt]
    rext = [view(off, 2 * sess.layer(li)["rows"]) for li, off in rows_scanned]
    sess.download()
    out += [d[k].numpy().copy() for cl in lay for d in cl for k in ("w", "bias")]
    return res, out, rext


def _compare(make, one_group, params, monkeypatch, nan=False, prefix=16, correct=True):
    """The three runs on identical bits; returns the prefix run's result."""
    pr, a, ra = _run(make, one_group, params, "prefix", monkeypatch, prefix, correct)
    fu, b, rb = _run(make, one_group, params, "full", monkeypatch, prefix, correct)
    ps, c, _ = _run(make, one_group, params, "per_sweep", monkeypatch, prefix, correct)
    assert fu.rows_streamed == FULL and ps.rows_streamed == FULL and ps.fused_sweeps == 0
    assert (pr.fused_sweeps, pr.bc_prepared) == (fu.fused_sweeps, fu.bc_prepared)
    for r in (fu, ps):
        assert (pr.n_sweeps, pr.converged) == (r.n_sweeps, r.converged)
        assert np.array_equal(pr.group_sweeps, r.group_sweeps), (pr.group_sweeps, r.group_sweeps)
    if pr.rows_streamed == STREAMED:
        assert pr.fused_sweeps == 2
    for other in (b, c):
        assert len(a) == len(other)
        for i, (x, y) in enumerate(zip(a, other)):
            assert np.array_equal(x, y, equal_nan=nan), i
    assert len(ra) == len(rb)
    for i, (x, y) in enumerate(zip(ra, rb)):
        assert np.array_equal(x, y, equal_nan=True), ("rext", i)
    np.testing.assert_allclose(pr.diffs, fu.diffs, rtol=1e-12, atol=0)
    np.testing.assert_allclose(pr.diffs, ps.diffs, rtol=1e-12, atol=0)
    return pr


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_stack_cases_prefix_equals_full_scan(case, monkeypatch):
    res = _compare(lambda: SC.chain_layers(case["chains"], case["seed"], case["edit"]), case["one_group"], case["params"],
                   monkeypatch, nan=case["nonfinite"], correct=case["correct"])
    assert res.rows_streamed in (STREAMED, UNDECIDED, HOST_FULL, FULL)
    print(case["name"], res.rows_streamed, res.fused_sweeps, list(res.group_sweeps))


def _prefix_equalized(blocks, rows=16):
    """STACK_BLOCKS behind identity BNs, where in the blocks listed the first `rows` channels are already equalized: row c of
    the first conv and input column c of the second both have range 1, so s1 is 1 to within rounding and those channels'
    terms of the guard's bound are ~0 - a prefix of 16 rows cannot decide, the other channels still move."""
    def make():
        lay = SC.chain_layers(SC.STACK_BLOCKS)
        for b, cl in enumerate(lay):
            for d in cl:
                n = d["w"].shape[0]
                d["gamma"], d["beta"], d["mean"], d["var"] = torch.ones(n), torch.zeros(n), torch.zeros(n), torch.ones(n)
                d["bn_eps"] = 0.0
            if b in blocks:
                w1, w2 = cl[0]["w"].clone(), cl[1]["w"].clone()
                for c in range(rows):
                    w1[c] /= (w1[c].max() - w1[c].min())
                    w2[:, c] /= (w2[:, c].max() - w2[:, c].min())
                cl[0]["w"], cl[1]["w"] = w1, w2
        return lay
    return make


@pytest.mark.parametrize("name,make,params,fused,streamed", [
    ("default", FRESH, {}, True, STREAMED),
    ("recalibrated", _recalibrated(range(len(SC.STACK_BLOCKS))), {}, False, UNDECIDED),
    ("one_recalibrated_among_fresh", _recalibrated([2]), {}, False, UNDECIDED),
    ("prefix_equalized", _prefix_equalized(range(len(SC.STACK_BLOCKS))), {}, True, UNDECIDED),
    ("one_prefix_equalized_among_fresh", _prefix_equalized([1]), {}, True, UNDECIDED),
    ("threshold_stops_after_sweep_1", FRESH, dict(converge_thres=1.0), False, UNDECIDED),
    ("converge_count_1", FRESH, dict(converge_count=1), False, HOST_FULL),
    ("max_sweeps_1", FRESH, dict(max_sweeps=1), False, HOST_FULL),
    ("max_sweeps_3", FRESH, dict(converge_thres=0.0, converge_count=3, max_sweeps=3), True, STREAMED),
    ("s_lo_0", FRESH, dict(s_range=(0.0, 1e8)), True, HOST_FULL),
    ("s_hi_inf", FRESH, dict(s_range=(1e-8, float("inf"))), True, HOST_FULL),
], ids=lambda v: v if isinstance(v, str) else None)
def test_prefix_guard_both_sides(name, make, params, fused, streamed, monkeypatch):
    res = _compare(make, False, params, monkeypatch)
    assert res.fused_sweeps == (2 if fused else 0), name
    assert res.rows_streamed == streamed, (name, res.rows_streamed)


@pytest.mark.parametrize("prefix", [1, 16, 4096])
def test_prefix_sizes(prefix, monkeypatch):
    """One row, the default, and more rows than any first conv has (the fold then scans every row: nothing is left to
    complete)."""
    res = _compare(FRESH, False, {}, monkeypatch, prefix=prefix)
    assert res.fused_sweeps == 2
    if prefix >= 512:
        assert res.rows_streamed == FULL
    else:
        assert res.rows_streamed in (STREAMED, UNDECIDED)


def test_prefix_larger_than_small_blocks(monkeypatch):
    """Blocks of fewer rows than the prefix next to larger ones: only the larger ones hold a prefix."""
    chains = [((8, 16, 3, 3), (12, 8, 3, 3)), ((96, 64, 3, 3), (200, 96, 1, 1)), ((4, 4, 1, 1), (8, 4, 3, 3))]
    res = _compare(lambda: SC.chain_layers(chains), False, {}, monkeypatch, prefix=16)
    assert res.rows_streamed in (STREAMED, UNDECIDED)
