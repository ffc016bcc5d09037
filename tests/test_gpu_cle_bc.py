"""-m gpu: the bias correction computed inside k_cle_stack's fused pass (plan_bias_correct(cle_plan=...), DfqCleResult.bc_prepared,
DFQ_BC_PREPARED) against k_bc_stream after the equalization, on identical input bits.  Every problem runs twice: with the
correction attached to the equalization and with it planned on its own.  Weights, biases, both layers' fake_weight /
fake_bias, S, and the correction's delta, E[x] and per-tensor range are bit-identical; the correction is prepared exactly when
the fused pass ran and every group stopped after sweep 2, and anything between the equalization and the correction sends it
down the full path."""
import numpy as np
import pytest

import stack_cases as SC
from test_gpu_cle_fuse import FRESH, _recalibrated
from test_gpu_engine import _bind_chains

pytestmark = pytest.mark.gpu


def _run(make, one_group, params, attach, monkeypatch, bits=8, between=None, correct=True):
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_CLE_STACK", "1")
    monkeypatch.setenv("DFQ_BC_STREAM", "1")        # the full correction on k_bc_stream whatever the size
    p = dict(SC.DEFAULT_PARAMS, **params)
    lay = make()
    sess = Session()
    rels, groups, folds, items = _bind_chains(sess, lay, one_group, p["signed"])
    cle = sess.plan_cle(rels, groups=groups)
    fold = sess.plan_bn_fold(folds, cle_plan=cle)
    bc = sess.plan_bias_correct(items, cle_plan=cle if attach else None)
    assert bc["attached"] == attach
    sess.upload()
    sess.run_bn_fold(fold)
    res = sess.run_cle_plan(cle, s_range=p["s_range"], converge_thres=p["converge_thres"], converge_count=p["converge_count"],
                            signed=p["signed"], eps=p["eps"], max_sweeps=p["max_sweeps"], cols_ready=fold["scanned"])
    if between is not None:
        between(sess, folds)
    if correct:
        sess.run_bias_correct_plan(bc, bits, col_hints=sess.cle_col_hints(cle, res))
    view = lambda off, n: sess.view(int(off), int(n)).cpu().numpy().copy()
    out = [view(o, sess.layer(r[0])["rows"]) for o, r in zip(cle["s_offs"], rels)]
    out += [view(d[k], d["w"].shape[0]) for cl in lay for d in cl for k in ("fake_w_off", "fake_b_off")]
    if correct:
        bt = bc["bt"]
        out += [view(b["delta_off"], sess.layer(int(b["layer"]))["rows"]) for b in bt]
        out += [view(b["expect_off"], b["expect_len"]) for b in bt] + [view(b["minmax_off"], 2) for b in bt]
    sess.download()
    out += [d[k].numpy().copy() for cl in lay for d in cl for k in ("w", "bias")]
    return res, out, [view(b["minmax_off"], 2) for b in bc["bt"]]


def _compare(make, one_group, params, monkeypatch, nan=False, **kw):
    """Returns (attached run's result, the per-tensor ranges it left)."""
    at, a, mm = _run(make, one_group, params, True, monkeypatch, **kw)
    de, b, _ = _run(make, one_group, params, False, monkeypatch, **kw)
    assert not de.bc_prepared
    assert at.bc_prepared == (at.fused_sweeps == 2 and bool(np.all(at.group_sweeps == 2))), (at.fused_sweeps, at.group_sweeps)
    assert (at.fused_sweeps, at.n_sweeps, at.converged) == (de.fused_sweeps, de.n_sweeps, de.converged)
    assert np.array_equal(at.group_sweeps, de.group_sweeps)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y, equal_nan=nan), i
    return at, mm


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_stack_cases_attached_equals_stream(case, monkeypatch):
    res, _ = _compare(lambda: SC.chain_layers(case["chains"], case["seed"], case["edit"]), case["one_group"], case["params"],
                      monkeypatch, nan=case["nonfinite"])
    print(case["name"], "prepared" if res.bc_prepared else "full", res.fused_sweeps, list(res.group_sweeps))


# every group stops after sweep 2 on the cap (threshold 0: the rule never ends it first), the fused pass runs
TWO = dict(converge_thres=0.0, converge_count=3, max_sweeps=2)


@pytest.mark.parametrize("name,make,params,prepared", [
    ("default", FRESH, {}, None),
    ("recalibrated", _recalibrated(range(len(SC.STACK_BLOCKS))), {}, False),
    ("one_recalibrated_among_fresh", _recalibrated([2]), {}, False),
    ("threshold_stops_after_sweep_1", FRESH, dict(converge_thres=1.0), False),
    ("converge_count_1", FRESH, dict(converge_count=1), False),
    ("max_sweeps_1", FRESH, dict(max_sweeps=1), False),
    ("max_sweeps_3", FRESH, dict(converge_thres=0.0, converge_count=3, max_sweeps=3), False),
    ("max_sweeps_2", FRESH, TWO, True),
    ("max_sweeps_2_signed", FRESH, dict(TWO, signed=True), True),
], ids=lambda v: v if isinstance(v, str) else None)
def test_guard_both_sides(name, make, params, prepared, monkeypatch):
    res, _ = _compare(make, False, params, monkeypatch)
    if prepared is not None:
        assert res.bc_prepared == prepared, (name, res.fused_sweeps, res.group_sweeps)


def _tiny_second(make):
    """Block 0's second conv scaled by 1e-30: a per-tensor range whose quantization step lies below bc_fast_quant's exponent
    window.  With s_range (1, 1) the equalization keeps the weights, and max_sweeps 2 stops every group after sweep 2."""
    def mk():
        lay = make()
        lay[0][1]["w"] = (lay[0][1]["w"] * 1e-30).contiguous()
        return lay
    return mk


def test_ieee_chain_inside_the_fused_pass(monkeypatch):
    res, mm = _compare(_tiny_second(FRESH), False, dict(s_range=(1.0, 1.0), converge_thres=-1.0, max_sweeps=2), monkeypatch)
    assert res.bc_prepared
    scale = np.float32((np.float64(mm[0][1]) - np.float64(mm[0][0])) / 255.0)
    assert ((int(scale.view(np.uint32)) >> 23) & 0xff) < 40          # bc_fast_quant refuses block 0: mode 1
    scale1 = np.float32((np.float64(mm[1][1]) - np.float64(mm[1][0])) / 255.0)
    assert 40 <= ((int(scale1.view(np.uint32)) >> 23) & 0xff) <= 200    # ... and takes the others


def test_other_num_bits_at_commit_runs_the_full_path(monkeypatch):
    res, _ = _compare(FRESH, False, TWO, monkeypatch, bits=4)
    assert res.bc_prepared          # prepared at 8 bits, committed at 4: the full correction ran (same bits as without)


@pytest.mark.parametrize("what", ["fold", "quantize"])
def test_a_call_between_runs_the_full_path(what, monkeypatch):
    def between(sess, folds):
        if what == "fold":       # the first conv of chain 0 folded once more: its BN vectors, hence E[x], change
            sess.run_bn_fold(sess.plan_bn_fold([folds[0]]))
        else:
            sess.run_quantize([(folds[0]["fake_b_off"], 8, 4, False)])
    res, _ = _compare(FRESH, False, TWO, monkeypatch, between=between)
    assert res.bc_prepared


def test_attached_but_never_corrected(monkeypatch):
    res, _ = _compare(FRESH, False, TWO, monkeypatch, correct=False)
    assert res.bc_prepared
