"""Host side of the deferred fold's row prefix, on the oracle-backed stand-in (tests/fakelib_rowstream.py): the fold plan scans
the first DFQ_ROW_PREFIX rows of every `first` layer and every row of every `second` layer, run_cle_plan hands the prefix over
in DfqLayer.rext_rows, and the result reports which way the guard went (DfqCleResult.rows_streamed)."""
import numpy as np
import pytest
import torch

import fakelib_rowstream
from dfq_b200 import _lib
from dfq_b200.workload import DeviceStack

f32 = np.float32


def _run(monkeypatch, prefix=None, C=32, **kw):
    from dfq_b200.engine import Session
    if prefix is not None:
        monkeypatch.setenv("DFQ_ROW_PREFIX", str(prefix))
    fake = fakelib_rowstream.install(monkeypatch)
    sess = Session()
    st = DeviceStack(sess, 3, C, 3, seed=9)
    st.generate()
    sess.run_bn_fold(st.fold_plan)
    res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"], **kw)
    return fake, sess, st, res


def test_abi_table_layouts():
    assert _lib.ABI_VERSION == 11
    assert _lib.LAYER_DT.fields["rext_rows"][1] == 80 and _lib.LAYER_DT.itemsize == 88
    assert _lib.FOLD_DT.fields["row_prefix"][1] == 80 and _lib.FOLD_DT.itemsize == 88
    assert _lib.CLE_RESULT_DT.fields["rows_streamed"][1] == 536 and _lib.CLE_RESULT_DT.itemsize == 544
    assert (_lib.ROWS_FULL, _lib.ROWS_STREAMED, _lib.ROWS_UNDECIDED, _lib.ROWS_HOST_FULL) == (0, 1, 2, 3)


@pytest.mark.parametrize("prefix,C", [(None, 32), (1, 32), (0, 32), (16, 8)])
def test_fold_plan_scans_a_prefix_of_first_layers_and_all_of_second_layers(prefix, C, monkeypatch):
    fake, sess, st, res = _run(monkeypatch, prefix, C)
    plan = st.fold_plan
    p = 16 if prefix is None else prefix
    assert plan["row_prefix"] == p
    first, second = st.layers[0::2], st.layers[1::2]
    ft = plan["ft"]
    for f in ft:
        li = int(f["layer"])
        if li in first:
            assert f["scan_rows"] == 1 and f["row_prefix"] == p and f["scan_go"] == 0
        else:
            assert li in second and f["scan_rows"] == 0 and f["scan_go"] > 0
    # the layer table the equalization gets carries the prefix of every first layer
    lt = plan["_pending_lt"]
    assert all(lt["flags"][li] & _lib.LAYER_ROWS_READY and lt["rext_rows"][li] == p for li in first)
    assert all(lt["rext_rows"][li] == 0 for li in second)
    scanned = fakelib_rowstream.prefix_rows(C, p)
    # the equalization got the prefix in the layer table and reports the branch
    expect = _lib.ROWS_FULL if scanned == C else (_lib.ROWS_STREAMED, _lib.ROWS_UNDECIDED)
    if scanned == C:
        assert res.rows_streamed == expect
    else:
        assert res.rows_streamed in expect
    assert res.fused_sweeps == 2 and list(res.group_sweeps) == [2, 2, 2]


def test_prefix_run_equals_full_scan_run(monkeypatch):
    _, _, st, res = _run(monkeypatch, 16)
    _, _, su, ru = _run(monkeypatch, 0)
    assert res.rows_streamed == _lib.ROWS_STREAMED and ru.rows_streamed == _lib.ROWS_FULL
    assert (res.fused_sweeps, list(res.group_sweeps)) == (ru.fused_sweeps, list(ru.group_sweeps))
    assert torch.equal(st.state(), su.state()) and torch.equal(st.scale_state(), su.scale_state())


def test_the_stand_in_reports_each_branch(monkeypatch):
    # the prefix cannot show sweep 1 moves enough: the rest is scanned, the full guard refuses
    _, _, _, res = _run(monkeypatch, 16, converge_thres=1.0)
    assert res.rows_streamed == _lib.ROWS_UNDECIDED and res.fused_sweeps == 0
    # no fused pass possible: the host scans the rest first
    _, _, _, res = _run(monkeypatch, 16, converge_count=1)
    assert res.rows_streamed == _lib.ROWS_HOST_FULL and res.fused_sweeps == 0


def test_prefix_guard_sides():
    g = np.random.default_rng(3)
    C = 64
    w1 = (g.standard_normal((C, C * 9)) * 10 ** g.uniform(-1, 1, (C, 1))).astype(f32)
    w2 = g.standard_normal((C, C, 9)).astype(f32)
    assert fakelib_rowstream.prefix_guard([(0, w1, w2)], 16)
    assert not fakelib_rowstream.prefix_guard([(0, w1, w2)], 16, converge_thres=1.0)
    # the first 16 channels equalized already (row and column ranges 1): their terms vanish, the prefix cannot decide
    e1, e2 = w1.copy(), w2.copy()
    for c in range(16):
        e1[c] /= e1[c].max() - e1[c].min()
        e2[:, c] /= e2[:, c].max() - e2[:, c].min()
    assert not fakelib_rowstream.prefix_guard([(0, e1, e2)], 16)
    assert fakelib_rowstream.prefix_guard([(0, e1, e2)], 32)
