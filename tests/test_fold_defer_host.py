"""Host side of the deferred BN fold, on the oracle-backed stand-in (tests/fakelib_defer.py): plan_bn_fold defers exactly when
the library reports that the equalization plan runs on the stack kernel, run_cle_plan hands the pending layers over, any other
session call completes the fold first, and the outcome equals the undeferred step."""
import numpy as np
import pytest
import torch

import fakelib_defer
from dfq_b200 import _lib
from dfq_b200.workload import DeviceStack


def _stack(monkeypatch, takes, n_blocks=3, channels=8, k=3):
    from dfq_b200.engine import Session
    fake = fakelib_defer.install(monkeypatch, takes=takes)
    sess = Session()
    st = DeviceStack(sess, n_blocks, channels, k, seed=9)
    st.generate()
    return fake, sess, st


@pytest.mark.parametrize("takes", [True, False])
def test_plan_defers_exactly_when_the_library_takes_the_stack_kernel(takes, monkeypatch):
    fake, sess, st = _stack(monkeypatch, takes)
    plan = st.fold_plan
    assert "dfq_cle_takes_stack" in fake.calls
    assert [d[0] for d in plan["deferred"]] == (list(st.layers) if takes else [])
    assert set(plan["ft"]["mode"].tolist()) == ({_lib.FOLD_DEFER} if takes else {_lib.FOLD_FULL})
    # a fold without an equalization plan never asks and never defers
    n_asks = fake.calls.count("dfq_cle_takes_stack")
    assert sess.plan_bn_fold([dict(layer=st.layers[0], bn_eps=1e-5)])["deferred"] == []
    assert fake.calls.count("dfq_cle_takes_stack") == n_asks


def _run(monkeypatch, takes):
    fake, sess, st = _stack(monkeypatch, takes)
    res = st.run()
    return fake, sess, st, res


def test_deferred_step_equals_the_undeferred_step(monkeypatch):
    fd, sd, std, rd = _run(monkeypatch, True)
    fu, su, stu, ru = _run(monkeypatch, False)
    assert torch.equal(std.state(), stu.state()) and torch.equal(std.scale_state(), stu.scale_state())
    assert np.array_equal(rd.group_sweeps, ru.group_sweeps)
    # the deferred step: one fold call (DEFER, no extra APPLY pass), the equalization gets every deferred layer as pending
    assert fd.fold_modes == [[_lib.FOLD_DEFER] * len(std.layers)]
    assert fd.pending_seen == [list(std.layers)]
    assert fu.fold_modes == [[_lib.FOLD_FULL] * len(stu.layers)] and fu.pending_seen == [[]]
    assert not sd.fold_pending


@pytest.mark.parametrize("call", ["view", "download", "bias_correct", "quantize", "fold", "other_plan"])
def test_other_session_calls_complete_a_pending_fold(call, monkeypatch):
    fu, su, stu = _stack(monkeypatch, False)
    su.run_bn_fold(stu.fold_plan)
    folded = stu.state().clone()
    fake, sess, st = _stack(monkeypatch, True)
    sess.run_bn_fold(st.fold_plan)
    assert sess.fold_pending
    if call == "view":
        sess.view(0, 1)
    elif call == "download":
        sess.download()
    elif call == "bias_correct":
        sess.run_bias_correct_plan(st.bc_plan, 8)
    elif call == "quantize":
        sess.run_quantize([(st.w_begin, 4, 8, False)])
    elif call == "fold":
        sess.run_bn_fold([])            # nothing to fold: no call at all, the pending one stays
        assert sess.fold_pending
        sess.run_bn_fold(st.fold_plan)
        assert sess.fold_pending        # the second deferred fold is pending now, the first was completed
        sess.finish_fold()
    elif call == "other_plan":
        other = sess.plan_cle(st.cle_plan["relations"], groups=list(range(st.n_blocks)))
        sess.run_cle_plan(other, max_sweeps=1)
    assert not sess.fold_pending
    assert fake.fold_modes[1] == [_lib.FOLD_APPLY] * len(st.layers)
    if call in ("view", "download"):
        assert torch.equal(st.state(), folded)
