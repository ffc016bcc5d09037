"""Host side of the bias correction computed in the equalization's fused pass, on the oracle-backed stand-in
(tests/fakelib_bc.py): plan_bias_correct attaches exactly the corrections the stack kernel can compute, run_cle_plan hands
them over, run_bias_correct_plan only retires the deltas right after a prepared run at the same num_bits, and every other
session call in between sends it down the full correction - with the same results as a step that never attaches."""
import pytest
import torch

import fakelib_bc
from dfq_b200.workload import DeviceStack


def _stack(monkeypatch, n_blocks=3, channels=8, k=3, takes=True):
    from dfq_b200.engine import Session
    fake = fakelib_bc.install(monkeypatch, takes=takes)
    sess = Session()
    st = DeviceStack(sess, n_blocks, channels, k, seed=9)
    st.generate()
    return fake, sess, st


def _detached(sess, st):
    """The same stack's correction planned without cle_plan (the full path only), and nothing attached to its equalization."""
    st.cle_plan.pop("bc")
    items = [dict(layer=st.layers[2 * b + 1], signed=False, level=0, next_bn_b_off=st.vec[2 * b + 1]["fake_b"],
                  terms=[dict(bn_w_off=st.vec[2 * b]["fake_w"], bn_b_off=st.vec[2 * b]["fake_b"], n=st.C, relu=True, op="set")])
             for b in range(st.n_blocks)]
    plan = sess.plan_bias_correct(items)
    assert not plan["attached"]
    return plan


def _step(sess, st, bits=8, between=None, hints=True, bc_plan=None):
    sess.run_bn_fold(st.fold_plan)
    res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"])
    if between is not None:
        between()
    sess.run_bias_correct_plan(bc_plan or st.bc_plan, bits, col_hints=sess.cle_col_hints(st.cle_plan, res) if hints else None)
    return res


def test_device_stack_attaches_and_the_step_only_retires(monkeypatch):
    fake, sess, st = _stack(monkeypatch)
    assert st.bc_plan["attached"] and st.cle_plan["bc"]["plan"] is st.bc_plan and st.cle_plan["bc"]["num_bits"] == 8
    res = st.run()
    assert res.fused_sweeps == 2 and res.bc_prepared and fake.attached == [st.n_blocks]
    assert fake.retired == 1
    # the same step with the correction planned apart: full correction, same bits
    fu, su, stu = _stack(monkeypatch)
    _step(su, stu, bc_plan=_detached(su, stu))
    assert fu.retired == 0 and fu.attached == [0]
    assert torch.equal(st.state(), stu.state()) and torch.equal(st.scale_state(), stu.scale_state())


def _reference(monkeypatch, bits=8, between=None):
    fu, su, stu = _stack(monkeypatch)
    _step(su, stu, bits, between=(lambda: between(su, stu)) if between else None, bc_plan=_detached(su, stu))
    return stu.state().clone()


def _fold(st, i):
    v = st.vec[i]
    return dict(layer=st.layers[i], bn_eps=1e-5, gamma_off=v["gamma"], beta_off=v["beta"], mean_off=v["mean"], var_off=v["var"],
                fake_w_off=v["fake_w"], fake_b_off=v["fake_b"])


@pytest.mark.parametrize("case", ["bits", "quantize", "fold", "view", "no_hints"])
def test_anything_in_between_runs_the_full_correction(case, monkeypatch):
    bits = 4 if case == "bits" else 8
    quant = lambda s, t: s.run_quantize([(t.w_begin, 4, 8, False)])
    between = {"quantize": quant, "fold": lambda s, t: s.run_bn_fold([_fold(t, 0)]),
               "view": lambda s, t: s.view(0, 1)}.get(case)
    fake, sess, st = _stack(monkeypatch)
    res = _step(sess, st, bits, between=(lambda: between(sess, st)) if between else None, hints=case != "no_hints")
    assert res.bc_prepared
    assert fake.retired == 0
    want = _reference(monkeypatch, bits, between)
    assert torch.equal(st.state(), want)


def test_attached_but_never_corrected_leaves_the_biases_alone(monkeypatch):
    fake, sess, st = _stack(monkeypatch)
    sess.run_bn_fold(st.fold_plan)
    res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"])
    assert res.bc_prepared
    fu, su, stu = _stack(monkeypatch)
    stu.cle_plan.pop("bc")
    su.run_bn_fold(stu.fold_plan)
    su.run_cle_plan(stu.cle_plan, cols_ready=stu.fold_plan["scanned"])
    assert fu.attached == [0]
    assert torch.equal(st.channel_state(), stu.channel_state()) and torch.equal(st.state(), stu.state())


def test_a_correction_is_prepared_only_after_two_fused_sweeps(monkeypatch):
    fake, sess, st = _stack(monkeypatch)
    res = st.run(converge_thres=1.0)        # every group stops after sweep 1: no fused pass
    assert res.fused_sweeps == 0 and not res.bc_prepared and fake.retired == 0
    # a library that does not take the stack kernel never gets the correction
    fn, sn, stn = _stack(monkeypatch, takes=False)
    rn = stn.run()
    assert not rn.bc_prepared and fn.attached == [0] and fn.retired == 0


def test_only_what_the_fused_pass_can_compute_is_attached(monkeypatch):
    fake, sess, st = _stack(monkeypatch)

    def item(b, **kw):
        d = dict(layer=st.layers[2 * b + 1], signed=False, level=0, next_bn_b_off=-1,
                 terms=[dict(bn_w_off=st.vec[2 * b]["fake_w"], bn_b_off=st.vec[2 * b]["fake_b"], n=st.C, relu=True, op="set")])
        d.update(kw)
        return d

    plan = lambda items: sess.plan_bias_correct(items, cle_plan=dict(st.cle_plan))
    assert plan([item(0), item(1, signed=True)])["attached"]
    assert not plan([item(0), item(1, level=1)])["attached"]                 # two levels
    assert not plan([item(0, raw_sum=True)])["attached"]                      # bias absorption
    assert not plan([item(0, add=True)])["attached"]
    assert not plan([item(0), item(0)])["attached"]                           # a layer twice
    assert not plan([item(0, layer=st.layers[0])])["attached"]                # a `first` layer
    two = [dict(bn_w_off=st.vec[0]["fake_w"], bn_b_off=st.vec[0]["fake_b"], n=st.C, relu=True, op="set")] * 2
    two[1] = dict(two[1], op="cat")
    assert not plan([item(0, terms=two)])["attached"]                         # E[x] longer than the input
