"""The BN fold deferred into the equalization's first sweep (DFQ_FOLD_DEFER / DFQ_LAYER_FOLD_PENDING).

When the library reports that an equalization plan runs on k_cle_stack, plan_bn_fold(folds, cle_plan=...) defers the fold's
weight pass: the fold call does the [rows]-vector work and a read-only scan of the second layers, and the first sweep multiplies
every row by its factor as it reads it.  Every element goes through the same fp32 operations in the same order as
fold-then-sweep, so the deferred run must equal the undeferred one bit for bit - and a pending fold must never be lost,
whichever path dfq_cle_run takes and whatever the session is asked to do in between."""
import numpy as np
import pytest
import torch

from test_gpu_engine import STACK_BLOCKS, _chains_session, _oracle_chains

pytestmark = pytest.mark.gpu


def _stack(n_blocks, channels, k, seed, defer, monkeypatch, stack_env):
    """A DeviceStack whose fold plan is (defer) or is not deferred; stack_env: DFQ_CLE_STACK while the equalization runs."""
    from dfq_b200.engine import Session
    from dfq_b200.workload import DeviceStack
    # the plan defers exactly when the library would take the plan on k_cle_stack: DFQ_CLE_STACK=0 at planning time keeps the
    # undeferred fold (with its column scan, so that k_cle_stack can still take the plan when it runs)
    if defer:
        monkeypatch.delenv("DFQ_CLE_STACK", raising=False) if stack_env is None else monkeypatch.setenv("DFQ_CLE_STACK", stack_env)
    else:
        monkeypatch.setenv("DFQ_CLE_STACK", "0")
    sess = Session()
    st = DeviceStack(sess, n_blocks, channels, k, seed=seed)
    assert bool(st.fold_plan["deferred"]) == defer, st.fold_plan["deferred"][:4]
    st.generate()
    if stack_env is None:
        monkeypatch.delenv("DFQ_CLE_STACK", raising=False)
    else:
        monkeypatch.setenv("DFQ_CLE_STACK", stack_env)
    return sess, st


def _step(sess, st):
    sess.run_bn_fold(st.fold_plan)
    assert sess.fold_pending == bool(st.fold_plan["deferred"])
    res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"])
    assert not sess.fold_pending
    return res


def _outcome(sess, st, res):
    return st.state().clone(), st.scale_state().clone(), res.group_sweeps.copy(), res.n_sweeps, res.converged


def _assert_same(a, b):
    assert a[3] == b[3] and a[4] and b[4] and np.array_equal(a[2], b[2]), (a[2], b[2])
    assert torch.equal(a[0], b[0]), "weights / biases / BN vectors differ"
    assert torch.equal(a[1], b[1]), "S differs"


def _oracle_ends(st, pristine, after, res):
    from oracle import stack_check
    for b in sorted({0, st.n_blocks - 1}):
        r = stack_check.compare_block(st.block_arrays(pristine, b), st.block_arrays(after, b))
        assert r["weights_bit_exact"] and r["vectors_bit_exact"] and r["sweeps"] == int(res.group_sweeps[b]), (b, r)


@pytest.mark.parametrize("n_blocks,channels,k,stack_env", [
    (40, 512, 3, None),        # large enough for the library to pick k_cle_stack on its own
    (5, 64, 3, "1"),           # several rows per tile (576-float rows)
    (5, 128, 1, "1"),          # pointwise blocks: 128-float rows, 32 rows per tile
    (5, 96, 3, "1"),           # 864-float rows
])
def test_deferred_fold_equals_the_undeferred_fold(n_blocks, channels, k, stack_env, monkeypatch):
    """Deferred and undeferred fold through k_cle_stack on the same bits: whole state (weights, biases, BN vectors), S and the
    sweeps per group identical; also identical to the plain fold (no column scan) on k_cle_engine; first and last block
    against the oracle."""
    outs = []
    for defer in (True, False):
        sess, st = _stack(n_blocks, channels, k, 11, defer, monkeypatch, stack_env)
        pristine = st.state().clone()
        outs.append(_outcome(sess, st, _step(sess, st)))
    _assert_same(outs[0], outs[1])
    # the plain fold (no cle_plan: no scan, nothing deferred) and the engine
    from dfq_b200.engine import Session
    from dfq_b200.workload import DeviceStack
    monkeypatch.setenv("DFQ_CLE_STACK", "0")
    sess = Session()
    st = DeviceStack(sess, n_blocks, channels, k, seed=11)
    plain = sess.plan_bn_fold([dict(layer=li, bn_eps=1e-5, gamma_off=v["gamma"], beta_off=v["beta"], mean_off=v["mean"],
                                    var_off=v["var"], fake_w_off=v["fake_w"], fake_b_off=v["fake_b"])
                               for li, v in zip(st.layers, st.vec)])
    assert not plain["deferred"]
    st.generate()
    sess.run_bn_fold(plain)
    res = sess.run_cle_plan(st.cle_plan)
    _assert_same(outs[0], _outcome(sess, st, res))
    _oracle_ends(st, pristine, outs[0][0], res)


@pytest.mark.parametrize("one_group", [False, True])
def test_deferred_fold_on_a_heterogeneous_stack(one_group, monkeypatch):
    """Unlike blocks (non-square, 3x3 next to 1x1, partial tiles, the 512-column / 4608-float edge, 36-float rows) in one launch:
    the forced k_cle_stack run defers its fold (plan_bn_fold sees DFQ_CLE_STACK=1) and equals the forced k_cle_engine run, which
    does not, and the oracle."""
    runs = [_chains_session(STACK_BLOCKS, one_group, v, "stream", v == "1", monkeypatch) for v in ("1", "0")]
    (before, a1, r1, d1, e1, s1), (_, a0, r0, d0, e0, s0) = runs
    assert np.array_equal(r1.group_sweeps, r0.group_sweeps)
    for x, y in zip(a1, a0):
        for p, q in zip(x, y):
            for key in p:
                assert np.array_equal(p[key], q[key]), key
    for x, y in zip(s1 + d1 + e1, s0 + d0 + e0):
        assert np.array_equal(x, y)
    layers, bns, sweeps = _oracle_chains(before, one_group)[:3]
    assert list(r1.group_sweeps) == (sweeps[:1] if one_group else sweeps)
    for b, cl in enumerate(a1):
        assert np.array_equal(cl[0]["w"], layers[2 * b].w) and np.array_equal(cl[1]["w"], layers[2 * b + 1].w.reshape(cl[1]["w"].shape))


def test_heterogeneous_stack_plan_defers_when_forced(monkeypatch):
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_CLE_STACK", "1")
    sess = Session()
    rels, folds = [], []
    for shapes in STACK_BLOCKS:
        ids = []
        for s in shapes:
            li = sess.add_layer(torch.randn(*s), None)
            n = s[0]
            folds.append(dict(layer=li, bn_eps=1e-5, gamma_off=sess.alloc(n), beta_off=sess.alloc(n), mean_off=sess.alloc(n),
                              var_off=sess.alloc(n), fake_w_off=sess.alloc(n), fake_b_off=sess.alloc(n)))
            ids.append(li)
        rels.append((ids[0], ids[1], folds[-2]["fake_w_off"], folds[-2]["fake_b_off"]))
    cle = sess.plan_cle(rels, groups=list(range(len(rels))))
    assert len(sess.plan_bn_fold(folds, cle_plan=cle)["deferred"]) == len(folds)
    monkeypatch.setenv("DFQ_CLE_STACK", "0")
    assert sess.plan_bn_fold(folds, cle_plan=cle)["deferred"] == []


def _folded_reference(n_blocks, channels, k, monkeypatch):
    """State after a plain (undeferred) fold: what every completed deferred fold must leave."""
    from dfq_b200.engine import Session
    from dfq_b200.workload import DeviceStack
    monkeypatch.setenv("DFQ_CLE_STACK", "0")
    sess = Session()
    st = DeviceStack(sess, n_blocks, channels, k, seed=3)
    st.generate()
    sess.run_bn_fold(st.fold_plan)
    return st.state().clone()


def test_pending_fold_on_the_engine_path(monkeypatch):
    """A deferred plan whose equalization then runs on k_cle_engine (DFQ_CLE_STACK=0 at run time): dfq_cle_run applies the fold
    before the engine starts - the result equals the undeferred run on the engine."""
    ref = []
    for defer in (True, False):
        sess, st = _stack(5, 64, 3, 11, defer, monkeypatch, "1")
        monkeypatch.setenv("DFQ_CLE_STACK", "0")
        ref.append(_outcome(sess, st, _step(sess, st)))
    _assert_same(ref[0], ref[1])


@pytest.mark.parametrize("thres,count", [(10.0, 20), (2e-7, 0)])
def test_pending_fold_when_no_sweep_runs(thres, count, monkeypatch):
    """An exit rule that is false before any sweep (converge_thres >= 10, converge_count <= 0): no sweep runs, and the weights
    still come out folded."""
    folded = _folded_reference(5, 64, 3, monkeypatch)
    sess, st = _stack(5, 64, 3, 3, True, monkeypatch, "1")
    sess.run_bn_fold(st.fold_plan)
    assert sess.fold_pending
    res = sess.run_cle_plan(st.cle_plan, converge_thres=thres, converge_count=count, cols_ready=st.fold_plan["scanned"])
    assert res.n_sweeps == 0 and not sess.fold_pending
    assert torch.equal(st.state(), folded)


def test_other_calls_see_folded_weights(monkeypatch):
    """Session calls between the deferred fold and the equalization complete the fold first: a view of the arena, a download,
    the bias correction - and a later run_cle_plan of the same plan then equalizes the folded weights normally."""
    folded = _folded_reference(5, 64, 3, monkeypatch)
    sess, st = _stack(5, 64, 3, 3, True, monkeypatch, "1")
    sess.run_bn_fold(st.fold_plan)
    assert sess.fold_pending
    assert torch.equal(st.state(), folded) and not sess.fold_pending        # view()
    # ... and the equalization after it equals the undeferred step
    res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"])
    ref_sess, ref_st = _stack(5, 64, 3, 3, False, monkeypatch, "1")
    _assert_same(_outcome(sess, st, res), _outcome(ref_sess, ref_st, _step(ref_sess, ref_st)))
    # bias correction with a fold pending: corrects the folded weights
    sess, st = _stack(5, 64, 3, 3, True, monkeypatch, "1")
    sess.run_bn_fold(st.fold_plan)
    sess.run_bias_correct_plan(st.bc_plan, 8)
    assert not sess.fold_pending
    ref_sess, ref_st = _stack(5, 64, 3, 3, False, monkeypatch, "1")
    ref_sess.run_bn_fold(ref_st.fold_plan)
    ref_sess.run_bias_correct_plan(ref_st.bc_plan, 8)
    assert torch.equal(st.state(), ref_st.state())


def test_host_stack_calibrator_output_unchanged(monkeypatch):
    """HostStackCalibrator (chunks streamed through arena slots, each slot's step deferred) gives the same host image as the
    same chunks calibrated with the fold undeferred."""
    from dfq_b200.workload import HostStackCalibrator
    dev = torch.device("cuda", torch.cuda.current_device())
    outs = []
    for defer in (True, False):
        monkeypatch.setenv("DFQ_CLE_STACK", "1" if defer else "0")
        hc = HostStackCalibrator(dev, chunk_blocks=4, channels=64, k=3, n_slots=3)
        assert all(bool(s.fold_plan["deferred"]) == defer for s in hc.slots)
        monkeypatch.setenv("DFQ_CLE_STACK", "1")
        for s in hc.slots:
            s.generate()
        n_chunks = 5
        host_in = torch.empty(n_chunks * hc.chunk_floats, dtype=torch.float32, pin_memory=True)
        host_out = torch.empty_like(host_in).pin_memory()
        for i in range(n_chunks):
            host_in[i * hc.chunk_floats:(i + 1) * hc.chunk_floats].copy_(hc.slots[i % len(hc.slots)].state())
        torch.cuda.synchronize()
        hc.run(host_in, host_out)
        torch.cuda.synchronize()
        outs.append(host_out.clone())
    assert torch.equal(outs[0], outs[1])
