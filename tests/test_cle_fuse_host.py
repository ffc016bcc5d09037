"""Host side of the first two equalization sweeps in one pass, on the oracle-backed stand-in (tests/fakelib_fuse.py): a
deferred fold scans the row extrema of exactly the plan's `first` layers, run_cle_plan hands them over as ROWS_READY, the
result reports the fused pass, and the guard refuses on both of its sides."""
import numpy as np
import pytest
import torch

import fakelib_fuse
from dfq_b200 import _lib
from dfq_b200.workload import DeviceStack
from oracle import dfq_oracle as O

f32 = np.float32


def _run(monkeypatch, takes, **kw):
    from dfq_b200.engine import Session
    fake = fakelib_fuse.install(monkeypatch, takes=takes)
    sess = Session()
    st = DeviceStack(sess, 3, 8, 3, seed=9)
    st.generate()
    res = st.run(**kw)
    return fake, sess, st, res


def test_deferred_fold_scans_first_layer_rows_and_the_equalization_fuses(monkeypatch):
    fake, sess, st, res = _run(monkeypatch, True)
    plan = st.fold_plan
    first = st.layers[0::2]
    assert [r[0] for r in plan["rows_scanned"]] == first
    ft = plan["ft"]
    assert [int(f["layer"]) for f in ft if f["scan_rows"]] == first
    assert all(plan["lt"]["rext_off"][li] == off for li, off in plan["rows_scanned"])
    assert len({off for _, off in plan["rows_scanned"]}) == len(first)
    assert res.fused_sweeps == 2 and list(res.group_sweeps) == [2, 2, 2]
    # the undeferred fold scans no rows and the equalization runs one pass per sweep, to the same state
    fu, su, stu, ru = _run(monkeypatch, False)
    assert stu.fold_plan["rows_scanned"] == [] and not stu.fold_plan["ft"]["scan_rows"].any()
    assert ru.fused_sweeps == 0
    assert torch.equal(st.state(), stu.state()) and torch.equal(st.scale_state(), stu.scale_state())


def test_threshold_that_stops_after_one_sweep_is_refused(monkeypatch):
    _, _, _, res = _run(monkeypatch, True, converge_thres=1.0)
    assert res.fused_sweeps == 0 and list(res.group_sweeps) == [1, 1, 1]


def _block(seed, C=16, kk=9):
    g = np.random.default_rng(seed)
    w1 = (g.standard_normal((C, C * kk)) * 10 ** g.uniform(-1, 1, (C, 1))).astype(f32)
    w2 = g.standard_normal((C, C, kk)).astype(f32)
    return w1, w2


def _equalized(w1, w2, sweeps):
    l1, l2 = O.OLayer(w1.reshape(w1.shape[0], -1, 9).copy(), np.zeros(w1.shape[0], f32)), O.OLayer(w2.copy(), np.zeros(w2.shape[0], f32))
    O.cross_layer_equalization([l1, l2], [(None, None)], [O.ORelation(0, 1, 0)], max_sweeps=sweeps)
    return l1.w.reshape(w1.shape), l2.w


def test_guard_both_sides():
    fresh = [(g, *_block(g)) for g in range(3)]
    assert fakelib_fuse.fuse_guard(fresh)
    # the exit rule's other ways out after sweep 1
    assert not fakelib_fuse.fuse_guard(fresh, converge_count=1)
    assert not fakelib_fuse.fuse_guard(fresh, max_sweeps=1)
    assert fakelib_fuse.fuse_guard(fresh, max_sweeps=3)
    # a block that is equalized already: sweep 1 moves it by a few ulps, the reference stops there, and its sweep 2 is no
    # identity - refused, alone and among fresh blocks
    again = (7, *_equalized(*_block(7), None))
    assert not fakelib_fuse.fuse_guard([again])
    assert not fakelib_fuse.fuse_guard(fresh + [again])
    # a column of zeros gives s = 0: clamped to a positive s_lo it is fine, with s_lo = 0 the monotonicity argument fails
    w1, w2 = _block(3)
    w2[:, 5, :] = 0
    assert fakelib_fuse.fuse_guard([(0, w1, w2)])
    assert not fakelib_fuse.fuse_guard([(0, w1, w2)], s_range=(0.0, 1e8))
