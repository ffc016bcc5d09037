"""CPU guards of the k_cle_stack edge cases (tests/stack_cases.py, run on the GPU by tests/test_gpu_stack_edges.py): from the
oracle alone, every case reaches what its comment claims - sweep counts, clamps, negative fold factors, zero rows, inf biases,
subnormals - is a problem the stack kernel takes, stops on its own, and never lets an exit comparison come so close to its
constant that the kernels' different summation order of the sweep metric could flip it."""
import numpy as np
import pytest

import stack_cases as SC
from oracle import dfq_oracle as O
from test_boundary_guards import _source_value

MARGIN = 1e-3          # relative distance of every exit comparison from its constant (stack_cases.exit_trace)
FLT_MIN = np.finfo(np.float32).tiny


def _record(monkeypatch):
    """Wraps the oracle's per-relation steps: which clamps solve_scale took, and whether a subnormal weight ever existed."""
    seen = dict(hi=False, lo=False, subnormal=False)
    solve, equalize = O.solve_scale, O.layer_equalization

    def solve_rec(r1, r2, s_range=(1e-8, 1e8), eps=0, sqrt_fn=None):
        s, inv = solve(r1, r2, s_range, eps, sqrt_fn)
        seen["hi"] |= bool((s == np.float32(s_range[1])).any())
        seen["lo"] |= bool((s == np.float32(s_range[0])).any())
        return s, inv

    def sub(a):
        a = np.abs(a)
        return bool(((a > 0) & (a < FLT_MIN)).any())

    def equalize_rec(w1, w2, *a, **k):
        seen["subnormal"] |= sub(w1) or sub(w2)
        S = equalize(w1, w2, *a, **k)
        seen["subnormal"] |= sub(w1) or sub(w2)
        return S
    monkeypatch.setattr(O, "solve_scale", solve_rec)
    monkeypatch.setattr(O, "layer_equalization", equalize_rec)
    return seen


def _folded(before):
    return [[O.bn_fold(d["w"], d["bias"], d["gamma"], d["beta"], d["mean"], d["var"], d["bn_eps"]) for d in cl] for cl in before]


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_case_reaches_what_it_claims(case, monkeypatch):
    _, before = SC.case_data(case)
    seen = _record(monkeypatch)
    with np.errstate(all="ignore"):
        layers, bns, sweeps, diffs, S = SC.oracle_chains(before, case["one_group"], case["params"])
    claims, p = case["claims"], dict(SC.DEFAULT_PARAMS, **case["params"])
    traces = [SC.exit_trace(d, case["params"]) for d in diffs]
    assert len(sweeps) == (1 if case["one_group"] else len(case["chains"]))
    # ---- sweeps ----
    if "distinct_stops" in claims:
        assert len(set(sweeps)) >= claims["distinct_stops"], sweeps
    if "parities" in claims:
        assert {n % 2 for n in sweeps} == claims["parities"], sweeps
    assert max(sweeps) >= claims.get("min_sweeps", 1), sweeps
    if claims.get("capped"):
        assert set(sweeps) == {p["max_sweeps"]} and not any(c for c, _ in traces), sweeps
    else:
        assert all(c for c, _ in traces), "a group ended on max_sweeps, not on the exit rule"
    if max(sweeps) <= 2:    # the default-parameter blocks stop after two sweeps: whatever else the case claims is its point
        assert set(claims) - {"min_sweeps"}, "a case that only repeats the existing two-sweep blocks"
    # ---- ingredients ----
    if claims.get("clamp_hi"):
        assert seen["hi"], "no channel clamped at s_hi"
    if claims.get("clamp_lo"):
        assert seen["lo"], "no channel clamped at s_lo"
    if claims.get("subnormal"):
        assert seen["subnormal"], "no subnormal weight in any sweep"
    folded = _folded(before)
    if claims.get("zero_rows"):
        assert any((np.abs(f[0][0].reshape(f[0][0].shape[0], -1)).max(axis=1) == 0).any() for f in folded)
    if claims.get("inf_bias"):
        assert any(np.isinf(layers[2 * b].b).any() for b in range(len(before)))
        assert case["nonfinite"] and not case["correct"]
    if claims.get("negative_factors"):
        # the extrema of fl(w * f) with f < 0 are not those of fl(w * |f|): a fold that swapped them or took |f| shows
        swapped = False
        for cl in before:
            d = cl[1]
            f = d["gamma"] / np.sqrt(d["var"] + np.float32(d["bn_eps"])).astype(np.float32)
            assert (f < 0).any()
            w = d["w"].reshape(d["w"].shape[0], d["w"].shape[1], -1)
            a, b = w * f.reshape(-1, 1, 1), w * np.abs(f).reshape(-1, 1, 1)
            swapped |= not np.array_equal(a.min(axis=(0, 2)), b.min(axis=(0, 2)))
        assert swapped
    if claims.get("signed_ranges"):
        # max |w| is not max - min: the unsigned ranges give other scales
        with np.errstate(all="ignore"):
            S_unsigned = SC.oracle_chains(before, case["one_group"], dict(case["params"], signed=False))[4]
        assert not all(np.array_equal(a, b) for a, b in zip(S, S_unsigned))
    # finite results exactly where the case says so (the GPU test compares with equal_nan only there)
    finite = all(np.isfinite(l.w).all() and np.isfinite(l.b).all() for l in layers) and all(np.isfinite(v).all() for b in bns for v in b)
    assert finite != case["nonfinite"]


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_case_is_a_stack_kernel_problem(case):
    """Two-layer chains, ungrouped, 3x3 or 1x1 taps, rows of a multiple of 4 floats and at most kStageFloats, at most kBcExCols
    second-layer columns: the conditions of cle_engine.cu::stack_ineligible."""
    stage, ex_cols = _source_value("rowpipe.cuh", "kStageFloats"), _source_value("bc_stream.cuh", "kBcExCols")
    for shapes in case["chains"]:
        assert len(shapes) == 2
        (c1, *_), (_, j2, *k2) = shapes
        assert c1 == j2, "grouped relation"
        for s in shapes:
            kk = int(np.prod(s[2:])) if len(s) > 2 else 1
            assert kk in (1, 9) and (s[1] * kk) % 4 == 0 and s[1] * kk <= stage, s
        assert j2 <= ex_cols


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_exit_comparisons_keep_a_margin_and_runs_terminate(case):
    """In every sweep of every group, |diff - diff_tmp| is at least MARGIN (relative) away from 1e-9 and diff_tmp at least
    MARGIN away from converge_thres: the kernels' metric (fp32 partial sums per lane, then float64) cannot stop a group one
    sweep early or late.  Without max_sweeps every group stops on its own within 200 sweeps (never on the kernels' 4096 cap)."""
    _, before = SC.case_data(case)
    params = dict(case["params"], max_sweeps=0)
    with np.errstate(all="ignore"):
        _, _, sweeps, diffs, _ = SC.oracle_chains(before, case["one_group"], params)
    assert max(sweeps) <= 200, sweeps
    for g, d in enumerate(diffs):
        converged, margins = SC.exit_trace(d, params)
        assert converged
        worst = min(min(m) for m in margins)
        assert worst >= MARGIN, (g, worst, int(np.argmin([min(m) for m in margins])))
