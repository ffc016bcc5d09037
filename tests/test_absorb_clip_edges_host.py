"""CPU guards of the absorption-and-clipping edge cases (tests/absorb_clip_edges.py, run on the GPU by
tests/test_gpu_absorb_clip_edges.py): from the oracle alone, every case reaches what its claims name - c positive, exactly
zero, NaN or inf; clip bounds on weight values, biting on one side or none, a zero or constant range, subnormal bounds;
degenerate, non-finite and signed-zero taps; ranges that send k_bc_stream to the IEEE chain - and the chains take every
branch of both correction kernels."""
import numpy as np
import pytest

import absorb_clip_edges as AE
import stack_cases as SC
from test_boundary_guards import _source_value

FLT_MIN = np.finfo(np.float32).tiny
KNOWN = {"zero_rows", "subnormal_taps", "bound_is_weight", "bites_lo", "bites_hi", "c_positive", "negative_factors",
         "zero_fake_weight", "range_zero", "negative_zero_taps", "zero_var", "range_constant", "no_weight_inside", "clip_noop",
         "c_exact_zero", "subnormal_bounds", "nan_taps", "inf_taps", "c_nan", "c_inf", "ieee_chain"}


def _weights(folded, corrected_only=False):
    return [l[0] for cl in folded for k, l in enumerate(cl) if k >= 1 or not corrected_only]


@pytest.mark.parametrize("case", AE.CASES, ids=[c["name"] for c in AE.CASES])
def test_case_reaches_what_it_claims(case):
    claims = case["claims"]
    assert set(claims) <= KNOWN, set(claims) - KNOWN
    folded = AE.folded_chains(case)
    clip = AE.clip_of(case, folded)
    vec = AE.absorb_vectors(folded, case["N"])
    cs = [c for rel in vec for c, _ in rel]
    ws = _weights(folded)
    finite = np.concatenate([w[np.isfinite(w)].ravel() for w in ws])
    if clip is not None:
        lo, hi = np.float32(clip[0]), np.float32(clip[1])
        assert np.isfinite(lo) and np.isfinite(hi) and lo <= hi       # what the entry accepts
    # ---- c ----
    if claims.get("c_positive"):
        assert all((c > 0).any() for rel in vec for c, _ in rel), "a relation without a positive c"
    if claims.get("c_exact_zero"):
        hits = 0
        for cl, rel in zip(folded, vec):
            for k, (c, _) in enumerate(rel):
                fw, fb = cl[k][2], cl[k][3]
                m = (fb == (np.float32(case["N"]) * fw).astype(np.float32)) & (fb != 0)
                assert (c[m] == 0).all() and not np.signbit(c[m]).any()
                hits += int(m.sum())
                assert ((c > 0) & (c < 1e-5 * np.abs(fb))).any(), "no c one ulp above zero"
        assert hits > 0
    if claims.get("c_nan"):
        assert any(np.isnan(c).any() for c in cs)
    if claims.get("c_inf"):
        assert any(np.isposinf(c).any() for c in cs)
        assert all(np.isfinite(l[2]).all() for cl in folded for l in cl)   # N * fake_weight overflows, not the data
    # ---- the clip ----
    every = np.concatenate([w.ravel() for w in ws])       # NaN compares False: only what the clip moves
    if "bites_lo" in claims:
        assert bool((every < lo).any()) == claims["bites_lo"]
    if "bites_hi" in claims:
        assert bool((every > hi).any()) == claims["bites_hi"]
    if claims.get("bound_is_weight"):
        w = folded[0][1][0]
        assert (w == lo).any() and (w == hi).any() and lo < hi
    if claims.get("range_zero"):
        assert lo == 0 and hi == 0
    if claims.get("range_constant"):
        assert lo == hi and lo != 0
    if claims.get("no_weight_inside"):
        assert not ((finite >= lo) & (finite <= hi)).any()
    if claims.get("clip_noop"):
        assert all(np.array_equal(AE.clipped(w, clip).view(np.uint32), w.view(np.uint32)) for w in ws)
    if claims.get("subnormal_bounds"):
        assert 0 < abs(lo) < FLT_MIN and 0 < abs(hi) < FLT_MIN
    if claims.get("ieee_chain"):
        refused = [AE.fast_quant_refuses(*np.clip(np.array([np.fmin.reduce(w.ravel()), np.fmax.reduce(w.ravel())], np.float32), lo, hi))
                   for w in _weights(folded, corrected_only=True)]
        assert any(refused), "bc_fast_quant takes every corrected layer"
    # ---- the data ----
    if claims.get("zero_rows"):
        assert any((np.abs(w.reshape(w.shape[0], -1)).max(axis=1) == 0).any() for w in ws)
    if claims.get("subnormal_taps"):
        assert any(((np.abs(w) > 0) & (np.abs(w) < FLT_MIN)).any() for w in ws)
    if claims.get("negative_zero_taps"):
        assert any(((w == 0) & np.signbit(w)).any() for w in ws)
    if claims.get("nan_taps"):
        assert all(np.isnan(w).any() for w in _weights(folded, corrected_only=True))
    if claims.get("inf_taps"):
        assert all(np.isposinf(w).any() and np.isneginf(w).any() for w in _weights(folded, corrected_only=True))
    lay = SC.chain_layers(case["chains"], case["seed"], case["edit"])
    if claims.get("negative_factors"):
        assert any((d["gamma"] < 0).any() for cl in lay for d in cl)
    if claims.get("zero_fake_weight"):
        assert any((l[2] == 0).any() for cl in folded for l in cl[:-1])
    if claims.get("zero_var"):
        assert any((d["var"] == 0).any() and d["bn_eps"] == 1e-3 for cl in lay for d in cl)


def test_chains_take_every_branch_of_both_kernels():
    """k_bc_engine: tiles of several rows (a warp per row) and of one row; k_bc_stream: staged rows, TK_PLAIN rows and
    TK_DIRECT rows; E[x] cached (<= kBcExCols columns) and not; a depthwise and a grouped (wc_so > 1) second layer; a layer
    with both an input and an output relation (AcSlot.sub_c_off) next to first layers without an entry (first_bias)."""
    stage, max_rows = _source_value("rowpipe.cuh", "kStageFloats"), _source_value("rowpipe.cuh", "DFQ_PIPE_MAX_ROWS")
    ex_cols = _source_value("bc_stream.cuh", "kBcExCols")
    seen = set()
    for shapes in AE.CHAINS:
        for k in range(1, len(shapes)):
            rows, cols = shapes[k][0], shapes[k][1]
            kk = int(np.prod(shapes[k][2:])) if len(shapes[k]) > 2 else 1
            row_len = cols * kk
            per_tile = 1 if row_len > stage else min(stage // row_len, max_rows)
            seen.add("multi_row" if per_tile > 1 else "single_row")
            seen.add("direct" if row_len > stage else ("plain" if row_len % 4 else "bulk"))
            seen.add("ex_cached" if cols <= ex_cols else "ex_global")
            groups = shapes[k - 1][0] // cols
            if groups == rows and cols == 1:
                seen.add("depthwise")
            elif groups > 1 and rows // groups > 1:
                seen.add("grouped_wc_so")
            if k < len(shapes) - 1:
                seen.add("sub_c")
    assert seen >= {"multi_row", "single_row", "direct", "plain", "bulk", "ex_cached", "ex_global", "depthwise", "grouped_wc_so",
                    "sub_c"}, seen


def test_cases_cover_the_issue_list():
    """N = 3, 0, -0.25 and an overflowing N; each kind of clip range at least once."""
    assert {3.0, 0.0, -0.25, -3e38} <= {c["N"] for c in AE.CASES}
    claims = set().union(*(c["claims"] for c in AE.CASES))
    assert {"bound_is_weight", "range_zero", "range_constant", "no_weight_inside", "clip_noop", "subnormal_bounds",
            "ieee_chain", "c_nan", "c_inf", "c_exact_zero", "nan_taps", "inf_taps"} <= claims
    assert any(c["clip"] is None for c in AE.CASES)
    assert any(c["claims"].get("bites_hi") and c["claims"].get("bites_lo") is False for c in AE.CASES)
