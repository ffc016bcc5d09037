"""Bytes actually moved per calibration step of the synthetic stack (bench.py's workload) and the bandwidth they take.

bench.py's `roofline.whole_step` counts the unfused algorithm, 26 B per weight: fold 8 + two sweeps 16 + correction 2.  With
the fold deferred into the first sweep (plan_bn_fold(..., cle_plan=...) when the stack kernel takes the plan) a step moves
  fold       read-only scan of the second convs (column extrema) and of the first P rows of the first convs (row extrema,
             DFQ_ROW_PREFIX, default 16): 2 B + 2 P / rows B per weight, 2.06 B at P = 16 of 512 rows
  equalize   8 B per weight per pass over the weights (read + write); the first pass applies sweeps 1 and 2 when the
             stack kernel's guard accepts (CleResult.fused_sweeps = 2), every later sweep is a pass of its own.  When the
             prefix does not decide the guard (CleResult.rows_streamed != ROWS_STREAMED) the kernel first reads the other
             rows of the first convs: 2 (rows - P) / rows B per weight more
  correct    0 B per weight when the equalization computed it in its fused pass (CleResult.bc_prepared: the correction
             planned with cle_plan=..., every group stopped after sweep 2) and only the deltas are retired; otherwise it
             reads the second conv once: 2 B per weight averaged over both convs
i.e. about 10.06 B per weight at 2 fused sweeps (12.06 B when the correction reads the weights again).  This prints those
bytes and the achieved TB/s of each phase and of the whole step, per phase timed with CUDA events like bench.py (state
restored from a pristine copy, untimed, before every step).  `prefix_margin`: the smallest ratio over all blocks of the
guard's bound from the row prefix to 2 x converge_thres (above 1: the prefix decides for every block).

    python tools/bench_fold_defer.py [--pairs 2048] [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dfq_b200.engine import Session          # noqa: E402
from dfq_b200.workload import DeviceStack    # noqa: E402
from dfq_b200._lib import ROWS_STREAMED       # noqa: E402


def prefix_margin(sess, st, pristine, thres=2e-7, s_range=(1e-8, 1e8)):
    """min over blocks of the guard's bound from the scanned row prefix (cle_engine.cu fuse_guard_scan<true>: fuse_term_bound
    over rows / columns [0, P)) / (2 x thres), from the extrema the fold leaves.  None without a prefix."""
    fp = st.fold_plan
    if not fp["rows_scanned"] or not fp.get("row_prefix"):
        return None
    st.state().copy_(pristine)
    sess.run_bn_fold(fp)
    torch.cuda.synchronize()
    arena, lt, rt = sess.arena, st.cle_plan["lt"], st.cle_plan["rt"]
    P = min(int(fp["row_prefix"]), st.C)
    idx = torch.arange(P, device=arena.device)
    out = []
    for li, off in fp["rows_scanned"]:
        l = lt[li]
        l2 = lt[int(rt[int(l["rel_out"])]["second"])]
        rmn, rmx = arena[off + idx], arena[off + int(l["rows"]) + idx]
        cmn, cmx = arena[int(l2["cmin_off"]) + idx], arena[int(l2["cmax_off"]) + idx]
        r1, r2 = rmx - rmn, cmx - cmn
        s = (1.0 / r1) * torch.sqrt(r1 * r2)
        s = torch.where(torch.isnan(s) | (s >= s_range[1]), torch.full_like(s, s_range[1]), s).clamp_min(s_range[0])
        inv = 1.0 / s

        def bound(mn, mx, f):
            m = torch.maximum(mn.abs(), mx.abs()).double()
            t = m * ((f.double() - 1.0).abs() - 2.0 ** -24 * f.double()) - 2.0 ** -149
            return torch.where((t > 0) & (t < 1e300), t, torch.zeros_like(t))
        n1 = float(l["rows"]) * float(l["cols"]) * float(l["kk"])
        n2 = float(l2["rows"]) * float(l2["cols"]) * float(l2["kk"])
        out.append(bound(rmn, rmx, s).sum() / n1 + bound(cmn, cmx, inv).sum() / n2)
    sess.finish_fold()
    return float(torch.stack(out).min()) / (2.0 * thres)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    sess = Session()
    st = DeviceStack(sess, args.pairs // 2, 512, 3, seed=1234)      # a block = two Conv+BN pairs
    st.generate()
    pristine = st.state().clone()
    deferred = bool(st.fold_plan["deferred"])
    margin = prefix_margin(sess, st, pristine)
    times, res = [], None
    for i in range(args.warmup + args.steps):
        st.state().copy_(pristine)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        sess.run_bn_fold(st.fold_plan)
        ev[1].record()
        res = sess.run_cle_plan(st.cle_plan, cols_ready=st.fold_plan["scanned"])
        ev[2].record()
        sess.run_bias_correct_plan(st.bc_plan, 8, col_hints=sess.cle_col_hints(st.cle_plan, res))
        ev[3].record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            times.append([ev[k].elapsed_time(ev[k + 1]) for k in range(3)])
    fold_ms, cle_ms, bc_ms = (sum(t[k] for t in times) / len(times) for k in range(3))
    n = st.N * st.n_layers                          # weights of the stack
    sweeps = int(res.n_sweeps)
    rows_scanned = bool(st.fold_plan["rows_scanned"])
    # read-only scan of both convs / of the second convs only / read + write of every weight
    rows = st.C
    prefix = min(int(st.fold_plan.get("row_prefix", 0)) or rows, rows) if rows_scanned else 0
    fold_b = ((2.0 + 2.0 * prefix / rows) if rows_scanned else 2.0 if deferred else 8.0) * n
    passes = sweeps - 1 if res.fused_sweeps == 2 else sweeps
    cle_b = 8.0 * passes * n
    if rows_scanned and res.rows_streamed != ROWS_STREAMED:
        cle_b += 2.0 * (rows - prefix) / rows * n      # the kernel reads the rows the prefix left out
    bc_b = 0.0 if res.bc_prepared else 2.0 * n
    step_ms = fold_ms + cle_ms + bc_ms
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    out = {"gpu": props.name, "pairs": st.n_layers, "sweeps": sweeps, "fold_deferred": deferred,
           "fused_sweeps": res.fused_sweeps, "passes": passes, "bc_prepared": res.bc_prepared, "row_prefix": prefix,
           "rows_streamed": res.rows_streamed, "prefix_margin": margin,
           "bytes_per_weight": {"fold": fold_b / n, "equalize": cle_b / n, "correct": bc_b / n,
                                "step": (fold_b + cle_b + bc_b) / n},
           "ms": {"fold": fold_ms, "equalize": cle_ms, "correct": bc_ms, "step": step_ms},
           "TB/s": {"fold": fold_b / (fold_ms * 1e-3) / 1e12, "equalize": cle_b / (cle_ms * 1e-3) / 1e12,
                    "correct": (bc_b / (bc_ms * 1e-3) / 1e12) if bc_b else None, "step": (fold_b + cle_b + bc_b) / (step_ms * 1e-3) / 1e12}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
