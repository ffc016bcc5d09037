"""Bytes actually moved per calibration step of the synthetic stack (bench.py's workload) and the bandwidth they take.

bench.py's `roofline.whole_step` counts the unfused algorithm, 26 B per weight: fold 8 + two sweeps 16 + correction 2.  With
the fold deferred into the first sweep (plan_bn_fold(..., cle_plan=...) when the stack kernel takes the plan) a step moves
  fold       read-only scan of the second conv: 4 B per second-conv weight = 2 B per weight averaged over both convs
  equalize   8 B per weight per sweep (read + write)
  correct    reads the second conv once: 2 B per weight averaged
i.e. 20 B per weight at 2 sweeps.  This prints those bytes and the achieved TB/s of the fold scan and of the whole step, per
phase timed with CUDA events like bench.py (state restored from a pristine copy, untimed, before every step).

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
    fold_b = (2.0 if deferred else 8.0) * n         # scan of the second convs / read + write of every weight
    cle_b = 8.0 * sweeps * n
    bc_b = 2.0 * n
    step_ms = fold_ms + cle_ms + bc_ms
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    out = {"gpu": props.name, "pairs": st.n_layers, "sweeps": sweeps, "fold_deferred": deferred,
           "bytes_per_weight": {"fold": fold_b / n, "equalize": cle_b / n, "correct": bc_b / n,
                                "step": (fold_b + cle_b + bc_b) / n},
           "ms": {"fold": fold_ms, "equalize": cle_ms, "correct": bc_ms, "step": step_ms},
           "TB/s": {"fold": fold_b / (fold_ms * 1e-3) / 1e12, "equalize": cle_b / (cle_ms * 1e-3) / 1e12,
                    "correct": bc_b / (bc_ms * 1e-3) / 1e12, "step": (fold_b + cle_b + bc_b) / (step_ms * 1e-3) / 1e12}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
