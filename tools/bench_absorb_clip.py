"""Bias absorption and weight clipping inside GraphCalibration's residency against the separate calls.

Three arms, alternated step by step on freshly built (seeded, CPU-resident) models, as the mains calibrate them:
  fused     GraphCalibration.run(absorption=True, clip_weight=(lo, hi), correction=True, quantize_bits=(8, 16))
  separate  merge_batchnorm -> cross_layer_equalization -> bias_absorption -> clip_weight -> bias_correction ->
            quantize_targ_layer (main_cls.py:149-181), each call staging the model to the GPU and back
  plain     GraphCalibration.run(correction=True, quantize_bits=(8, 16)) without the two flags
on the config-5 synthetic stack (Conv+BN+ReLU -> Conv+BN blocks: every relation absorbs) and on the MobileNetV2 topology
of tests/golden.  Per arm: wall time of the whole calibration (host clock around work that ends in a
device synchronise), then, in a profiled run of its own, the kernel time per kernel name.  Bytes per weight are those the
absorption, clip and correction move (4 B per weight read, 4 B per clamped weight written); the check that the fused and the
separate arm leave the same model is made on the timed outputs.

    python tools/bench_absorb_clip.py [--blocks 8] [--channels 512] [--steps 3] [--warmup 1] [--clip 0.05] [--n 0]
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dfq_b200 import dfq, workload                       # noqa: E402
from dfq_b200.calibrate import GraphCalibration         # noqa: E402
from dfq_b200.utils import layer_transform as LT        # noqa: E402
from dfq_b200.utils.relation import create_relation     # noqa: E402

TARG = [nn.Conv2d, nn.Linear]
GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def arm(name, g, b, clip, n):
    if name == "separate":
        LT.merge_batchnorm(None, g, b, TARG)
        rels = create_relation(g, b, TARG)
        dfq.cross_layer_equalization(g, rels, TARG)
        dfq.bias_absorption(g, rels, b, n)
        dfq.clip_weight(g, [-clip, clip], TARG)
        dfq.bias_correction(g, b, TARG)
        LT.quantize_targ_layer(g, 8, 16, TARG)
    elif name == "fused":
        GraphCalibration(g, b, TARG).run(absorption=True, absorption_n=n, clip_weight=(-clip, clip), quantize_bits=(8, 16))
    else:
        GraphCalibration(g, b, TARG).run(quantize_bits=(8, 16))


def state(g):
    out = []
    for m in g.values():
        if type(m) in TARG:
            out += [m.weight.detach().clone(), m.bias.detach().clone()]
        elif isinstance(m, nn.BatchNorm2d) and hasattr(m, "fake_bias"):
            out += [m.fake_weight.clone(), m.fake_bias.clone()]
    return out


def run_model(label, topo, args):
    import torch.profiler as P
    names = ["fused", "separate", "plain"]
    times = {k: [] for k in names}
    equal = True
    for step in range(args.warmup + args.steps):
        outs = {}
        for name in names:
            g, b, _ = workload.build_graph(topo, seed=args.seed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            arm(name, g, b, args.clip, args.n)
            torch.cuda.synchronize()
            if step >= args.warmup:
                times[name].append(time.perf_counter() - t0)
            outs[name] = state(g)
        equal = equal and all(np.array_equal(x.numpy(), y.numpy()) for x, y in zip(outs["fused"], outs["separate"]))
        equal = equal and len(outs["fused"]) == len(outs["separate"])
    # per-kernel time, one profiled call per arm (after the timed ones: tracing slows the host)
    kernels = {}
    for name in names:
        g, b, _ = workload.build_graph(topo, seed=args.seed)
        with P.profile(activities=[P.ProfilerActivity.CUDA]) as prof:
            arm(name, g, b, args.clip, args.n)
            torch.cuda.synchronize()
        per = collections.Counter()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                per[e.name.split("(")[0][:60]] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        kernels[name] = {k: round(v / 1e3, 3) for k, v in per.most_common(12)}     # ms
    # bytes per weight of absorption + clip + correction: fused reads every corrected weight once and writes the clamped
    # ones; separate reads the absorbing seconds, reads and writes every weight (clip) and reads the corrected ones again
    g, b, _ = workload.build_graph(topo, seed=args.seed)
    GraphCalibration(g, b, TARG).run(absorption=True, absorption_n=args.n, quantize_bits=None, correction=False)
    w = torch.cat([m.weight.detach().reshape(-1) for m in g.values() if type(m) in TARG])
    clamped = float(((w < -args.clip) | (w > args.clip)).float().mean())
    return dict(model=label, weights=int(w.numel()), clamped_fraction=round(clamped, 4),
                wall_ms={k: round(1e3 * float(np.median(v)), 2) for k, v in times.items()},
                kernel_ms=kernels, fused_equals_separate=bool(equal),
                bytes_per_weight=dict(fused=round(4 + 4 * clamped, 3), separate_upper=16.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--channels", type=int, default=512)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--clip", type=float, default=0.05)
    ap.add_argument("--n", type=float, default=0.0, help="absorption N (the mains' 3 absorbs nothing on seeded BNs)")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures on the GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = dict(gpu=q[0] if q else torch.cuda.get_device_name(), args=vars(args), results=[])
    res["results"].append(run_model("stack_%dx%d" % (2 * args.blocks, args.channels),
                                    workload.stack_topology(args.blocks, channels=args.channels), args))
    res["results"].append(run_model("mobilenetv2", workload.load_topology(os.path.join(GOLD, "topology_mobilenetv2.json")), args))
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
