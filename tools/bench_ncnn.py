"""Images/s of the reference's int8 ncnn MobileNetV2 (model_quant_relu_equal, staged in oracle/_ref by build()) at one batch
size, three arms timed alternately in one run:

    interpreter   tests/ncnn_int8_case.Int8Net with Int8Conv2d / Int8Linear executors, its mean replaced by ncnn.PlaneMean
    per-layer     ncnn.load: one Int8Conv2d per weighted layer, fp32 between layers
    chained       int8.chain_int8(ncnn.load(...), residual=True, pool_cat=True): int8 codes between layers

The logits (blob 781) of the three arms are asserted equal, bit for bit, on every timed batch.  The card's name and power
limit are read in the same call.  Prints one JSON line.

    python tools/bench_ncnn.py [--batch 256] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_int8 import card  # noqa: E402

import ncnn_int8_case as case  # noqa: E402


def interpreter_arm():
    """The interpreter on GPU int8 layers built from the .bin's codes, with ncnn's plane mean before its InnerProduct."""
    from dfq_b200 import int8, ncnn
    net = case.Int8Net()
    mods = [int8.Int8Conv2d.from_codes(s["codes"], s["bias"], s["in_scale"], s["w_scales"], s["stride"], s["pad"],
                                       s["dilation"], s["groups"]) for s in net.specs]
    execute = lambda s, x: mods[s["index"]](x)                  # noqa: E731
    mean = ncnn.PlaneMean(False)
    fc = next(l["spec"] for l in net.layers if l["name"] == "781")

    def run(x):
        v = mean(net.forward(x, execute, upto="779")["779"])
        return execute(fc, v.reshape(v.shape[0], -1, 1, 1)).reshape(v.shape[0], -1)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ncnn needs a CUDA device")
    if case.paths() is None:
        raise SystemExit("the reference's int8 ncnn model is not staged in oracle/_ref (run __graft_entry__.build())")
    from dfq_b200 import int8, ncnn
    per_layer = ncnn.load(*case.paths(), outputs="781")
    chained = int8.chain_int8(ncnn.load(*case.paths(), outputs="781"), residual=True, pool_cat=True)
    arms = {"interpreter": interpreter_arm(), "per_layer": per_layer, "chained": chained}
    g = torch.Generator().manual_seed(0)
    batches = [torch.randn(a.batch, 3, 224, 224, generator=g).cuda() for _ in range(2)]
    times = {k: [] for k in arms}
    with torch.no_grad():
        for step in range(a.warmup + a.steps):
            x = batches[step % 2]
            logits = {}
            for name, f in arms.items():                         # alternately, one batch each
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                logits[name] = f(x)
                stop.record()
                stop.synchronize()
                if step >= a.warmup:
                    times[name].append(start.elapsed_time(stop) / 1e3)
            ref = logits["per_layer"]
            equal = {k: bool(torch.equal(v, ref)) for k, v in logits.items()}
            assert all(equal.values()), "logits differ at step %d: %s" % (step, equal)
    res = {"card": card(), "batch": a.batch, "steps": a.steps, "logits_equal_every_batch": True}
    for name, t in times.items():
        t = sorted(t)
        res[name] = {"images_per_s_median": round(a.batch / t[len(t) // 2], 1), "ms_median": round(t[len(t) // 2] * 1e3, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
