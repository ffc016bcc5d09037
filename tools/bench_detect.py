"""SSD post-processing throughput on the H100: the reference-style per-image CPU post-processing against
dfq_b200.detect.postprocess on the device; prints one JSON line.

    python tools/bench_detect.py [--batches 256,1] [--reps 20] [--cpu-images 32] [--nms hard,soft] [--soft-cpu-images 2]

Two workloads at each batch size: `ssd_lite_int8`, the outputs of the SSD-Lite of tests/ssd_lite_like.py (seeded
weights, chained with int8.chain_int8(..., layout=True), 300x300 inputs) with the priors of mobilenetv1_ssd_config - a
random network keeps nearly every prior as a candidate of every class; and `peaked`, synthetic softmax scores with about
20 candidates per class, closer to a trained model.  Arms: `cpu`, the decode on the GPU then, image by image on the CPU,
threshold, stable sort and hard NMS in torch ops (tests/ssd_postprocess_oracle.py, reached through
tests/ssd_soft_nms_oracle.py; what Predictor.predict runs), timed over the first --cpu-images images of the batch;
`gpu`, postprocess on the whole batch (host wall clock to its result, and CUDA events), plus the per-kernel times from
torch.profiler.  `with_network` adds the chained network's time for the batch.  With hard NMS the kept boxes, labels and
probs of the two arms are asserted equal on every timed batch (on the CPU arm's images).  The card's name and power
limit are read in the same run.  Needs a CUDA device; writes nothing.

`--nms soft` times postprocess(nms_method="soft") instead, on a third workload as well, `seeded`: the seeded
SSD-Lite-shaped outputs tools/make_golden.py makes (about 800 candidates per class).  Its CPU arm runs the soft NMS of
tests/ssd_soft_nms_oracle.py on the CPU (the loop of box_utils.soft_nms) over the first --soft-cpu-images images.  The
scores may differ in their last bits, where CUDA's expf and torch's CPU exp differ, and such a difference can change a
later pick: `same_boxes_images` counts the compared images whose boxes and labels are equal, and `prob_max_ulp` is the
largest score difference among them.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_int8 import card  # noqa: E402

import ssd_soft_nms_oracle as SO  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "ref_ssd_postprocess.npz")


def _network(batch):
    """(chained SSD-Lite, input, priors, cv, sv)."""
    from dfq_b200 import int8
    import test_gpu_int8_layout as GL
    model, _ = GL._net("ssd", 2, 300, is_test=True)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
    z = np.load(GOLD)
    x = torch.randn(batch, 3, 300, 300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    return gm, x, torch.from_numpy(z["priors"]).cuda(), *(float(v) for v in z["variances"])


def _peaked(batch, P, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(batch, P, 21, device="cuda", generator=g)
    logits[..., 0] += 8.1          # ~20 of 3,000 priors above 0.01 per class
    return torch.softmax(logits, 2), torch.randn(batch, P, 4, device="cuda", generator=g) * 0.7


def _seeded(batch, P, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(batch, P, 21, device="cuda", generator=g) * 2.5
    logits[..., 0] += 5.0
    return torch.softmax(logits, 2), torch.randn(batch, P, 4, device="cuda", generator=g) * 0.7


def _ulps(a, b):
    ia, ib = (t.numpy().view(np.int32).astype(np.int64) for t in (a, b))
    ia, ib = (np.where(i < 0, np.int64(-2 ** 31) - i, i) for i in (ia, ib))
    return int(np.abs(ia - ib).max()) if ia.size else 0


def _events(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _wall(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / reps


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("k_ssd_decode", "k_ssd_nms", "k_ssd_scan", "k_ssd_compact", "k_ssd_soft"):
            if k in e.key:
                out[k + "_us"] = round(e.device_time_total / max(e.count, 1), 1)
    return out


def run(name, scores, loc, pri, cv, sv, net_ms, reps, cpu_images, nms="hard"):
    from dfq_b200 import detect
    B = scores.shape[0]
    post = lambda: detect.postprocess(scores, loc, pri, cv, sv, nms_method=nms)   # noqa: E731
    gpu_ms = _wall(post, reps)
    gpu_ev_ms = _events(post, reps)
    det = post()
    n = min(B, cpu_images)
    t = time.perf_counter()
    want = SO.predict(scores[:n], loc[:n], pri, cv, sv, nms_method=nms)
    cpu_ms = (time.perf_counter() - t) * 1e3 / n
    got = det.per_image()[:n]
    extra = {}
    if nms == "soft":
        same = [g[0].shape == w[0].shape and torch.equal(g[0], w[0]) and torch.equal(g[1], w[1])
                for g, w in zip(got, want)]
        extra["same_boxes_images"] = sum(same)
        extra["prob_max_ulp"] = max([_ulps(g[2], w[2]) for g, w, ok in zip(got, want, same) if ok] or [0])
    else:
        assert all(all(torch.equal(a, b) for a, b in zip(g, w)) for g, w in zip(got, want)), "arms differ"
    kept = det.offsets.diff().float().mean().item()
    return {"workload": name, "nms": nms, "batch": B, "kept_boxes_per_image": round(kept, 1), "parity_images": n, **extra,
            "cpu": {"ms_per_image": round(cpu_ms, 2), "images_per_s": round(1e3 / cpu_ms, 1),
                    "with_network_images_per_s": round(B * 1e3 / (net_ms + cpu_ms * B), 1)},
            "gpu": {"ms_per_batch_wall": round(gpu_ms, 3), "ms_per_batch_events": round(gpu_ev_ms, 3),
                    "images_per_s": round(B * 1e3 / gpu_ms, 1),
                    "with_network_images_per_s": round(B * 1e3 / (net_ms + gpu_ms), 1), **_kernels(post)},
            "network_ms_per_batch": round(net_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-images", type=int, default=32)
    ap.add_argument("--nms", default="hard", help="comma-separated: hard, soft")
    ap.add_argument("--soft-cpu-images", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detect needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "torch_cpu_threads": torch.get_num_threads(), "results": []}
    for B in (int(b) for b in a.batches.split(",")):
        gm, x, pri, cv, sv = _network(B)
        with torch.no_grad():
            net_ms = _events(lambda: gm(x), a.reps)
            scores, loc = gm(x)
            for nms in a.nms.split(","):
                ci = a.cpu_images if nms == "hard" else a.soft_cpu_images
                res["results"].append(run("ssd_lite_int8", scores, loc, pri, cv, sv, net_ms, a.reps, ci, nms))
                s, l = _peaked(B, pri.shape[0])
                res["results"].append(run("peaked", s, l, pri, cv, sv, net_ms, a.reps, ci, nms))
                if nms == "soft":
                    s, l = _seeded(B, pri.shape[0])
                    res["results"].append(run("seeded", s, l, pri, cv, sv, net_ms, a.reps, ci, nms))
        del gm, x
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
