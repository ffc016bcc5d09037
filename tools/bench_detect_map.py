"""VOC average-precision throughput on the H100: main_ssd.py's per-detection evaluation loop on the CPU against
dfq_b200.detect.Evaluator on the device; prints one JSON line.

    python tools/bench_detect_map.py [--kept 333,1636] [--cpu-images 24] [--batch 256] [--reps 5]

Workload: a VOC2007-test-sized set of 4,952 images and 21 classes, seeded annotations with difficult flags and detections
made of jittered copies of the annotations plus clutter, at about --kept detections per image (the kept-box counts
tools/bench_detect.py measured).  Arms:
  `cpu`        tests/ssd_map_oracle.py with the reference's structure - each detection through the text line main_ssd.py
               writes and reads back, then one Python step per detection - timed on the first --cpu-images images and
               reported per detection;
  `gpu`        Evaluator.add_batch per batch of --batch images plus one average_precision(), over all 4,952 images (the
               batches are on the device beforehand), host wall clock;
  `pipeline`   the chained SSD-Lite of tests/ssd_lite_like.py + postprocess + add_batch on batches of --batch images, in
               images/s, against the same pipeline without the evaluator.
The APs of the CPU and GPU arms are asserted equal on the CPU arm's images, and the pipeline's on its first images.  The
card's name and power limit are read in the same run.  Needs a CUDA device; writes nothing.
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

import map_scenes as MS  # noqa: E402
import ssd_map_oracle as O  # noqa: E402

IMAGES, CLASSES = 4952, 21


def _equal(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def _gpu_eval(batches, use_2007=True):
    from dfq_b200 import detect
    ev = detect.Evaluator(CLASSES, 0.5, use_2007)
    for det, gt in batches:
        ev.add_batch(det, gt)
    return ev.average_precision()


def run_set(kept, cpu_images, batch, reps):
    from dfq_b200 import detect
    gts, dets = MS.scene(IMAGES, CLASSES, seed=kept, max_gt=8, copies=4, clutter=2 * kept - 20, difficult=0.1)
    D = sum(l.numel() for _, l, _ in dets)
    batches = [(MS.detections(dets[a:a + batch], "cuda"), detect.ground_truth(gts[a:a + batch], "cuda"))
               for a in range(0, IMAGES, batch)]
    out = {"kept_per_image": round(D / IMAGES, 1), "detections": D}
    for use_2007 in (True, False):
        _gpu_eval(batches, use_2007)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(reps):
            _gpu_eval(batches, use_2007)
        gpu_ms = (time.perf_counter() - t) * 1e3 / reps
        out["gpu_2007" if use_2007 else "gpu_area"] = {"ms_per_set": round(gpu_ms, 2),
                                                       "ns_per_detection": round(gpu_ms * 1e6 / D, 2)}
    sd, sg = dets[:cpu_images], gts[:cpu_images]
    n = sum(l.numel() for _, l, _ in sd)
    t = time.perf_counter()
    want, _ = O.average_precision(sd, sg, CLASSES, 0.5, True, text=True)
    cpu_s = time.perf_counter() - t
    got = _gpu_eval([(MS.detections(sd, "cuda"), detect.ground_truth(sg, "cuda"))])
    assert _equal(got, want), "arms differ"
    out["cpu"] = {"images": cpu_images, "detections": n, "us_per_detection": round(cpu_s * 1e6 / n, 1),
                  "projected_s_per_set": round(cpu_s / n * D, 1)}
    out["speedup_2007"] = round(cpu_s / n * D * 1e3 / out["gpu_2007"]["ms_per_set"], 1)
    return out


def run_pipeline(batch, reps, parity_images=8):
    from dfq_b200 import detect, int8
    import test_detect_host as TH
    import test_gpu_int8_layout as GL
    model, _ = GL._net("ssd", 2, 300, is_test=True)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
    z, t, cv, sv = TH.fixture()
    pri = t["priors"].cuda()
    x = torch.randn(batch, 3, 300, 300, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    sizes = torch.tensor([[500, 375]], device="cuda").expand(batch, 2).contiguous()
    gts, _ = MS.scene(batch, CLASSES, seed=2, max_gt=8, copies=0, clutter=0)
    gt = detect.ground_truth(gts, "cuda")
    ev = detect.Evaluator(CLASSES)

    def step(evaluate):
        with torch.no_grad():
            det = detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
        if evaluate:
            ev.add_batch(det, gt)
        return det

    res = {}
    for evaluate in (False, True):
        step(evaluate)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            step(evaluate)
        ev.average_precision() if evaluate else torch.cuda.synchronize()
        res["with_evaluator" if evaluate else "without_evaluator"] = round(batch * reps / (time.perf_counter() - t0), 1)
    det = step(False)
    per = det.per_image()[:parity_images]
    one = detect.Evaluator(CLASSES)
    one.add_batch(MS.detections(per, "cuda"), detect.ground_truth(gts[:parity_images], "cuda"))
    assert _equal(one.average_precision(), O.average_precision(per, gts[:parity_images], CLASSES)[0]), "arms differ"
    res["kept_per_image"] = round(det.offsets.diff().float().mean().item(), 1)
    return {"batch": batch, "images_per_s": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kept", default="333,1636")
    ap.add_argument("--cpu-images", type=int, default=24)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detect_map needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "images": IMAGES, "classes": CLASSES, "sets": {}}
    for k in (int(v) for v in a.kept.split(",")):
        res["sets"][str(k)] = run_set(k, a.cpu_images, a.batch, a.reps)
    res["pipeline"] = run_pipeline(a.batch, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
