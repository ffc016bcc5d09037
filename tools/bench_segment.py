"""Segmentation evaluation throughput on the H100: the reference's per-batch evaluation work against the best torch-only
GPU path and dfq_b200.segment; prints one JSON line.

    python tools/bench_segment.py [--batches 8,32] [--steps 10] [--warmup 2]

Workload: the DeepLab-v3+ of tests/deeplab_mobilenet_padded.py in the reference's evaluation state (tests/
affine_observed_state.py: replace_op() active, observers calibrated), converted with int8.convert_affine and chained with
int8.chain_affine(residual=True, concat=True, fold_pads=True), at 513x513.  Inputs are seeded; labels are seeded, VOC-like
float32 maps (what the reference's dataset yields): mostly background, a few classes in blocks, 255 borders.  Two input
batches alternate.  Arms, each producing the same confusion matrix:
  reference    the full model, torch.max(logits, 1)[1], both maps copied to the host and cast to uint8, then the
               Evaluator's mask and np.bincount (forward_all's per-batch work; its copy of the images to the host is left
               out)
  torch_gpu    the full model, torch.max and a masked torch.bincount on the device
  segment      split_upsample's head, then Evaluator.add_logits
Per arm: images/s of the whole step (host clock, ending in a device synchronise), the post-network time alone (host clock
for the reference arm, CUDA events for the others, on logits computed beforehand), and the bytes each post-network step
moves, computed from shapes.  A separate torch.profiler run gives the kernel times of torch_gpu's interpolate + max +
bincount against k_seg_argmax.  The per-batch matrices of the three arms are asserted equal on every timed batch.  The
card's name and power limit are read in the same run; the calibration's progress messages go to stderr.  Needs a CUDA
device; writes nothing.
"""
import argparse
import contextlib
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_int8 import card  # noqa: E402

C, S = 21, 513


def _labels(B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.zeros(B, S, S, device="cuda")
    for n in range(B):
        for _ in range(3):
            c = int(torch.randint(1, C, (1,), device="cuda", generator=g))
            y, x, h, w = (int(v) for v in torch.randint(0, 300, (4,), device="cuda", generator=g))
            lab[n, y:y + h // 2 + 20, x:x + w // 2 + 20] = c
    lab[:, :4] = 255.
    lab[:, -4:] = 255.
    lab[:, :, :4] = 255.
    lab[:, :, -4:] = 255.
    return lab


def _host_matrix(gt, pred):
    """The reference's Evaluator._generate_matrix on uint8 maps."""
    mask = (gt >= 0) & (gt < C)
    return np.bincount(C * gt[mask].astype(int) + pred[mask], minlength=C * C).reshape(C, C)


def _torch_matrix(labels, pred):
    ok = (labels > -1) & (labels < 256)
    gt = labels.long()                                      # in range: truncation toward zero, as astype(np.uint8)
    keep = ok & (gt >= 0) & (gt < C)
    idx = torch.where(keep, C * gt + pred, C * C)
    return torch.bincount(idx.view(-1), minlength=C * C + 1)[:C * C].view(C, C)


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


def _kernels(fns):
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        rows = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                rows[e.key[:80]] = round(e.device_time_total / 5, 1)
        out[name] = {"kernels_us_per_batch": rows, "total_us_per_batch": round(sum(rows.values()), 1)}
    return out


def _bytes(B, h, w):
    """Main-memory traffic of the post-network step per batch, from shapes (the largest tensors only)."""
    low, full, px = 4 * B * C * h * w, 4 * B * C * S * S, B * S * S
    return {"reference": {"device": full + full + 12 * px, "to_host": 8 * px + 4 * px,
                          "note": "interpolate writes the logits, max reads them and writes values + indices; both maps "
                                  "go to the host"},
            "torch_gpu": {"device": low + full + full + 12 * px + 4 * px + 8 * px + 8 * px,
                          "note": "interpolate, max (values + indices), the mask and bincount's index map"},
            "segment": {"device": low + 4 * px + 8 * C * C,
                        "note": "the low-resolution logits once (L2-resident), the labels, the matrix"}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_segment needs a CUDA device")
    import affine_observed_state
    from dfq_b200 import int8, segment
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": card(), "size": S, "classes": C, "results": []}
    with contextlib.redirect_stdout(sys.stderr), \
            affine_observed_state.evaluation_state("deeplab", size=S, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
        head, ac = segment.split_upsample(gm)
        for B in (int(b) for b in a.batches.split(",")):
            g = torch.Generator(device="cuda").manual_seed(B)
            xs = [torch.randn(B, 3, S, S, device="cuda", generator=g).clamp_(-2.5, 2.5) for _ in range(2)]
            labs = [_labels(B, B + i) for i in range(2)]
            ev = segment.Evaluator(C)
            got = {"reference": [], "torch_gpu": [], "segment": []}

            def ref_step(i):
                with torch.no_grad():
                    out = gm(xs[i % 2])
                pred = torch.max(out, 1)[1].cpu().numpy().astype(np.uint8)
                lab = labs[i % 2].cpu().numpy().astype(np.uint8)
                return _host_matrix(lab, pred)

            def torch_step(i):
                with torch.no_grad():
                    out = gm(xs[i % 2])
                return _torch_matrix(labs[i % 2], torch.max(out, 1)[1])

            def seg_step(i):
                with torch.no_grad():
                    low = head(xs[i % 2])
                before = ev.counts.clone() if ev.counts is not None else None
                ev.add_logits(labs[i % 2], low, align_corners=ac)
                return ev.counts - before if before is not None else ev.counts.clone()

            arms = {}
            for name, step in (("reference", ref_step), ("torch_gpu", torch_step), ("segment", seg_step)):
                for i in range(a.warmup):
                    step(i)
                torch.cuda.synchronize()
                t = time.perf_counter()
                for i in range(a.steps):
                    got[name].append(step(i))
                torch.cuda.synchronize()
                arms[name] = {"images_per_s": round(B * a.steps / (time.perf_counter() - t), 1)}
            for i in range(a.steps):
                r = got["reference"][i]
                assert np.array_equal(got["torch_gpu"][i].cpu().numpy(), r), ("torch_gpu", B, i)
                assert np.array_equal(got["segment"][i].cpu().numpy(), r), ("segment", B, i)
            # the post-network step alone, on logits computed beforehand
            with torch.no_grad():
                full, low = gm(xs[0]), head(xs[0])
            lab = labs[0]

            def ref_post():
                pred = torch.max(full, 1)[1].cpu().numpy().astype(np.uint8)
                return _host_matrix(lab.cpu().numpy().astype(np.uint8), pred)
            ref_post()
            t = time.perf_counter()
            for _ in range(a.steps):
                ref_post()
            arms["reference"]["post_network_ms"] = round((time.perf_counter() - t) * 1e3 / a.steps, 3)
            arms["torch_gpu"]["post_network_ms"] = round(_events(lambda: _torch_matrix(lab, torch.max(full, 1)[1]),
                                                                 a.steps), 3)
            arms["torch_gpu"]["post_network_from_low_ms"] = round(_events(lambda: _torch_matrix(lab, torch.max(
                F.interpolate(low, (S, S), mode="bilinear", align_corners=ac), 1)[1]), a.steps), 3)
            arms["segment"]["post_network_ms"] = round(_events(lambda: ev.add_logits(lab, low, align_corners=ac),
                                                               a.steps), 3)
            with torch.no_grad():
                net_ms = _events(lambda: gm(xs[0]), a.steps)
                head_ms = _events(lambda: head(xs[0]), a.steps)
            res["results"].append({
                "batch": B, "network_ms": round(net_ms, 3), "head_ms": round(head_ms, 3), "arms": arms,
                "bytes_per_batch": _bytes(B, *low.shape[2:]), "parity_batches": a.steps,
                "profile": _kernels({
                    "torch_gpu": lambda: _torch_matrix(lab, torch.max(F.interpolate(low, (S, S), mode="bilinear",
                                                                                    align_corners=ac), 1)[1]),
                    "segment": lambda: ev.add_logits(lab, low, align_corners=ac)})})
            del xs, labs, full, low, got
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
