"""Seeded inputs of dfq_b200.detect.Evaluator for the tests and tools/bench_detect_map.py: the committed fixture
tests/golden/ref_ssd_map.npz, and VOC-like scenes of annotations and detections (jittered copies of the annotations plus
clutter) with the layout postprocess returns."""
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ssd_map.npz")


def split(offsets, *arrays):
    """Per-image slices of flat arrays."""
    return [tuple(a[s:e] for a in arrays) for s, e in zip(offsets[:-1], offsets[1:])]


def fixture():
    """(z, num_classes, gts [(boxes, labels, difficult)] per image, dets [(boxes, labels, probs) tensors] per image)."""
    z = np.load(GOLD)
    gts = split(z["gt_offsets"], z["gt_boxes"], z["gt_labels"], z["gt_difficult"])
    dets = [tuple(torch.from_numpy(a) for a in t)
            for t in split(z["det_offsets"], z["det_boxes"], z["det_labels"], z["det_probs"])]
    return z, int(z["num_classes"]), gts, dets


def scene(N, C, seed, max_gt=6, copies=3, clutter=8, empty=0.1, ties=False, difficult=0.15):
    """N images of C classes: up to max_gt annotated boxes per image (a fraction `empty` of the images has none), each
    with up to `copies` jittered detections, plus up to `clutter` random detections.  Pixel boxes in 0 .. 500.  Scores are
    rounded to 1/64 when ties is set, so that equal scores are common.  Detection rows are ordered as postprocess orders
    them: class ascending, score descending (equal scores in generation order)."""
    g = np.random.default_rng(seed)
    gts, dets = [], []
    for _ in range(N):
        k = 0 if g.random() < empty else int(g.integers(1, max_gt + 1))
        xy = g.uniform(0, 400, (k, 2))
        wh = g.uniform(8, 250, (k, 2))
        boxes = np.concatenate([xy, np.minimum(xy + wh, 500)], 1).astype(np.float32)
        labels = g.integers(1, C, k).astype(np.int64)
        diff = (g.random(k) < difficult).astype(np.uint8)
        gts.append((boxes, labels, diff))
        n_copies = g.integers(0, copies + 1, k)
        src = np.repeat(np.arange(k), n_copies)
        jit = boxes[src] + g.normal(0, 0.08, (len(src), 4)) * np.tile(boxes[src, 2:] - boxes[src, :2], 2)
        m = int(g.integers(0, clutter + 1))
        cxy = g.uniform(0, 450, (m, 2))
        clut = np.concatenate([cxy, cxy + g.uniform(5, 120, (m, 2))], 1)
        rb = np.concatenate([jit, clut]).astype(np.float32).reshape(-1, 4)
        rl = np.concatenate([labels[src], g.integers(1, C, m)]).astype(np.int64)
        scores = g.uniform(0.011, 1.0, len(rl)).astype(np.float32)
        if ties:
            scores = np.round(scores * 64).astype(np.float32) / 64
        order = np.lexsort((-scores, rl))                # stable: equal scores keep generation order
        dets.append((torch.from_numpy(rb[order].copy()), torch.from_numpy(rl[order].copy()),
                     torch.from_numpy(scores[order].copy())))
    return gts, dets


def detections(dets, device):
    """A detect.Detections of per-image (boxes, labels, probs)."""
    from dfq_b200 import detect
    offs = torch.tensor(np.cumsum([0] + [l.numel() for _, l, _ in dets]), dtype=torch.int64)
    cat = [torch.cat([d[i].reshape(-1, 4) if i == 0 else d[i].reshape(-1) for d in dets]) for i in range(3)]
    return detect.Detections(cat[0].float().contiguous().to(device), cat[1].long().to(device), cat[2].float().to(device),
                             offs.to(device))
