"""PNG label decoding on the H100 against Pillow; prints one JSON line.

    python tools/bench_png.py [--batches 8,32,256] [--reps 20] [--loop-batches 12]

Inputs are seeded VOC-like label maps of the sizes tools/bench_preprocess.py uses (500 x 375, 375 x 500, 500 x 333,
333 x 500, 500 x 486): class blobs with 255 borders on a flat background, saved by Pillow in P mode with its defaults.
Reported: Pillow's decode rate (np.array(Image.open(...))) on one core of this host; the device time of k_png_inflate
and k_png_unfilter per batch of each size (torch.profiler, in a run of its own); the wall time of
preprocess.voc_segmentation per batch of 32 with JPEG images and labels given as arrays against labels given as PNG bytes
(CUDA events around the calls, so the parse, the gather and the copy are in them); and main_seg.py's evaluation loop at
its 2 DataLoader workers with the chained affine int8 DeepLab-v3+ of tests/affine_observed_state.py (513, TF32 off) and
segment.Evaluator.add_logits behind it, for three kinds of worker:
  reference     Pillow decodes the JPEG and the label, the reference transform (FixScaleCrop + Normalize) runs there
  jpeg_bytes    the worker returns the JPEG's bytes and the label decoded by Pillow; voc_segmentation decodes the JPEG
  both_bytes    the worker returns both files' bytes; voc_segmentation decodes both on the device
Every timed output is asserted equal: the decoded labels to Pillow's, the calls' outputs to the array path's, and the
loop's network inputs, labels and confusion counts across the three kinds of worker.  The card's name and power limit
are read in the same run.  Needs a CUDA device; writes nothing.
"""
import argparse
import io
import json
import os
import sys
import time

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench_preprocess as BP  # noqa: E402
from bench_int8 import card  # noqa: E402
from dfq_b200 import jpeg, png, preprocess as P  # noqa: E402
import jpeg_corpus as JC  # noqa: E402
import png_corpus as PC  # noqa: E402

VOC = [(375, 500), (500, 375), (333, 500), (500, 333), (500, 486)]


def _labels(n, seed):
    return [PC.pil_p(PC.voc_label(*VOC[i % len(VOC)], seed + i)) for i in range(n)]


def _pillow_rate(items):
    t = time.perf_counter()
    for d in items:
        np.array(Image.open(io.BytesIO(d)))
    return len(items) / (time.perf_counter() - t)


def _kernel_us(items, want, reps):
    from torch.profiler import ProfilerActivity, profile
    png.decode(items)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        outs = [png.decode(items) for _ in range(reps)]
        torch.cuda.synchronize()
    for o in outs:                                        # every timed call's labels
        assert all(torch.equal(a, w) for a, w in zip(o, want))
    out = {}
    for e in prof.key_averages():
        for k in ("k_png_inflate", "k_png_unfilter"):
            if k in e.key:
                out[k] = round(e.device_time_total / reps, 1)
    return out


def _call_ms(images, labels, want, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    P.voc_segmentation(images, labels)
    torch.cuda.synchronize()
    s.record()
    outs = [P.voc_segmentation(images, labels) for _ in range(reps)]
    e.record()
    torch.cuda.synchronize()
    for x, y in outs:
        assert torch.equal(x, want[0]) and torch.equal(y, want[1])
    return round(s.elapsed_time(e) / reps, 3)


class _Seg(torch.utils.data.Dataset):
    """main_seg.py's evaluation items as one kind of worker returns them."""

    def __init__(self, items, kind):
        self.items, self.kind = items, kind

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        jpg, lab = self.items[i]
        if self.kind == "both_bytes":
            return jpg, lab
        label = np.array(Image.open(io.BytesIO(lab)))
        if self.kind == "jpeg_bytes":
            return jpg, torch.from_numpy(label)
        return BP._seg(Image.open(io.BytesIO(jpg)).convert("RGB"), label)


def _collate(batch):
    if isinstance(batch[0][0], torch.Tensor) and batch[0][0].dim() == 3:
        return torch.stack([b[0] for b in batch]), torch.stack([b[1] for b in batch])
    return [b[0] for b in batch], [b[1] for b in batch]


def _seg_loop(items, batch, workers):
    """images/s of the three kinds of worker with the chained DeepLab and the evaluator behind the loop."""
    import contextlib
    import affine_observed_state
    from dfq_b200 import int8, segment
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    with contextlib.redirect_stdout(sys.stderr), \
            affine_observed_state.evaluation_state("deeplab", size=513, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        head, ac = segment.split_upsample(int8.chain_affine(model, residual=True, concat=True, fold_pads=True))
        out, seen = {"workers": workers, "batch": batch}, []
        for kind in ("reference", "jpeg_bytes", "both_bytes"):
            dl = torch.utils.data.DataLoader(_Seg(items, kind), batch_size=batch, num_workers=workers, collate_fn=_collate,
                                             persistent_workers=False, prefetch_factor=2)
            got, t0 = [], None
            for i, (x, y) in enumerate(dl):
                if i == 1:                                # the first batch carries the workers' start-up
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                if kind == "reference":
                    x, y = x.cuda(non_blocking=True), y.cuda(non_blocking=True)
                else:
                    x, y = P.voc_segmentation(x, y)
                ev = segment.Evaluator(21)
                with torch.no_grad():
                    ev.add_logits(y, head(x), align_corners=ac)
                got.append((x, y, ev.counts))
            torch.cuda.synchronize()
            out[kind + "_img_s"] = round((len(items) - batch) / (time.perf_counter() - t0), 1)
            seen.append(got)
        for r, j, b in zip(*seen):                        # every batch: inputs, labels and counts equal across kinds
            for k in range(3):
                assert torch.equal(r[k], j[k]) and torch.equal(r[k], b[k])
        png.check()
        jpeg.check()
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,32,256")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--loop-batches", type=int, default=12)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    items = _labels(256, 7)
    want = [np.array(Image.open(io.BytesIO(d))) for d in items]
    res["label_bytes_mean"] = round(float(np.mean([len(d) for d in items])), 1)
    res["pillow_labels_per_s_one_core"] = round(_pillow_rate(items), 1)
    for n in [int(v) for v in a.batches.split(",")]:
        outs = png.decode(items[:n])
        for w, o in zip(want, outs):
            assert torch.equal(o.cpu(), torch.from_numpy(w))
        png.check()
        res["device_us_batch_%d" % n] = _kernel_us(items[:n], outs, a.reps)
        png.check()
    jp = [JC.pil(JC.picture(h, w, i), quality=90) for i, (h, w) in enumerate(VOC * 7)][:32]
    labs, arrs = items[:32], want[:32]
    x, y = P.voc_segmentation(jp, arrs)
    xb, yb = P.voc_segmentation(jp, labs)
    assert torch.equal(x, xb) and torch.equal(y, yb)
    res["voc_segmentation_ms_batch_32"] = {"labels_as_arrays": _call_ms(jp, arrs, (x, y), a.reps),
                                           "labels_as_png_bytes": _call_ms(jp, labs, (x, y), a.reps)}
    png.check()
    jpeg.check()
    n = 16 * a.loop_batches
    jl = BP._jpegs(VOC, n, 11)
    loop_items = [(j, PC.pil_p(PC.voc_label(*l.shape, 500 + i))) for i, (j, l) in enumerate(jl)]
    res["seg_loop_deeplab"] = _seg_loop(loop_items, 16, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
