"""Evaluation preprocessing throughput on the H100: the reference's CPU transforms in DataLoader workers against workers
that only decode, followed by dfq_b200.preprocess, and workers that only read the file, followed by the device decode of
dfq_b200.jpeg and dfq_b200.preprocess; prints one JSON line.

    python tools/bench_preprocess.py [--batch 64] [--batches 12] [--workers 1,2,4,8]

Inputs are seeded synthetic JPEGs encoded here (quality 90): VOC-like sizes (500 x 375, 375 x 500, 500 x 333, 333 x 500,
486 x 500) for segmentation and SSD, ImageNet-like sizes (500 x 375 to 1280 x 960) for classification.  Per main and
arm, at each worker count: images/s of the loop that takes each batch to the device (host clock, ending in a device
synchronise).  Arms:
  reference   workers decode with PIL and run the reference's transform (torchvision Compose, FixScaleCrop + Normalize,
              cv2.resize + SubtractMeans + / std), the batch is copied to the device
  gpu         workers decode only; dfq_b200.preprocess forms the batch on the device
  bytes       workers return the file's bytes; dfq_b200.preprocess decodes them on the device and forms the batch
All arms' outputs are asserted equal on every timed batch.  Without a network behind the loop the rate is the ceiling the
input pipeline puts on an evaluation.  With --network, each main's loop is also timed at its own worker count with the
chained affine int8 network (tests/affine_observed_state.py: MobileNetV2 at 224, DeepLab-v3+ at 513, SSD-Lite at 300,
TF32 off) and the matching evaluation step behind it: the logits, segment.Evaluator.add_logits, detect.postprocess.
Per main also: the whole preprocessing call per batch (CUDA events around calls on batches decoded beforehand, so the
gather and the copy are in it) and the kernel alone (torch.profiler's device time of k_pre_resample, in a run of its own:
events cannot bracket a kernel that the call enqueues behind its copy).  The card's name and power limit are read in the
same run.  For the bytes arm also: the corpus's compressed / decoded byte ratio, the call time at batch 64 and 256, the
device time of each decode phase (k_jpeg_huff, k_jpeg_idct, k_jpeg_color) and of k_pre_resample, and Pillow's decode
rate on one core of this host for scale.  Needs a CUDA device; writes nothing.
"""
import argparse
import io
import json
import os
import sys
import time

import cv2
import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_int8 import card  # noqa: E402
from dfq_b200 import preprocess as P  # noqa: E402

VOC = [(375, 500), (500, 375), (333, 500), (500, 333), (500, 486)]
IMAGENET = [(375, 500), (500, 375), (480, 640), (960, 1280), (333, 500)]
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _jpegs(sizes, n, seed):
    g = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        yy, xx = np.mgrid[0:h, 0:w]
        a = 127.5 + 100 * np.sin(xx[..., None] * (0.02 + 0.01 * np.arange(3)) + yy[..., None] * 0.015)
        a = np.clip(a + g.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)
        lab = (np.arange(w)[None, :] // 40 % 21 + np.zeros((h, 1), np.int64)).astype(np.uint8)
        lab[:4] = 255
        b = io.BytesIO()
        Image.fromarray(a).save(b, "JPEG", quality=90)
        out.append((b.getvalue(), lab))
    return out


class _Set(torch.utils.data.Dataset):
    def __init__(self, items, main, mode):
        self.items, self.main, self.mode = items, main, mode

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        jpg, lab = self.items[i]
        if self.mode == "bytes":
            return jpg, lab
        img = Image.open(io.BytesIO(jpg)).convert("RGB")
        if self.mode == "gpu":                          # tensors: they leave the worker through shared memory
            return torch.from_numpy(np.asarray(img)), torch.from_numpy(lab)
        if self.main == "cls":
            return _cls()(img), lab
        if self.main == "seg":
            return _seg(img, lab), None                 # (image, label) pair: _collate_ref stacks both
        return _ssd(np.asarray(img)), lab


def _cls():
    from torchvision import transforms
    return transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224), transforms.ToTensor(),
                               transforms.Normalize(MEAN, STD)])


def _seg(img, lab):
    """FixScaleCrop(513) + Normalize + ToTensor, as custom_transforms states them."""
    w, h = img.size
    oh, ow = (513, int(1.0 * w * 513 / h)) if w > h else (int(1.0 * h * 513 / w), 513)
    x1, y1 = int(round((ow - 513) / 2.)), int(round((oh - 513) / 2.))
    im = img.resize((ow, oh), Image.BILINEAR).crop((x1, y1, x1 + 513, y1 + 513))
    lb = Image.fromarray(lab).resize((ow, oh), Image.NEAREST).crop((x1, y1, x1 + 513, y1 + 513))
    x = np.array(im).astype(np.float32)
    x /= 255.0
    x -= MEAN
    x /= STD
    return torch.from_numpy(x.transpose(2, 0, 1).copy()), torch.from_numpy(np.array(lb).astype(np.float32))


def _ssd(a):
    x = cv2.resize(a, (300, 300)).astype(np.float32) - np.array([127, 127, 127], np.float32)
    return torch.from_numpy(x / 128.0).permute(2, 0, 1)


def _collate_ref(batch):
    if isinstance(batch[0][0], tuple):
        return torch.stack([b[0][0] for b in batch]), torch.stack([b[0][1] for b in batch])
    return torch.stack([b[0] for b in batch]), None


def _collate_list(batch):
    return [b[0] for b in batch], [b[1] for b in batch]


def _gpu(main, imgs, labs):
    if main == "cls":
        return P.imagenet(imgs), None
    if main == "seg":
        return P.voc_segmentation(imgs, labs)
    return P.ssd(imgs, mean=(127, 127, 127))[0], None


def _loop(main, items, batch, workers, mode, consume=None):
    transform = mode == "reference"
    dl = torch.utils.data.DataLoader(_Set(items, main, mode), batch_size=batch, num_workers=workers,
                                     collate_fn=_collate_ref if transform else _collate_list,
                                     persistent_workers=False, prefetch_factor=2)
    outs = []
    t0 = None
    for i, (x, y) in enumerate(dl):
        if i == 1:                                        # the first batch carries the workers' start-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        if transform:
            x = x.cuda(non_blocking=True)
            y = y.cuda(non_blocking=True) if y is not None else None
        else:
            x, y = _gpu(main, x, y)
        if consume is None:
            outs.append((x, y))
        else:
            outs.append(consume(x, y))
    torch.cuda.synchronize()
    return (len(items) - batch) / (time.perf_counter() - t0), outs


def _with_network(main, items, batch, workers):
    """images/s of both arms at `workers` with the chained int8 network and the evaluation step behind the loop."""
    import contextlib
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_observed_state
    from dfq_b200 import detect, int8, segment
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    net, size = {"cls": ("mobilenet_v2", 224), "seg": ("deeplab", 513), "ssd": ("ssd", 300)}[main]
    with contextlib.redirect_stdout(sys.stderr), \
            affine_observed_state.evaluation_state(net, size=size, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        if main == "cls":
            gm = int8.chain_affine(model, residual=True)

            def consume(x, y):
                with torch.no_grad():
                    return gm(x)
        elif main == "seg":
            head, ac = segment.split_upsample(int8.chain_affine(model, residual=True, concat=True, fold_pads=True))

            def consume(x, y):
                ev = segment.Evaluator(21)
                with torch.no_grad():
                    ev.add_logits(y, head(x), align_corners=ac)
                return ev.counts
        else:
            from test_detect_host import fixture
            _, t, cv, sv = fixture()
            pri = t["priors"].cuda()
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True, heads=True)

            def consume(x, y):
                with torch.no_grad():
                    return detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv).boxes
        out = {}
        rates = []
        for mode in ("reference", "gpu", "bytes"):
            rate, outs = _loop(main, items, batch, workers, mode, consume)
            rates.append(outs)
            out[mode + "_img_s"] = round(rate, 1)
        for o0, o1, o2 in zip(*rates):
            assert torch.equal(o0, o1) and torch.equal(o0, o2), main
        out["workers"] = workers
        return out


def _bytes_arm(main, items, labs, batch):
    """The device decode: byte ratio, call time at batch 64 and 256 (and `batch`), per-phase kernel times, Pillow's rate."""
    from torch.profiler import ProfilerActivity, profile
    from dfq_b200 import jpeg
    dec = [np.asarray(Image.open(io.BytesIO(j)).convert("RGB")) for j, _ in items]
    out = {"compressed_over_decoded": round(sum(len(j) for j, _ in items) / sum(d.nbytes for d in dec), 4)}
    t0 = time.perf_counter()
    for j, _ in items[:64]:
        np.asarray(Image.open(io.BytesIO(j)).convert("RGB"))
    out["pillow_decode_img_s_one_core"] = round(64 / (time.perf_counter() - t0), 1)
    for n in sorted({64, 256, batch}):
        js = [items[i % len(items)][0] for i in range(n)]
        ls = [items[i % len(items)][1] for i in range(n)]
        ds = [dec[i % len(items)] for i in range(n)]
        want = _gpu(main, ds, ls)
        got = _gpu(main, js, ls)
        assert torch.equal(want[0], got[0]) and (want[1] is None or torch.equal(want[1], got[1])), (main, n)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(10):
            _gpu(main, js, ls)
        ev[1].record()
        torch.cuda.synchronize()
        row = {"call_ms": round(ev[0].elapsed_time(ev[1]) / 10, 3)}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                _gpu(main, js, ls)
            torch.cuda.synchronize()
        for k in ("k_jpeg_huff", "k_jpeg_idct", "k_jpeg_color", "k_pre_resample"):
            t = [e.device_time for e in prof.events() if k in e.name]
            row[k + "_ms"] = round(sum(t) / max(len(t), 1) / 1e3, 3)
        out["batch_%d" % n] = row
    jpeg.check()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--workers", default="1,2,4,8")
    ap.add_argument("--network", action="store_true")
    a = ap.parse_args()
    workers = [int(w) for w in a.workers.split(",")]
    res = {"card": card(), "batch": a.batch, "batches": a.batches, "mains": {}}
    for main, sizes, own in (("cls", IMAGENET, 4), ("seg", VOC, 2), ("ssd", VOC, 1)):
        items = _jpegs(sizes, a.batch * a.batches, seed=len(main))
        r = {"main_workers": own}
        for w in sorted(set(workers + [own])):
            ref_rate, ref_out = _loop(main, items, a.batch, w, "reference")
            gpu_rate, gpu_out = _loop(main, items, a.batch, w, "gpu")
            byte_rate, byte_out = _loop(main, items, a.batch, w, "bytes")
            for (x0, y0), (x1, y1), (x2, y2) in zip(ref_out, gpu_out, byte_out):
                assert torch.equal(x0, x1) and (y0 is None or torch.equal(y0, y1)), (main, w)
                assert torch.equal(x0, x2) and (y0 is None or torch.equal(y0, y2)), (main, w)
            r["workers_%d" % w] = {"reference_img_s": round(ref_rate, 1), "gpu_img_s": round(gpu_rate, 1),
                                   "bytes_img_s": round(byte_rate, 1)}
        dec = [np.asarray(Image.open(io.BytesIO(j)).convert("RGB")) for j, _ in items[:a.batch]]
        labs = [l for _, l in items[:a.batch]]
        for _ in range(3):
            _gpu(main, dec, labs)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(20):
            _gpu(main, dec, labs)
        ev[1].record()
        torch.cuda.synchronize()
        r["call_ms_per_batch"] = round(ev[0].elapsed_time(ev[1]) / 20, 3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                _gpu(main, dec, labs)
            torch.cuda.synchronize()
        k = [e.device_time for e in prof.events() if "k_pre_resample" in e.name]
        r["kernel_ms_per_batch"] = round(sum(k) / max(len(k), 1) / 1e3, 3)
        r["bytes"] = _bytes_arm(main, items, labs, a.batch)
        if a.network:
            r["with_network"] = _with_network(main, items, a.batch, own)
        res["mains"][main] = r
        print(main, json.dumps(r), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
