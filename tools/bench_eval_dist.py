"""Sharded evaluation throughput: the three mains' evaluation loops split over ranks with dfq_b200.dist.shard and merged
with the evaluators' all_reduce; prints one JSON line.

    python tools/bench_eval_dist.py [--images 512] [--batch 32] [--worlds 1,2,4,8]

Per main, seeded synthetic JPEGs (tools/bench_preprocess.py's: ImageNet-like sizes for classification, VOC-like sizes
with VOC-like labels for segmentation), and for SSD seeded ground truth (tests/map_scenes.py's scenes, as
tools/bench_detect_map.py makes them).  Each rank runs the whole loop on its shard: the file's bytes, preprocess.* (device
decode and resize), the chained affine int8 network (tests/affine_observed_state.py: MobileNetV2 at 224, DeepLab-v3+ at
513, SSD-Lite at 300, TF32 off, calibrated once and loaded by every rank from int8.save's file), detect.postprocess for
SSD, then the evaluator; after the loop, all_reduce.  Reported per world size: images/s of each rank over its shard (host
clock from a barrier to the end of its loop, ending in a device synchronise), the aggregate rate (all images over the
slowest rank's time), the all_reduce time, and whether the reduced metric equals the world-1 metric bit for bit (a run
where it does not fails).

One process per GPU with NCCL for every world size up to the number of GPUs.  On a machine with fewer GPUs than a world
size, that size runs with its ranks sharing the GPUs under gloo (the collectives stage through the host) and is reported
as "shared_gpu"; such rates say what several processes feeding one card reach, not how sharding scales over cards, and
multi-GPU scaling is then reported as "not measured".  The card's name and power limit are read in the same run.  Needs
a CUDA device; writes only to a temporary directory.
"""
import argparse
import contextlib
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TESTS = os.path.join(ROOT, "tests")
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, TESTS)

MAINS = ("cls", "seg", "ssd")


def _inputs(main, n):
    """(JPEG bytes, labels) of n seeded images: ImageNet class indices, VOC label planes or SSD ground truth."""
    from bench_preprocess import IMAGENET, VOC, _jpegs
    items = _jpegs(IMAGENET if main == "cls" else VOC, n, seed=len(main))
    data = [j for j, _ in items]
    if main == "cls":
        return data, torch.from_numpy(np.random.default_rng(1).integers(0, 1000, n))
    if main == "seg":
        return data, [lab for _, lab in items]
    import map_scenes as MS
    return data, MS.scene(n, 21, seed=3)[0]


def _build(tmp):
    """The chained affine int8 networks, saved under tmp."""
    import affine_observed_state
    from dfq_b200 import int8
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    for main, net, size, flags in (("cls", "mobilenet_v2", 224, dict(residual=True)),
                                   ("seg", "deeplab", 513, dict(residual=True, concat=True, fold_pads=True)),
                                   ("ssd", "ssd", 300, dict(residual=True, concat=True, fold_pads=True, heads=True))):
        with contextlib.redirect_stdout(sys.stderr), \
                affine_observed_state.evaluation_state(net, size=size, batch=4) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            int8.save(int8.chain_affine(model, **flags), os.path.join(tmp, main + ".pt"))


def _loop(main, tmp, data, labels, rng, batch):
    """The main's evaluation loop over the images of rng; returns (evaluator, seconds from the barrier to the end)."""
    import torch.distributed as dist
    from dfq_b200 import classify, detect, int8, jpeg, preprocess as P, segment
    from test_detect_host import fixture
    gm = int8.load(os.path.join(tmp, main + ".pt"))
    if main == "seg":
        gm, ac = segment.split_upsample(gm)
    _, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    ev = {"cls": lambda: classify.Evaluator(1000), "seg": lambda: segment.Evaluator(21),
          "ssd": lambda: detect.Evaluator(21)}[main]()

    def step(b, ev):
        with torch.no_grad():
            if main == "cls":
                ev.add_logits(gm(P.imagenet([data[i] for i in b])), labels[b])
            elif main == "seg":
                x, y = P.voc_segmentation([data[i] for i in b], [labels[i] for i in b])
                ev.add_logits(y, gm(x), align_corners=ac)
            else:
                x, sizes = P.ssd([data[i] for i in b], mean=np.array([127, 127, 127]), std=128.0)
                det = detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
                ev.add_batch(det, detect.ground_truth([labels[i] for i in b], "cuda"))
    batches = [list(rng[i:i + batch]) for i in range(0, len(rng), batch)]
    warm = {"cls": lambda: classify.Evaluator(1000), "seg": lambda: segment.Evaluator(21),
            "ssd": lambda: detect.Evaluator(21)}[main]()
    step(list(range(min(batch, len(data)))), warm)                 # warm-up on an evaluator that is thrown away
    torch.cuda.synchronize()
    if dist.is_initialized():
        dist.barrier()
    t0 = time.perf_counter()
    for b in batches:
        step(b, ev)
    jpeg.check()
    torch.cuda.synchronize()
    return ev, time.perf_counter() - t0


def _metric(main, ev):
    if main == "cls":
        return {"accuracy": float(ev.accuracy()), "counts": [int(ev.num_correct), ev.num_total]}
    if main == "seg":
        return {"miou": float(ev.Mean_Intersection_over_Union()), "matrix": ev.confusion_matrix.tolist()}
    return {"aps": [None if np.isnan(a) else float(a) for a in ev.average_precision()]}


def _worker(rank, world, port, backend, tmp, images, batch):
    import torch.distributed as dist
    from dfq_b200 import dist as ddist
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dist.init_process_group(backend, init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        out = {}
        for main in MAINS:
            data, labels = _inputs(main, images)
            rng = ddist.shard(images)
            ev, sec = _loop(main, tmp, data, labels, rng, batch)
            dist.barrier()
            t0 = time.perf_counter()
            red = ev.all_reduce()
            torch.cuda.synchronize()
            ar = time.perf_counter() - t0
            out[main] = {"images": len(rng), "seconds": sec, "all_reduce_ms": 1e3 * ar, "metric": _metric(main, red)}
        with open(os.path.join(tmp, "rank%d_world%d.json" % (rank, world)), "w") as f:
            json.dump(out, f)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--worlds", default="1,2,4,8")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_dist.py needs a CUDA device")
    from bench_int8 import card
    gpus = torch.cuda.device_count()
    res = {"card": card(), "gpus": gpus, "images": a.images, "batch": a.batch, "worlds": {}}
    with tempfile.TemporaryDirectory() as tmp:
        _build(tmp)
        torch.cuda.empty_cache()
        base = None
        for w in [int(v) for v in a.worlds.split(",")]:
            backend = "nccl" if w <= gpus else "gloo"
            port = 29500 + (os.getpid() % 2000) + w
            mp.spawn(_worker, args=(w, port, backend, tmp, a.images, a.batch), nprocs=w, join=True)
            ranks = []
            for r in range(w):
                with open(os.path.join(tmp, "rank%d_world%d.json" % (r, w))) as f:
                    ranks.append(json.load(f))
            row = {"backend": backend, "placement": "one_gpu_per_rank" if w <= gpus else "shared_gpu"}
            for main in MAINS:
                metrics = [rk[main]["metric"] for rk in ranks]
                if base is None or main not in base:
                    base = base or {}
                    base[main] = metrics[0]
                equal = all(m == base[main] for m in metrics)
                if not equal:
                    raise SystemExit("world %d, %s: the reduced metric differs from the world-1 metric" % (w, main))
                slowest = max(rk[main]["seconds"] for rk in ranks)
                row[main] = {"per_rank_img_s": [round(rk[main]["images"] / rk[main]["seconds"], 1) for rk in ranks],
                             "aggregate_img_s": round(a.images / slowest, 1),
                             "all_reduce_ms": round(max(rk[main]["all_reduce_ms"] for rk in ranks), 3),
                             "metric_equals_world_1": equal}
            res["worlds"][str(w)] = row
            print(w, json.dumps(row), file=sys.stderr)
        res["metric_world_1"] = {m: {k: v for k, v in base[m].items() if k != "matrix"} for m in MAINS}
    if gpus < 2:
        res["multi_gpu_scaling"] = "not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
