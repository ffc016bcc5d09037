"""-m gpu, one GPU, several processes: sharded evaluation reduced with all_reduce equals one process, bit for bit.

Worker processes share cuda:0 with gloo (NCCL refuses several ranks on one device; the reductions then stage through the
host, dfq_b200/dist.py::_all_gather_flat) and run the real kernels on their dist.shard of the data:
  * 4 ranks, uneven and empty shards: classify counts, the segment confusion matrix and its four metrics, and the detect
    average precisions and match flags (NaN included) on seeded scenes whose probabilities are int8-like multiples of
    1/256, so equal scores are everywhere and cross the shard boundaries;
  * 3 ranks end to end: JPEG bytes through preprocess, the chained affine MobileNetV2, DeepLab-v3+ and SSD-Lite (saved by
    the parent with int8.save, loaded by every rank), postprocess and the evaluators, against one process over the same
    batches."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
NC, NS, ND = 100, 21, 21
SIZES = {"uneven": (1001, 7, 27), "empty": (3, 2, 3)}      # dataset sizes (classify, segment, detect); 4 ranks


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def _data(case):
    import map_scenes as MS
    n_cls, n_seg, n_det = SIZES[case]
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(n_cls, NC, device="cuda", generator=g)
    x[::4, 7] = x[::4].max(1)[0]
    y = torch.randint(-1, NC + 1, (n_cls,), device="cuda", generator=g)
    y[::2] = torch.max(x, 1)[1][::2]
    sx = torch.randn(n_seg, NS, 17, 17, device="cuda", generator=g)
    sy = torch.randint(0, 23, (n_seg, 65, 65), device="cuda", generator=g).to(torch.uint8)
    gts, dets = MS.scene(n_det, ND, seed=21, max_gt=8, copies=4, clutter=20, difficult=0.2)
    for n, (b, l, d) in enumerate(gts):                            # class ND - 1 has no ground truth: NaN
        gts[n] = (b, np.where(l == ND - 1, 1, l), d)
    for n, (b, l, p) in enumerate(dets):                           # int8-like probabilities: many equal scores
        dets[n] = (b, l, torch.round(p * 256) / 256)
    return x, y, sx, sy, gts, dets


def _evaluate(data, ranges, batch=4):
    import map_scenes as MS
    from dfq_b200 import classify, detect, segment
    x, y, sx, sy, gts, dets = data
    ce, se, de = classify.Evaluator(NC), segment.Evaluator(NS), detect.Evaluator(ND)
    for r, ev in zip(ranges, (ce, se, de)):
        for i in range(r.start, r.stop, batch):
            b = list(range(i, min(i + batch, r.stop)))
            if ev is ce:
                ce.add_logits(x[b].contiguous(), y[b].cpu())
            elif ev is se:
                se.add_logits(sy[b].contiguous(), sx[b].contiguous(), align_corners=True)
            else:
                de.add_batch(MS.detections([dets[k] for k in b], "cuda"), detect.ground_truth([gts[k] for k in b], "cuda"))
    return ce, se, de


def _results(ce, se, de):
    return {"correct": np.array(ce.num_correct), "total": np.array(ce.num_total), "acc": np.array(ce.accuracy()),
            "matrix": se.confusion_matrix, "pa": np.array(se.Pixel_Accuracy()), "pac": np.array(se.Pixel_Accuracy_Class()),
            "miou": np.array(se.Mean_Intersection_over_Union()),
            "fwiou": np.array(se.Frequency_Weighted_Intersection_over_Union()),
            "aps": de.average_precision(), "flags": de.match_flags.cpu().numpy()}


def _worker(rank, world, port, out_dir, fn):
    sys.path.insert(0, ROOT); sys.path.insert(0, TESTS)
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **globals()[fn](out_dir))
    finally:
        dist.destroy_process_group()


def _reductions(out_dir):
    from dfq_b200 import dist as ddist
    out = {}
    for case, sizes in SIZES.items():
        evs = _evaluate(_data(case), [ddist.shard(n) for n in sizes])
        for k, v in _results(*[ev.all_reduce() for ev in evs]).items():
            out[case + "_" + k] = v
        out[case + "_own"] = np.array([evs[0].num_total, int(evs[1].confusion_matrix.sum() > 0), evs[2]._count])
    return out


@pytest.mark.timeout(900)
def test_four_ranks_reduce_to_one_process(tmp_path):
    sys.path.insert(0, TESTS)
    world = 4
    port = 29500 + (os.getpid() % 2000) + 89
    mp.spawn(_worker, args=(world, port, str(tmp_path), "_reductions"), nprocs=world, join=True)
    for case, sizes in SIZES.items():
        alone = _results(*_evaluate(_data(case), [range(n) for n in sizes]))
        assert np.isnan(alone["aps"]).any() and not np.isnan(alone["aps"]).all()
        assert int(alone["correct"]) > 0 and alone["matrix"].sum() > 0 and alone["flags"].size > 0
        owns = []
        for r in range(world):
            d = np.load(tmp_path / ("rank%d.npz" % r))
            for k, v in alone.items():
                assert _same(d[case + "_" + k], v), (case, r, k)
            owns.append(d[case + "_own"])
        if case == "empty":                                        # rank 3 added nothing, rank 2 no segmentation
            assert owns[3].tolist() == [0, 0, 0] and owns[2][1] == 0
        else:
            assert len({int(o[0]) for o in owns}) == 2             # uneven: 251, 250, 250, 250


# ---- end to end from JPEG bytes --------------------------------------------------------------------------------------------
N_E2E = 7


def _e2e_inputs():
    import map_scenes as MS
    from test_gpu_jpeg import _batch
    items, _, labels = _batch(N_E2E, 31)
    gts, _ = MS.scene(N_E2E, 21, seed=12)
    return items, labels, gts


def _e2e(out_dir, batches=None):
    """The three mains' loops over `batches` (lists of image indices; this rank's dist.shard in one batch when None), the
    models loaded from out_dir, then all_reduce when run under a process group."""
    import torch.distributed as dist
    from dfq_b200 import classify, detect, dist as ddist, int8, preprocess as P, segment
    from test_detect_host import fixture
    items, labels, gts = _e2e_inputs()
    cls_labels = torch.from_numpy(np.load(os.path.join(out_dir, "cls_labels.npy")))
    if batches is None:
        batches = [list(ddist.shard(N_E2E))]
    batches = [b for b in batches if b]
    mbv2 = int8.load(os.path.join(out_dir, "mbv2.pt"))
    head, ac = segment.split_upsample(int8.load(os.path.join(out_dir, "deeplab.pt")))
    ssd = int8.load(os.path.join(out_dir, "ssd.pt"))
    _, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    ce, se, de = classify.Evaluator(1000), segment.Evaluator(21), detect.Evaluator(21)
    with torch.no_grad():
        for b in batches:
            ce.add_logits(mbv2(P.imagenet([items[i] for i in b])), cls_labels[b])
            x, y = P.voc_segmentation([items[i] for i in b], [labels[i] for i in b], crop_size=129)
            se.add_logits(y, head(x), align_corners=ac)
            x, sizes = P.ssd([items[i] for i in b], mean=np.array([127, 127, 127]), std=128.0)
            det = detect.postprocess(*ssd(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
            de.add_batch(det, detect.ground_truth([gts[i] for i in b], "cuda"))
    from dfq_b200 import jpeg
    jpeg.check()
    if dist.is_initialized():
        ce, se, de = ce.all_reduce(), se.all_reduce(), de.all_reduce()
    return {"correct": np.array(ce.num_correct), "total": np.array(ce.num_total), "matrix": se.confusion_matrix,
            "miou": np.array(se.Mean_Intersection_over_Union()), "aps": de.average_precision(),
            "flags": de.match_flags.cpu().numpy()}


@pytest.mark.timeout(1800)
def test_chained_networks_over_three_ranks_equal_one_process(tmp_path):
    sys.path.insert(0, TESTS)
    import affine_observed_state
    from dfq_b200 import classify, int8, preprocess as P
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("mobilenet_v2", size=224) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            int8.save(int8.chain_affine(model, residual=True), tmp_path / "mbv2.pt")
        with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            int8.save(int8.chain_affine(model, residual=True, concat=True, fold_pads=True), tmp_path / "deeplab.pt")
        with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            int8.save(int8.chain_affine(model, residual=True, concat=True, fold_pads=True, heads=True),
                      tmp_path / "ssd.pt")
        # labels: half the images labelled with the network's own prediction, so that the count is not zero
        items, _, _ = _e2e_inputs()
        with torch.no_grad():
            pred = classify.predict(int8.load(tmp_path / "mbv2.pt")(P.imagenet(items))).cpu()
        lab = torch.randint(0, 1000, (N_E2E,), generator=torch.Generator().manual_seed(2))
        lab[::2] = pred[::2]
        np.save(tmp_path / "cls_labels.npy", lab.numpy())
        world = 3
        shards = [[0, 1, 2], [3, 4], [5, 6]]                       # dist.shard(7) on ranks 0, 1 and 2: one batch each
        alone = _e2e(str(tmp_path), shards)
        port = 29500 + (os.getpid() % 2000) + 97
        mp.spawn(_worker, args=(world, port, str(tmp_path), "_e2e"), nprocs=world, join=True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    assert int(alone["correct"]) > 0 and alone["matrix"].sum() > 0 and alone["flags"].size > 0
    for r in range(world):
        d = np.load(tmp_path / ("rank%d.npz" % r))
        for k, v in alone.items():
            assert _same(d[k], v), (r, k)
