"""Sharded evaluation on the CPU: dist.shard's split, and the all_reduce of classify, segment and detect evaluators over 2
gloo ranks, each fed its shard, equal to one evaluator fed every batch in dataset order - uneven and empty shards,
detections of equal score on both sides of the shard boundary, a bad label flagged on one rank only, and a union over
the detection limit.  The arithmetic runs in the oracle-backed twins (tests/fakelib_classify.py, fakelib_segment.py,
fakelib_detect_map.py); the -m gpu suite runs the kernels (tests/test_gpu_dist_eval.py)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NC, NS, ND = 5, 5, 6          # classes of the three evaluators
BATCH = 3
CASES = {"uneven": (14, 9, 11), "empty": (1, 1, 1)}     # dataset sizes (classify, segment, detect) per case


def _shard_check(n, world):
    from dfq_b200 import dist as ddist
    got = []
    for rank in range(world):
        ddist._world_rank = lambda group=None, r=rank: (world, r)
        got.append(ddist.shard(n))
    sizes = [len(r) for r in got]
    assert [i for r in got for i in r] == list(range(n)), (n, world)
    assert all(r.step == 1 for r in got)
    assert sizes == sorted(sizes, reverse=True) and sizes[0] - sizes[-1] <= 1, (n, world, sizes)
    assert sum(s == sizes[0] for s in sizes) == (world if n % world == 0 else n % world)


def test_shard_covers_the_dataset_once_in_order(monkeypatch):
    from dfq_b200 import dist as ddist
    assert ddist.shard(7) == range(7) and ddist.shard(0) == range(0)        # no process group
    real = ddist._world_rank
    try:
        for world in range(1, 10):
            for n in range(0, 1001):
                _shard_check(n, world)
    finally:
        ddist._world_rank = real
    for bad in (-1, 2.0, True, "3"):
        with pytest.raises(ValueError, match="non-negative int"):
            ddist.shard(bad)


# ---- the data: seeded, the same in every process -------------------------------------------------------------------------
def _data(case, bad_rank1=False):
    import map_scenes as MS
    n_cls, n_seg, n_det = CASES[case]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n_cls, NC, generator=g)
    x[::2, 1] = x[::2, 0]                                             # ties
    x[3::5, 2] = float("nan")
    y = torch.randint(-1, NC + 1, (n_cls,), generator=g)
    y[::3] = torch.max(x, 1)[1][::3]
    sx = torch.randn(n_seg, NS, 4, 4, generator=g)
    sy = torch.randint(0, NS + 2, (n_seg, 7, 7), generator=g).to(torch.uint8)
    gts, dets = MS.scene(n_det, ND, seed=8, ties=True)
    if bad_rank1:
        b, l, d = gts[-1]
        gts[-1] = (np.concatenate([b, b[:1] * 0 + 1]), np.concatenate([l, [ND]]), np.concatenate([d, [0]]))
    return x, y, sx, sy, gts, dets


def _batches(r):
    return [list(r[i:i + BATCH]) for i in range(0, len(r), BATCH)]


def _evaluate(data, ranges):
    """The three evaluators fed the items of ranges (classify, segment, detect) in batches of BATCH."""
    import map_scenes as MS
    from dfq_b200 import classify, detect, segment
    x, y, sx, sy, gts, dets = data
    ce, se, de = classify.Evaluator(NC), segment.Evaluator(NS), detect.Evaluator(ND)
    for b in _batches(ranges[0]):
        ce.add_logits(x[b].contiguous(), y[b].contiguous())
    for b in _batches(ranges[1]):
        se.add_logits(sy[b].contiguous(), sx[b].contiguous(), align_corners=True)
    for b in _batches(ranges[2]):
        de.add_batch(MS.detections([dets[i] for i in b], "cpu"), detect.ground_truth([gts[i] for i in b], "cpu"))
    return ce, se, de


def _results(ce, se, de):
    out = {"cls": np.array([int(ce.num_correct), ce.num_total]), "seg": se.confusion_matrix,
           "flags": de.match_flags.numpy().copy(), "keys": de._keys[:de._count].numpy().copy() if de._count else
           np.zeros(0, np.int64), "gt_count": de._gt_count.numpy().copy() if de._gt_count is not None else np.zeros(ND)}
    try:
        out["aps"] = de.average_precision()
    except Exception as e:                          # noqa: BLE001 - the message is compared
        out["aps_error"] = np.array(str(e))
    return out


class _Fakes:
    """One stand-in for the library holding the three evaluators' twins: the classification and segmentation entries go
    to their twins, everything else to the detection twin."""
    ROUTES = {"dfq_cls_count": 0, "dfq_seg_argmax": 1}

    def __init__(self):
        import fakelib_classify, fakelib_detect_map, fakelib_segment
        self.parts = [fakelib_classify.FakeClassifyLib(), fakelib_segment.FakeSegmentLib(),
                      fakelib_detect_map.FakeDetectMapLib()]

    def __getattr__(self, name):
        return getattr(self.parts[self.ROUTES.get(name, 2)], name)


def _install(mpatch):
    import fakelib
    from dfq_b200 import _lib, dist as ddist
    fakelib.install(mpatch)
    fakes = _Fakes()
    mpatch.setattr(_lib, "load", lambda build_if_missing=True: fakes)
    mpatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    mpatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    mpatch.setattr(ddist, "_idle_device", lambda: torch.device("cpu"))


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist

    class _MP:
        def setattr(self, obj, name, value):
            setattr(obj, name, value)
    _install(_MP())
    from dfq_b200 import detect, dist as ddist
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        for case in CASES:
            for bad in (False, True):
                data = _data(case, bad)
                evs = _evaluate(data, [ddist.shard(n) for n in CASES[case]])
                red = [ev.all_reduce() for ev in evs]
                again = [ev.all_reduce() for ev in evs]                 # the evaluators are left as they were
                out = _results(*red)
                for k, v in _results(*again).items():
                    out["again_" + k] = v
                for k, v in _results(*evs).items():
                    out["own_" + k] = v
                if case == "uneven" and not bad:
                    limit = detect.MAX_MAP_DETECTIONS
                    detect.MAX_MAP_DETECTIONS = red[2]._count - 1
                    try:
                        evs[2].all_reduce()
                    except Exception as e:              # noqa: BLE001 - the message is compared
                        out["limit_error"] = np.array(str(e))
                    finally:
                        detect.MAX_MAP_DETECTIONS = limit
                np.savez(os.path.join(out_dir, "%s%d_rank%d.npz" % (case, bad, rank)), **out)
    finally:
        dist.destroy_process_group()


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


@pytest.mark.timeout(900)
def test_two_rank_reductions_equal_one_process(monkeypatch, tmp_path):
    import map_scenes as MS
    from dfq_b200 import dist as ddist
    port = 29500 + (os.getpid() % 2000) + 83
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    _install(monkeypatch)
    for case, sizes in CASES.items():
        for bad in (False, True):
            data = _data(case, bad)
            alone = _results(*_evaluate(data, [range(n) for n in sizes]))
            assert ("aps_error" in alone) == bad, (case, bad)
            own = []
            for rank in (0, 1):
                got = np.load(tmp_path / ("%s%d_rank%d.npz" % (case, bad, rank)))
                for k, v in alone.items():
                    assert k in got.files and _same(got[k], v), (case, bad, rank, k)
                    assert _same(got["again_" + k], v), (case, bad, rank, "again", k)
                own.append(got)
            # each rank's own evaluator still holds its shard only
            assert own[0]["own_cls"][1] + own[1]["own_cls"][1] == alone["cls"][1]
            assert np.array_equal(own[0]["own_seg"] + own[1]["own_seg"], alone["seg"])
            assert own[0]["own_flags"].size + own[1]["own_flags"].size == alone["flags"].size
            if case == "empty":
                assert own[1]["own_cls"][1] == 0 and own[1]["own_flags"].size == 0 and own[1]["own_seg"].sum() == 0
            if bad:
                assert "ground-truth label" in str(alone["aps_error"])
            if bad and case == "uneven":                # flagged on rank 1 only, raised by the union on both
                assert "own_aps_error" not in own[0].files and "own_aps_error" in own[1].files
            if case == "uneven" and not bad:
                for g in own:
                    assert "MAX_MAP_DETECTIONS" in str(g["limit_error"])
                # detections of equal score and class on both sides of the shard boundary
                _, _, _, _, gts, dets = data
                cut = (sizes[2] + 1) // 2
                left = {(int(c), float(p)) for _, l, s in dets[:cut] for c, p in zip(l, s)}
                right = {(int(c), float(p)) for _, l, s in dets[cut:] for c, p in zip(l, s)}
                assert left & right, "the scene must tie scores across the boundary"
                assert alone["cls"][1] == sizes[0] and alone["seg"].sum() > 0 and alone["flags"].size > 0
