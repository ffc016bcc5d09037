"""dfq_b200.detect's VOC average precision on the CPU: the oracle of tests/ssd_map_oracle.py against main_ssd.py's
compute_average_precision_per_class (the fixture tests/golden/ref_ssd_map.npz, and live where the reference checkout is
present), every rule of DESIGN.md section 3.11 decided by the fixture, ground_truth's packing, and the Evaluator wrapper
through the oracle-backed twins of tests/fakelib_detect_map.py: its checks, every refusal, batching, the KeyError-class
rule and the host's last sums."""
import os
import sys

import numpy as np
import pytest
import torch

import fakelib_detect_map
import map_scenes as MS
import ssd_map_oracle as O
from dfq_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _oracle(broken=None, text=False):
    z, C, gts, dets = MS.fixture()
    return [O.average_precision(dets, gts, C, float(t), bool(u), text=text, broken=broken)[0] for t, u in z["configs"]]


def test_oracle_equals_the_fixture():
    z = MS.fixture()[0]
    for text in (False, True):
        for k, aps in enumerate(_oracle(text=text)):
            assert _same(aps, z["aps_%d" % k]), (k, text)
    nan = [np.isnan(z["aps_%d" % k]) for k in range(4)]
    assert nan[0][1] and nan[0][3] and not nan[1][3]           # a best detection on a difficult box: NaN under 2007 only
    assert all(n[7] for n in nan)                               # class 8: no ground truth (KeyError in the reference)


@pytest.mark.parametrize("rule", sorted(O.BROKEN))
def test_the_fixture_decides_every_rule(rule):
    z = MS.fixture()[0]
    got = _oracle(broken=rule)
    assert not all(_same(a, z["aps_%d" % k]) for k, a in enumerate(got)), O.BROKEN[rule]


def test_live_against_the_reference():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import refenv
    if not refenv.available():
        pytest.skip("no reference checkout")
    refenv.install()
    saved, cwd = sys.argv, os.getcwd()
    sys.argv = ["main_ssd.py"]
    try:
        os.chdir(refenv.REF_ROOT)
        import main_ssd
    finally:
        sys.argv = saved
        os.chdir(cwd)
    import tempfile
    gts, dets = MS.scene(40, 7, seed=4, difficult=0.3)
    for n in range(40):                                         # the reference's order among ties is arbitrary
        dets[n] = (dets[n][0], dets[n][1], dets[n][2] + torch.arange(dets[n][2].numel()) * 1e-6 + n * 1e-4)

    class Dataset:
        ids = ["%06d" % n for n in range(40)]

        def __len__(self):
            return 40

        def get_annotation(self, i):
            return self.ids[i], gts[i]
    stat, boxes, diffs = main_ssd.group_annotation_by_class(Dataset())
    with tempfile.TemporaryDirectory() as tmp:
        for c in range(1, 7):
            with open(os.path.join(tmp, "%d.txt" % c), "w") as f:
                for n, (b, l, p) in enumerate(dets):
                    for i in np.nonzero(l.numpy() == c)[0]:
                        row = torch.cat([p[i:i + 1], b[i] + 1.0]).numpy()
                        print(Dataset.ids[n] + " " + " ".join(str(v) for v in row), file=f)
        for thr, use_2007 in ((0.5, True), (0.55, False)):
            with np.errstate(all="ignore"):
                want = [main_ssd.compute_average_precision_per_class(stat[c], boxes[c], diffs[c],
                                                                     os.path.join(tmp, "%d.txt" % c), thr, use_2007)
                        for c in range(1, 7)]
            got = O.average_precision(dets, gts, 7, thr, use_2007)[0]
            assert _same(got, want)
            assert _same(O.mean_average_precision(got), sum(want) / len(want))


def test_ground_truth_packing(monkeypatch):
    fakelib_detect_map.install(monkeypatch)
    from dfq_b200 import detect
    anns = [(np.array([[1, 2, 3, 4], [5, 6, 7, 8]], np.float32), np.array([3, 1]), np.array([0, 2], np.uint8)),
            (np.array([], np.float32), np.array([], np.int64), np.array([], np.uint8)),
            (torch.tensor([[9., 9., 10., 10.]]), torch.tensor([2], dtype=torch.int32), torch.tensor([True]))]
    gt = detect.ground_truth(anns, "cpu")
    assert gt.boxes.dtype == torch.float32 and gt.boxes.tolist() == [[1, 2, 3, 4], [5, 6, 7, 8], [9, 9, 10, 10]]
    assert gt.labels.dtype == torch.int64 and gt.labels.tolist() == [3, 1, 2]
    assert gt.difficult.dtype == torch.uint8 and gt.difficult.tolist() == [0, 1, 1]
    assert gt.offsets.dtype == torch.int64 and gt.offsets.tolist() == [0, 2, 2, 3]
    assert gt.boxes.data_ptr() % 16 == 0
    empty = detect.ground_truth([anns[1]], "cpu")
    assert empty.boxes.shape == (0, 4) and empty.offsets.tolist() == [0, 0]
    for bad, msg in [([], "at least one image"), ([(np.zeros((1, 4)), np.ones(1), np.zeros(1))], "float32"),
                     ([(np.zeros((1, 4), np.float32), np.ones(2), np.zeros(1))], "labels of shape"),
                     ([(np.zeros((1, 3), np.float32), np.ones(1), np.zeros(1))], r"\[k, 4\]"),
                     ([(np.zeros((1, 4), np.float32), np.ones(1) * 0.5, np.zeros(1))], "integers"),
                     ([(np.zeros((1, 4), np.float32),)], "triple")]:
        with pytest.raises(_lib.DfqError, match=msg):
            detect.ground_truth(bad, "cpu")


def _evaluator(monkeypatch, gts, dets, C, thr=0.5, use_2007=True, batches=1):
    from dfq_b200 import detect
    ev = detect.Evaluator(C, thr, use_2007)
    bounds = np.linspace(0, len(gts), batches + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        ev.add_batch(MS.detections(dets[a:b], "cpu"), detect.ground_truth(gts[a:b], "cpu"))
    return ev


@pytest.mark.parametrize("k", range(4))
def test_wrapper_gives_the_fixture_aps(monkeypatch, k):
    fakelib_detect_map.install(monkeypatch)
    z, C, gts, dets = MS.fixture()
    thr, use_2007 = z["configs"][k]
    ev = _evaluator(monkeypatch, gts, dets, C, float(thr), bool(use_2007), batches=3)
    assert _same(ev.average_precision(), z["aps_%d" % k])
    with pytest.raises(_lib.DfqError, match="class 8 has no non-difficult ground truth"):
        ev.mean_average_precision()


@pytest.mark.parametrize("use_2007", [True, False])
def test_wrapper_batches_growth_reset_and_mean(monkeypatch, use_2007):
    fakelib_detect_map.install(monkeypatch)
    from dfq_b200 import detect
    gts, dets = MS.scene(30, 6, seed=8, ties=True, clutter=5000)
    want, flags = O.average_precision(dets, gts, 6, 0.5, use_2007)
    ev = _evaluator(monkeypatch, gts, dets, 6, 0.5, use_2007, batches=5)   # grows past the first 65,536 rows
    assert ev._keys.shape[0] > 1 << 16
    assert _same(ev.average_precision(), want)
    assert np.array_equal(ev.match_flags.numpy(), flags)
    assert ev.mean_average_precision() == O.mean_average_precision(want)
    ev.reset()
    assert np.isnan(ev.average_precision()).all() and ev.match_flags.numel() == 0
    ev.add_batch(MS.detections(dets, "cpu"), detect.ground_truth(gts, "cpu"))
    assert _same(ev.average_precision(), want)


def test_host_sums_follow_the_reference(monkeypatch):
    """The 2007 sum is sequential in Python floats and the area sum numpy's pairwise .sum() of the terms in order; a class
    without detections is a Python float under 2007, as the reference's loop leaves it, so sum(aps) takes the same path."""
    fakelib_detect_map.install(monkeypatch)
    gts, dets = MS.scene(12, 4, seed=6, clutter=200)
    gts.append((np.array([[0, 0, 10, 10]], np.float32), np.array([4]), np.array([0], np.uint8)))
    dets = [(b, l.masked_fill(l == 4, 3), p) for b, l, p in dets] + [(torch.zeros(0, 4), torch.zeros(0, dtype=torch.int64),
                                                                     torch.zeros(0))]
    for use_2007 in (True, False):
        ev = _evaluator(monkeypatch, gts, dets, 5, 0.5, use_2007)
        aps, _ = ev._aps()
        want, _ = O.average_precision(dets, gts, 5, 0.5, use_2007)
        assert [type(a) for a in aps] == [type(w) for w in want]
        assert _same(aps, want) and aps[3] == 0.0
        assert ev.mean_average_precision() == sum(want) / len(want)


def test_wrapper_refusals(monkeypatch):
    fake = fakelib_detect_map.install(monkeypatch)
    from dfq_b200 import detect
    for bad in (1, 4097, True, 2.0):
        with pytest.raises(_lib.DfqError, match="num_classes"):
            detect.Evaluator(bad)
    with pytest.raises(_lib.DfqError, match="iou_threshold"):
        detect.Evaluator(21, "0.5")
    with pytest.raises(_lib.DfqError, match="use_2007_metric"):
        detect.Evaluator(21, 0.5, 1)
    gts, dets = MS.scene(3, 5, seed=2, empty=0.0)
    det, gt = MS.detections(dets, "cpu"), detect.ground_truth(gts, "cpu")
    ev = detect.Evaluator(5)
    D = det.labels.numel()
    cases = [
        (dict(det=(det.boxes, det.labels, det.probs, det.offsets)), "gt must be a detect.GroundTruth"),
        (dict(det_boxes=det.boxes.double()), "det.boxes must be torch.float32"),
        (dict(det_boxes=det.boxes[:, :3]), r"det.boxes must have shape"),
        (dict(det_labels=det.labels.int()), "det.labels must be torch.int64"),
        (dict(det_probs=det.probs[:-1]), "det.boxes must have shape"),
        (dict(det_offsets=det.offsets[:-1]), "gt.offsets must have shape"),
        (dict(gt_difficult=gt.difficult.bool()), "gt.difficult must be torch.uint8"),
        (dict(gt_labels=gt.labels[:-1]), "gt.boxes must have shape"),
        (dict(det_boxes=torch.zeros(4 * D + 1)[1:].view(D, 4)), "16-byte aligned"),
    ]
    for change, msg in cases:
        d = dict(det_boxes=det.boxes, det_labels=det.labels, det_probs=det.probs, det_offsets=det.offsets,
                 gt_boxes=gt.boxes, gt_labels=gt.labels, gt_difficult=gt.difficult, gt_offsets=gt.offsets)
        if "det" in change:
            a, b = change["det"], None
        else:
            d.update(change)
            a = detect.Detections(d["det_boxes"], d["det_labels"], d["det_probs"], d["det_offsets"])
            b = detect.GroundTruth(d["gt_boxes"], d["gt_labels"], d["gt_difficult"], d["gt_offsets"])
        with pytest.raises(_lib.DfqError, match=msg):
            ev.add_batch(detect.Detections(*a) if isinstance(a, tuple) else a, b)
    assert "dfq_map_match" not in fake.calls              # every refusal before any launch
    ev._count = 2 ** 31 - 1                               # the detection limit, without adding two billion rows
    with pytest.raises(_lib.DfqError, match="above the limit"):
        ev.add_batch(det, gt)


@pytest.mark.parametrize("case,msg", [("det_label", "detection label"), ("gt_label", "ground-truth label"),
                                      ("det_offsets", "detection offsets"), ("gt_offsets", "ground-truth offsets")])
def test_device_flagged_errors(monkeypatch, case, msg):
    fakelib_detect_map.install(monkeypatch)
    from dfq_b200 import detect
    gts, dets = MS.scene(4, 5, seed=3, empty=0.0)
    det, gt = MS.detections(dets, "cpu"), detect.ground_truth(gts, "cpu")
    {"det_label": lambda: det.labels.__setitem__(0, 5), "gt_label": lambda: gt.labels.__setitem__(0, -1),
     "det_offsets": lambda: det.offsets.__setitem__(1, -1), "gt_offsets": lambda: gt.offsets.__setitem__(-1, 0)}[case]()
    ev = detect.Evaluator(5)
    ev.add_batch(det, gt)
    with pytest.raises(_lib.DfqError, match=msg):
        ev.average_precision()


def test_library_refusals(monkeypatch):
    fake = fakelib_detect_map.install(monkeypatch)
    z = torch.zeros(16, dtype=torch.int64)
    p = z.data_ptr()
    assert fake.dfq_map_match(None, None, None, p, 0, None, None, None, p, 0, 1, 4097, 0.5, None, None, p, p, None) == -2
    assert fake.dfq_map_match(None, None, None, p, 0, None, None, None, p, 0, 1, 1, 0.5, None, None, p, p, None) == -1
    assert fake.dfq_map_match(None, None, None, p, 1, None, None, None, p, 0, 1, 5, 0.5, None, None, p, p, None) == -1
    assert fake.dfq_map_curve(None, None, 0, 5, p, 1, p, 43, p, None) == -1
    assert fake.dfq_map_curve(p, p, 2 ** 31, 5, p, 0, p, 44, p, None) == -2
    assert fake.dfq_map_curve(None, None, 0, 5, p, 2, p, 44, p, None) == -1
    assert [r[1] for r in fake.refusals] == [-2, -1, -1, -1, -2, -1]
