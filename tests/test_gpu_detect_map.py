"""dfq_b200.detect.Evaluator on the H100: the fixture's APs (the reference's own compute_average_precision_per_class),
seeded batches and the per-detection verdicts bit for bit against the stable oracle of tests/ssd_map_oracle.py, batching
and reset, a run of several million detections, no host synchronisation, the device-flagged errors and the limits, and
end to end behind the chained SSD-Lite of tests/ssd_lite_like.py."""
import numpy as np
import pytest
import torch

import map_scenes as MS
import ssd_map_oracle as O
from dfq_b200 import _lib

pytestmark = pytest.mark.gpu

def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _evaluate(gts, dets, C, thr=0.5, use_2007=True, batches=1):
    from dfq_b200 import detect
    ev = detect.Evaluator(C, thr, use_2007)
    bounds = np.linspace(0, len(gts), batches + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        if a < b:
            ev.add_batch(MS.detections(dets[a:b], "cuda"), detect.ground_truth(gts[a:b], "cuda"))
    return ev


@pytest.mark.parametrize("k", range(4))
def test_fixture_inputs_give_the_fixture_aps(k):
    z, C, gts, dets = MS.fixture()
    thr, use_2007 = z["configs"][k]
    ev = _evaluate(gts, dets, C, float(thr), bool(use_2007))
    aps = ev.average_precision()
    assert _same(aps, z["aps_%d" % k]), (aps, z["aps_%d" % k])
    _, want = O.average_precision(dets, gts, C, float(thr), bool(use_2007))
    assert np.array_equal(ev.match_flags.cpu().numpy(), want)


@pytest.mark.parametrize("N,C,ties", [(1, 2, False), (1, 21, True), (256, 2, True), (256, 21, False), (256, 21, True),
                                      (64, 91, False), (48, 601, True)])
@pytest.mark.parametrize("thr,use_2007", [(0.5, True), (0.55, False)])
def test_seeded_batches_match_the_oracle(N, C, ties, thr, use_2007):
    gts, dets = MS.scene(N, C, seed=N * 1000 + C, ties=ties)
    ev = _evaluate(gts, dets, C, thr, use_2007)
    want, flags = O.average_precision(dets, gts, C, thr, use_2007)
    assert _same(ev.average_precision(), want)
    assert np.array_equal(ev.match_flags.cpu().numpy(), flags)
    if not any(np.isnan(want)):
        assert ev.mean_average_precision() == O.mean_average_precision(want)


@pytest.mark.parametrize("use_2007", [True, False])
def test_batches_and_reset(use_2007):
    gts, dets = MS.scene(300, 21, seed=5, ties=True)
    one = _evaluate(gts, dets, 21, 0.5, use_2007)
    many = _evaluate(gts, dets, 21, 0.5, use_2007, batches=7)
    assert _same(one.average_precision(), many.average_precision())
    assert torch.equal(one.match_flags, many.match_flags)
    want = one.average_precision()
    from dfq_b200 import detect
    many.reset()
    assert np.isnan(many.average_precision()).all()          # nothing added: no class has ground truth
    many.add_batch(MS.detections(dets, "cuda"), detect.ground_truth(gts, "cuda"))
    assert _same(many.average_precision(), want)


def test_several_million_detections():
    """4,952 images with about 600 detections each, in batches of 256: equal to one batch, and the curve equal to numpy's
    on the device's own verdicts (the per-detection oracle is checked on a sample of images)."""
    from dfq_b200 import detect
    gts, dets = MS.scene(4952, 21, seed=9, max_gt=30, copies=12, clutter=1000, ties=True)
    D = sum(l.numel() for _, l, _ in dets)
    assert D > 2_500_000
    for use_2007 in (True, False):
        ev = _evaluate(gts, dets, 21, 0.5, use_2007, batches=20)
        aps = ev.average_precision()
        flags = ev.match_flags.cpu().numpy()
        labels = torch.cat([l for _, l, _ in dets]).numpy()
        probs = torch.cat([p for _, _, p in dets]).numpy().astype(np.float64)
        num_true = np.bincount(np.concatenate([l[d == 0] for _, l, d in gts]), minlength=21)
        want = []
        for c in range(1, 21):
            idx = np.nonzero(labels == c)[0]
            idx = idx[np.argsort(-probs[idx], kind="stable")]
            tp, fp = np.cumsum(flags[idx] == 1).astype(np.float64), np.cumsum(flags[idx] == 2).astype(np.float64)
            with np.errstate(invalid="ignore"):
                precision = tp / (tp + fp)
            recall = tp / num_true[c]
            want.append(O.voc2007_ap(precision, recall) if use_2007 else O.area_ap(precision, recall))
        assert _same(aps, want)
    sample = list(range(0, 4952, 619))
    part = detect.Evaluator(21)
    part.add_batch(MS.detections([dets[i] for i in sample], "cuda"), detect.ground_truth([gts[i] for i in sample], "cuda"))
    w, f = O.average_precision([dets[i] for i in sample], [gts[i] for i in sample], 21)
    assert _same(part.average_precision(), w) and np.array_equal(part.match_flags.cpu().numpy(), f)


def test_no_host_synchronisation():
    from dfq_b200 import detect
    gts, dets = MS.scene(256, 21, seed=3)
    ev = detect.Evaluator(21)
    det, gt = MS.detections(dets, "cuda"), detect.ground_truth(gts, "cuda")
    ev.add_batch(det, gt)                                 # first call: allocation and library load
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            ev.add_batch(det, gt)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    want, _ = O.average_precision(dets * 4, gts * 4, 21)
    assert _same(ev.average_precision(), want)


@pytest.mark.parametrize("case,msg", [
    ("det_label_0", "detection label"), ("det_label_C", "detection label"), ("gt_label_C", "ground-truth label"),
    ("gt_label_neg", "ground-truth label"), ("det_offsets", "detection offsets"), ("gt_offsets", "ground-truth offsets")])
def test_device_flagged_errors_raise_at_average_precision(case, msg):
    from dfq_b200 import detect
    gts, dets = MS.scene(8, 5, seed=1, empty=0.0)
    det, gt = MS.detections(dets, "cuda"), detect.ground_truth(gts, "cuda")
    if case == "det_label_0":
        det.labels[0] = 0
    elif case == "det_label_C":
        det.labels[-1] = 5
    elif case == "gt_label_C":
        gt.labels[0] = 5
    elif case == "gt_label_neg":
        gt.labels[-1] = -1
    elif case == "det_offsets":
        det.offsets[3] = det.offsets[4] + 1
    else:
        gt.offsets[-1] = gt.offsets[-1] - 1
    ev = detect.Evaluator(5)
    ev.add_batch(det, gt)                                 # accepted: the check needs device data
    with pytest.raises(_lib.DfqError, match=msg):
        ev.average_precision()
    ev.reset()
    ev.add_batch(MS.detections(dets, "cuda"), detect.ground_truth(gts, "cuda"))
    want, _ = O.average_precision(dets, gts, 5)
    assert _same(ev.average_precision(), want)


def test_limits_and_refusals():
    import ctypes as C
    from dfq_b200 import detect
    lib = _lib.load()
    gts, dets = MS.scene(4, 4096, seed=2)
    ev = _evaluate(gts, dets, 4096)                       # the class limit itself
    want, _ = O.average_precision(dets, gts, 4096)
    assert _same(ev.average_precision(), want)
    with pytest.raises(_lib.DfqError, match="num_classes"):
        detect.Evaluator(4097)
    cnt = torch.zeros(4097, dtype=torch.int64, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    off = torch.zeros(2, dtype=torch.int64, device="cuda")
    st = _lib.stream_ptr()
    p = lambda t: C.c_void_p(t.data_ptr())               # noqa: E731
    rc = lib.dfq_map_match(None, None, None, p(off), 0, None, None, None, p(off), 0, 1, 4097, 0.5, None, None, p(cnt),
                           p(err), st)
    assert rc != 0 and "above the limit 4096" in lib.dfq_last_error().decode()
    rc = lib.dfq_map_match(None, None, None, p(off), 1, None, None, None, p(off), 0, 1, 21, 0.5, None, None, p(cnt),
                           p(err), st)
    assert rc != 0 and "non-NULL" in lib.dfq_last_error().decode()
    out = torch.zeros(10, dtype=torch.float64, device="cuda")
    rc = lib.dfq_map_curve(None, None, 0, 21, p(cnt), 1, p(out), 10, p(cnt), st)
    assert rc != 0 and "at least 220" in lib.dfq_last_error().decode()
    rc = lib.dfq_map_curve(p(cnt), p(cnt), 1 << 31, 21, p(cnt), 1, p(out), 1 << 20, p(cnt), st)
    assert rc != 0 and "above the limit" in lib.dfq_last_error().decode()
    torch.cuda.synchronize()
    assert int(err.item()) == 0 and int(cnt.sum()) == 0   # refused calls wrote nothing


# ---- end to end on SSD-Lite -------------------------------------------------------------------------------------------------
def _end_to_end(m, x):
    """postprocess + Evaluator behind the model, against the oracle on det.per_image(), with annotations made from the
    picks (jittered) and random boxes."""
    from dfq_b200 import detect
    import test_detect_host as TH
    z, t, cv, sv = TH.fixture()
    pri = t["priors"].cuda()
    sizes = torch.tensor([[300, 300], [640, 480]], device="cuda")[:x.shape[0]]
    with torch.no_grad():
        det = detect.postprocess(*m(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
    per = det.per_image()
    g = np.random.default_rng(int(det.boxes.shape[0]))
    gts = []
    for b, l, p in per:
        b, l = b.reshape(-1, 4).numpy(), l.reshape(-1).long().numpy()
        pick = g.random(len(l)) < 0.05
        boxes = b[pick] + g.normal(0, 3, (int(pick.sum()), 4)).astype(np.float32)
        extra = g.uniform(0, 250, (3, 2))
        boxes = np.concatenate([boxes, np.concatenate([extra, extra + 40], 1)]).astype(np.float32)
        labels = np.concatenate([l[pick], g.integers(1, 21, 3)]).astype(np.int64)
        gts.append((boxes, labels, (g.random(len(labels)) < 0.15).astype(np.uint8)))
    for use_2007 in (True, False):
        ev = detect.Evaluator(21, 0.5, use_2007)
        ev.add_batch(det, detect.ground_truth(gts, "cuda"))
        want, flags = O.average_precision(per, gts, 21, 0.5, use_2007)
        assert _same(ev.average_precision(), want)
        assert np.array_equal(ev.match_flags.cpu().numpy(), flags)
        assert (flags == 1).any()


def test_ssd_lite_ncnn_chain_and_loaded(tmp_path):
    from dfq_b200 import int8
    import test_gpu_int8_layout as GL
    model, x = GL._net("ssd", 2, 300, is_test=True)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
    _end_to_end(gm, x)
    int8.save(gm, tmp_path / "ssd.pt")
    _end_to_end(int8.load(tmp_path / "ssd.pt"), x)


def test_ssd_lite_affine_chain_and_loaded(tmp_path):
    import affine_observed_state
    from dfq_b200 import int8
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True, heads=True)
            g = torch.Generator(device="cuda").manual_seed(2)
            x = torch.randn(2, 3, 300, 300, device="cuda", generator=g).clamp_(-2.5, 2.5)
            _end_to_end(gm, x)
            int8.save(gm, tmp_path / "ssd_affine.pt")
            _end_to_end(int8.load(tmp_path / "ssd_affine.pt"), x)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
