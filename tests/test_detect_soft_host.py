"""dfq_b200.detect's soft NMS on the CPU: the oracle of tests/ssd_soft_nms_oracle.py against the reference's
Predictor(nms_method="soft").predict (the fixture tests/golden/ref_ssd_soft_nms.npz) and against box_utils.soft_nms live
where the reference checkout is present, on the edge cases of tests/soft_nms_cases.py; and postprocess(nms_method="soft")
through the oracle-backed twins of tests/fakelib_detect_soft.py - the output layout, every refusal, and the hard path
left as it was."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import fakelib_detect_soft
import soft_nms_cases
import ssd_soft_nms_oracle as SO
from dfq_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_ssd_soft_nms.npz")
REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")
HAVE_REF = os.path.isfile(os.path.join(REF, "utils", "detection", "box_utils.py"))


def fixture():
    z = np.load(GOLD)
    t = {k: torch.from_numpy(z[k]) for k in ("scores", "locations", "priors", "image_sizes")}
    cv, sv = (float(v) for v in z["variances"])
    return z, t, cv, sv


def _triples(z, k):
    offs = z["offsets_%d" % k]
    return [(z["boxes_%d" % k][a:b], z["labels_%d" % k][a:b], z["probs_%d" % k][a:b]) for a, b in zip(offs[:-1], offs[1:])]


def _eq(g, w):
    if g.dtype != w.dtype or g.shape != w.shape:
        return False
    return bool(((g == w) | (g.isnan() & w.isnan())).all()) if g.is_floating_point() else torch.equal(g, w)


def _box_utils():
    sys.path.insert(0, REF)
    try:
        from utils.detection import box_utils
    finally:
        sys.path.remove(REF)
    return box_utils


# ---- the oracle against the reference ------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(3))
def test_oracle_matches_the_reference_fixture(k):
    z, t, cv, sv = fixture()
    top_k, sigma = int(z["top_ks"][k]), float(z["sigma"])
    got = SO.predict(t["scores"], t["locations"], t["priors"], cv, sv, t["image_sizes"], prob_threshold=0.01,
                     top_k=top_k, nms_method="soft", sigma=sigma)
    for n, (g, (b, l, p)) in enumerate(zip(got, _triples(z, k))):
        want = (torch.from_numpy(b), torch.from_numpy(l), torch.from_numpy(p))
        assert all(_eq(a, w) for a, w in zip(g, want)), (k, n)
    assert 7 not in got[1][1].tolist() and 7 in got[0][1].tolist()               # a class without candidates
    if top_k > 0:
        assert all(np.bincount(l.numpy()).max() <= top_k for _, l, _ in got)


def test_fixture_sigma_is_not_a_power_of_two():
    z = np.load(GOLD)
    assert math.frexp(float(z["sigma"]))[0] != 0.5 and sorted(z["top_ks"].tolist()) == [-1, 1, 5]


def _soft_ref(box_utils, boxes, scores, thr, sigma, top_k):
    rows = box_utils.soft_nms(torch.cat([boxes, scores.unsqueeze(1)], 1), thr, sigma, top_k)
    return rows.reshape(-1, 5)


@pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present")
@pytest.mark.filterwarnings("ignore::UserWarning")
@pytest.mark.parametrize("name", [s[0] for s in soft_nms_cases.scenes()])
@pytest.mark.parametrize("top_k", [1, 5, -1])
def test_oracle_matches_box_utils_soft_nms_live(name, top_k):
    box_utils = _box_utils()
    _, s, b = next(sc for sc in soft_nms_cases.scenes() if sc[0] == name)
    thr, sigma = soft_nms_cases.THR, soft_nms_cases.SIGMA
    segments = 0
    for c in range(1, s.shape[2]):
        keep = s[0, :, c] > thr
        if not keep.any():
            continue
        segments += 1
        got = SO.soft_nms(b[0, keep], s[0, keep, c], thr, sigma, top_k)
        want = _soft_ref(box_utils, b[0, keep].clone(), s[0, keep, c].clone(), thr, sigma, top_k)
        assert _eq(got, want), (name, c)
    assert segments


@pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present")
@pytest.mark.filterwarnings("ignore::UserWarning")
@pytest.mark.parametrize("seed", [21, 22])
def test_oracle_matches_box_utils_soft_nms_on_seeded_outputs(seed):
    box_utils = _box_utils()
    z, t, cv, sv = fixture()
    g = torch.Generator().manual_seed(seed)
    P = t["priors"].shape[0]
    scores = torch.softmax(torch.randn(1, P, 4, generator=g) * 3 + torch.tensor([5., 0, 0, 0]), dim=2)
    boxes = SO.decode(torch.randn(1, P, 4, generator=g), t["priors"], cv, sv)
    for sigma in (0.5, 0.3, 1.7):
        for c in range(1, 4):
            keep = scores[0, :, c] > 0.01
            got = SO.soft_nms(boxes[0, keep], scores[0, keep, c], 0.01, sigma, -1)
            want = _soft_ref(box_utils, boxes[0, keep].clone(), scores[0, keep, c].clone(), 0.01, sigma, -1)
            assert _eq(got, want), (sigma, c)


def test_edge_scenes_reach_their_cases():
    """The claims of soft_nms_cases hold: ties, a single candidate, a score one ulp above the threshold decaying out,
    non-finite boxes turning scores NaN, and a crowded class losing many rows per step."""
    sc = {name: (s, b) for name, s, b in soft_nms_cases.scenes()}
    thr, sigma = soft_nms_cases.THR, soft_nms_cases.SIGMA
    s, b = sc["single_and_threshold"]
    assert int((s[0, :, 1] > thr).sum()) == 1 and int((s[0, :, 3] > thr).sum()) == 2
    rows = SO.soft_nms(b[0, s[0, :, 3] > thr], s[0, s[0, :, 3] > thr, 3], thr, sigma, -1)
    assert rows.shape[0] == 1                                 # the identical box decayed below the threshold
    s, b = sc["ties"]
    keep = s[0, :, 1] > thr
    rows = SO.soft_nms(b[0, keep], s[0, keep, 1], thr, sigma, 1)
    assert torch.equal(rows[0, :4], b[0, 0])                   # the first of the tied maxima
    s, b = sc["all_candidates_crowded"]
    assert bool((s[0, :, 1] > thr).all())
    rows = SO.soft_nms(b[0], s[0, :, 1], thr, sigma, -1)
    assert rows.shape[0] < s.shape[1] // 2
    s, b = sc["nonfinite_scores"]
    rows = SO.soft_nms(b[0, s[0, :, 1] > thr], s[0, s[0, :, 1] > thr, 1], thr, sigma, -1)
    assert math.isinf(rows[0, 4].item())


# ---- the host path through the twins ---------------------------------------------------------------------------------------
def _inputs(z, t):
    cv, sv = (float(v) for v in z["variances"])
    return t["scores"].clone(), t["locations"].clone(), t["priors"].clone(), cv, sv


@pytest.mark.parametrize("k", range(3))
def test_postprocess_soft_matches_the_oracle_through_the_twins(monkeypatch, k):
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    z, t, cv, sv = fixture()
    top_k, sigma = int(z["top_ks"][k]), float(z["sigma"])
    scores, locations, priors, cv, sv = _inputs(z, t)
    sizes = t["image_sizes"].clone()
    det = detect.postprocess(scores, (locations, priors, cv, sv), image_sizes=sizes, top_k=top_k, nms_method="soft",
                             sigma=sigma)
    assert fake.calls == ["dfq_ssd_decode", "dfq_ssd_soft_nms", "dfq_ssd_soft_compact"]
    want = SO.predict(scores, locations, priors, cv, sv, sizes, prob_threshold=0.01, top_k=top_k, nms_method="soft",
                      sigma=sigma)
    for n, (g, w) in enumerate(zip(det.per_image(), want)):
        assert all(_eq(a, b) for a, b in zip(g, w)), n
    assert det.offsets.tolist() == z["offsets_%d" % k].tolist()


def test_postprocess_soft_on_edge_scenes_through_the_twins(monkeypatch):
    from dfq_b200 import detect
    fakelib_detect_soft.install(monkeypatch)
    for name, s, b in soft_nms_cases.scenes():
        P = s.shape[1]
        # boxes enter through the decode: zero locations on priors that are the boxes in centre form give them back
        # only approximately, so these scenes go through the twin's entries with the boxes themselves
        lib = _lib.load()
        d, _ = detect._descriptor(torch.zeros(1, P, 4), torch.zeros(P, 4), 0.1, 0.2, s.shape[2], soft_nms_cases.THR)
        S = s.shape[2] - 1
        cand, cnt, off = torch.empty(S, dtype=torch.int32), torch.empty(S, dtype=torch.int32), \
            torch.empty(S + 1, dtype=torch.int64)
        assert lib.dfq_ssd_soft_nms(detect._ptr(s), detect._ptr(b), detect._ptr(cand), detect._ptr(cnt),
                                    detect._ptr(off), _lib.table_ptr(d), soft_nms_cases.SIGMA, None) == 0
        T = int(off[-1])
        ob, ol, op = torch.empty(max(T, 1), 4), torch.empty(max(T, 1), dtype=torch.int64), torch.empty(max(T, 1))
        assert lib.dfq_ssd_soft_compact(detect._ptr(s), detect._ptr(b), detect._ptr(cand), detect._ptr(off), None,
                                        detect._ptr(ob), detect._ptr(ol), detect._ptr(op), _lib.table_ptr(d),
                                        soft_nms_cases.SIGMA, None) == 0
        want = SO.predict_one(s[0], b[0], prob_threshold=soft_nms_cases.THR, nms_method="soft",
                              sigma=soft_nms_cases.SIGMA)
        if T == 0:
            assert want[0].numel() == 0, name
        else:
            assert _eq(ob[:T], want[0]) and torch.equal(ol[:T], want[1]) and _eq(op[:T], want[2]), name
        assert cand.tolist() == [int((s[0, :, c] > soft_nms_cases.THR).sum()) for c in range(1, s.shape[2])], name


def test_postprocess_soft_without_detections_and_without_sizes(monkeypatch):
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    z, t, cv, sv = fixture()
    scores, locations, priors, cv, sv = _inputs(z, t)
    det = detect.postprocess(scores, locations, priors, cv, sv, prob_threshold=1.0, nms_method="soft")
    assert det.boxes.shape == (0, 4) and det.offsets.tolist() == [0, 0, 0]
    assert fake.calls == ["dfq_ssd_decode", "dfq_ssd_soft_nms"]               # nothing to compact
    assert [tuple(x.numel() for x in tr) for tr in det.per_image()] == [(0, 0, 0)] * 2
    det = detect.postprocess(scores[:1], locations[:1], priors, cv, sv, top_k=1, nms_method="soft", sigma=2)
    want = SO.predict(scores[:1], locations[:1], priors, cv, sv, prob_threshold=0.01, top_k=1, nms_method="soft",
                      sigma=2.0)[0]
    assert all(_eq(a, b) for a, b in zip(det.per_image()[0], want))


@pytest.mark.parametrize("method", [None, "hard"])
def test_hard_path_unchanged(monkeypatch, method):
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    z, t, cv, sv = fixture()
    scores, locations, priors, cv, sv = _inputs(z, t)
    kw = {} if method is None else dict(nms_method=method)
    det = detect.postprocess(scores, locations, priors, cv, sv, sigma=float("nan"), **kw)   # sigma is not read
    assert fake.calls == ["dfq_ssd_decode", "dfq_ssd_nms", "dfq_ssd_compact"]
    want = SO.predict(scores, locations, priors, cv, sv, prob_threshold=0.01)
    for g, w in zip(det.per_image(), want):
        assert all(_eq(a, b) for a, b in zip(g, w))


# ---- refusals --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["Soft", "greedy", "", 1, True])
def test_refuses_an_unknown_nms_method(monkeypatch, method):
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    z, t, cv, sv = fixture()
    scores, locations, priors, cv, sv = _inputs(z, t)
    with pytest.raises(_lib.DfqError, match="nms_method must be None, 'hard' or 'soft'"):
        detect.postprocess(scores, locations, priors, cv, sv, nms_method=method)
    assert fake.calls == []


@pytest.mark.parametrize("sigma", [0, 0.0, -0.5, -0.0, float("nan"), float("inf"), -float("inf"), 1e39, 1e-50, "0.5",
                                   None, True, torch.tensor(0.5)])
def test_refuses_a_sigma_that_is_not_finite_and_positive(monkeypatch, sigma):
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    z, t, cv, sv = fixture()
    scores, locations, priors, cv, sv = _inputs(z, t)
    with pytest.raises(_lib.DfqError, match="sigma must be a finite positive number"):
        detect.postprocess(scores, locations, priors, cv, sv, nms_method="soft", sigma=sigma)
    assert fake.calls == []


def _entry_desc(priors, classes, **desc):
    from dfq_b200 import detect
    d, _ = detect._descriptor(torch.zeros(1, priors, 4), torch.zeros(priors, 4), 0.1, 0.2, classes, 0.01)
    for k, v in desc.items():
        d[0][k] = v
    return d


@pytest.mark.parametrize("what,reason", [
    ("null_desc", "descriptor is NULL"), ("N", "N and P must be positive"), ("P", "N and P must be positive"),
    ("prior_batch", "prior_batch must be 1 or N"), ("C", "C must be at least 2"),
    ("sigma0", "sigma must be a finite positive number"), ("sigma_nan", "sigma must be a finite positive number"),
    ("sigma_inf", "sigma must be a finite positive number"), ("null_scores", "NULL or misaligned pointer"),
    ("null_out", "NULL or misaligned pointer")])
def test_entry_refusals_of_the_twin(monkeypatch, what, reason):
    """The twins refuse what dfq_ssd_soft_nms / dfq_ssd_soft_compact refuse (tests/test_gpu_detect_soft.py checks the
    library's own refusals with the same cases)."""
    from dfq_b200 import detect
    fake = fakelib_detect_soft.install(monkeypatch)
    s, b = torch.rand(1, 8, 3), torch.rand(1, 8, 4)
    desc = dict(N=0) if what == "N" else dict(P=0) if what == "P" else dict(prior_batch=2) if what == "prior_batch" \
        else dict(C=1) if what == "C" else {}
    d = _entry_desc(8, 3, **desc)
    sigma = {"sigma0": 0.0, "sigma_nan": float("nan"), "sigma_inf": float("inf")}.get(what, 0.5)
    lib = _lib.load()
    dp = None if what == "null_desc" else _lib.table_ptr(d)
    cand, cnt, off = torch.zeros(2, dtype=torch.int32), torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.int64)
    sp = None if what == "null_scores" else detect._ptr(s)
    rc = lib.dfq_ssd_soft_nms(sp, detect._ptr(b), detect._ptr(cand), detect._ptr(cnt), detect._ptr(off), dp, sigma, None)
    if what != "null_out":
        assert rc == fakelib_detect_soft.E_ARG and fake.refusals[-1][2] == reason
    ob, ol, op = torch.zeros(4, 4), torch.zeros(4, dtype=torch.int64), torch.zeros(4)
    rc = lib.dfq_ssd_soft_compact(sp, detect._ptr(b), detect._ptr(cand), detect._ptr(off), None, detect._ptr(ob),
                                  None if what == "null_out" else detect._ptr(ol), detect._ptr(op), dp, sigma, None)
    assert rc == fakelib_detect_soft.E_ARG and fake.refusals[-1] == ("dfq_ssd_soft_compact", rc, reason)
