"""dfq_b200.detect on the CPU: the oracle of tests/ssd_postprocess_oracle.py against the reference's Predictor.predict
(the fixture tests/golden/ref_ssd_postprocess.npz, and live where the reference checkout is present), and the host wrapper
through the oracle-backed twins of tests/fakelib_detect.py - argument checks, every refusal, the output layout and the empty
cases."""
import os
import sys

import numpy as np
import pytest
import torch

import fakelib_detect
import ssd_postprocess_oracle as SO
from dfq_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_ssd_postprocess.npz")


def fixture():
    z = np.load(GOLD)
    t = {k: torch.from_numpy(z[k]) for k in ("scores", "locations", "priors", "image_sizes")}
    cv, sv = (float(v) for v in z["variances"])
    return z, t, cv, sv


def _triples(z, k):
    offs = z["offsets_%d" % k]
    return [(z["boxes_%d" % k][a:b], z["labels_%d" % k][a:b], z["probs_%d" % k][a:b]) for a, b in zip(offs[:-1], offs[1:])]


def _same(got, want):
    """One image's (boxes, labels, probs) triples equal, dtypes and shapes included; NaN equals NaN (a NaN box can be
    picked)."""
    def eq(g, w):
        if g.dtype != w.dtype or g.shape != w.shape:
            return False
        return bool(((g == w) | (g.isnan() & w.isnan())).all()) if g.is_floating_point() else torch.equal(g, w)
    return all(eq(g, w) for g, w in zip(got, want))


# ---- the oracle against the reference --------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(4))
def test_oracle_matches_the_reference_fixture(k):
    z, t, cv, sv = fixture()
    top_k, cand = (int(v) for v in z["configs"][k])
    got = SO.predict(t["scores"], t["locations"], t["priors"], cv, sv, t["image_sizes"], prob_threshold=0.01,
                     iou_threshold=float(z["iou_threshold"]), candidate_size=cand, top_k=top_k)
    for n, (g, (b, l, p)) in enumerate(zip(got, _triples(z, k))):
        if b.shape[0] == 0:
            assert _same(g, (torch.tensor([]),) * 3), n
        else:
            assert _same(g, (torch.from_numpy(b), torch.from_numpy(l), torch.from_numpy(p))), (k, n)
    assert [g[0].shape[0] for g in got][2] == 0                                  # an image without detections
    assert 5 not in got[0][1].tolist() and 5 in got[1][1].tolist()               # a class without candidates


REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "utils", "detection", "box_utils.py")),
                    reason="reference checkout not present")
@pytest.mark.parametrize("seed", [11, 12, 13])
def test_oracle_matches_box_utils_live(seed):
    sys.path.insert(0, REF)
    try:
        from utils.detection import box_utils
    finally:
        sys.path.remove(REF)
    z, t, cv, sv = fixture()
    g = torch.Generator().manual_seed(seed)
    P = t["priors"].shape[0]
    scores = torch.softmax(torch.randn(1, P, 6, generator=g) * 3 + torch.tensor([4., 0, 0, 0, 0, 0]), dim=2)
    locations = torch.randn(1, P, 4, generator=g)
    boxes = box_utils.center_form_to_corner_form(box_utils.convert_locations_to_boxes(locations, t["priors"], cv, sv))
    assert torch.equal(boxes, SO.decode(locations, t["priors"], cv, sv))
    for top_k, cand in ((-1, 200), (3, 50), (-1, 1)):
        for c in range(1, 6):
            s = scores[0, :, c]
            keep = s > 0.01
            assert torch.unique(s[keep]).numel() == int(keep.sum())
            bp = torch.cat([boxes[0, keep], s[keep, None]], 1)
            want = box_utils.hard_nms(bp, 0.45, top_k, cand)
            picks = SO.hard_nms(boxes[0, keep], s[keep], 0.45, top_k, cand)
            got = torch.cat([boxes[0, keep][picks], s[keep][picks, None]], 1)
            assert torch.equal(got, want), (seed, top_k, cand, c)


def test_oracle_stable_order_and_signed_zero():
    """Equal scores keep prior order, -0.0 ties +0.0, NaN is never a candidate and NaN IoUs drop the box."""
    boxes = torch.tensor([[0, 0, 1, 1], [5, 5, 6, 6], [0, 0, 1, 1], [9, 9, 10, 10]], dtype=torch.float32)
    scores = torch.tensor([0.5, 0.5, 0.5, 0.25])
    assert SO.hard_nms(boxes, scores, 0.45).tolist() == [0, 1, 3]
    z = torch.tensor([-0.0, 0.0, -0.0])
    assert SO.hard_nms(boxes[:3] + torch.arange(3.).view(3, 1) * 10, z, 0.45).tolist() == [0, 1, 2]
    nan_box = torch.tensor([[0, 0, 1, 1], [float("nan"), 0, 1, 1], [3, 3, 4, 4]], dtype=torch.float32)
    assert SO.hard_nms(nan_box, torch.tensor([0.9, 0.8, 0.7]), 0.45).tolist() == [0, 2]


# ---- the host wrapper through the twins -------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(4))
@pytest.mark.parametrize("tuple_form", [False, True])
def test_postprocess_through_the_twins_matches_the_oracle(monkeypatch, k, tuple_form):
    from dfq_b200 import detect
    fake = fakelib_detect.install(monkeypatch)
    z, t, cv, sv = fixture()
    top_k, cand = (int(v) for v in z["configs"][k])
    kw = dict(iou_threshold=0.45, candidate_size=cand, top_k=top_k)
    if tuple_form:
        det = detect.postprocess(t["scores"], (t["locations"], t["priors"], cv, sv), image_sizes=t["image_sizes"], **kw)
    else:
        det = detect.postprocess(t["scores"], t["locations"], t["priors"].unsqueeze(0), cv, sv, t["image_sizes"], **kw)
    assert fake.calls == ["dfq_ssd_decode", "dfq_ssd_nms", "dfq_ssd_compact"]
    T = int(z["offsets_%d" % k][-1])
    assert det.boxes.shape == (T, 4) and det.boxes.dtype == torch.float32
    assert det.labels.shape == (T,) and det.labels.dtype == torch.int64
    assert det.probs.shape == (T,) and det.probs.dtype == torch.float32
    assert det.offsets.dtype == torch.int64 and det.offsets.tolist() == z["offsets_%d" % k].tolist()
    want = SO.predict(t["scores"], t["locations"], t["priors"], cv, sv, t["image_sizes"], **kw)
    for n, (g, w) in enumerate(zip(det.per_image(), want)):
        assert _same(g, w), n


def test_postprocess_without_sizes_and_priors_per_image(monkeypatch):
    from dfq_b200 import detect
    fakelib_detect.install(monkeypatch)
    z, t, cv, sv = fixture()
    pri = t["priors"].unsqueeze(0).repeat(3, 1, 1).contiguous()
    pri[1] *= 0.5
    det = detect.postprocess(t["scores"], t["locations"], pri, cv, sv, top_k=2)
    want = SO.predict(t["scores"], t["locations"], pri, cv, sv, top_k=2)
    for g, w in zip(det.per_image(), want):
        assert _same(g, w)
    assert torch.equal(detect.decode_boxes(t["locations"], pri, cv, sv), SO.decode(t["locations"], pri, cv, sv))


def test_empty_batch_skips_compaction(monkeypatch):
    from dfq_b200 import detect
    fake = fakelib_detect.install(monkeypatch)
    z, t, cv, sv = fixture()
    det = detect.postprocess(t["scores"][2:], t["locations"][2:], t["priors"], cv, sv)
    assert fake.calls == ["dfq_ssd_decode", "dfq_ssd_nms"]
    assert det.boxes.shape == (0, 4) and det.labels.shape == (0,) and det.probs.shape == (0,)
    assert det.offsets.tolist() == [0, 0]
    (b, l, p), = det.per_image()
    assert _same((b, l, p), (torch.tensor([]),) * 3)


def _inputs(N=2, P=7, C=3):
    g = torch.Generator().manual_seed(0)
    return (torch.softmax(torch.randn(N, P, C, generator=g), 2), torch.randn(N, P, 4, generator=g),
            torch.rand(P, 4, generator=g) + 0.1)


def _refused(monkeypatch, match, *args, **kw):
    from dfq_b200 import detect
    fake = fakelib_detect.install(monkeypatch)
    with pytest.raises(_lib.DfqError, match=match):
        detect.postprocess(*args, **kw)
    return fake


@pytest.mark.parametrize("case,match", [
    ("cand0", "candidate_size"), ("cand_float", "candidate_size"), ("top_k", "top_k"), ("C1", "at least 2 classes"),
    ("scores_dtype", "scores must be float32"), ("loc_dtype", "locations must be float32"),
    ("pri_dtype", "priors must be float32"), ("scores_nc", "scores must be contiguous"),
    ("loc_nc", "locations must be contiguous"), ("scores_shape", "scores must have shape"),
    ("loc_shape", "locations must have shape"), ("loc_np", "locations must have shape"),
    ("pri_shape", "priors must have shape"), ("pri_batch", "batch of 1 or N"), ("sizes_shape", "image_sizes"),
    ("no_priors", "needs priors"), ("both", "tuple"), ("not_tensor", "scores must be a torch.Tensor"),
])
def test_refusals_name_the_argument(monkeypatch, case, match):
    s, l, p = _inputs()
    kw = {}
    if case == "cand0":
        kw["candidate_size"] = 0
    elif case == "cand_float":
        kw["candidate_size"] = 2.0
    elif case == "top_k":
        kw["top_k"] = 1.5
    elif case == "C1":
        s = s[..., :1].contiguous()
    elif case == "scores_dtype":
        s = s.double()
    elif case == "loc_dtype":
        l = l.half()
    elif case == "pri_dtype":
        p = p.double()
    elif case == "scores_nc":
        s = s.transpose(0, 1).contiguous().transpose(0, 1)
    elif case == "loc_nc":
        l = torch.randn(2, 4, 7).transpose(1, 2)
    elif case == "scores_shape":
        s = s[0]
    elif case == "loc_shape":
        l = torch.randn(2, 7, 5)
    elif case == "loc_np":
        l, p = torch.randn(2, 6, 4), torch.rand(6, 4)
    elif case == "pri_shape":
        p = torch.rand(6, 4)
    elif case == "pri_batch":
        p = torch.rand(3, 7, 4)
    elif case == "sizes_shape":
        kw["image_sizes"] = torch.ones(2, 3)
    elif case == "not_tensor":
        s = s.numpy()
    if case == "no_priors":
        fake = _refused(monkeypatch, match, s, l, None, 0.1, 0.2, **kw)
    elif case == "both":
        fake = _refused(monkeypatch, match, s, (l, p, 0.1, 0.2), p, **kw)
    else:
        fake = _refused(monkeypatch, match, s, l, p, 0.1, 0.2, **kw)
    assert fake.calls == []


def test_candidate_size_above_the_limit_is_refused_by_the_library(monkeypatch):
    s, l, p = _inputs()
    fake = _refused(monkeypatch, "dfq_ssd_nms", s, l, p, 0.1, 0.2, candidate_size=1025)
    assert fake.refusals == [("dfq_ssd_nms", fakelib_detect.E_UNSUPPORTED, "candidate_size is above the limit")]
    from dfq_b200 import detect
    det = detect.postprocess(s, l, p, 0.1, 0.2, candidate_size=1024, prob_threshold=0.0)
    assert det.offsets.shape == (3,)


def test_cpu_tensors_are_refused():
    from dfq_b200 import detect
    s, l, p = _inputs()
    with pytest.raises(_lib.DfqError, match="scores must be on the GPU"):
        detect.postprocess(s, l, p, 0.1, 0.2)
    with pytest.raises(_lib.DfqError, match="locations must be on the GPU"):
        detect.decode_boxes(l, p, 0.1, 0.2)


def test_descriptor_layout():
    assert _lib.SSD_NMS_DT.itemsize == 40 and _lib.SSD_NMS_DT.fields["center_variance"][1] == 16
    assert _lib.SSD_NMS_DT.fields["candidate_size"][1] == 32 and list(_lib.EXPECTED_SIZES)[-1] == "DfqSsdNms"
