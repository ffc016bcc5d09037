"""dfq_b200.detect on the H100: the decode bit for bit against torch's CUDA ops, postprocess bit for bit against the stable
oracle of tests/ssd_postprocess_oracle.py (the reference's fixture inputs, ties, degenerate boxes and scores, the limits),
and end to end on the SSD-Lite of tests/ssd_lite_like.py chained under both int8 schemes and loaded back."""
import numpy as np
import pytest
import torch

import ssd_postprocess_oracle as SO
from test_detect_host import _same, fixture

pytestmark = pytest.mark.gpu

CV, SV = 0.1, 0.2


def _bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _check(scores, locations, priors, sizes=None, cv=CV, sv=SV, **kw):
    """postprocess against the oracle image by image (the oracle decodes on the GPU, as the predictor does); returns the
    Detections."""
    from dfq_b200 import detect
    det = detect.postprocess(scores, locations, priors, cv, sv, sizes, **kw)
    want = SO.predict(scores, locations, priors, cv, sv, sizes, **kw)
    got = det.per_image()
    assert len(got) == len(want)
    for n, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), (n, kw, [(x.shape, y.shape) for x, y in zip(g, w)])
    offs = det.offsets.cpu()
    assert offs[0] == 0 and offs[-1] == det.boxes.shape[0] and det.boxes.is_cuda
    return det


def _rand(N, P, C, seed, temp=2.5, bg=5.0, spread=0.7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(N, P, C, device="cuda", generator=g) * temp
    logits[..., 0] += bg
    scores = torch.softmax(logits, 2)
    locations = torch.randn(N, P, 4, device="cuda", generator=g) * spread
    priors = torch.rand(P, 4, device="cuda", generator=g) * torch.tensor([1, 1, 0.5, 0.5], device="cuda") + 0.01
    return scores, locations, priors


# ---- decode -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 3000, 8732, 20001])
@pytest.mark.parametrize("prior_shape", ["P4", "1P4", "NP4"])
def test_decode_is_torch_bit_for_bit(P, prior_shape):
    from dfq_b200 import detect
    N = 3
    g = torch.Generator(device="cuda").manual_seed(P)
    loc = torch.randn(N, P, 4, device="cuda", generator=g) * 3
    pri = torch.rand(N if prior_shape == "NP4" else 1, P, 4, device="cuda", generator=g)
    special = torch.tensor([float("nan"), -0.0, 0.0, 1e-40, -1e-40, 500.0, -500.0, float("inf"), -float("inf"), 1e30],
                           device="cuda")
    flat = loc.view(-1)
    k = min(flat.numel(), 4 * special.numel())
    flat[:k] = special.repeat(4)[:k]                      # specials in every coordinate: exp overflow to inf, NaN, ...
    pri.view(-1)[:min(pri.numel(), 6)] = torch.tensor([0.0, -0.0, 1e-40, 0.5, float("nan"), 2.0],
                                                      device="cuda")[:min(pri.numel(), 6)]
    p = pri[0] if prior_shape == "P4" else pri
    for cv, sv in ((CV, SV), (0.13, 0.37)):
        got = detect.decode_boxes(loc, p, cv, sv)
        assert _bits(got, SO.decode(loc, p, cv, sv)), (P, prior_shape, cv, sv)


# ---- NMS against the oracle -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(4))
def test_reference_fixture_inputs(k):
    z, t, cv, sv = fixture()
    top_k, cand = (int(v) for v in z["configs"][k])
    t = {n: v.cuda() for n, v in t.items()}
    det = _check(t["scores"], t["locations"], t["priors"], t["image_sizes"], cv, sv, candidate_size=cand, top_k=top_k)
    assert det.offsets.tolist() == z["offsets_%d" % k].tolist()


@pytest.mark.parametrize("N,C,seed", [(1, 2, 1), (1, 21, 2), (2, 91, 3), (256, 21, 4)])
def test_seeded_batches_and_class_counts(N, C, seed):
    # peaked enough that the 256-image batch keeps a few candidates per class (the oracle runs one pick at a time)
    scores, loc, pri = _rand(N, 3000, C, seed, temp=1.5 if N < 256 else 1.0, bg=3.0 if N < 256 else 9.0)
    sizes = torch.randint(100, 1000, (N, 2), device="cuda")
    _check(scores, loc, pri, sizes)
    if N < 256:
        _check(scores, loc, pri, top_k=3, iou_threshold=0.3)


def test_vgg_prior_count():
    scores, loc, pri = _rand(2, 8732, 21, 5)
    _check(scores, loc, pri, candidate_size=300)


def test_heavy_ties_follow_prior_order():
    scores, loc, pri = _rand(2, 3000, 21, 6, temp=1.0, bg=1.0)
    scores = (scores * 64).floor() / 64                   # a few distinct values per class
    det = _check(scores, loc, pri, prob_threshold=0.0)
    assert det.boxes.shape[0] > 0


def test_identical_boxes_give_one_pick_per_class():
    scores, _, _ = _rand(3, 500, 21, 7, temp=1.0, bg=0.0)
    loc = torch.zeros(3, 500, 4, device="cuda")
    pri = torch.tensor([0.5, 0.5, 0.2, 0.2], device="cuda").expand(500, 4).contiguous()
    det = _check(scores, loc, pri)
    assert det.boxes.shape[0] == 3 * 20


def test_disjoint_boxes_keep_candidate_size():
    side = 40
    P = side * side
    ys, xs = torch.meshgrid(torch.arange(side), torch.arange(side), indexing="ij")
    pri = torch.stack([(xs.reshape(-1) + 0.5) / side, (ys.reshape(-1) + 0.5) / side,
                       torch.full((P,), 0.5 / side), torch.full((P,), 0.5 / side)], 1).float().cuda()
    scores, _, _ = _rand(2, P, 4, 8, temp=0.5, bg=0.0)
    loc = torch.zeros(2, P, 4, device="cuda")
    for cand in (1, 200, 1024):
        det = _check(scores, loc, pri, candidate_size=cand)
        assert det.boxes.shape[0] == 2 * 3 * cand


def test_fewer_candidates_than_candidate_size():
    scores, loc, pri = _rand(3, 3000, 21, 9, temp=1.0, bg=8.0)
    keep = (scores[..., 1:] > 0.01).sum(1)
    assert 0 < keep.max() < 200
    _check(scores, loc, pri)


def test_scores_at_the_threshold():
    scores, loc, pri = _rand(2, 1000, 5, 10)
    thr = np.float32(0.01)
    scores[:, ::3, 1:] = float(thr)                      # exactly fp32(0.01): not a candidate
    scores[:, 1::3, 1:] = float(np.nextafter(thr, np.float32(1)))
    det = _check(scores, loc, pri)
    assert det.boxes.shape[0] > 0


def test_nan_and_inf_scores_and_boxes():
    scores, loc, pri = _rand(2, 3000, 21, 11)
    g = torch.Generator(device="cuda").manual_seed(11)
    for v in (float("nan"), float("inf"), -float("inf"), -0.0):
        idx = torch.randint(0, scores.numel(), (300,), device="cuda", generator=g)
        scores.view(-1)[idx] = v
        idx = torch.randint(0, loc.numel(), (300,), device="cuda", generator=g)
        loc.view(-1)[idx] = v if v != -0.0 else 200.0    # 200 * 0.2: exp overflows to inf
    det = _check(scores, loc, pri)
    assert det.boxes.isnan().any() and det.probs.isinf().any()
    _check(scores, loc, pri, prob_threshold=-1.0, candidate_size=50)


def test_zero_area_boxes():
    scores, loc, pri = _rand(2, 2000, 21, 12)
    pri[::2, 2] = 0.0
    pri[1::4, 3] = 0.0
    _check(scores, loc, pri)


@pytest.mark.parametrize("iou", [0.0, 1.0])
def test_iou_threshold_extremes(iou):
    scores, loc, pri = _rand(2, 3000, 21, 13, temp=1.0, bg=4.0)
    _check(scores, loc, pri, iou_threshold=iou)


def test_candidate_size_limit():
    from dfq_b200 import _lib, detect
    scores, loc, pri = _rand(1, 3000, 6, 14, temp=1.0, bg=0.0)
    _check(scores, loc, pri, candidate_size=1024)
    _check(scores, loc, pri, candidate_size=1)
    with pytest.raises(_lib.DfqError, match="candidate_size 1025 is above the limit"):
        detect.postprocess(scores, loc, pri, CV, SV, candidate_size=1025)


# ---- end to end on SSD-Lite -------------------------------------------------------------------------------------------------
def _end_to_end(m, x):
    from dfq_b200 import detect
    z, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    sizes = torch.tensor([[300, 300], [640, 480]], device="cuda")[:x.shape[0]]
    with torch.no_grad():
        out = m(x)
        scores, loc = out
        det = detect.postprocess(*out, priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
        want = SO.predict(scores, loc, pri, cv, sv, sizes)
    got = det.per_image()
    for n, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), n
    assert det.boxes.shape[0] > 0
    return det


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
