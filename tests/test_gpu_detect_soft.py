"""dfq_b200.detect.postprocess(nms_method="soft") on the H100: bit for bit against the soft NMS of
tests/ssd_soft_nms_oracle.py run on CUDA tensors (torch's CUDA exp), over batch sizes, class counts, prior counts,
the edge scenes of tests/soft_nms_cases.py and both sides of every launch the kernel chooses between (up to 1,024
candidates on a small CTA, up to 11,264 in one CTA's shared memory, beyond that in global memory); against the
reference's CPU fixture within a stated ULP bound on the scores; one host synchronisation per call; the library's
refusals; and end to end behind the chained SSD-Lite of tests/ssd_lite_like.py into detect.Evaluator."""
import warnings

import numpy as np
import pytest
import torch

import soft_nms_cases
import ssd_map_oracle as O
import ssd_soft_nms_oracle as SO
from test_detect_soft_host import _eq, _triples, fixture

pytestmark = pytest.mark.gpu

CV, SV = 0.1, 0.2
SMALL_ROWS, LARGE_ROWS = 1024, 11264       # the kernel's launch boundaries (k_ssd_soft in detect.cu)

# The largest difference, in units in the last place, between the scores of the device path and those of the reference's
# CPU soft NMS on the fixture (ref_ssd_soft_nms.npz), as measured on an H100: 19 ulp at top_k -1, 1 at top_k 5, 0 at
# top_k 1.  It comes from exp alone: torch's CPU exp and CUDA's expf differ in the last bit on some arguments, and a
# score rescored many times carries each step's difference into the next.  No pick, box or label differs.
FIXTURE_ULP_BOUND = 19


def _same_image(g, w):
    return all(_eq(a, b) for a, b in zip(g, w))


def _direct(scores, boxes, thr, sigma, top_k=-1, sizes=None):
    """dfq_ssd_soft_nms + dfq_ssd_soft_compact on decoded boxes given as they are: [(boxes, labels, probs)] per image,
    and the candidate counts."""
    from dfq_b200 import _lib, detect
    N, P, C = scores.shape
    d, _ = detect._descriptor(torch.zeros(N, P, 4, device="cuda"), torch.zeros(P, 4, device="cuda"), CV, SV, C, thr,
                              0.45, 200, top_k)
    lib, st, dp = _lib.load(), _lib.stream_ptr(), _lib.table_ptr(d)
    S = N * (C - 1)
    cand = torch.empty(S, dtype=torch.int32, device="cuda")
    cnt = torch.empty(S, dtype=torch.int32, device="cuda")
    off = torch.empty(S + 1, dtype=torch.int64, device="cuda")
    _lib.check(lib.dfq_ssd_soft_nms(detect._ptr(scores), detect._ptr(boxes), detect._ptr(cand), detect._ptr(cnt),
                                    detect._ptr(off), dp, sigma, st), "dfq_ssd_soft_nms")
    T = int(off[-1])
    sizes = sizes.to(torch.float32).contiguous() if sizes is not None else None
    ob = torch.empty(max(T, 1), 4, device="cuda")
    ol = torch.empty(max(T, 1), dtype=torch.int64, device="cuda")
    op = torch.empty(max(T, 1), device="cuda")
    if T:
        _lib.check(lib.dfq_ssd_soft_compact(detect._ptr(scores), detect._ptr(boxes), detect._ptr(cand), detect._ptr(off),
                                            detect._ptr(sizes), detect._ptr(ob), detect._ptr(ol), detect._ptr(op), dp,
                                            sigma, st), "dfq_ssd_soft_compact")
    det = detect.Detections(ob[:T], ol[:T], op[:T], off[::C - 1])
    assert cnt.sum().item() == T
    return det.per_image(), cand.cpu()


def _check_direct(scores, boxes, thr=0.01, sigma=0.5, top_k=-1, sizes=None):
    got, cand = _direct(scores, boxes, thr, sigma, top_k, sizes)
    sz = sizes.cpu().tolist() if sizes is not None else [None] * scores.shape[0]
    for n in range(scores.shape[0]):
        want = SO.predict_one(scores[n], boxes[n], sz[n], prob_threshold=thr, top_k=top_k, nms_method="soft",
                              sigma=sigma, device="cuda")
        assert _same_image(got[n], want), (n, [x.shape for x in got[n]], [x.shape for x in want])
    return got, cand


def _check(scores, locations, priors, sizes=None, **kw):
    """postprocess(nms_method="soft") against the oracle on CUDA tensors, image by image."""
    from dfq_b200 import detect
    det = detect.postprocess(scores, locations, priors, CV, SV, sizes, nms_method="soft", **kw)
    kw = dict(kw)
    sigma = kw.pop("sigma", 0.5)
    boxes = SO.decode(locations, priors, CV, SV)
    sz = sizes.cpu().tolist() if sizes is not None else [None] * scores.shape[0]
    got = det.per_image()
    for n in range(scores.shape[0]):
        want = SO.predict_one(scores[n], boxes[n], sz[n], nms_method="soft", sigma=sigma, device="cuda", **kw)
        assert _same_image(got[n], want), n
    offs = det.offsets.cpu()
    assert offs[0] == 0 and offs[-1] == det.boxes.shape[0]
    return det


def _rand(N, P, C, seed, temp=2.5, bg=5.0, spread=0.7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(N, P, C, device="cuda", generator=g) * temp
    logits[..., 0] += bg
    scores = torch.softmax(logits, 2)
    locations = torch.randn(N, P, 4, device="cuda", generator=g) * spread
    priors = torch.rand(P, 4, device="cuda", generator=g) * torch.tensor([1, 1, 0.5, 0.5], device="cuda") + 0.01
    return scores, locations, priors


def _boxes(P, seed, spread=1.0, size=0.3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.rand(P, 2, device="cuda", generator=g) * spread
    wh = torch.rand(P, 2, device="cuda", generator=g) * size + 0.005
    return torch.cat([c - wh / 2, c + wh / 2], 1)


# ---- against the oracle on CUDA ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,C,P,seed,temp,bg", [(1, 2, 1, 1, 2.5, 0.0), (1, 21, 3000, 2, 2.5, 5.0),
                                                (7, 21, 3000, 3, 1.5, 4.0), (2, 91, 3000, 4, 1.5, 3.0),
                                                (256, 21, 3000, 5, 1.0, 9.0), (1, 21, 8732, 6, 2.0, 6.0),
                                                (1, 2, 20001, 7, 2.0, 3.0)])
@pytest.mark.parametrize("top_k", [-1, 5])
def test_seeded_batches_match_the_oracle(N, C, P, seed, temp, bg, top_k):
    scores, loc, pri = _rand(N, P, C, seed, temp, bg)
    sizes = torch.randint(100, 900, (N, 2), device="cuda")
    _check(scores, loc, pri, sizes, top_k=top_k, sigma=0.3)


@pytest.mark.parametrize("sigma", [0.5, 0.3, 2.0, 1e-3])
def test_sigmas(sigma):
    scores, loc, pri = _rand(3, 3000, 21, 11, 2.0, 5.0)
    _check(scores, loc, pri, sigma=sigma)


@pytest.mark.parametrize("name", [s[0] for s in soft_nms_cases.scenes()])
@pytest.mark.parametrize("top_k", [1, 5, -1])
def test_edge_scenes(name, top_k):
    _, s, b = next(sc for sc in soft_nms_cases.scenes() if sc[0] == name)
    _check_direct(s.cuda(), b.cuda(), soft_nms_cases.THR, soft_nms_cases.SIGMA, top_k,
                  torch.tensor([[640, 480]], device="cuda"))


def _segment(P, m, seed, spread, size):
    """One image, C = 2: m candidates spread over P priors (every prior when m == P)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.zeros(1, P, 2, device="cuda")
    idx = torch.randperm(P, device="cuda", generator=g)[:m]
    s[0, idx, 1] = torch.rand(m, device="cuda", generator=g) * 0.9 + 0.05
    s[0, :, 0] = 1 - s[0, :, 1]
    return s, _boxes(P, seed + 1, spread, size).unsqueeze(0)


@pytest.mark.parametrize("P,m", [(3000, SMALL_ROWS), (3000, SMALL_ROWS + 1), (8732, 8732), (20001, LARGE_ROWS),
                                 (20001, LARGE_ROWS + 1), (20001, 20001)])
@pytest.mark.parametrize("top_k", [50, -1])
def test_both_sides_of_each_launch_boundary(P, m, top_k):
    """Segments with exactly the candidates a launch holds and one more; the full segments are crowded so that rows decay
    out at every step."""
    s, b = _segment(P, m, P + m, 0.6 if top_k < 0 else 1.0, 0.2)
    _, cand = _check_direct(s, b, 0.01, 0.5, top_k)
    assert cand.tolist() == [m]


def test_launches_share_one_batch():
    """Segments of all three sizes in one call, in a class order that interleaves them."""
    P = 12000
    g = torch.Generator(device="cuda").manual_seed(5)
    s = torch.zeros(2, P, 5, device="cuda")
    for n, ms in enumerate(((10, 12000, 900, 0), (2000, 5, 11500, 1))):
        for c, m in enumerate(ms, 1):
            idx = torch.randperm(P, device="cuda", generator=g)[:m]
            s[n, idx, c] = torch.rand(m, device="cuda", generator=g) * 0.5 + 0.02
    b = torch.stack([_boxes(P, 8, 0.5, 0.2), _boxes(P, 9, 0.5, 0.2)])
    _, cand = _check_direct(s, b, 0.01, 0.5, 20)
    assert cand.tolist() == [10, 12000, 900, 0, 2000, 5, 11500, 1]


def test_disjoint_boxes_pick_every_candidate_in_score_order():
    P = 4000
    s = torch.zeros(1, P, 2, device="cuda")
    s[0, :, 1] = torch.linspace(0.02, 0.9, P, device="cuda").flip(0)[torch.randperm(P, device="cuda")]
    x = torch.arange(P, device="cuda", dtype=torch.float32) * 2
    b = torch.stack([x, x, x + 1, x + 1], 1).unsqueeze(0)
    got, _ = _check_direct(s, b)
    assert got[0][0].shape[0] == P and torch.equal(got[0][2], s[0, :, 1].sort(descending=True).values.cpu())


# ---- against the reference's CPU fixture --------------------------------------------------------------------------------------
def _ulps(a, b):
    ia = a.numpy().view(np.int32).astype(np.int64)
    ib = b.numpy().view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 31) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 31) - ib, ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("k", range(3))
def test_reference_fixture_within_the_exp_bound(k):
    """The kernel on the boxes the fixture's predictor decoded (on the CPU, so the decode's own exp does not enter):
    the same picks in the same order, equal boxes and labels, scores within FIXTURE_ULP_BOUND."""
    z, t, cv, sv = fixture()
    top_k, sigma = int(z["top_ks"][k]), float(z["sigma"])
    boxes = SO.decode(t["locations"], t["priors"], cv, sv)
    got, _ = _direct(t["scores"].cuda(), boxes.cuda(), 0.01, sigma, top_k, t["image_sizes"].cuda())
    worst = 0
    for n, (g, (b, l, p)) in enumerate(zip(got, _triples(z, k))):
        b, l, p = torch.from_numpy(b), torch.from_numpy(l), torch.from_numpy(p)
        assert g[0].shape == b.shape, (k, n, g[0].shape, b.shape)
        rows = ((g[0] != b).any(1) | (g[1] != l)).nonzero().flatten().tolist()
        assert not rows, "image %d: pick %d differs from the reference: got %s class %d, want %s class %d" % (
            n, rows[0], g[0][rows[0]].tolist(), g[1][rows[0]], b[rows[0]].tolist(), l[rows[0]])
        u = _ulps(g[2], p)
        worst = max(worst, int(u.max()) if u.size else 0)
    print("soft NMS fixture %d: largest score difference %d ulp" % (k, worst))
    assert worst <= FIXTURE_ULP_BOUND


# ---- host synchronisation, refusals ----------------------------------------------------------------------------------------
def test_one_host_synchronisation_per_call():
    from dfq_b200 import detect
    scores, loc, pri = _rand(16, 3000, 21, 12, 2.0, 5.0)
    sizes = torch.randint(100, 900, (16, 2), device="cuda")
    detect.postprocess(scores, loc, pri, CV, SV, sizes, nms_method="soft")          # warm
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            detect.postprocess(scores, loc, pri, CV, SV, sizes, nms_method="soft")
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]


def test_library_refusals():
    from dfq_b200 import _lib, detect
    lib = _lib.load()
    N, P, C = 1, 8, 3
    s, b = torch.rand(N, P, C, device="cuda"), torch.rand(N, P, 4, device="cuda")
    cand = torch.zeros(2, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    off = torch.zeros(3, dtype=torch.int64, device="cuda")
    ob, ol, op = torch.zeros(4, 4, device="cuda"), torch.zeros(4, dtype=torch.int64, device="cuda"), \
        torch.zeros(4, device="cuda")
    P_ = detect._ptr
    E_ARG = -1

    def last_error():
        return lib.dfq_last_error().decode()

    def desc(**kv):
        d, _ = detect._descriptor(torch.zeros(N, P, 4, device="cuda"), torch.zeros(P, 4, device="cuda"), CV, SV, C, 0.01)
        for k, v in kv.items():
            d[0][k] = v
        return d

    cases = [(None, 0.5, "descriptor is NULL"), (desc(N=0), 0.5, "N and P must be positive"),
             (desc(P=0), 0.5, "N and P must be positive"), (desc(prior_batch=2), 0.5, "prior_batch must be 1 or N"),
             (desc(C=1), 0.5, "C must be at least 2"), (desc(), 0.0, "sigma must be a finite positive number"),
             (desc(), -1.0, "sigma must be a finite positive number"),
             (desc(), float("nan"), "sigma must be a finite positive number"),
             (desc(), float("inf"), "sigma must be a finite positive number")]
    for d, sigma, msg in cases:
        dp = _lib.table_ptr(d) if d is not None else None
        for rc in (lib.dfq_ssd_soft_nms(P_(s), P_(b), P_(cand), P_(cnt), P_(off), dp, sigma, _lib.stream_ptr()),
                   lib.dfq_ssd_soft_compact(P_(s), P_(b), P_(cand), P_(off), None, P_(ob), P_(ol), P_(op), dp, sigma,
                                            _lib.stream_ptr())):
            assert rc == E_ARG and msg in last_error(), (msg, last_error())
    dp = _lib.table_ptr(desc())
    assert lib.dfq_ssd_soft_nms(P_(s), P_(b), None, P_(cnt), P_(off), dp, 0.5, _lib.stream_ptr()) == E_ARG
    assert "every pointer must be non-NULL" in last_error()
    bb = torch.zeros(N * P * 4 + 1, device="cuda")[1:]
    assert lib.dfq_ssd_soft_nms(P_(s), P_(bb), P_(cand), P_(cnt), P_(off), dp, 0.5, _lib.stream_ptr()) == E_ARG
    assert lib.dfq_ssd_soft_compact(P_(s), P_(b), P_(cand), P_(off), None, P_(ob), None, P_(op), dp, 0.5,
                                    _lib.stream_ptr()) == E_ARG
    assert "every pointer but image_sizes must be non-NULL" in last_error()
    obb = torch.zeros(17, device="cuda")[1:]
    assert lib.dfq_ssd_soft_compact(P_(s), P_(b), P_(cand), P_(off), None, P_(obb), P_(ol), P_(op), dp, 0.5,
                                    _lib.stream_ptr()) == E_ARG


# ---- end to end on SSD-Lite ----------------------------------------------------------------------------------------------------
def _end_to_end(m, x):
    """postprocess(nms_method="soft") + Evaluator behind the model: the detections equal the oracle's, and the APs equal
    those of the oracle's detections through tests/ssd_map_oracle.py."""
    from dfq_b200 import detect
    z, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    sizes = torch.tensor([[300, 300], [640, 480]], device="cuda")[:x.shape[0]]
    with torch.no_grad():
        scores, loc = m(x)
        det = detect.postprocess(scores, loc, priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes,
                                 nms_method="soft")
        boxes = SO.decode(loc, pri, cv, sv)
    per = det.per_image()
    want = [SO.predict_one(scores[n], boxes[n], sizes[n].tolist(), nms_method="soft", device="cuda")
            for n in range(x.shape[0])]
    for n, (g, w) in enumerate(zip(per, want)):
        assert _same_image(g, w), n
    assert det.boxes.shape[0] > 0
    g = np.random.default_rng(int(det.boxes.shape[0]))
    gts = []
    for b, l, p in want:
        b, l = b.reshape(-1, 4).numpy(), l.reshape(-1).long().numpy()
        pick = g.random(len(l)) < 0.05
        boxes_ = b[pick] + g.normal(0, 3, (int(pick.sum()), 4)).astype(np.float32)
        extra = g.uniform(0, 250, (3, 2))
        boxes_ = np.concatenate([boxes_, np.concatenate([extra, extra + 40], 1)]).astype(np.float32)
        labels = np.concatenate([l[pick], g.integers(1, 21, 3)]).astype(np.int64)
        gts.append((boxes_, labels, (g.random(len(labels)) < 0.15).astype(np.uint8)))
    for use_2007 in (True, False):
        ev = detect.Evaluator(21, 0.5, use_2007)
        ev.add_batch(det, detect.ground_truth(gts, "cuda"))
        aps, flags = O.average_precision(want, gts, 21, 0.5, use_2007)
        got = ev.average_precision()
        assert np.array_equal(np.asarray(got, np.float64), np.asarray(aps, np.float64), equal_nan=True)
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
