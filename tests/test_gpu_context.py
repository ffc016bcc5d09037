"""Every device entry point off its usual setting: on a side stream while the default stream is busy, on two streams
interleaved, from concurrent host threads, and on a GPU that is not the current one.  Each result is compared bit for bit
with the same call made on the default stream of cuda:0 from one thread, which the other suites pin to the oracles and
the libraries.  DESIGN.md, "Launch context", states the rules these check."""
import contextlib
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus  # noqa: E402
import map_scenes  # noqa: E402
import png_corpus  # noqa: E402
import preprocess_cases as PC  # noqa: E402
from test_gpu_detect import _rand  # noqa: E402
from dfq_b200 import _lib  # noqa: E402

pytestmark = pytest.mark.gpu
SPIN = 2_000_000_000        # cycles of torch.cuda._sleep: about 1 s of a busy default stream at 1.98 GHz, bounded


# ---- comparison ----------------------------------------------------------------------------------------------------------
def _flat(x):
    """Tensors, arrays and numbers of a result, in order (Detections and dataclasses by field)."""
    if isinstance(x, (list, tuple)):
        return [v for e in x for v in _flat(e)]
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _flat(x[k])]
    if hasattr(x, "__dataclass_fields__"):
        return [v for k in x.__dataclass_fields__ for v in _flat(getattr(x, k))]
    return [x]


def _bits(v):
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu()
        if v.dtype == torch.float32:
            v = v.view(torch.int32)
        elif v.dtype == torch.float64:
            v = v.view(torch.int64)
        return ("t", v.dtype, tuple(v.shape), v.numpy().tobytes())
    if isinstance(v, np.ndarray) or isinstance(v, (float, np.floating)):
        a = np.ascontiguousarray(v)
        return ("a", a.dtype.str, a.shape, a.tobytes())
    return ("o", v)


def _same(a, b):
    fa, fb = _flat(a), _flat(b)
    return len(fa) == len(fb) and all(_bits(x) == _bits(y) for x, y in zip(fa, fb))


# ---- the workloads -----------------------------------------------------------------------------------------------------------
def _jpegs():
    return [b for _, b in jpeg_corpus.corpus(big=False)]


def _pngs():
    out = []
    for k, (_, b) in enumerate(png_corpus.corpus(big=False)):
        h, w = png_corpus.pillow(b).shape[:2]
        out.append((PC.image(h, w, k), b))
    return out


class Work:
    """The calls of one batch size N; each method makes its calls on the current device's current stream and returns the
    results.  Inputs are made once on the default stream of the current device."""

    def __init__(self, N, seed, P=3000, jp=None, pn=None):
        self.N, self.dev = N, torch.device("cuda", torch.cuda.current_device())
        g = np.random.default_rng(seed)
        jp = jp if jp is not None else _jpegs()
        pn = pn if pn is not None else _pngs()
        self.images = [jp[int(i)] if i % 2 else PC.image(int(g.integers(60, 500)), int(g.integers(60, 500)), seed + i)
                       for i in g.integers(0, len(jp), N)]
        pick = [pn[int(i)] for i in g.integers(0, len(pn), min(N, 8))]
        self.seg_images, self.seg_labels = [p[0] for p in pick], [p[1] for p in pick]
        self.det = _rand(N, P, 21, seed)
        self.cls_logits = torch.randn(N, 1000, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
        self.cls_labels = torch.randint(0, 1000, (N,), generator=torch.Generator().manual_seed(seed))
        self.seg_logits = torch.randn(N, 21, 17, 23, device="cuda", generator=torch.Generator("cuda").manual_seed(seed + 1))
        self.seg_target = torch.randint(0, 22, (N, 65, 89), device="cuda", dtype=torch.uint8,
                                        generator=torch.Generator("cuda").manual_seed(seed + 2))
        gts, dets = map_scenes.scene(N, 21, seed)
        self.gts, self.dets = gts, dets
        torch.cuda.synchronize()

    def preprocess(self):
        from dfq_b200 import preprocess as P
        seg, lab = P.voc_segmentation(self.seg_images, self.seg_labels, crop_size=129)
        return P.imagenet(self.images), seg, lab, P.ssd(self.images)

    def decode(self):
        from dfq_b200 import jpeg, png
        return jpeg.decode([b for b in self.images if isinstance(b, bytes)] or _jpegs()[:1]), png.decode(self.seg_labels)

    def hard(self):
        from dfq_b200 import detect
        s, l, p = self.det
        return detect.postprocess(s, l, priors=p, center_variance=0.1, size_variance=0.2, top_k=50)

    def soft(self):
        from dfq_b200 import detect
        s, l, p = self.det
        return detect.postprocess(s, l, priors=p, center_variance=0.1, size_variance=0.2, prob_threshold=0.3,
                                  nms_method="soft", sigma=0.5, top_k=20)

    def predict(self):
        from dfq_b200 import classify, detect, segment
        s, l, p = self.det
        return (classify.predict(self.cls_logits), segment.predict(self.seg_logits, (65, 89), align_corners=False),
                detect.decode_boxes(l, p, 0.1, 0.2))

    def evaluators(self):
        """The evaluators fed here; read() gives their results (call it after the feeding stream has been waited for)."""
        from dfq_b200 import classify, detect, segment
        c, s, d = classify.Evaluator(1000), segment.Evaluator(21), detect.Evaluator(21)
        c.add_logits(self.cls_logits, self.cls_labels)
        s.add_logits(self.seg_target, self.seg_logits, align_corners=True)
        d.add_batch(map_scenes.detections(self.dets, self.dev), detect.ground_truth(self.gts, self.dev))
        return c, s, d

    @staticmethod
    def read(evs):
        c, s, d = evs
        return int(c.num_correct), s.confusion_matrix, d.average_precision()

    def plane_mean(self):
        from dfq_b200 import ncnn
        return ncnn.PlaneMean(True)(self.seg_logits), ncnn.PlaneMean(False, out_scale=9.0)(self.seg_logits)

    CALLS = ("preprocess", "decode", "hard", "soft", "predict", "plane_mean")

    def all(self):
        return {k: getattr(self, k)() for k in self.CALLS}


@contextlib.contextmanager
def _chain(scheme):
    """(chained MobileNetV2, input batch) of one int8 scheme, built on the default stream of cuda:0; run it inside."""
    import affine_observed_state
    from dfq_b200 import int8
    with affine_observed_state.evaluation_state("mobilenet_v2", size=64, batch=4) as (model, qgraph, qtarg):
        if scheme == "affine":
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True)
        else:
            int8.convert_to_int8(model, qgraph, qtarg)
            gm = int8.chain_int8(model, residual=True)
        x = torch.randn(4, 3, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        yield gm, x


# ---- side stream -------------------------------------------------------------------------------------------------------------
def side_stream_trace(what):
    """Each call family of `what` ("work": every Work call and the evaluators' adds; "affine" / "ncnn": the chained
    MobileNetV2) made on a stream of its own while the default stream spins, under one CUDA profiler session.  Every
    kernel, copy and memset in the Kineto trace must be on the family's stream: the only event on the default stream is
    the spin.  The results must equal the same calls made before on the default stream.  Run in a fresh interpreter, so
    that the profiler session is the process's only one."""
    import json
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    with contextlib.ExitStack() as stack:
        if what == "work":
            work = Work(30, 3)
            fams = {k: getattr(work, k) for k in Work.CALLS}
            fams["evaluators"] = work.evaluators
        else:
            gm, x = stack.enter_context(_chain(what))
            stack.enter_context(torch.no_grad())
            fams = {"chain": lambda: gm(x)}
        want = {k: f() for k, f in fams.items()}
        if "evaluators" in want:
            want["evaluators"] = Work.read(want["evaluators"])
        torch.cuda.synchronize()
        streams = {k: torch.cuda.Stream() for k in fams}
        got = {}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(4 * SPIN)
            for k, f in fams.items():
                with torch.cuda.stream(streams[k]):
                    torch.cuda._sleep(1)                   # marks the family's stream in the trace
                    got[k] = f()
                streams[k].synchronize()                   # families in turn: their marks are in launch order
            spinning = not torch.cuda.current_stream().query()
            torch.cuda.synchronize()
        if "evaluators" in got:                            # read on the default stream, after the spin
            got["evaluators"] = Work.read(got["evaluators"])
        with tempfile.TemporaryDirectory() as d:
            prof.export_chrome_trace(os.path.join(d, "trace.json"))
            with open(os.path.join(d, "trace.json")) as f:
                events = json.load(f)["traceEvents"]
    assert spinning, "the default stream finished its spin before the calls on the side streams did"
    for k in want:
        assert _same(got[k], want[k]), k
    dev = sorted((e for e in events if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["ts"])
    spins = [e for e in dev if "spin" in e["name"]]
    assert len(spins) == len(fams) + 1, [(e["name"], e["args"]["stream"], e["dur"]) for e in spins]
    default = max(spins, key=lambda e: e["dur"])
    marks = [e for e in spins if e is not default]
    fam_stream = dict(zip(fams, (e["args"]["stream"] for e in marks)))
    assert len(set(fam_stream.values())) == len(fams) and default["args"]["stream"] not in fam_stream.values(), fam_stream
    where = {}
    for e in dev:
        if e is not default and e not in marks:
            where.setdefault(e["args"]["stream"], []).append(e["name"])
    stray = {st: names[:5] for st, names in where.items() if st not in fam_stream.values()}
    assert not stray, "events off the families' streams (default stream %s): %s" % (default["args"]["stream"], stray)
    for k, st in fam_stream.items():
        assert where.get(st), "%s issued nothing on its stream" % k


@pytest.mark.parametrize("what", ["work", "affine", "ncnn"])
def test_side_stream_trace(what):
    _subprocess("side_stream_trace", what)


# ---- two streams interleaved -------------------------------------------------------------------------------------------------
def test_two_streams_interleaved_without_waits():
    """Two batches enqueued alternately on two streams, ten rounds, no waits: the descriptor ring wraps under both streams,
    the preprocessing staging blocks are reused across them, and postprocess reads its pick count back on each."""
    jp, pn = _jpegs(), _pngs()
    a, b = Work(7, 11, jp=jp, pn=pn), Work(30, 12, P=8732, jp=jp, pn=pn)
    want = [a.all(), b.all()]
    torch.cuda.synchronize()
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    got = [[], []]
    for _ in range(10):
        for k, (w, s) in enumerate(((a, sa), (b, sb))):
            with torch.cuda.stream(s):
                got[k].append(w.all())
    torch.cuda.synchronize()
    for k in range(2):
        for r, g in enumerate(got[k]):
            for call in Work.CALLS:
                assert _same(g[call], want[k][call]), (k, r, call)


# ---- host threads --------------------------------------------------------------------------------------------------------------
def _threads(fns):
    errors = []

    def run(fn):
        try:
            fn()
        except BaseException as e:             # reported by the main thread
            errors.append(e)
    ts = [threading.Thread(target=run, args=(fn,)) for fn in fns]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0]


def test_four_host_threads_with_their_own_streams():
    jp, pn = _jpegs(), _pngs()
    works = [Work(n, 20 + n, jp=jp, pn=pn) for n in (1, 7, 30, 256)]
    with _chain("affine") as (gm, x):
        _threads_with_int8(works, gm, x)


def _threads_with_int8(works, gm, x):
    with torch.no_grad():
        want_int8 = gm(x)
    calls = Work.CALLS + ("evaluators", "int8")
    want = []
    for w in works:
        d = w.all()
        d["evaluators"] = Work.read(w.evaluators())
        want.append(d)
    torch.cuda.synchronize()
    bad = []

    def worker(k):
        w, s = works[k], torch.cuda.Stream()
        for i in range(20):
            call = calls[(i + k) % len(calls)]
            with torch.cuda.stream(s), torch.no_grad():
                if call == "int8":
                    out = gm(x)
                elif call == "evaluators":
                    evs = w.evaluators()
                    s.synchronize()
                    out = Work.read(evs)
                else:
                    out = getattr(w, call)()
                bad_n = -(1000 * (k + 1) + i)       # refused on purpose: the message is this thread's, not another's
                with pytest.raises(_lib.DfqError, match=r"N and C must be positive, got %d and 5$" % bad_n):
                    _lib.check(_lib.load().dfq_cls_count(w.cls_logits.data_ptr(), None, w.cls_logits.data_ptr(), None,
                                                         bad_n, 5, _lib.stream_ptr()), "dfq_cls_count")
            s.synchronize()
            if not _same(out, want_int8 if call == "int8" else want[k][call]):
                bad.append((k, i, call))

    _threads([lambda k=k: worker(k) for k in range(4)])
    assert not bad, bad


def _calibrate(seed, device):
    """A BN fold, equalization and bias correction of a 3-layer chain through engine.Session (one read-back per
    equalization); returns the weights and biases."""
    from dfq_b200.engine import Session
    g = torch.Generator().manual_seed(seed)
    shapes = [(32, 3, 3, 3), (32, 1, 3, 3), (16, 32, 1, 1)]
    ws = [torch.randn(*s, generator=g) for s in shapes]
    bs = [torch.randn(s[0], generator=g) for s in shapes]
    bn = [dict(gamma=torch.rand(s[0], generator=g) + 0.5, beta=torch.randn(s[0], generator=g) * 0.3,
               mean=torch.randn(s[0], generator=g) * 0.1, var=torch.rand(s[0], generator=g) + 0.5) for s in shapes]
    sess = Session(device)
    ids = [sess.add_layer(w, b) for w, b in zip(ws, bs)]
    vec = [dict((k, sess.bind(v[k], False)) for k in ("gamma", "beta", "mean", "var")) for v in bn]
    for v, s in zip(vec, shapes):
        v["fake_w"] = sess.alloc(s[0]); v["fake_b"] = sess.alloc(s[0])
    folds = [dict(layer=li, bn_eps=1e-5, gamma_off=v["gamma"], beta_off=v["beta"], mean_off=v["mean"], var_off=v["var"],
                  fake_w_off=v["fake_w"], fake_b_off=v["fake_b"]) for li, v in zip(ids, vec)]
    cle = sess.plan_cle([(ids[0], ids[1], vec[0]["fake_w"], vec[0]["fake_b"]),
                         (ids[1], ids[2], vec[1]["fake_w"], vec[1]["fake_b"])])
    fold = sess.plan_bn_fold(folds, cle_plan=cle)
    bc = sess.plan_bias_correct([dict(layer=ids[i], signed=False, level=i, next_bn_b_off=vec[i]["fake_b"],
                                      terms=[dict(bn_w_off=vec[i - 1]["fake_w"], bn_b_off=vec[i - 1]["fake_b"],
                                                  n=shapes[i - 1][0], relu=True, op="set")]) for i in (1, 2)])
    sess.upload()
    sess.run_bn_fold(fold)
    res = sess.run_cle_plan(cle, cols_ready=fold["scanned"])
    sess.run_bias_correct_plan(bc, 8, col_hints=sess.cle_col_hints(cle, res))
    sess.download()
    return [w.clone() for w in ws] + [b.clone() for b in bs] + [res.n_sweeps]


def test_six_host_threads_calibrate_at_once():
    """Six threads calibrating at once, each on its own stream and each first holding its stream with a spin, so that up
    to six equalization read-backs can be waiting at once, more than the four mapped slots (the ones past the ring go
    through cudaMemcpyAsync).  Which path each read-back took is not observed here; every thread must get its own
    sequential result."""
    dev = torch.device("cuda", 0)
    want = [_calibrate(k, dev) for k in range(6)]
    bad = []

    def worker(k):
        s = torch.cuda.Stream()
        for r in range(5):
            with torch.cuda.stream(s):
                torch.cuda._sleep(SPIN // 20)
                got = _calibrate(k, dev)
            if not _same(got, want[k]):
                bad.append((k, r))

    _threads([lambda k=k: worker(k) for k in range(6)])
    assert not bad, bad


# ---- a second GPU --------------------------------------------------------------------------------------------------------------
def _subprocess_code(name, *args):
    """The program that runs test_gpu_context.<name>(*args) in a fresh interpreter."""
    here = os.path.dirname(os.path.abspath(__file__))
    return "import sys\nsys.path[:0] = [%r, %r]\nimport test_gpu_context\ntest_gpu_context.%s(*%r)\n" % (
        here, os.path.join(here, ".."), name, args)


def _subprocess(name, *args):
    """Run test_gpu_context.<name>(*args) in a fresh interpreter: cuda:0 is then really the first device used, and
    nothing it does is left in this process."""
    r = subprocess.run([sys.executable, "-c", _subprocess_code(name, *args)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def second_gpu():
    """Every entry point under torch.cuda.device(1) after cuda:0 was used, then on cuda:0 again: the results equal
    cuda:0's, with the outputs on cuda:1."""
    def on(dev, w):
        with torch.cuda.device(dev):
            d = w.all()
            evs = w.evaluators()
            torch.cuda.synchronize(dev)
            d["evaluators"] = Work.read(evs)
            d["calibrate"] = _calibrate(4, torch.device("cuda", dev))
        return d
    with torch.cuda.device(0):
        w0 = Work(7, 31)
        want = on(0, w0)
    with torch.cuda.device(1):
        w1 = Work(7, 31)
    got1 = on(1, w1)
    again0 = on(0, w0)
    for k in want:
        assert _same(got1[k], want[k]), k
        assert _same(again0[k], want[k]), k
    for v in _flat(got1):
        if isinstance(v, torch.Tensor) and v.is_cuda:
            assert v.device == torch.device("cuda", 1), v.device


def follow_inputs():
    """Tensors on cuda:1 while cuda:0 is current: the calls follow them, and an evaluator fed on cuda:1 keeps refusing a
    batch on cuda:0."""
    from dfq_b200 import detect
    with torch.cuda.device(1):
        w1 = Work(7, 41)
    w0 = Work(7, 41)
    torch.cuda.set_device(0)
    for call in ("hard", "soft", "predict", "plane_mean"):
        want = getattr(w0, call)()
        got = getattr(w1, call)()             # tensors on cuda:1, cuda:0 current
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        assert _same(got, want), call
        for v in _flat(got):
            if isinstance(v, torch.Tensor) and v.is_cuda:
                assert v.device == torch.device("cuda", 1), (call, v.device)
    evs = w1.evaluators()
    torch.cuda.synchronize(1)
    assert _same(Work.read(evs), Work.read(w0.evaluators()))
    c, s, d = evs
    for fn, msg in ((lambda: c.add_logits(w0.cls_logits, w0.cls_labels), "the evaluator counts on cuda:1"),
                    (lambda: s.add_logits(w0.seg_target, w0.seg_logits, align_corners=True),
                     "the evaluator counts on cuda:1"),
                    (lambda: d.add_batch(map_scenes.detections(w0.dets, "cuda:0"), detect.ground_truth(w0.gts, "cuda:0")),
                     "expected cuda:1")):
        with pytest.raises(_lib.DfqError, match=msg):
            fn()


SUBPROCESS_BODIES = ("side_stream_trace", "second_gpu", "follow_inputs")
TWO_GPUS = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs: device 1 after device 0")


@TWO_GPUS
def test_every_entry_point_on_device_1_after_device_0():
    _subprocess("second_gpu")


@TWO_GPUS
def test_inputs_on_device_1_are_followed_while_device_0_is_current():
    _subprocess("follow_inputs")
