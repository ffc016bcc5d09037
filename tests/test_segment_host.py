"""dfq_b200.segment on the CPU: the oracle of tests/segment_oracle.py against the reference's forward_all / Evaluator (the
fixture tests/golden/ref_seg_eval.npz, and live where the reference checkout is present), the Evaluator's metrics, the
host wrappers through the oracle-backed twin of tests/fakelib_segment.py with every refusal, and split_upsample on every
graph form it takes."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F

import fakelib_segment
import segment_oracle as SO
from dfq_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_seg_eval.npz")
REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")
MATRICES = ("matrix_0", "matrix_1", "matrix_2", "matrix_empty")


def _metrics(ev):
    return np.array([ev.Pixel_Accuracy(), ev.Pixel_Accuracy_Class(), ev.Mean_Intersection_over_Union(),
                     ev.Frequency_Weighted_Intersection_over_Union()])


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


def _with_counts(m):
    from dfq_b200 import segment
    ev = segment.Evaluator(m.shape[0])
    ev.counts = torch.from_numpy(m.astype(np.int64))
    return ev


# ---- the oracle and the metrics against the reference ----------------------------------------------------------------------
def test_oracle_matches_the_reference_fixture():
    z = np.load(GOLD)
    total = np.zeros((21, 21), np.uint64)
    for b in range(3):
        pred = SO.predict(z["logits_%d" % b])
        assert np.array_equal(pred.astype(np.uint8), z["pred_%d" % b]), b
        total += SO.confusion(z["labels_%d" % b], pred, 21)
        assert np.array_equal(total.astype(np.float64), z["matrix_%d" % b]), b
    assert np.array_equal(SO.confusion(z["labels_2"], SO.predict(z["logits_2"]), 21), z["matrix_empty"])
    # what the fixture covers: tied maxima, fractional and negative float labels, a class absent from a batch
    x = z["logits_0"]
    assert ((x == x.max(1, keepdims=True)).sum(1) > 1).any()
    lab = z["labels_0"]
    assert (lab != np.trunc(lab)).any() and (lab < 0).any() and (lab == 255).any()
    assert not (z["labels_1"].astype(np.uint8) == 7).any() and (z["labels_2"] == 255).all()


@pytest.mark.parametrize("key", MATRICES)
def test_metrics_equal_the_fixture_bit_for_bit(key):
    z = np.load(GOLD)
    got = _metrics(_with_counts(z[key]))
    want = z["metrics" + key[len("matrix"):]]
    assert _same_bits(got, want), (got, want)
    if key == "matrix_empty":
        assert np.isnan(got[:3]).all() and got[3] == 0


def _reference_evaluator():
    sys.path.insert(0, REF)
    try:
        from utils.metrics import Evaluator
    finally:
        sys.path.remove(REF)
    return Evaluator


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "utils", "metrics.py")), reason="reference checkout not present")
@pytest.mark.parametrize("seed", [21, 22, 23])
def test_oracle_and_metrics_match_the_evaluator_live(seed):
    g = torch.Generator().manual_seed(seed)
    C = (2, 21, 150)[seed - 21]
    ref = _reference_evaluator()(C)
    total = np.zeros((C, C), np.uint64)
    for n, h, w in ((2, 17, 23), (1, 31, 9)):
        x = torch.randn(n, C, h, w, generator=g)
        x[:, 1:] = torch.round(x[:, 1:])
        labels = torch.randint(-3, C + 3, (n, h, w), generator=g).float() + torch.rand(n, h, w, generator=g) * 0.99
        labels[0, 0] = 255.
        pred = SO.predict(x.numpy())
        ref.add_batch(labels.numpy().astype(np.uint8), pred.astype(np.uint8))
        assert np.array_equal(torch.max(x, 1)[1].numpy(), pred)
        total += SO.confusion(labels.numpy(), pred, C)
        assert np.array_equal(total.astype(np.float64), ref.confusion_matrix)
    with np.errstate(all="ignore"):
        want = _metrics(ref)
    assert _same_bits(_metrics(_with_counts(total)), want)
    # a matrix with empty rows and columns (NaN per-class values)
    m = np.zeros((C, C))
    m[0, 0], m[0, 1 % C] = 5, 3
    ref.confusion_matrix = m
    with np.errstate(all="ignore"):
        assert _same_bits(_metrics(_with_counts(m)), _metrics(ref))


def test_float_labels_truncate_toward_zero_and_drop_the_rest():
    lab = np.array([-1.0, -0.5, -0.0, 0.99, 2.5, 254.9, 255.0, 255.99, 256.0, 300.0, np.nan, np.inf, -np.inf, 20.999],
                   np.float32)
    assert SO.label_index(lab, 21).tolist() == [-1, 0, 0, 0, 2, -1, -1, -1, -1, -1, -1, -1, -1, 20]
    assert SO.label_index(np.array([-1, 0, 20, 21, 255, -256], np.int64), 21).tolist() == [-1, 0, 20, -1, -1, -1]
    assert SO.label_index(np.array([0, 20, 21, 255], np.uint8), 21).tolist() == [0, 20, -1, -1]


def test_argmax_rule():
    nan, inf = np.nan, np.inf
    y = np.array([[1., 1.], [-0., 0.], [0., -0.], [nan, 5.], [2., nan], [nan, nan], [-inf, -inf], [inf, inf],
                  [1., 2.]], np.float32).T.reshape(1, 2, 1, 9)
    assert SO.argmax(y).reshape(-1).tolist() == [0, 0, 0, 0, 1, 0, 0, 0, 1]


# ---- the wrappers through the twin ------------------------------------------------------------------------------------------
def test_evaluator_through_the_twin_matches_the_fixture(monkeypatch):
    from dfq_b200 import segment
    fake = fakelib_segment.install(monkeypatch)
    z = np.load(GOLD)
    ev = segment.Evaluator(21)
    for b in range(3):
        ev.add_logits(torch.from_numpy(z["labels_%d" % b]), torch.from_numpy(z["logits_%d" % b]))
        m = ev.confusion_matrix
        assert m.dtype == np.float64 and np.array_equal(m, z["matrix_%d" % b]), b
        assert _same_bits(_metrics(ev), z["metrics_%d" % b]), b
    assert fake.calls == ["dfq_seg_argmax"] * 3
    ev.reset()
    assert not ev.confusion_matrix.any()
    ev.add_logits(torch.from_numpy(z["labels_2"]), torch.from_numpy(z["logits_2"]))
    assert _same_bits(_metrics(ev), z["metrics_empty"])


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int64, torch.float32])
@pytest.mark.parametrize("ac", [False, True])
def test_add_logits_resizes_to_the_labels(monkeypatch, dtype, ac):
    from dfq_b200 import segment
    fakelib_segment.install(monkeypatch)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 6, 7, generator=g)
    labels = torch.randint(-2, 8, (2, 13, 11), generator=g)
    labels = labels.clamp(min=0).to(dtype) if dtype == torch.uint8 else labels.to(dtype)
    ev = segment.Evaluator(5)
    ev.add_logits(labels, x, align_corners=ac)
    ev.add_logits(labels[:1].contiguous(), x[:1].contiguous(), align_corners=ac)
    want = SO.evaluate(labels.numpy(), x.numpy(), ac) + SO.evaluate(labels[:1].numpy(), x[:1].numpy(), ac)
    assert np.array_equal(ev.confusion_matrix, want.astype(np.float64))


def test_predict_through_the_twin(monkeypatch):
    from dfq_b200 import segment
    fake = fakelib_segment.install(monkeypatch)
    x = torch.randn(3, 4, 5, 6, generator=torch.Generator().manual_seed(4))
    p = segment.predict(x)
    assert p.dtype == torch.int64 and p.shape == (3, 5, 6) and torch.equal(p, torch.max(x, 1)[1])
    assert torch.equal(segment.predict(x, (5, 6)), p)
    assert torch.equal(segment.predict(x, torch.Size([9, 4]), True), torch.from_numpy(SO.predict(x.numpy(), (9, 4), True)))
    assert fake.calls == ["dfq_seg_argmax"] * 3


def _good():
    g = torch.Generator().manual_seed(6)
    return torch.randint(0, 4, (2, 9, 10), generator=g).to(torch.uint8), torch.randn(2, 4, 3, 5, generator=g)


@pytest.mark.parametrize("case,match", [
    ("c_mismatch", "evaluator counts 4"), ("fp16", "logits must be float32"), ("logits_nc", "logits must be contiguous"),
    ("labels_nc", "labels must be contiguous"), ("labels_dtype", "labels must be uint8, int64 or float32"),
    ("labels_shape", "labels must have shape"), ("logits_shape", r"logits must have shape \[N, C, H, W\]"),
    ("no_ac", "align_corners must be True or False"), ("ac_int", "align_corners must be True or False"),
    ("cross_device", "labels are on meta"), ("not_tensor", "labels must be a torch.Tensor"),
])
def test_add_logits_refusals_touch_nothing(monkeypatch, case, match):
    from dfq_b200 import segment
    fake = fakelib_segment.install(monkeypatch)
    labels, x = _good()
    ev = segment.Evaluator(4)
    ev.add_logits(labels, x, align_corners=False)
    before, lab0, x0 = ev.counts.clone(), labels.clone(), x.clone()
    ac = False
    if case == "c_mismatch":
        x = torch.randn(2, 5, 3, 5)
    elif case == "fp16":
        x = x.half()
    elif case == "logits_nc":
        x = x.transpose(2, 3).contiguous().transpose(2, 3)
    elif case == "labels_nc":
        labels = labels.transpose(1, 2).contiguous().transpose(1, 2)
    elif case == "labels_dtype":
        labels = labels.int()
    elif case == "labels_shape":
        labels = labels[:1]
    elif case == "logits_shape":
        x = x[0]
    elif case == "no_ac":
        ac = None
    elif case == "ac_int":
        ac = 1
    elif case == "cross_device":
        labels = torch.empty(2, 9, 10, dtype=torch.uint8, device="meta")
    elif case == "not_tensor":
        labels = labels.numpy()
    with pytest.raises(_lib.DfqError, match=match):
        ev.add_logits(labels, x, align_corners=ac)
    assert fake.calls == ["dfq_seg_argmax"] and torch.equal(ev.counts, before)
    lab_now = _good()[0]
    assert torch.equal(lab_now, lab0) and torch.equal(_good()[1], x0)


def test_evaluator_on_another_device_is_refused(monkeypatch):
    from dfq_b200 import segment
    fakelib_segment.install(monkeypatch)
    labels, x = _good()
    ev = segment.Evaluator(4)
    ev.counts = torch.zeros(4, 4, dtype=torch.int64, device="meta")
    with pytest.raises(_lib.DfqError, match="counts on meta"):
        ev.add_logits(labels, x, align_corners=False)


def test_too_many_classes_is_refused(monkeypatch):
    from dfq_b200 import segment
    fake = fakelib_segment.install(monkeypatch)
    for bad in (0, 161, 2.0, True):
        with pytest.raises(_lib.DfqError, match="num_class"):
            segment.Evaluator(bad)
    with pytest.raises(_lib.DfqError, match="dfq_seg_argmax"):
        segment.predict(torch.zeros(1, 161, 2, 2))
    assert fake.refusals == [("dfq_seg_argmax", fakelib_segment.E_UNSUPPORTED, "C is above the limit")]
    assert segment.predict(torch.zeros(1, 160, 2, 2)).shape == (1, 2, 2)


@pytest.mark.parametrize("size", [(3,), (0, 4), (2.0, 3), (True, 3), "ab", 7])
def test_predict_refuses_bad_sizes(monkeypatch, size):
    from dfq_b200 import segment
    fake = fakelib_segment.install(monkeypatch)
    with pytest.raises(_lib.DfqError, match="size must be"):
        segment.predict(torch.zeros(1, 2, 3, 4), size, True)
    assert fake.calls == []


def test_library_refusals_write_nothing(monkeypatch):
    """The twin's refusals, the library's: labels without counts, neither output, an unknown label type, a count that
    overlaps the logits; the outputs keep their contents."""
    import ctypes as C
    fake = fakelib_segment.install(monkeypatch)
    x = torch.randn(1, 3, 2, 2)
    labels = torch.zeros(1, 2, 2, dtype=torch.uint8)
    pred = torch.full((1, 2, 2), -7, dtype=torch.int64)
    count = torch.full((3, 3), 5, dtype=torch.int64)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731

    def call(lab, pr, cnt, **kw):
        d = np.zeros(1, _lib.SEG_ARGMAX_DT)
        f = dict(N=1, C=3, H=2, W=2, OH=2, OW=2, align_corners=0, label_type=0)
        f.update(kw)
        d[0] = tuple(f[k] for k in _lib.SEG_ARGMAX_DT.names)
        return fake.dfq_seg_argmax(p(x), p(lab), p(pr), p(cnt), _lib.table_ptr(d), None)
    assert call(labels, pred, None) == fakelib_segment.E_ARG
    assert call(None, None, None) == fakelib_segment.E_ARG
    assert call(labels, pred, count, label_type=3) == fakelib_segment.E_ARG
    assert call(labels, pred, count, align_corners=2) == fakelib_segment.E_ARG
    assert call(labels, pred, count, OH=0) == fakelib_segment.E_ARG
    over = torch.zeros(64, dtype=torch.int64)
    x = over[:6].view(torch.float32).view(1, 3, 2, 2)
    assert call(labels, pred, over[2:11]) == fakelib_segment.E_ARG
    assert (pred == -7).all() and (count == 5).all()
    assert len(fake.refusals) == 6


def test_cpu_tensors_are_refused():
    from dfq_b200 import segment
    with pytest.raises(_lib.DfqError, match="logits must be on the GPU"):
        segment.predict(torch.zeros(1, 2, 3, 3))
    with pytest.raises(_lib.DfqError, match="logits must be on the GPU"):
        segment.Evaluator(2).add_logits(torch.zeros(1, 3, 3, dtype=torch.uint8), torch.zeros(1, 2, 3, 3))


def test_descriptor_layout():
    assert _lib.SEG_ARGMAX_DT.itemsize == _lib.SEG_ARGMAX_SIZE == 32 and _lib.SEG_ARGMAX_DT.names[-1] == "label_type"
    assert _lib.SEG_ARGMAX_DT.fields["OH"][1] == 16 and _lib.SEG_ARGMAX_INDEX == len(_lib.EXPECTED_SIZES) == 19
    assert _lib.SIGNATURES["dfq_seg_argmax"][-1] is _lib.SIGNATURES["dfq_ssd_decode"][-1]


def test_descriptor_size_matches_the_library():
    """The compiled sizeof(DfqSegArgmax) (no GPU needed: the library only has to load)."""
    lib = _lib.load(build_if_missing=False)
    assert lib.dfq_struct_size(_lib.SEG_ARGMAX_INDEX) == _lib.SEG_ARGMAX_SIZE
    assert lib.dfq_struct_size(_lib.SEG_ARGMAX_INDEX + 1) == -1


# ---- split_upsample -------------------------------------------------------------------------------------------------------
class _Net(nn.Module):
    def __init__(self, how="interpolate", ac=True):
        super().__init__()
        self.conv = nn.Conv2d(3, 4, 3, stride=4, padding=1)
        self.up = nn.Upsample(size=(17, 19), mode="bilinear", align_corners=ac)
        self.how, self.ac = how, ac

    def forward(self, x):
        y = self.conv(x)
        if self.how == "upsample":
            return self.up(y)
        return F.interpolate(y, size=x.size()[2:], mode="bilinear", align_corners=self.ac)


def _check_split(gm, x, ac):
    from dfq_b200 import segment
    code = gm.code
    head, got_ac = segment.split_upsample(gm)
    assert got_ac is ac and gm.code == code
    with torch.no_grad():
        want = gm(x)
        y = head(x)
    assert torch.equal(F.interpolate(y, size=want.shape[2:], mode="bilinear", align_corners=ac), want)
    assert not [n for n in head.graph.nodes if n.op == "call_method" and n.target == "size"]
    assert not [n for n in head.graph.nodes if n.op == "call_function" and "interpolate" in str(n.target)]
    return head


@pytest.mark.parametrize("ac", [True, False])
def test_split_upsample_of_a_traced_fp32_model(ac):
    x = torch.randn(2, 3, 17, 19)
    _check_split(fx.symbolic_trace(_Net(ac=ac).eval()), x, ac)
    _check_split(fx.symbolic_trace(_Net("upsample", ac).eval()), x, ac)


def test_split_upsample_while_replace_op_is_active():
    """A graph traced before replace_op() names the raw F.interpolate, which is not F.interpolate while it is active."""
    from dfq_b200.utils import layer_transform as LT
    gm = fx.symbolic_trace(_Net().eval())
    prev = LT.module_tensor_op
    LT.replace_op()
    try:
        assert F.interpolate is not LT.raw_func_op["interpolate"]
        from dfq_b200 import segment
        head, ac = segment.split_upsample(gm)
        assert ac is True and head.graph.output_node().args[0].target == "conv"
    finally:
        LT.restore_op()
        LT.module_tensor_op = prev


def test_split_upsample_keeps_an_observer_and_takes_the_raw_op():
    """The form chain_affine and int8.load leave: an observer module (here a clamp standing in for the GPU-only
    QuantMeasure) in front of int8._raw_interpolate."""
    from dfq_b200 import int8
    gm = fx.symbolic_trace(_Net().eval())
    gm.add_module("obs", nn.Hardtanh(-0.5, 0.5))
    for n in list(gm.graph.nodes):
        if n.op == "call_function" and n.target is F.interpolate:
            with gm.graph.inserting_before(n):
                o = gm.graph.call_module("obs", (n.args[0],))
            n.args = (o,) + tuple(n.args[1:])
            n.target = int8._raw_interpolate
    gm.recompile()
    head = _check_split(gm, torch.randn(2, 3, 17, 19), True)
    assert head.graph.output_node().args[0].target == "obs"
    # the chaining rules do not take the raw op: their matcher is unchanged
    node = next(n for n in gm.graph.nodes if n.target is int8._raw_interpolate)
    assert int8._bilinear_upsample(node, dict(gm.named_modules()), raw=True) is None


class _Bad(nn.Module):
    def __init__(self, how):
        super().__init__()
        self.how = how
        self.conv = nn.Conv2d(3, 4, 1)

    def forward(self, x):
        y = self.conv(x)
        if self.how == "tuple":
            return y, y
        if self.how == "nearest":
            return F.interpolate(y, size=x.size()[2:], mode="nearest")
        if self.how == "scale":
            return F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=False)
        if self.how == "no_ac":
            return F.interpolate(y, size=x.size()[2:], mode="bilinear")
        return y


@pytest.mark.parametrize("how", ["tuple", "nearest", "scale", "no_ac", "conv"])
def test_split_upsample_refusals_name_the_output(how):
    from dfq_b200 import segment
    gm = fx.symbolic_trace(_Bad(how))
    code = gm.code
    with pytest.raises(_lib.DfqError, match="output"):
        segment.split_upsample(gm)
    assert gm.code == code
    with pytest.raises(_lib.DfqError, match="GraphModule"):
        segment.split_upsample(_Bad(how))
