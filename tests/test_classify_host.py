"""dfq_b200.classify on the CPU through the oracle-backed twin of tests/fakelib_classify.py: the argmax rule of DESIGN.md
section 4 restated in numpy, the host path (types, shapes, labels on the logits' device or the CPU), accuracy()'s value
and type against main_cls.py inference_all's own expression, reset, and every refusal by name."""
import numpy as np
import pytest
import torch

import fakelib_classify
from dfq_b200 import _lib


def _logits(N, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C, generator=g)
    if C >= 3:
        x[::3, 1] = x[::3, 0]                       # ties
        x[1::5, :] = 0.0
        x[1::5, C - 1] = -0.0                       # -0.0 against +0.0
        x[2::7, C // 2] = float("nan")
        x[3::7, 0] = float("inf")
    return x


def test_argmax_rule():
    nan, inf = float("nan"), float("inf")
    rows = [[1., 3., 3.], [nan, 5., nan], [2., nan, nan], [-0., 0., -0.], [0., -0., 0.], [-inf, -inf, -inf],
            [1.4e-45, 3e-45, 3e-45], [inf, nan, inf], [nan, nan, nan], [-1., -2., inf]]
    assert fakelib_classify.argmax_rows(np.array(rows, np.float32)).tolist() == [1, 0, 1, 0, 0, 0, 1, 1, 0, 2]


def test_host_path_and_accuracy(monkeypatch):
    fake = fakelib_classify.install(monkeypatch)
    from dfq_b200 import classify
    ev = classify.Evaluator(31)
    num_correct, num_total = 0, 0
    for n, N in enumerate((1, 7, 256)):
        x = _logits(N, 31, n)
        y = torch.from_numpy(np.random.default_rng(n).integers(-2, 33, N))      # some labels out of range
        y[::2] = torch.max(x, 1)[1][::2]
        ev.add_logits(x, y)
        pred = torch.max(x, 1)[1].numpy()                 # main_cls.py inference_all, line for line
        num_correct += np.sum(pred == y.numpy())
        num_total += x.shape[0]
        p = classify.predict(x)
        assert p.dtype == torch.int64 and torch.equal(p, torch.from_numpy(fakelib_classify.argmax_rows(x.numpy())))
        assert torch.equal(ev.predict(x), p)
    assert type(ev.num_correct) is np.int64 and ev.num_correct == num_correct
    assert type(ev.num_total) is int and ev.num_total == num_total == 264
    acc = ev.accuracy()
    want = num_correct / num_total
    assert type(acc) is type(want) is np.float64 and acc == want
    assert fake.calls.count("dfq_cls_count") == 9 and not fake.refusals
    ev.reset()
    assert ev.num_correct == 0 and ev.num_total == 0


def test_labels_from_another_device_go_up_pinned(monkeypatch):
    fakelib_classify.install(monkeypatch)
    from dfq_b200 import classify
    moved = []
    real_to = torch.Tensor.to

    def to(self, *a, **k):
        moved.append(k.get("non_blocking"))
        return real_to(self, "cpu")

    class Dev:                  # logits that report a device other than the labels'
        type = "cuda"

        def __eq__(self, other):
            return isinstance(other, Dev)

        def __ne__(self, other):
            return not self == other
    x, y = _logits(5, 4, 0), torch.tensor([0, 1, 2, 3, 9])
    monkeypatch.setattr(torch.Tensor, "to", to)
    monkeypatch.setattr(torch.Tensor, "device", property(lambda self: Dev() if self.dtype == torch.float32 else
                                                         torch.device("cpu")))
    monkeypatch.setattr(torch, "zeros", lambda *a, device=None, **k: torch.empty(*a, **k).zero_())
    ev = classify.Evaluator(4)
    ev.add_logits(x, y)
    assert moved == [True]
    assert ev.num_correct == int((torch.max(x, 1)[1] == y).sum())


def test_zero_batches_and_one_class(monkeypatch):
    fakelib_classify.install(monkeypatch)
    from dfq_b200 import classify
    ev = classify.Evaluator(1)
    with pytest.raises(_lib.DfqError, match="no batch was added"):
        ev.accuracy()
    assert ev.num_correct == 0 and type(ev.num_correct) is np.int64
    ev.add_logits(torch.tensor([[float("nan")], [-1.0], [2.0]]), torch.tensor([0, 1, 0]))
    assert ev.num_correct == 2 and ev.accuracy() == np.float64(2) / 3


def test_refusals(monkeypatch):
    fakelib_classify.install(monkeypatch)
    from dfq_b200 import classify
    for bad in (0, -1, True, 2.0, "10", 2 ** 31):
        with pytest.raises(_lib.DfqError, match="num_classes must be an int"):
            classify.Evaluator(bad)
    ev = classify.Evaluator(4)
    x, y = _logits(3, 4, 1), torch.tensor([0, 1, 2])
    cases = [((x.numpy(), y), "logits must be a torch.Tensor"), ((x.double(), y), "logits must be float32"),
             ((x[0], y), r"logits must have shape \[N, C\]"), ((x[:0], y[:0]), r"logits must have shape \[N, C\]"),
             ((torch.randn(3, 8)[:, ::2], y), "logits must be contiguous"),
             ((torch.randn(3, 5), y), "logits have 5 classes, the evaluator counts 4"),
             ((x, [0, 1, 2]), "labels must be a torch.Tensor"), ((x, y.int()), "labels must be int64"),
             ((x, y[:2]), r"labels must have shape \[3\]"), ((x, y.view(3, 1)), r"labels must have shape \[3\]"),
             ((x, torch.arange(6)[::2]), "labels must be contiguous"),
             ((x, y.to("meta")), "labels are on meta")]
    for args, msg in cases:
        with pytest.raises(_lib.DfqError, match=msg):
            ev.add_logits(*args)
    assert ev.num_total == 0 and ev._correct is None
    for bad, msg in ((x.numpy(), "logits must be a torch.Tensor"), (x.half(), "logits must be float32"),
                     (x.view(1, 3, 4), r"shape \[N, C\]")):
        with pytest.raises(_lib.DfqError, match=msg):
            classify.predict(bad)


def test_library_refusals(monkeypatch):
    fake = fakelib_classify.install(monkeypatch)
    lib = fake
    x = torch.zeros(4, 3)
    p = torch.zeros(4, dtype=torch.int64)
    c = torch.zeros(1, dtype=torch.int64)
    y = torch.zeros(4, dtype=torch.int64)
    X, P, Cp, Y = (t.data_ptr() for t in (x, p, c, y))
    for args, reason in [((X, Y, P, Cp, 0, 3), "positive"), ((X, Y, P, Cp, 4, 0), "positive"),
                         ((0, Y, P, Cp, 4, 3), "logits is NULL"), ((X, Y, P, 0, 4, 3), "both be given"),
                         ((X, 0, 0, 0, 4, 3), "neither"), ((X + 2, Y, P, Cp, 4, 3), "misaligned"),
                         ((X, Y, X, Cp, 4, 3), "overlap"), ((X, Y, P, P + 8, 4, 3), "overlap"),
                         ((X, Y, P, Cp, 2 ** 40, 2 ** 21), "2^60")]:
        fake.refusals.clear()
        assert lib.dfq_cls_count(*args, None) != 0
        assert reason in fake.refusals[0][2], (args, fake.refusals)
    assert lib.dfq_cls_count(X, Y, P, Cp, 4, 3, None) == 0 and int(c) == 4 and p.tolist() == [0] * 4
