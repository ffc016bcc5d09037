"""tests/fakelib.py's stand-in for libdfq_sm90.so, extended by a host twin of dfq_cls_count: torch's CUDA max(dim) rule
restated in numpy, the counts in the library's layout, and the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.classify through it inside a test, so its argument checks, label
handling and buffer plumbing run without a GPU.
"""
import numpy as np
import torch

import fakelib
from dfq_b200 import _lib
from fakelib import _floats, _val
from fakelib_int8 import E_UNSUPPORTED, _array

E_ARG = -1


def argmax_rows(x):
    """int64 [N]: per row, the first NaN's index when the row has one, else the first index of the largest value (-0.0
    equal to +0.0) - torch.max(x, 1)[1] on CUDA (DESIGN.md section 4)."""
    x = np.asarray(x, np.float32)
    nan = np.isnan(x)
    first_nan = nan.argmax(1)
    best = np.where(nan, -np.inf, x).max(1, keepdims=True)
    first_max = (np.where(nan, False, x == best)).argmax(1)
    return np.where(nan.any(1), first_nan, first_max).astype(np.int64)


def _overlap(a, na, b, nb):
    return bool(a and b and a < b + nb and b < a + na)


class FakeClassifyLib(fakelib.FakeLib):
    def __init__(self, sqrt_fn=None):
        super().__init__(sqrt_fn)
        self.refusals = []          # (entry, code, reason) of every refused call

    def _refuse(self, code, reason):
        self.refusals.append(("dfq_cls_count", code, reason))
        return code

    def dfq_cls_count(self, x_p, lab_p, pred_p, cor_p, N, C, stream):
        self.calls.append("dfq_cls_count")
        x_p, lab_p, pred_p, cor_p = (int(_val(v) or 0) for v in (x_p, lab_p, pred_p, cor_p))
        if N < 1 or C < 1:
            return self._refuse(E_ARG, "N and C must be positive")
        if N * C >= 2 ** 60:
            return self._refuse(E_UNSUPPORTED, "2^60 logits or more")
        if not x_p:
            return self._refuse(E_ARG, "logits is NULL")
        if bool(lab_p) != bool(cor_p):
            return self._refuse(E_ARG, "labels and correct must both be given or both be NULL")
        if not (pred_p or cor_p):
            return self._refuse(E_ARG, "neither pred nor correct is given")
        if x_p % 4 or lab_p % 8 or pred_p % 8 or cor_p % 8:
            return self._refuse(E_ARG, "misaligned pointer")
        nx, nl, npr = 4 * N * C, 8 * N if lab_p else 0, 8 * N if pred_p else 0
        if _overlap(cor_p, 8, x_p, nx) or _overlap(cor_p, 8, lab_p, nl) or _overlap(cor_p, 8, pred_p, npr) or \
                _overlap(pred_p, npr, x_p, nx) or _overlap(pred_p, npr, lab_p, nl):
            return self._refuse(E_ARG, "correct and pred must not overlap the other buffers")
        pred = argmax_rows(_floats(x_p, N * C).reshape(N, C))
        if pred_p:
            _array(pred_p, N, np.int64)[...] = pred
        if cor_p:
            _array(cor_p, 1, np.int64)[...] += int((pred == _array(lab_p, N, np.int64)).sum())
        return 0


def install(monkeypatch):
    """fakelib.install() with the classification twin; every tensor counts as a CUDA tensor and pinning is a no-op while
    it is active."""
    fakelib.install(monkeypatch)
    fake = FakeClassifyLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return fake
