"""tests/fakelib.py's stand-in for libdfq_sm90.so, extended by a host twin of dfq_seg_argmax computed by
tests/segment_oracle.py, with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.segment through it inside a test, so its argument checks and buffer
plumbing run without a GPU.
"""
import numpy as np
import torch

import fakelib
import segment_oracle as SO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import E_UNSUPPORTED, _array

E_ARG = -1
MAX_CLASSES = 160
LABEL_DTYPES = {_lib.SEG_LABEL_U8: np.uint8, _lib.SEG_LABEL_I64: np.int64, _lib.SEG_LABEL_F32: np.float32}


def _overlap(a, na, b, nb):
    return bool(a and b and a < b + nb and b < a + na)


class FakeSegmentLib(fakelib.FakeLib):
    def __init__(self, sqrt_fn=None):
        super().__init__(sqrt_fn)
        self.refusals = []          # (entry, code, reason) of every refused call

    def _refuse(self, code, reason):
        self.refusals.append(("dfq_seg_argmax", code, reason))
        return code

    def dfq_seg_argmax(self, x_p, lab_p, pred_p, cnt_p, d_p, stream):
        self.calls.append("dfq_seg_argmax")
        if not _val(d_p):
            return self._refuse(E_ARG, "descriptor is NULL")
        d = _table(d_p, 1, _lib.SEG_ARGMAX_DT)[0]
        N, C, H, W, OH, OW, ac, lt = (int(d[k]) for k in _lib.SEG_ARGMAX_DT.names)
        x_p, lab_p, pred_p, cnt_p = (int(_val(v) or 0) for v in (x_p, lab_p, pred_p, cnt_p))
        if min(N, C, H, W, OH, OW) < 1:
            return self._refuse(E_ARG, "sizes must be positive")
        if ac not in (0, 1):
            return self._refuse(E_ARG, "align_corners must be 0 or 1")
        if lt not in LABEL_DTYPES:
            return self._refuse(E_ARG, "unknown label_type")
        if C > MAX_CLASSES:
            return self._refuse(E_UNSUPPORTED, "C is above the limit")
        if not x_p or bool(lab_p) != bool(cnt_p) or not (pred_p or cnt_p):
            return self._refuse(E_ARG, "missing buffer")
        ls = np.dtype(LABEL_DTYPES[lt]).itemsize
        if x_p % 4 or pred_p % 8 or cnt_p % 8 or lab_p % ls:
            return self._refuse(E_ARG, "misaligned pointer")
        px = N * OH * OW
        nx, nl, npr, nc = 4 * N * C * H * W, ls * px if lab_p else 0, 8 * px if pred_p else 0, 8 * C * C
        if _overlap(cnt_p, nc, x_p, nx) or _overlap(cnt_p, nc, lab_p, nl) or _overlap(cnt_p, nc, pred_p, npr) or \
                _overlap(pred_p, npr, x_p, nx) or _overlap(pred_p, npr, lab_p, nl):
            return self._refuse(E_ARG, "count and pred must not overlap the other buffers")
        x = _floats(x_p, N * C * H * W).reshape(N, C, H, W)
        pred = SO.predict(x, (OH, OW), ac)
        if pred_p:
            _array(pred_p, px, np.int64)[...] = pred.reshape(-1)
        if cnt_p:
            labels = _array(lab_p, px, LABEL_DTYPES[lt]).reshape(N, OH, OW)
            _array(cnt_p, C * C, np.uint64)[...] += SO.confusion(labels, pred, C).reshape(-1)
        return 0


def install(monkeypatch):
    """fakelib.install() with the segmentation twin; every tensor counts as a CUDA tensor while it is active."""
    fakelib.install(monkeypatch)
    fake = FakeSegmentLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return fake
