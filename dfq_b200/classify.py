"""Classification evaluation on the GPU: main_cls.py's top-1 accuracy, counted on the device.

The reference evaluates a classifier in main_cls.py inference_all: per batch, torch.max(logits, 1)[1] goes to the host and
numpy counts it against the labels, one host synchronisation per batch.  Here one kernel (dfq_cls_count) takes each row's
argmax with torch's CUDA rule and adds the rows whose label equals it to a counter kept on the device; nothing goes to the
host until the accuracy is read.

    ev = classify.Evaluator(1000)
    for images, labels in loader:
        ev.add_logits(model(images.cuda()), labels)
    print(ev.accuracy())
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

__all__ = ["Evaluator", "predict"]

MAX_CLASSES = 2 ** 31 - 1


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _logits(x):
    if not isinstance(x, torch.Tensor):
        raise _lib.DfqError("logits must be a torch.Tensor, got %s" % type(x).__name__)
    if not x.is_cuda:
        raise _lib.DfqError("logits must be on the GPU (no CPU fallback), got %s" % x.device)
    if x.dtype != torch.float32:
        raise _lib.DfqError("logits must be float32, got %s" % x.dtype)
    if x.dim() != 2 or min(x.shape) < 1:
        raise _lib.DfqError("logits must have shape [N, C] with N, C >= 1, got %s" % (tuple(x.shape),))
    if not x.is_contiguous():
        raise _lib.DfqError("logits must be contiguous")
    return x


def _run(logits, labels, pred, correct):
    N, C_ = logits.shape
    _lib.check(_lib.load().dfq_cls_count(_ptr(logits), _ptr(labels), _ptr(pred), _ptr(correct), N, C_,
                                         _lib.stream_ptr()), "dfq_cls_count")


def predict(logits) -> torch.Tensor:
    """int64 [N]: torch.max(logits, 1)[1] bit for bit (DESIGN.md section 4 has the rule for ties, NaN and -0.0).  logits:
    contiguous fp32 [N, C] on the GPU.  Does not synchronise with the host."""
    logits = _logits(logits)
    pred = torch.empty(logits.shape[0], dtype=torch.int64, device=logits.device)
    _run(logits, None, pred, None)
    return pred


class Evaluator:
    """main_cls.py inference_all's count with the counting on the GPU.  add_logits counts a batch; num_correct, num_total
    and accuracy() are what the main's num_correct, num_total and acc hold after the same batches, with the same types.
    The correct count is kept as int64 on the device of the first batch and never leaves it between batches."""

    def __init__(self, num_classes):
        if not isinstance(num_classes, int) or isinstance(num_classes, bool) or not 1 <= num_classes <= MAX_CLASSES:
            raise _lib.DfqError("num_classes must be an int in 1 .. %d, got %r" % (MAX_CLASSES, num_classes))
        self.num_classes = num_classes
        self.device = None
        self._correct = None
        self.num_total = 0

    def add_logits(self, logits, labels):
        """Count one batch: the rows of logits fp32 [N, num_classes] (contiguous, on the GPU) whose argmax equals the label.
        labels: int64 [N], on the CPU (as ImageFolder yields them) or on the logits' GPU.  A label outside
        0 .. num_classes - 1 counts as wrong, as pred == label does.  CPU labels go up through page-locked memory in one
        asynchronous copy.  Does not synchronise with the host."""
        N, C_ = _logits(logits).shape
        if C_ != self.num_classes:
            raise _lib.DfqError("logits have %d classes, the evaluator counts %d" % (C_, self.num_classes))
        if not isinstance(labels, torch.Tensor):
            raise _lib.DfqError("labels must be a torch.Tensor, got %s" % type(labels).__name__)
        if labels.dtype != torch.int64:
            raise _lib.DfqError("labels must be int64, got %s" % labels.dtype)
        if tuple(labels.shape) != (N,):
            raise _lib.DfqError("labels must have shape [%d], got %s" % (N, tuple(labels.shape)))
        if labels.device != logits.device and labels.device.type != "cpu":
            raise _lib.DfqError("labels are on %s, logits on %s: labels must be on the CPU or the logits' GPU"
                                % (labels.device, logits.device))
        if self.device is not None and self.device != logits.device:
            raise _lib.DfqError("the evaluator counts on %s, logits are on %s" % (self.device, logits.device))
        if labels.device != logits.device:
            labels = labels.contiguous().pin_memory().to(logits.device, non_blocking=True)
        elif not labels.is_contiguous():
            raise _lib.DfqError("labels must be contiguous")
        if self._correct is None:
            self.device = logits.device
            self._correct = torch.zeros(1, dtype=torch.int64, device=logits.device)
        _run(logits, labels, None, self._correct)
        self.num_total += N

    def predict(self, logits) -> torch.Tensor:
        """classify.predict(logits)."""
        return predict(logits)

    def reset(self):
        """Forget every batch added."""
        if self._correct is not None:
            self._correct.zero_()
        self.num_total = 0

    @property
    def num_correct(self):
        """numpy int64: the rows counted correct, as the main's np.sum(pred == label) totals give it (one read-back)."""
        return np.int64(0 if self._correct is None else int(self._correct.cpu()[0]))

    def accuracy(self):
        """numpy float64: num_correct / num_total, the main's acc with its types (numpy int64 over a Python int).  DfqError
        when nothing was added, where the main divides 0 by 0."""
        if self.num_total == 0:
            raise _lib.DfqError("classify.Evaluator: no batch was added (the main's acc would divide 0 by 0)")
        return self.num_correct / self.num_total

    def all_reduce(self, group=None) -> "Evaluator":
        """A new Evaluator holding the counts of every rank of `group` (the default group when None), on every rank; this
        one is left as it is.  Every rank must call it, also a rank that added no batch.  The counts are sums of int64,
        so the result is what one process adding every rank's batches holds.  See dist.shard for the split."""
        from . import dist as ddist
        dev = self.device if self.device is not None else ddist._idle_device()
        send = torch.zeros(2, dtype=torch.int64, device=dev)
        if self._correct is not None:
            send[:1].copy_(self._correct)
        send[1] = self.num_total
        total = ddist._gather_rows(send, group).sum(0)
        out = Evaluator(self.num_classes)
        out.device, out._correct = dev, total[:1].clone()
        out.num_total = int(total[1])
        return out
