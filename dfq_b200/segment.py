"""Segmentation evaluation on the GPU: predictions and the reference's confusion-matrix metrics, fused with the final
bilinear resize.

The reference evaluates a segmentation network in utils/segmentation/utils.py forward_all: the network's last op resizes
the logits to the input size (F.interpolate, bilinear), torch.max(logits, 1)[1] forms the label map, and the predictions
and labels go to the host as uint8, where utils/metrics.py Evaluator counts them with numpy.  Here one kernel does all of
that from the low-resolution logits: it resizes them through each output pixel's bilinear taps, bit for bit torch's CUDA
resize, takes the argmax with torch's CUDA rule, and adds the pixel to a confusion matrix kept on the device.  The
full-resolution logits never exist, and nothing goes to the host until a metric is read.

    head, ac = segment.split_upsample(chained)        # or int8.load(...), or fx.symbolic_trace(fp32_model)
    ev = segment.Evaluator(21)
    for images, labels in loader:
        ev.add_logits(labels.cuda(), head(images.cuda()), align_corners=ac)
    print(ev.Mean_Intersection_over_Union())
"""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np
import torch
import torch.fx as fx

from . import _lib

__all__ = ["Evaluator", "predict", "split_upsample"]

MAX_CLASSES = 160
_LABEL_TYPES = {torch.uint8: _lib.SEG_LABEL_U8, torch.int64: _lib.SEG_LABEL_I64, torch.float32: _lib.SEG_LABEL_F32}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _logits(x):
    if not isinstance(x, torch.Tensor):
        raise _lib.DfqError("logits must be a torch.Tensor, got %s" % type(x).__name__)
    if not x.is_cuda:
        raise _lib.DfqError("logits must be on the GPU (no CPU fallback), got %s" % x.device)
    if x.dtype != torch.float32:
        raise _lib.DfqError("logits must be float32, got %s" % x.dtype)
    if x.dim() != 4 or min(x.shape) < 1:
        raise _lib.DfqError("logits must have shape [N, C, H, W] with every size >= 1, got %s" % (tuple(x.shape),))
    if not x.is_contiguous():
        raise _lib.DfqError("logits must be contiguous")
    return x


def _size(size, H, W, align_corners):
    """(OH, OW, align_corners as 0 / 1) of a resize of [H, W] to `size` (None: no resize)."""
    if size is None:
        return H, W, 0
    if isinstance(size, torch.Size) or (isinstance(size, (tuple, list)) and len(size) == 2):
        size = tuple(size)
    if not (isinstance(size, tuple) and len(size) == 2 and
            all(isinstance(v, int) and not isinstance(v, bool) and v >= 1 for v in size)):
        raise _lib.DfqError("size must be None or a pair of positive ints, got %r" % (size,))
    if size != (H, W) and align_corners is not True and align_corners is not False:
        raise _lib.DfqError("align_corners must be True or False when the size changes (%d x %d -> %d x %d), got %r"
                            % (H, W, size[0], size[1], align_corners))
    return size[0], size[1], int(bool(align_corners))


def _run(logits, labels, pred, count, OH, OW, ac, label_type):
    N, C_, H, W = logits.shape
    d = np.zeros(1, _lib.SEG_ARGMAX_DT)
    d[0] = (N, C_, H, W, OH, OW, ac, label_type)
    _lib.check(_lib.load().dfq_seg_argmax(_ptr(logits), _ptr(labels), _ptr(pred), _ptr(count), _lib.table_ptr(d),
                                          _lib.stream_ptr()), "dfq_seg_argmax")


def predict(logits, size=None, align_corners=None) -> torch.Tensor:
    """int64 [N, OH, OW]: torch.max(F.interpolate(logits, size, mode="bilinear", align_corners=align_corners), 1)[1] bit for
    bit, or torch.max(logits, 1)[1] when size is None or logits' own [H, W].  logits: contiguous fp32 [N, C, H, W] on the
    GPU, C at most 160.  align_corners must be True or False when the size changes.  Does not synchronise with the host."""
    N, C_, H, W = _logits(logits).shape
    OH, OW, ac = _size(size, H, W, align_corners)
    pred = torch.empty(N, OH, OW, dtype=torch.int64, device=logits.device)
    _run(logits, None, pred, None, OH, OW, ac, _lib.SEG_LABEL_U8)
    return pred


class Evaluator:
    """utils/metrics.py Evaluator with the counting on the GPU.  add_logits counts a batch from the network's logits;
    confusion_matrix and the four metrics read the matrix back, and are what the reference's methods compute on the same
    matrix, NaN included.  The matrix is kept as int64 [num_class, num_class] on the device of the first batch and never
    leaves it between batches."""

    def __init__(self, num_class):
        if not isinstance(num_class, int) or isinstance(num_class, bool) or not 1 <= num_class <= MAX_CLASSES:
            raise _lib.DfqError("num_class must be an int in 1 .. %d, got %r" % (MAX_CLASSES, num_class))
        self.num_class = num_class
        self.counts = None

    def add_logits(self, labels, logits, align_corners=None):
        """Count one batch: logits fp32 [N, num_class, h, w] are resized bilinearly to the labels' [H, W] (not resized when
        they have that size already), and each pixel whose label passes the reference's mask 0 <= label < num_class adds
        one to [label, argmax].  labels [N, H, W]: uint8 or int64, counted as given; or float32, as the reference's dataset
        yields them, truncated toward zero as astype(np.uint8) does for -1 < v < 256, any other value (NaN included)
        ignored.  Both on the same GPU, contiguous.  Does not synchronise with the host."""
        N, C_, H, W = _logits(logits).shape
        if C_ != self.num_class:
            raise _lib.DfqError("logits have %d classes, the evaluator counts %d" % (C_, self.num_class))
        if not isinstance(labels, torch.Tensor):
            raise _lib.DfqError("labels must be a torch.Tensor, got %s" % type(labels).__name__)
        if labels.dtype not in _LABEL_TYPES:
            raise _lib.DfqError("labels must be uint8, int64 or float32, got %s" % labels.dtype)
        if labels.device != logits.device:
            raise _lib.DfqError("labels are on %s, logits on %s" % (labels.device, logits.device))
        if labels.dim() != 3 or labels.shape[0] != N or min(labels.shape) < 1:
            raise _lib.DfqError("labels must have shape [%d, H, W], got %s" % (N, tuple(labels.shape)))
        if not labels.is_contiguous():
            raise _lib.DfqError("labels must be contiguous")
        if self.counts is not None and self.counts.device != logits.device:
            raise _lib.DfqError("the evaluator counts on %s, logits are on %s" % (self.counts.device, logits.device))
        OH, OW, ac = _size(tuple(labels.shape[1:]), H, W, align_corners)
        if self.counts is None:
            self.counts = torch.zeros(C_, C_, dtype=torch.int64, device=logits.device)
        _run(logits, labels, None, self.counts, OH, OW, ac, _LABEL_TYPES[labels.dtype])

    def reset(self):
        """Clear the counts."""
        if self.counts is not None:
            self.counts.zero_()

    def all_reduce(self, group=None) -> "Evaluator":
        """A new Evaluator whose matrix is the sum of every rank's in `group` (the default group when None), on every rank;
        this one is left as it is.  Every rank must call it, also a rank that added no batch.  The matrix is int64, so the
        sum is exact: the result is what one process adding every rank's batches holds.  See dist.shard for the split."""
        from . import dist as ddist
        dev = self.counts.device if self.counts is not None else ddist._idle_device()
        send = self.counts if self.counts is not None else \
            torch.zeros(self.num_class, self.num_class, dtype=torch.int64, device=dev)
        out = Evaluator(self.num_class)
        out.counts = ddist._gather_rows(send.reshape(-1), group).sum(0).view(self.num_class, self.num_class)
        return out

    @property
    def confusion_matrix(self):
        """float64 numpy [num_class, num_class], rows the labels and columns the predictions, as the reference keeps it."""
        if self.counts is None:
            return np.zeros((self.num_class,) * 2)
        return self.counts.cpu().numpy().astype(np.float64)

    # The metrics: the reference's formulas on the float64 matrix, in its operation order.
    def Pixel_Accuracy(self):
        m = self.confusion_matrix
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.diag(m).sum() / m.sum()

    def Pixel_Accuracy_Class(self):
        m = self.confusion_matrix
        with np.errstate(divide="ignore", invalid="ignore"):
            return _nanmean(np.diag(m) / m.sum(axis=1))

    @staticmethod
    def _iou(m):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.diag(m) / (np.sum(m, axis=1) + np.sum(m, axis=0) - np.diag(m))

    def Mean_Intersection_over_Union(self):
        return _nanmean(self._iou(self.confusion_matrix))

    def Frequency_Weighted_Intersection_over_Union(self):
        m = self.confusion_matrix
        with np.errstate(divide="ignore", invalid="ignore"):
            freq = np.sum(m, axis=1) / np.sum(m)
            iu = self._iou(m)
            seen = freq > 0
            return (freq[seen] * iu[seen]).sum()


def _nanmean(v):
    """np.nanmean, quiet about an all-NaN input (NaN, as the reference gets with a warning)."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return np.nanmean(v)


def split_upsample(gm):
    """(head, align_corners) of a GraphModule whose single output is a bilinear resize of one tensor: head is a new
    GraphModule returning that resize's input, with everything upstream of it (an observer in front of the resize
    included), and align_corners is the resize's.  The size-computation nodes only the resize used are dropped; gm is not
    modified.  The resize's size is not returned: under the reference's evaluation it is the input size, which is the
    label size, and Evaluator.add_logits takes it from the labels.

    gm: what int8.chain_int8 / chain_affine return, what int8.load returns, or torch.fx.symbolic_trace of an fp32 model -
    a resize by F.interpolate (patched by replace_op() or not), by the raw op those leave in a graph, or by nn.Upsample,
    mode "bilinear", to a given size, align_corners True or False.  Anything else raises DfqError naming the output."""
    from .int8 import _bilinear_upsample
    if not isinstance(gm, fx.GraphModule):
        raise _lib.DfqError("split_upsample takes a torch.fx.GraphModule, got %s" % type(gm).__name__)
    out = next(n for n in gm.graph.nodes if n.op == "output")
    res = out.args[0]
    if not isinstance(res, fx.Node):
        raise _lib.DfqError("split_upsample: the output %s is not a single tensor (%s)" % (out.name, type(res).__name__))
    found = _bilinear_upsample(res, dict(gm.named_modules()), raw=True, wrapped=True)
    if found is None:
        raise _lib.DfqError("split_upsample: the output %s is %s, not a bilinear resize of one tensor to a given size "
                            "with align_corners True or False" % (out.name, res.format_node()))
    graph = fx.Graph()
    env = {}
    graph.graph_copy(gm.graph, env)
    graph.output(env[res.args[0]])
    head = fx.GraphModule(gm, graph, type(gm).__name__ + "Head")
    stack = [env[res]]
    while stack:
        n = stack.pop()
        if n.users or n.op in ("placeholder", "output") or n.is_impure():
            continue
        ins = n.all_input_nodes
        graph.erase_node(n)
        stack.extend(ins)
    graph.lint()
    head.recompile()
    return head, found[1]
