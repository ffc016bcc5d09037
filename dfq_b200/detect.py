"""SSD post-processing and evaluation for whole batches on the GPU: box decoding, the reference's per-class hard NMS and
its VOC average precision.

`postprocess` returns, for every image of a batch, what the reference's `Predictor.predict`
(modeling/detection/predictor.py) returns for that image alone - the decode of utils/detection/box_utils.py bit for bit
with torch's CUDA ops, then per foreground class the threshold, the sort, the `candidate_size` cut and `hard_nms` - with
one difference: candidates of equal score are ordered by prior index (the reference's CPU sort is not stable, so its
order among equal scores is arbitrary).  Soft NMS is not offered (DESIGN.md section 8).

    scores, boxes = model(images)          # the reference's is_test form: boxes = (locations, priors, cv, sv)
    det = detect.postprocess(scores, boxes, image_sizes=sizes)
    for boxes, labels, probs in det.per_image():
        ...

`Evaluator` computes from those detections, batch by batch and without a host synchronisation until the end, the
per-class average precision main_ssd.py computes (compute_average_precision_per_class, DESIGN.md section 3.11):

    ev = detect.Evaluator(num_classes=21)
    for images, sizes, annotations in loader:
        ev.add_batch(detect.postprocess(*net(images), image_sizes=sizes), detect.ground_truth(annotations, "cuda"))
    aps = ev.average_precision()           # classes 1 .. C-1
    print(ev.mean_average_precision())
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

__all__ = ["Detections", "Evaluator", "GroundTruth", "decode_boxes", "ground_truth", "postprocess"]

MAX_MAP_CLASSES = 4096
MAX_MAP_DETECTIONS = 2 ** 31 - 1
MATCH_IGNORED, MATCH_TP, MATCH_FP = _lib.MAP_IGNORED, _lib.MAP_TP, _lib.MAP_FP


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _tensor(t, name, shape):
    """t as given when it is a contiguous fp32 CUDA tensor of `shape` (None in shape: any size >= 1), else DfqError."""
    if not isinstance(t, torch.Tensor):
        raise _lib.DfqError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    if not t.is_cuda:
        raise _lib.DfqError("%s must be on the GPU (no CPU fallback), got %s" % (name, t.device))
    if t.dtype != torch.float32:
        raise _lib.DfqError("%s must be float32, got %s" % (name, t.dtype))
    if t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)) or min(t.shape) < 1:
        raise _lib.DfqError("%s must have shape %s, got %s"
                            % (name, tuple("*" if s is None else s for s in shape), tuple(t.shape)))
    if not t.is_contiguous():
        raise _lib.DfqError("%s must be contiguous" % name)
    return t


def _descriptor(locations, priors, center_variance, size_variance, C_=2, prob_threshold=0., iou_threshold=0.,
                candidate_size=1, top_k=-1):
    N, P, _ = _tensor(locations, "locations", (None, None, 4)).shape
    if isinstance(priors, torch.Tensor) and priors.dim() == 2:
        priors = priors.unsqueeze(0)
    _tensor(priors, "priors", (None, P, 4))
    if priors.shape[0] not in (1, N):
        raise _lib.DfqError("priors must have a batch of 1 or N = %d, got %d" % (N, priors.shape[0]))
    if priors.device != locations.device:
        raise _lib.DfqError("priors are on %s, locations on %s" % (priors.device, locations.device))
    d = np.zeros(1, _lib.SSD_NMS_DT)
    d[0] = (N, P, C_, priors.shape[0], center_variance, size_variance, prob_threshold, iou_threshold, candidate_size, top_k)
    return d, priors


def decode_boxes(locations, priors, center_variance, size_variance):
    """Corner-form boxes fp32 [N, P, 4] of SSD regression outputs: box_utils.center_form_to_corner_form(
    box_utils.convert_locations_to_boxes(locations, priors, center_variance, size_variance)) bit for bit with torch on CUDA.
    locations fp32 [N, P, 4]; priors fp32 in centre form, [P, 4], [1, P, 4] or [N, P, 4]; the variances Python floats."""
    d, priors = _descriptor(locations, priors, center_variance, size_variance)
    boxes = torch.empty_like(locations)
    _lib.check(_lib.load().dfq_ssd_decode(_ptr(locations), _ptr(priors), _ptr(boxes), _lib.table_ptr(d), _lib.stream_ptr()),
               "dfq_ssd_decode")
    return boxes


@dataclass
class Detections:
    """The detections of a batch, on the device: image n's are rows offsets[n] .. offsets[n + 1] of boxes fp32 [T, 4]
    (corner form, times the image's width and height when sizes were given), labels int64 [T] and probs fp32 [T], classes
    ascending and, within a class, in pick order.  offsets is int64 [N + 1]."""
    boxes: torch.Tensor
    labels: torch.Tensor
    probs: torch.Tensor
    offsets: torch.Tensor

    def per_image(self):
        """[(boxes, labels, probs)] on the CPU, one triple per image, each exactly what Predictor.predict returns for that
        image - three empty torch.tensor([]) for an image without detections."""
        offs = self.offsets.cpu().tolist()
        boxes, labels, probs = self.boxes.cpu(), self.labels.cpu(), self.probs.cpu()
        out = []
        for a, b in zip(offs[:-1], offs[1:]):
            if a == b:
                out.append((torch.tensor([]), torch.tensor([]), torch.tensor([])))
            else:
                out.append((boxes[a:b], labels[a:b], probs[a:b]))
        return out


def postprocess(scores, locations, priors=None, center_variance=None, size_variance=None, image_sizes=None,
                prob_threshold=0.01, iou_threshold=0.45, candidate_size=200, top_k=-1) -> Detections:
    """Predictor.predict's post-processing (hard NMS) for a batch, on the GPU, with one host synchronisation.

    scores: softmax output fp32 [N, P, C], class 0 the background.  locations: fp32 [N, P, 4], or the tuple
    (locations, priors, center_variance, size_variance) that an SSD in the reference's is_test form returns next to the
    scores, so `postprocess(*model(images))` works; otherwise pass priors ([P, 4], [1, P, 4] or [N, P, 4], centre form) and
    the variances.  image_sizes: [N, 2] (width, height) per image on the GPU, any real dtype; the boxes are multiplied by
    them as Predictor.predict does (left relative when None).

    Per class c = 1 .. C-1: the priors with score > prob_threshold, the best candidate_size of them by score (equal scores
    by prior index), box_utils.hard_nms at iou_threshold stopping at top_k picks when top_k > 0.  Thresholds are taken as
    fp32, as torch compares an fp32 tensor with a Python float.  Predictor.predict(image, top_k, prob_threshold) falls back
    to its filter_threshold when prob_threshold is None or 0; pass that value here.  candidate_size is 1 .. 1024.
    """
    if isinstance(locations, (tuple, list)):
        if priors is not None or center_variance is not None or size_variance is not None:
            raise _lib.DfqError("locations is the (locations, priors, center_variance, size_variance) tuple: pass the "
                                "priors and variances there only")
        locations, priors, center_variance, size_variance = locations
    if priors is None or center_variance is None or size_variance is None:
        raise _lib.DfqError("postprocess needs priors, center_variance and size_variance")
    if not isinstance(candidate_size, int) or candidate_size < 1:
        raise _lib.DfqError("candidate_size must be an int >= 1, got %r" % (candidate_size,))
    if not isinstance(top_k, int):
        raise _lib.DfqError("top_k must be an int, got %r" % (top_k,))
    N, P, C_ = _tensor(scores, "scores", (None, None, None)).shape
    if C_ < 2:
        raise _lib.DfqError("scores must have at least 2 classes (background and one), got C = %d" % C_)
    d, priors = _descriptor(locations, priors, center_variance, size_variance, C_, prob_threshold, iou_threshold,
                            candidate_size, top_k)
    if tuple(locations.shape[:2]) != (N, P):
        raise _lib.DfqError("locations must have shape (%d, %d, 4) to match scores, got %s" % (N, P, tuple(locations.shape)))
    if locations.device != scores.device:
        raise _lib.DfqError("locations are on %s, scores on %s" % (locations.device, scores.device))
    if image_sizes is not None:
        if not isinstance(image_sizes, torch.Tensor) or not image_sizes.is_cuda or image_sizes.dtype.is_complex or \
                image_sizes.dtype == torch.bool or tuple(image_sizes.shape) != (N, 2):
            raise _lib.DfqError("image_sizes must be a real tensor [%d, 2] of (width, height) on the GPU, got %s"
                                % (N, tuple(image_sizes.shape) if isinstance(image_sizes, torch.Tensor) else image_sizes))
        image_sizes = image_sizes.to(device=scores.device, dtype=torch.float32).contiguous()
    lib, st, dp = _lib.load(), _lib.stream_ptr(), _lib.table_ptr(d)
    dev = scores.device
    boxes = torch.empty_like(locations)
    _lib.check(lib.dfq_ssd_decode(_ptr(locations), _ptr(priors), _ptr(boxes), dp, st), "dfq_ssd_decode")
    S, K = N * (C_ - 1), candidate_size
    slot_boxes = torch.empty(S, K, 4, dtype=torch.float32, device=dev)
    slot_probs = torch.empty(S, K, dtype=torch.float32, device=dev)
    counts = torch.empty(S, dtype=torch.int32, device=dev)
    seg_offsets = torch.empty(S + 1, dtype=torch.int64, device=dev)
    _lib.check(lib.dfq_ssd_nms(_ptr(scores), _ptr(boxes), _ptr(slot_boxes), _ptr(slot_probs), _ptr(counts),
                               _ptr(seg_offsets), dp, st), "dfq_ssd_nms")
    T = int(seg_offsets[-1])
    out_boxes = torch.empty(T, 4, dtype=torch.float32, device=dev)
    labels = torch.empty(T, dtype=torch.int64, device=dev)
    probs = torch.empty(T, dtype=torch.float32, device=dev)
    if T:
        _lib.check(lib.dfq_ssd_compact(_ptr(slot_boxes), _ptr(slot_probs), _ptr(counts), _ptr(seg_offsets),
                                       _ptr(image_sizes), _ptr(out_boxes), _ptr(labels), _ptr(probs), dp, st),
                   "dfq_ssd_compact")
    return Detections(out_boxes, labels, probs, seg_offsets[::C_ - 1])


# ---- VOC average precision -------------------------------------------------------------------------------------------

@dataclass
class GroundTruth:
    """The ground truth of a batch of N images, on the device: image n's boxes are rows offsets[n] .. offsets[n + 1] of
    boxes fp32 [G, 4] (0-based corner form, pixels, as VOCDataset.get_annotation returns them), labels int64 [G] and
    difficult uint8 [G] (non-zero: difficult), in annotation order.  offsets is int64 [N + 1]."""
    boxes: torch.Tensor
    labels: torch.Tensor
    difficult: torch.Tensor
    offsets: torch.Tensor


def ground_truth(annotations, device) -> GroundTruth:
    """A GroundTruth from the (boxes, labels, is_difficult) triples VOCDataset.get_annotation returns, one per image (numpy
    arrays or CPU tensors; an image may have no boxes), packed on the host and moved to `device` in one copy.  Boxes must be
    float32, as the dataset yields them; labels and difficult flags may be of any integer or bool type."""
    boxes, labels, difficult, offsets = [], [], [], [0]
    for n, ann in enumerate(annotations):
        if not isinstance(ann, (tuple, list)) or len(ann) != 3:
            raise _lib.DfqError("annotation %d must be a (boxes, labels, is_difficult) triple, got %s" % (n, type(ann).__name__))
        b, l, d = (np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v) for v in ann)
        if b.dtype != np.float32:
            raise _lib.DfqError("annotation %d: boxes must be float32, got %s" % (n, b.dtype))
        if b.size == 0:
            b = b.reshape(0, 4)
        if b.ndim != 2 or b.shape[1] != 4:
            raise _lib.DfqError("annotation %d: boxes must have shape [k, 4], got %s" % (n, b.shape))
        k = b.shape[0]
        if l.shape != (k,) or d.shape != (k,):
            raise _lib.DfqError("annotation %d: %d boxes, but labels of shape %s and is_difficult of shape %s"
                                % (n, k, l.shape, d.shape))
        if not (np.issubdtype(l.dtype, np.integer) or k == 0):
            raise _lib.DfqError("annotation %d: labels must be integers, got %s" % (n, l.dtype))
        if not (np.issubdtype(d.dtype, np.integer) or d.dtype == np.bool_ or k == 0):
            raise _lib.DfqError("annotation %d: is_difficult must be integers or bools, got %s" % (n, d.dtype))
        boxes.append(b); labels.append(l.astype(np.int64)); difficult.append((d != 0).astype(np.uint8))
        offsets.append(offsets[-1] + k)
    N, G = len(offsets) - 1, offsets[-1]
    if N < 1:
        raise _lib.DfqError("ground_truth needs at least one image")
    # one byte buffer: boxes at 0 (16-byte aligned), labels at 16 G, offsets at 24 G, difficult at 24 G + 8 (N + 1)
    o_lab, o_off, o_dif = 16 * G, 24 * G, 24 * G + 8 * (N + 1)
    host = np.empty(o_dif + G, np.uint8)
    host[:o_lab].view(np.float32)[:] = np.concatenate(boxes).reshape(-1) if G else []
    host[o_lab:o_off].view(np.int64)[:] = np.concatenate(labels) if G else []
    host[o_off:o_dif].view(np.int64)[:] = offsets
    host[o_dif:] = np.concatenate(difficult) if G else []
    buf = torch.from_numpy(host).to(device)
    return GroundTruth(buf[:o_lab].view(torch.float32).view(G, 4), buf[o_lab:o_off].view(torch.int64),
                       buf[o_dif:], buf[o_off:o_dif].view(torch.int64))


def _field(t, name, dtype, shape, device):
    """t, contiguous, when it is a tensor of `dtype` and `shape` on `device`, else DfqError."""
    if not isinstance(t, torch.Tensor):
        raise _lib.DfqError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    if not t.is_cuda:
        raise _lib.DfqError("%s must be on the GPU (no CPU fallback), got %s" % (name, t.device))
    if t.dtype != dtype:
        raise _lib.DfqError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if tuple(t.shape) != shape:
        raise _lib.DfqError("%s must have shape %s, got %s" % (name, shape, tuple(t.shape)))
    if t.device != device:
        raise _lib.DfqError("%s is on %s, expected %s" % (name, t.device, device))
    return t.contiguous()


_ERRORS = [(_lib.MAP_ERR_DET_LABEL, "a detection label outside 1 .. num_classes - 1"),
           (_lib.MAP_ERR_GT_LABEL, "a ground-truth label outside 0 .. num_classes - 1"),
           (_lib.MAP_ERR_DET_OFFSETS, "detection offsets that do not run from 0 to the detection count without decreasing"),
           (_lib.MAP_ERR_GT_OFFSETS, "ground-truth offsets that do not run from 0 to the box count without decreasing")]


class Evaluator:
    """main_ssd.py's per-class VOC average precision (compute_average_precision_per_class, DESIGN.md section 3.11) over the
    batches added, computed on the GPU.  The defaults are main_ssd.py's.

    add_batch matches each batch's detections against its ground truth as soon as they exist and appends them to buffers on
    the device, without synchronising with the host.  average_precision() sorts everything added and reads back the
    compact per-class results once.  The one intended difference from the reference: detections of equal score are taken
    in the order they were added (images in order, then row order within an image), where the reference's sort is not
    stable.  The accumulators live on the device of the first batch."""

    def __init__(self, num_classes=21, iou_threshold=0.5, use_2007_metric=True):
        if not isinstance(num_classes, int) or isinstance(num_classes, bool) or not 2 <= num_classes <= MAX_MAP_CLASSES:
            raise _lib.DfqError("num_classes must be an int in 2 .. %d, got %r" % (MAX_MAP_CLASSES, num_classes))
        if isinstance(iou_threshold, bool) or not isinstance(iou_threshold, (int, float)):
            raise _lib.DfqError("iou_threshold must be a real number, got %r" % (iou_threshold,))
        if not isinstance(use_2007_metric, bool):
            raise _lib.DfqError("use_2007_metric must be a bool, got %r" % (use_2007_metric,))
        self.num_classes = num_classes
        self.iou_threshold = float(iou_threshold)
        self.use_2007_metric = use_2007_metric
        self.device = None
        self._keys = self._flags = self._gt_count = self._error = None
        self.reset()

    def reset(self):
        """Forget every batch added."""
        self._count = 0          # detections added
        self._gt_total = 0       # ground-truth boxes added
        if self._gt_count is not None:
            self._gt_count.zero_()
            self._error.zero_()

    @property
    def match_flags(self):
        """The verdict of every detection added, uint8 on the device in the order added: MATCH_TP, MATCH_FP or MATCH_IGNORED
        (the best box was difficult)."""
        if self._flags is None:
            return torch.empty(0, dtype=torch.uint8)
        return self._flags[:self._count]

    def add_batch(self, det, gt):
        """Match a batch: det the Detections of N images with boxes in pixels (postprocess(..., image_sizes=...)), gt the
        GroundTruth of the same N images.  Shapes, dtypes and devices are checked here; labels and offsets are checked on
        the device, and average_precision() raises if they were wrong.  Does not synchronise with the host."""
        if not isinstance(det, Detections):
            raise _lib.DfqError("det must be a detect.Detections, got %s" % type(det).__name__)
        if not isinstance(gt, GroundTruth):
            raise _lib.DfqError("gt must be a detect.GroundTruth, got %s" % type(gt).__name__)
        if not isinstance(det.offsets, torch.Tensor) or det.offsets.dim() != 1 or det.offsets.shape[0] < 2:
            raise _lib.DfqError("det.offsets must be a tensor [N + 1] with N >= 1")
        if not isinstance(det.probs, torch.Tensor) or det.probs.dim() != 1:
            raise _lib.DfqError("det.probs must be a tensor [T]")
        if not isinstance(gt.labels, torch.Tensor) or gt.labels.dim() != 1:
            raise _lib.DfqError("gt.labels must be a tensor [G]")
        N, T, G = det.offsets.shape[0] - 1, det.probs.shape[0], gt.labels.shape[0]
        dev = self.device if self.device is not None else det.probs.device
        if not det.probs.is_cuda:
            raise _lib.DfqError("det.probs must be on the GPU (no CPU fallback), got %s" % det.probs.device)
        d_boxes = _field(det.boxes, "det.boxes", torch.float32, (T, 4), dev)
        d_labels = _field(det.labels, "det.labels", torch.int64, (T,), dev)
        d_probs = _field(det.probs, "det.probs", torch.float32, (T,), dev)
        d_offs = _field(det.offsets, "det.offsets", torch.int64, (N + 1,), dev)
        g_boxes = _field(gt.boxes, "gt.boxes", torch.float32, (G, 4), dev)
        g_labels = _field(gt.labels, "gt.labels", torch.int64, (G,), dev)
        g_diff = _field(gt.difficult, "gt.difficult", torch.uint8, (G,), dev)
        g_offs = _field(gt.offsets, "gt.offsets", torch.int64, (N + 1,), dev)
        for t, name in ((d_boxes, "det.boxes"), (g_boxes, "gt.boxes")):
            if t.numel() and t.data_ptr() % 16:
                raise _lib.DfqError("%s must be 16-byte aligned" % name)
        if self._count + T > MAX_MAP_DETECTIONS:
            raise _lib.DfqError("%d detections added in all, above the limit %d" % (self._count + T, MAX_MAP_DETECTIONS))
        if self._gt_count is None:
            self.device = dev
            self._gt_count = torch.zeros(self.num_classes, dtype=torch.int64, device=dev)
            self._error = torch.zeros(1, dtype=torch.int32, device=dev)
        self._reserve(self._count + T)
        lib = _lib.load()
        _lib.check(lib.dfq_map_match(
            _ptr(d_boxes), _ptr(d_labels), _ptr(d_probs), _ptr(d_offs), T, _ptr(g_boxes), _ptr(g_labels), _ptr(g_diff),
            _ptr(g_offs), G, N, self.num_classes, self.iou_threshold,
            C.c_void_p(self._keys.data_ptr() + 8 * self._count), C.c_void_p(self._flags.data_ptr() + self._count),
            _ptr(self._gt_count), _ptr(self._error), _lib.stream_ptr()), "dfq_map_match")
        self._count += T
        self._gt_total += G

    def all_reduce(self, group=None) -> "Evaluator":
        """A new Evaluator holding the batches of every rank of `group` (the default group when None), on every rank; this
        one is left as it is.  Every rank must call it, with the same num_classes, also a rank that added no batch.

        The match records (sort key and verdict of every detection) are concatenated in rank order, so with the dataset
        split by dist.shard they stand in dataset order, the order one process would have added them in.  dfq_map_curve's
        sort is stable, so detections of equal score then come out in the one-process order and average_precision() is
        bit for bit the one-process value.  The ground-truth counts are summed and the device error words OR-ed, so a bad
        label or offset on any rank raises in average_precision() on every rank.  Two all-gathers: the per-rank sizes with
        the counts and error word (one host synchronisation), then the records, padded to the longest rank's.  A union of
        more than MAX_MAP_DETECTIONS detections is refused on every rank."""
        from . import dist as ddist
        Cn = self.num_classes
        dev = self.device if self.device is not None else ddist._idle_device()
        head = torch.zeros(3 + Cn, dtype=torch.int64, device=dev)       # count, gt_total, error, gt_count [C]
        head[0], head[1] = self._count, self._gt_total
        if self._gt_count is not None:
            head[2:3].copy_(self._error)
            head[3:].copy_(self._gt_count)
        heads = ddist._gather_rows(head, group)
        sizes = heads[:, :2].cpu().tolist()
        counts = [c for c, _ in sizes]
        total = sum(counts)
        if total > MAX_MAP_DETECTIONS:
            raise _lib.DfqError("detect.Evaluator.all_reduce: the ranks hold %d detections in all (%s), above "
                                "MAX_MAP_DETECTIONS = %d" % (total, " + ".join(map(str, counts)), MAX_MAP_DETECTIONS))
        out = Evaluator(Cn, self.iou_threshold, self.use_2007_metric)
        out.device = dev
        out._gt_count = heads[:, 3:].sum(0)
        error = heads[0, 2]
        for r in range(1, heads.shape[0]):
            error = error | heads[r, 2]
        out._error = error.to(torch.int32).reshape(1)
        out._gt_total = sum(g for _, g in sizes)
        cap = max(counts)
        if cap:
            # one uint8 row per rank: keys (8 bytes each) then verdicts, padded to the longest rank's count and to 8 bytes
            send = torch.zeros(8 * cap + (cap + 7) // 8 * 8, dtype=torch.uint8, device=dev)
            if self._count:
                send[:8 * self._count].copy_(self._keys[:self._count].view(torch.uint8))
                send[8 * cap:8 * cap + self._count].copy_(self._flags[:self._count])
            recs = ddist._gather_rows(send, group)
            out._reserve(total)
            o = 0
            for r, c in enumerate(counts):
                if c:
                    out._keys[o:o + c].copy_(recs[r, :8 * c].view(torch.int64))
                    out._flags[o:o + c].copy_(recs[r, 8 * cap:8 * cap + c])
                    o += c
            out._count = total
        return out

    def _reserve(self, n):
        """Room for n detections in the accumulation buffers, grown on the device (no synchronisation)."""
        cap = 0 if self._keys is None else self._keys.shape[0]
        if n <= cap:
            return
        cap = max(n, 2 * cap, 1 << 16)
        keys = torch.empty(cap, dtype=torch.int64, device=self.device)
        flags = torch.empty(cap, dtype=torch.uint8, device=self.device)
        if self._count:
            keys[:self._count].copy_(self._keys[:self._count])
            flags[:self._count].copy_(self._flags[:self._count])
        self._keys, self._flags = keys, flags

    def _curve(self):
        """(gt_count, counts, out) on the host: dfq_map_curve's results, read back in one copy."""
        Cn = self.num_classes
        if self._gt_count is None:
            return np.zeros(Cn, np.int64), np.zeros(Cn, np.int64), np.zeros(11 * (Cn - 1))
        n_out = 11 * (Cn - 1) if self.use_2007_metric else self._gt_total + Cn
        # error (padded to 8 bytes), gt_count [C], counts [C], out [n_out]
        buf = torch.zeros(8 + 16 * Cn + 8 * n_out, dtype=torch.uint8, device=self.device)
        counts = buf[8 + 8 * Cn:8 + 16 * Cn].view(torch.int64)
        out = buf[8 + 16 * Cn:].view(torch.float64)
        D = self._count
        _lib.check(_lib.load().dfq_map_curve(
            _ptr(self._keys) if D else None, _ptr(self._flags) if D else None, D, Cn, _ptr(self._gt_count),
            int(self.use_2007_metric), _ptr(out), n_out, _ptr(counts), _lib.stream_ptr()), "dfq_map_curve")
        buf[:4].copy_(self._error.view(torch.uint8))
        buf[8:8 + 8 * Cn].copy_(self._gt_count.view(torch.uint8))
        host = buf.cpu().numpy()
        error = int(host[:4].view(np.int32)[0])
        if error:
            raise _lib.DfqError("detect.Evaluator: the batches added had %s"
                                % "; ".join(msg for bit, msg in _ERRORS if error & bit))
        return (host[8:8 + 8 * Cn].view(np.int64), host[8 + 8 * Cn:8 + 16 * Cn].view(np.int64),
                host[8 + 16 * Cn:].view(np.float64))

    def _aps(self):
        """(aps as the reference's own list, with its Python float / numpy float64 types, gt_count)."""
        gt_count, counts, out = self._curve()
        aps = []
        for c in range(1, self.num_classes):
            if gt_count[c] == 0:
                aps.append(float("nan"))                 # the reference raises KeyError for this class
            elif self.use_2007_metric:
                ap = 0.
                for p in out[11 * (c - 1):11 * c].tolist():
                    ap = ap + p / 11.
                aps.append(np.float64(ap) if counts[c] else ap)   # a class without detections never meets numpy
            else:
                base = c - 1 + int(gt_count[1:c].sum())
                aps.append(out[base:base + counts[c]].copy().sum())
        return aps, gt_count

    def average_precision(self):
        """float64 numpy [num_classes - 1]: compute_average_precision_per_class for classes 1 .. num_classes - 1, bit for
        bit, NaN included.  A class with no non-difficult ground truth, for which the reference raises KeyError, is NaN.
        Raises DfqError when a batch added had labels or offsets out of range."""
        return np.array(self._aps()[0], dtype=np.float64)

    def mean_average_precision(self):
        """sum(aps) / len(aps) as main_ssd.py prints it.  DfqError when a class has no non-difficult ground truth."""
        aps, gt_count = self._aps()
        missing = [c for c in range(1, self.num_classes) if gt_count[c] == 0]
        if missing:
            raise _lib.DfqError("class %d has no non-difficult ground truth (main_ssd.py raises KeyError for it)%s"
                                % (missing[0], "" if len(missing) == 1 else "; so do %d more" % (len(missing) - 1)))
        return sum(aps) / len(aps)
