"""SSD post-processing for whole batches on the GPU: box decoding and the reference's per-class hard NMS.

`postprocess` returns, for every image of a batch, what the reference's `Predictor.predict`
(modeling/detection/predictor.py) returns for that image alone - the decode of utils/detection/box_utils.py bit for bit
with torch's CUDA ops, then per foreground class the threshold, the sort, the `candidate_size` cut and `hard_nms` - with
one difference: candidates of equal score are ordered by prior index (the reference's CPU sort is not stable, so its
order among equal scores is arbitrary).  Soft NMS is not offered (DESIGN.md section 8).

    scores, boxes = model(images)          # the reference's is_test form: boxes = (locations, priors, cv, sv)
    det = detect.postprocess(scores, boxes, image_sizes=sizes)
    for boxes, labels, probs in det.per_image():
        ...
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

__all__ = ["Detections", "decode_boxes", "postprocess"]


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
