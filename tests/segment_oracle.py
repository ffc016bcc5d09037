"""Oracle of dfq_seg_argmax (dfq_b200.segment)  --  TEST INFRASTRUCTURE.

The kernel restated in numpy: the resize is tests/int8_upsample_oracle.py's restatement of torch's CUDA bilinear resize
(fma32 and its taps; a plain copy when the size does not change), the argmax torch's CUDA max(dim) rule (the first NaN
wins, otherwise the larger value, equal values keep the lower index), and the counts the reference's Evaluator mask on the
label as forward_all hands it over, with float32 labels truncated toward zero for -1 < v < 256 and dropped otherwise.
"""
import numpy as np

import int8_upsample_oracle as U

f32 = np.float32


def resize(x, OH, OW, align_corners):
    """F.interpolate(x, (OH, OW), mode="bilinear", align_corners=...) of fp32 x [N, C, H, W] on the GPU."""
    return U.i8_upsample_bilinear(np.asarray(x, f32), OH, OW, bool(align_corners))


def argmax(y):
    """torch.max(y, 1)[1] of y [N, C, H, W] on the GPU, int64 [N, H, W]."""
    best, arg = y[:, 0].copy(), np.zeros(y[:, 0].shape, np.int64)
    for c in range(1, y.shape[1]):
        v = y[:, c]
        take = ~np.isnan(best) & (np.isnan(v) | (v > best))
        best, arg = np.where(take, v, best), np.where(take, c, arg)
    return arg


def predict(x, size=None, align_corners=False):
    x = np.asarray(x, f32)
    if size is None:
        size = x.shape[2:]
    return argmax(resize(x, size[0], size[1], align_corners))


def label_index(labels, C):
    """The label of each pixel as the Evaluator counts it, -1 where its mask drops the pixel: uint8 and int64 labels as
    given, float32 truncated toward zero for -1 < v < 256 and dropped otherwise (NaN included)."""
    labels = np.asarray(labels)
    if labels.dtype == np.float32:
        with np.errstate(invalid="ignore"):
            ok = (labels > -1) & (labels < 256)
        v = np.where(ok, np.trunc(np.where(ok, labels, 0)), -1).astype(np.int64)
    elif labels.dtype in (np.uint8, np.int64):
        v = labels.astype(np.int64)
    else:
        raise TypeError(labels.dtype)
    return np.where((v >= 0) & (v < C), v, -1)


def confusion(labels, pred, C):
    """uint64 [C, C]: count[label][pred] over the pixels the mask keeps."""
    gt = label_index(labels, C).reshape(-1)
    keep = gt >= 0
    return np.bincount(C * gt[keep] + np.asarray(pred).reshape(-1)[keep], minlength=C * C).reshape(C, C).astype(np.uint64)


def evaluate(labels, x, align_corners=False):
    """The counts of one batch: logits x [N, C, h, w] resized to the labels' [N, H, W]."""
    labels = np.asarray(labels)
    return confusion(labels, predict(x, labels.shape[1:], align_corners), np.asarray(x).shape[1])
