"""The soft NMS of the reference's Predictor(nms_method="soft").predict (box_utils.soft_nms) restated in torch ops, from
the contract of dfq_b200.detect (DESIGN.md section 3.9), on top of the hard-NMS oracle of tests/ssd_postprocess_oracle.py
(its decode and iou_of, and its predict_one for nms_method None or "hard").

The decode runs on the device of its inputs (the predictor decodes on the GPU); the soft NMS on `device`: the CPU, as the
reference runs it, or CUDA, where torch's exp is CUDA's expf.
"""
import torch

import ssd_postprocess_oracle as base
from ssd_postprocess_oracle import decode, hard_nms, iou  # noqa: F401  (re-exported for the soft tests)


def soft_nms(boxes, scores, score_threshold, sigma=0.5, top_k=-1):
    """box_utils.soft_nms of one class's candidates boxes [M, 4], scores [M] (in prior order): the picks' rows
    (box, decayed score) [K, 5] in pick order, on the device of the inputs.  The divisor is a 0-dim tensor on that device,
    so the division is a true division on the CPU and on CUDA alike (a Python float divides as a reciprocal multiply on
    CUDA)."""
    rows = torch.cat([boxes, scores.unsqueeze(1)], dim=1)
    div = torch.tensor(sigma, dtype=rows.dtype, device=rows.device)
    picked = []
    while rows.shape[0] > 0:
        j = int(torch.argmax(rows[:, 4]))
        cur = rows[j].clone()
        picked.append(cur)
        if 0 < top_k == len(picked) or rows.shape[0] == 1:
            break
        rows[j] = rows[-1]
        rows = rows[:-1]
        ious = iou(rows[:, :4], cur[:4].unsqueeze(0))
        rows[:, 4] = rows[:, 4] * torch.exp(-(ious * ious) / div)
        rows = rows[rows[:, 4] > score_threshold]
    return torch.stack(picked) if picked else rows.new_zeros(0, 5)


def predict_one(scores, boxes, size=None, prob_threshold=0.01, iou_threshold=0.45, candidate_size=200, top_k=-1,
                nms_method=None, sigma=0.5, device="cpu"):
    """One image's (boxes, labels, probs) from its scores [P, C] and decoded boxes [P, 4], moved to the CPU first;
    size = (width, height) scales the boxes.  Three empty tensors when nothing is kept.  nms_method None or "hard" is
    ssd_postprocess_oracle.predict_one; "soft" runs soft_nms on `device` and brings the rows back."""
    if nms_method != "soft":
        return base.predict_one(scores, boxes, size, prob_threshold, iou_threshold, candidate_size, top_k)
    scores, boxes = scores.cpu(), boxes.cpu()
    rows, labels = [], []
    for c in range(1, scores.shape[1]):
        keep = scores[:, c] > prob_threshold
        probs = scores[keep, c]
        if probs.numel() == 0:
            continue
        picked = soft_nms(boxes[keep].to(device), probs.to(device), prob_threshold, sigma, top_k).cpu()
        rows.append(picked)
        labels += [c] * picked.shape[0]
    if not rows:
        return torch.tensor([]), torch.tensor([]), torch.tensor([])
    rows = torch.cat(rows)
    if size is not None:
        w, h = float(size[0]), float(size[1])
        rows[:, 0] *= w
        rows[:, 1] *= h
        rows[:, 2] *= w
        rows[:, 3] *= h
    return rows[:, :4], torch.tensor(labels), rows[:, 4]


def predict(scores, locations, priors, center_variance, size_variance, image_sizes=None, **kw):
    """[predict_one(...)] for every image of a batch; the decode on the inputs' device."""
    boxes = decode(locations, priors, center_variance, size_variance)
    sizes = image_sizes.cpu().tolist() if image_sizes is not None else [None] * scores.shape[0]
    return [predict_one(scores[n], boxes[n], sizes[n], **kw) for n in range(scores.shape[0])]
