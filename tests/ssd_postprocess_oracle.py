"""The SSD post-processing of the reference's Predictor.predict restated in torch ops, from the contract of
dfq_b200.detect (DESIGN.md section 3.9), with a stable sort: candidates of equal score keep prior order.

The decode runs on the device of its inputs (the predictor decodes on the GPU); everything after it on the CPU, as there.
"""
import torch


def decode(locations, priors, center_variance, size_variance):
    """Corner-form boxes [N, P, 4]: each op separately rounded, in the reference's order."""
    if priors.dim() == 2:
        priors = priors.unsqueeze(0)
    wh_prior, c_prior = priors[..., 2:], priors[..., :2]
    centre = (locations[..., :2] * center_variance) * wh_prior + c_prior
    size = torch.exp(locations[..., 2:] * size_variance) * wh_prior
    half = size / 2
    return torch.cat([centre - half, centre + half], dim=-1)


def iou(rest, cur):
    """IoU of every box of rest [M, 4] with cur [1, 4]: NaN-propagating max / min / clamp, rest's area first."""
    lt = torch.maximum(rest[:, :2], cur[:, :2])
    rb = torch.minimum(rest[:, 2:], cur[:, 2:])
    side = (rb - lt).clamp(min=0.0)
    inter = side[:, 0] * side[:, 1]
    s_rest = (rest[:, 2:] - rest[:, :2]).clamp(min=0.0)
    s_cur = (cur[:, 2:] - cur[:, :2]).clamp(min=0.0)
    return inter / (s_rest[:, 0] * s_rest[:, 1] + s_cur[:, 0] * s_cur[:, 1] - inter + 1e-5)


def hard_nms(boxes, scores, iou_threshold, top_k=-1, candidate_size=200):
    """Indices into boxes / scores (one class's candidates, CPU) of the picks, in pick order."""
    order = torch.sort(scores, descending=True, stable=True).indices[:candidate_size]
    picks = []
    while order.numel():
        first = order[0]
        picks.append(int(first))
        if 0 < top_k == len(picks):
            break
        order = order[1:]
        order = order[iou(boxes[order], boxes[first].unsqueeze(0)) <= iou_threshold]
    return torch.tensor(picks, dtype=torch.int64)


def predict_one(scores, boxes, size=None, prob_threshold=0.01, iou_threshold=0.45, candidate_size=200, top_k=-1):
    """One image's (boxes, labels, probs) from its scores [P, C] and decoded boxes [P, 4], moved to the CPU first;
    size = (width, height) scales the boxes.  Three empty tensors when nothing is kept."""
    scores, boxes = scores.cpu(), boxes.cpu()
    rows, labels = [], []
    for c in range(1, scores.shape[1]):
        keep = scores[:, c] > prob_threshold
        probs = scores[keep, c]
        if probs.numel() == 0:
            continue
        cand = boxes[keep]
        picks = hard_nms(cand, probs, iou_threshold, top_k, candidate_size)
        rows.append(torch.cat([cand[picks], probs[picks].unsqueeze(1)], dim=1))
        labels += [c] * picks.numel()
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
