"""main_ssd.py's VOC average precision (group_annotation_by_class, compute_average_precision_per_class and
utils/detection/measurements.py) restated in torch / numpy from the contract of dfq_b200.detect.Evaluator (DESIGN.md
section 3.11), with the reference's execution structure - one Python step per detection - and a stable sort: detections
of equal score keep the order they were added in.

`broken` runs the computation with one rule of DESIGN.md section 3.11 deliberately changed (see BROKEN); the tests use it
to show that the committed fixture decides every rule.
"""
import numpy as np
import torch

# rule name -> what the broken variant does instead
BROKEN = {
    "plus_one": "matches the box as given, not fl32(fl32(b + 1) - 1)",
    "fp32_threshold": "compares the IoU with the threshold in fp32",
    "double_claim": "counts every detection on an unmatched-or-matched box as a true positive",
    "difficult_skip": "takes the best non-difficult box instead of ignoring a detection whose best box is difficult",
    "last_max": "takes the last of equal IoUs",
    "nan_skip": "ignores NaN IoUs in the max / argmax",
    "no_gt_ignored": "ignores a detection on an image without ground truth of its class",
    "nanmax_2007": "ignores NaN precision in the VOC2007 maxima",
    "empty_nan": "gives a class without detections AP NaN",
}


def iou_of(box, gt, eps=1e-5):
    """IoU of box [1, 4] with every row of gt [G, 4], fp32: NaN-propagating max / min / clamp, box's area first."""
    lt = torch.max(box[..., :2], gt[..., :2])
    rb = torch.min(box[..., 2:], gt[..., 2:])
    side = torch.clamp(rb - lt, min=0.0)
    overlap = side[..., 0] * side[..., 1]
    s0 = torch.clamp(box[..., 2:] - box[..., :2], min=0.0)
    s1 = torch.clamp(gt[..., 2:] - gt[..., :2], min=0.0)
    return overlap / (s0[..., 0] * s0[..., 1] + s1[..., 0] * s1[..., 1] - overlap + eps)


def group_by_class(gts):
    """gts: [(boxes fp32 [k, 4], labels [k], difficult [k])] per image.  (num_true {class: count of non-difficult boxes},
    boxes {class: {image: fp32 tensor [m, 4]}}, difficult {class: {image: [flags]}}), annotation order kept."""
    num_true, boxes, difficult = {}, {}, {}
    for n, (b, l, d) in enumerate(gts):
        b = torch.as_tensor(np.asarray(b, np.float32).reshape(-1, 4))
        for i in range(b.shape[0]):
            c = int(l[i])
            if not d[i]:
                num_true[c] = num_true.get(c, 0) + 1
            boxes.setdefault(c, {}).setdefault(n, []).append(b[i])
            difficult.setdefault(c, {}).setdefault(n, []).append(int(d[i]))
    boxes = {c: {n: torch.stack(v) for n, v in per.items()} for c, per in boxes.items()}
    return num_true, boxes, difficult


def class_detections(dets, c, text=False, plus_one=True):
    """(image, score, box fp32 [1, 4], insertion index) of every detection of class c, in insertion order.  dets:
    [(boxes, labels, probs)] per image as Detections.per_image() returns them.  The box is as main_ssd.py reads it back:
    fl32(fl32(b + 1) - 1) (b itself when plus_one is False); with text=True it really goes through the text line the main
    writes and parses."""
    out, base = [], 0
    for n, (b, l, p) in enumerate(dets):
        b, l, p = b.reshape(-1, 4).float(), l.reshape(-1), p.reshape(-1).float()
        for i in range(l.numel()):
            if int(l[i]) == c:
                row = torch.cat([p[i:i + 1], b[i] + 1.0]).numpy()
                if text:
                    t = ("%d " % n + " ".join(str(v) for v in row)).split(" ")
                    score, box = float(t[1]), torch.tensor([float(v) for v in t[2:]]).unsqueeze(0)
                else:
                    score, box = float(row[0]), torch.from_numpy(row[1:]).unsqueeze(0)
                box -= 1.0
                if not plus_one:
                    box = b[i:i + 1].clone()
                out.append((n, score, box, base + i))
        base += l.numel()
    return out


def match_class(records, num_true, gt_boxes, difficult, iou_threshold, broken=None):
    """(true_positive, false_positive, verdicts {insertion index: 0 ignored / 1 TP / 2 FP}) of one class."""
    scores = np.array([r[1] for r in records])
    order = np.argsort(-scores, kind="stable")
    tp, fp = np.zeros(len(records)), np.zeros(len(records))
    matched, verdict = set(), {}
    for k, j in enumerate(order):
        n, _, box, idx = records[j]
        verdict[idx] = 0
        if n not in gt_boxes:
            if broken != "no_gt_ignored":
                fp[k] = 1
                verdict[idx] = 2
            continue
        ious = iou_of(box, gt_boxes[n])
        if broken == "nan_skip":
            ious = torch.nan_to_num(ious, nan=-1.0)
        if broken == "difficult_skip":
            ious = torch.where(torch.tensor(difficult[n], dtype=torch.bool), torch.full_like(ious, -1.0), ious)
        max_iou = torch.max(ious).item()
        max_arg = torch.argmax(ious).item()
        if broken == "last_max":
            max_arg = int(torch.nonzero(ious == ious.max()).max()) if not np.isnan(max_iou) else max_arg
        above = np.float32(max_iou) > np.float32(iou_threshold) if broken == "fp32_threshold" else max_iou > iou_threshold
        if above:
            if difficult[n][max_arg] == 0:
                if (n, max_arg) not in matched or broken == "double_claim":
                    tp[k] = 1
                    matched.add((n, max_arg))
                    verdict[idx] = 1
                else:
                    fp[k] = 1
                    verdict[idx] = 2
        else:
            fp[k] = 1
            verdict[idx] = 2
    return tp, fp, verdict


def voc2007_ap(precision, recall, broken=None):
    ap = 0.
    for t in np.arange(0., 1.1, 0.1):
        sel = precision[recall >= t]
        p = 0 if sel.size == 0 else (np.nanmax(sel) if broken == "nanmax_2007" and not np.isnan(sel).all() else np.max(sel))
        ap = ap + p / 11.
    return ap


def area_ap(precision, recall):
    p = np.concatenate([[0.0], precision, [0.0]])
    p = np.maximum.accumulate(p[::-1])[::-1]                   # the running maximum from the end, NaN-propagating
    r = np.concatenate([[0.0], recall, [1.0]])
    cp = np.where(r[1:] != r[:-1])[0]
    return ((r[cp + 1] - r[cp]) * p[cp + 1]).sum()


def average_precision(dets, gts, num_classes, iou_threshold=0.5, use_2007_metric=True, text=False, broken=None):
    """(aps [classes 1 .. C-1] with the reference's types - NaN for a class without non-difficult ground truth, where the
    reference raises KeyError -, verdicts uint8 [D] in insertion order)."""
    if broken is not None and broken not in BROKEN:
        raise ValueError(broken)
    num_true, gt_boxes, difficult = group_by_class(gts)
    D = sum(int(l.numel()) for _, l, _ in dets)
    verdicts = np.full(D, 2, np.uint8)
    aps = []
    for c in range(1, num_classes):
        records = class_detections(dets, c, text, plus_one=broken != "plus_one")
        if c not in num_true:
            aps.append(float("nan"))
            tp, fp, v = match_class(records, 1, gt_boxes.get(c, {}), difficult.get(c, {}), iou_threshold, broken)
        else:
            tp, fp, v = match_class(records, num_true[c], gt_boxes[c], difficult[c], iou_threshold, broken)
            tp, fp = tp.cumsum(), fp.cumsum()
            with np.errstate(divide="ignore", invalid="ignore"):
                precision = tp / (tp + fp)
            recall = tp / num_true[c]
            if broken == "empty_nan" and not records:
                aps.append(float("nan"))
            elif use_2007_metric:
                aps.append(voc2007_ap(precision, recall, broken))
            else:
                aps.append(area_ap(precision, recall))
        for idx, f in v.items():
            verdicts[idx] = f
    return aps, verdicts


def mean_average_precision(aps):
    return sum(aps) / len(aps)
