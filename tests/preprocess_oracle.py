"""numpy restatement of the reference's evaluation transforms: the three resamplers (Pillow bilinear, Pillow nearest, OpenCV
INTER_LINEAR on uint8) and the three normalisations (torchvision, custom_transforms.Normalize, SubtractMeans + / std).

Test infrastructure only, never imported by dfq_b200.  Every coefficient is formed by a literal translation of the
library's C loop, one output coordinate at a time, so the product's vectorised tables are checked against an independent
statement of the same rules; the oracle itself is checked byte for byte against PIL and cv2 in test_preprocess_host.py.
"""
import math

import numpy as np

PIL_BITS = 22          # Pillow's PRECISION_BITS for 8-bit images
CV_BITS = 11           # OpenCV's INTER_RESIZE_COEF_BITS


# ---- Pillow bilinear (Resample.c precompute_coeffs, ImagingResampleHorizontal/Vertical_8bpc) ---------------------------
def pil_coeffs(insz, outsz):
    """[(xmin, [int weights])] per output coordinate."""
    scale = insz / outsz
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    out = []
    for xx in range(outsz):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > insz:
            xmax = insz
        xmax -= xmin
        w, ww = [], 0.0
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * ss)
            v = 1.0 - t if t < 1.0 else 0.0
            w.append(v)
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        out.append((xmin, [int(-0.5 + v * (1 << PIL_BITS)) if v < 0 else int(0.5 + v * (1 << PIL_BITS)) for v in w]))
    return out


def _pil_pass(a, taps, axis):
    a = np.moveaxis(a, axis, 0).astype(np.int64)
    rows = []
    for xmin, w in taps:
        s = np.full(a.shape[1:], 1 << (PIL_BITS - 1), np.int64)
        for k, v in enumerate(w):
            s += a[xmin + k] * v
        rows.append(np.clip(s >> PIL_BITS, 0, 255))
    return np.moveaxis(np.stack(rows), 0, axis).astype(np.uint8)


def pil_bilinear(img, ow, oh):
    """Image.fromarray(img).resize((ow, oh), BILINEAR): horizontal pass first, the intermediate stored as uint8; a pass
    whose size does not change is skipped (its taps would be the identity anyway)."""
    h, w = img.shape[:2]
    out = img
    if ow != w:
        out = _pil_pass(out, pil_coeffs(w, ow), 1)
    if oh != h:
        out = _pil_pass(out, pil_coeffs(h, oh), 0)
    return np.ascontiguousarray(out)


# ---- Pillow nearest (Image.resize NEAREST -> ImagingTransform affine -> ImagingScaleAffine) ------------------------------
def pil_nearest_index(insz, outsz):
    """Source index per output coordinate: xo starts at a0 / 2 and is advanced by repeated double addition of
    a0 = insz / outsz; the index is (int)xo."""
    a0 = insz / outsz
    xo = 0.0 + a0 * 0.5
    idx = []
    for _ in range(outsz):
        idx.append(-1 if xo < 0.0 else int(xo))
        xo += a0
    return idx


def pil_nearest(lab, ow, oh):
    h, w = lab.shape[:2]
    if (ow, oh) == (w, h):
        return lab.copy()
    return lab[np.array(pil_nearest_index(h, oh))][:, np.array(pil_nearest_index(w, ow))]


# ---- OpenCV INTER_LINEAR on uint8 (resize.cpp: resize coefficient loop, HResizeLinear, VResizeLinearVec_32s8u) --------------
def _cv_round(v):
    return int(np.rint(np.float32(v)))        # saturate_cast<short>(float) = cvRound: round half to even


def cv_coeffs(insz, outsz, clamp):
    """[(s0, s1, c0, c1)] per output coordinate.  fx = (float)((d + 0.5) * scale - 0.5), sx = floor, fx -= sx in float.
    Horizontally (clamp) a tap before the first or past the last source pixel is moved onto it with fx = 0.  Vertically
    the source rows are clipped into the image but the coefficients are kept as computed: where an enlargement reaches
    past a border, both taps read the border row with (1 - fx, fx)."""
    scale = 1. / (outsz / insz)      # resize.cpp: inv_scale = (double)dsize / ssize, scale = 1. / inv_scale
    out = []
    for d in range(outsz):
        fx = np.float32((d + 0.5) * scale - 0.5)
        sx = math.floor(fx)
        fx = np.float32(fx - np.float32(sx))
        if clamp:
            if sx < 0:
                sx, fx = 0, np.float32(0)
            if sx >= insz - 1:
                sx, fx = insz - 1, np.float32(0)
        c0 = _cv_round(np.float32(np.float32(1.0) - fx) * np.float32(1 << CV_BITS))
        c1 = _cv_round(fx * np.float32(1 << CV_BITS))
        out.append((min(max(sx, 0), insz - 1), min(max(sx + 1, 0), insz - 1), c0, c1))
    return out


def cv_linear(img, ow, oh):
    """cv2.resize(img, (ow, oh)) for uint8 HWC: int32 horizontal sums S = a*c0 + b*c1 (a pixel past the right border
    contributes with a zero coefficient), then ((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16) + 2 >> 2 per output."""
    h, w = img.shape[:2]
    a = img.astype(np.int64)
    hx = np.stack([a[:, s0] * c0 + a[:, s1] * c1 for s0, s1, c0, c1 in cv_coeffs(w, ow, True)], 1)
    rows = []
    for s0, s1, b0, b1 in cv_coeffs(h, oh, False):
        rows.append(((((hx[s0] >> 4) * b0) >> 16) + (((hx[s1] >> 4) * b1) >> 16) + 2) >> 2)
    return np.clip(np.stack(rows), 0, 255).astype(np.uint8)


# ---- sizes and crops -------------------------------------------------------------------------------------------------
def imagenet_geometry(h, w, resize, crop):
    """torchvision Resize(resize) (the short side to resize, the long side int(resize * long / short)) and
    CenterCrop(crop) (int(round((size - crop) / 2.0)) per axis): (rh, rw, top, left)."""
    if w <= h:
        rw, rh = resize, int(resize * h / w)
    else:
        rh, rw = resize, int(resize * w / h)
    return rh, rw, int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0))


def fixscale_geometry(h, w, crop):
    """custom_transforms.FixScaleCrop: (oh, ow, y1, x1)."""
    if w > h:
        oh = crop
        ow = int(1.0 * w * oh / h)
    else:
        ow = crop
        oh = int(1.0 * h * ow / w)
    return oh, ow, int(round((oh - crop) / 2.)), int(round((ow - crop) / 2.))


# ---- the three transforms ----------------------------------------------------------------------------------------------
def imagenet(img, resize=256, crop=224, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
    """float32 [3, crop, crop]: ToTensor's x.float() / 255, then (t - mean) / std, every step in fp32."""
    rh, rw, top, left = imagenet_geometry(*img.shape[:2], resize, crop)
    r = pil_bilinear(img, rw, rh)[top:top + crop, left:left + crop]
    t = r.astype(np.float32).transpose(2, 0, 1) / np.float32(255)
    m = np.asarray(mean, np.float32)[:, None, None]
    s = np.asarray(std, np.float32)[:, None, None]
    return (t - m) / s


def voc_segmentation(img, label=None, crop=513, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
    """(float32 [3, crop, crop], float32 [crop, crop] or None): img / 255 in fp32, then - mean and / std in fp64, each
    rounded back to fp32 (numpy promotes the tuple to float64 and casts on the in-place store)."""
    oh, ow, y1, x1 = fixscale_geometry(*img.shape[:2], crop)
    r = pil_bilinear(img, ow, oh)[y1:y1 + crop, x1:x1 + crop].astype(np.float32)
    r = r / np.float32(255)
    r = (r.astype(np.float64) - np.asarray(mean, np.float64)).astype(np.float32)
    r = (r.astype(np.float64) / np.asarray(std, np.float64)).astype(np.float32)
    lab = None
    if label is not None:
        lab = pil_nearest(label, ow, oh)[y1:y1 + crop, x1:x1 + crop].astype(np.float32)
    return np.ascontiguousarray(r.transpose(2, 0, 1)), lab


def ssd(img, size=300, mean=127.0, std=128.0):
    """float32 [3, size, size]: float32(x) - float32(mean), then / std in fp32."""
    r = cv_linear(img, size, size).astype(np.float32) - np.asarray(mean, np.float32)
    r = r / np.float32(std)
    return np.ascontiguousarray(r.transpose(2, 0, 1))
