"""Evaluation preprocessing on the GPU: the reference's resize, crop and normalisation of decoded images, bit for bit.

The reference's three evaluation loops transform every decoded image on the CPU before the network sees it:
main_cls.py with torchvision Resize(256) -> CenterCrop(224) -> ToTensor -> Normalize (Pillow bilinear), main_seg.py with
custom_transforms FixScaleCrop(513) -> Normalize -> ToTensor (Pillow bilinear image, Pillow nearest label), and
main_ssd.py with PredictionTransform (cv2.resize INTER_LINEAR -> - mean -> / std).  Here the loader only decodes (or, with
dfq_b200.jpeg, only reads the file: JPEG bytes are decoded on the device into the same blob): the batch's
images, of any sizes, are gathered into one page-locked buffer, moved by one host-to-device copy, and one kernel launch
resizes, crops and normalises them into the NCHW float32 batch.  The resize coefficients are the libraries' own, formed on
the host by their rules; the arithmetic on the device is theirs step for step, so the output equals the CPU transform's.

    for images in loader:                              # collate_fn returns the decoded uint8 HWC arrays as a list
        x = preprocess.imagenet(images)                # [N, 3, 224, 224] on the current device
        logits = model(x)
"""
from __future__ import annotations

import ctypes as C
import functools
import numbers

import numpy as np
import torch

from . import _lib, jpeg, png

__all__ = ["imagenet", "voc_segmentation", "ssd"]

_IMAGENET_MEAN, _IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
_ALIGN = 64


# ---- tap tables: [out, K] int32 pairs {source index, weight}, padded with the last index at weight 0 ----------------------
def _pil_taps(insz, outsz):
    """Pillow's precompute_coeffs for BILINEAR (support 1, scaled by the reduction) and normalize_coeffs_8bpc."""
    scale = insz / outsz
    fs = max(scale, 1.0)
    center = (np.arange(outsz, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum((center - fs + 0.5).astype(np.int64), 0)
    cnt = np.minimum((center + fs + 0.5).astype(np.int64), insz) - xmin
    k = np.arange(int(cnt.max()))
    t = np.abs(((k[None, :] + xmin[:, None]) - center[:, None] + 0.5) * (1.0 / fs))
    w = np.where((t < 1.0) & (k[None, :] < cnt[:, None]), 1.0 - t, 0.0)
    ww = np.cumsum(w, axis=1)[:, -1:]                  # Pillow's sequential sum (the zero padding adds exact zeros)
    w = np.where(ww != 0.0, w / np.where(ww != 0.0, ww, 1.0), w)
    iw = np.where(w < 0, -0.5 + w * (1 << 22), 0.5 + w * (1 << 22)).astype(np.int64)   # C's (int): toward zero
    idx = xmin[:, None] + np.minimum(k[None, :], cnt[:, None] - 1)
    return _pairs(idx, iw)


@functools.lru_cache(maxsize=1024)
def _cv_taps(insz, outsz, clamp):
    """OpenCV resize's INTER_LINEAR coefficients on uint8: fx = (float)((d + 0.5) * scale - 0.5) with scale =
    1 / (out / in), floored, taps cvRound(fx * 2048) and cvRound((1 - fx) * 2048).  Columns (clamp) at or past a border
    take the border pixel with fx = 0; rows are clipped into the image with their coefficients kept."""
    scale = 1.0 / (outsz / insz)
    fx = ((np.arange(outsz, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    fx = fx - sx.astype(np.float32)
    if clamp:
        edge = (sx < 0) | (sx >= insz - 1)
        fx = np.where(edge, np.float32(0), fx)
        sx = np.where(sx < 0, 0, np.where(sx >= insz - 1, insz - 1, sx))
    c0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64)
    c1 = np.rint(fx * np.float32(2048)).astype(np.int64)
    idx = np.clip(np.stack([sx, sx + 1], 1), 0, insz - 1)
    return _pairs(idx, np.stack([c0, c1], 1))


def _nearest_index(insz, outsz):
    """Pillow's NEAREST resize (ImagingScaleAffine): the source coordinate starts at a / 2 and advances by repeated double
    additions of a = in / out (a cumulative sum, so the same roundings); the index is its truncation."""
    a = insz / outsz
    steps = np.full(outsz, a)
    steps[0] = 0.0 + a * 0.5
    return np.cumsum(steps).astype(np.int64).astype(np.int32)


def _pairs(idx, w):
    p = np.empty(idx.shape + (2,), np.int32)
    p[..., 0], p[..., 1] = idx, w
    return _readonly(p)


# ---- argument checks ---------------------------------------------------------------------------------------------------
def _images(images, what="images", planes=3):
    if isinstance(images, (np.ndarray, torch.Tensor, bytes, bytearray, memoryview)) or not hasattr(images, "__len__"):
        raise _lib.DfqError("%s must be a list of uint8 arrays, got %s" % (what, type(images).__name__))
    if len(images) == 0:
        raise _lib.DfqError("%s: the batch is empty" % what)
    out = []
    for i, a in enumerate(jpeg.parse(images, what) if planes else png.parse(images, what)):
        if isinstance(a, (jpeg._Jpeg, png._Png)):
            out.append(a)
            continue
        if isinstance(a, torch.Tensor):
            if a.device.type != "cpu":
                raise _lib.DfqError("%s[%d] is on %s: decoded images come from the host" % (what, i, a.device))
            if a.dtype != torch.uint8:
                raise _lib.DfqError("%s[%d] must be uint8, got %s" % (what, i, a.dtype))
            a = a.numpy()
        elif not isinstance(a, np.ndarray):
            raise _lib.DfqError("%s[%d] must be a numpy array, a CPU tensor%s, got %s"
                                % (what, i, " or JPEG bytes" if planes else " or PNG bytes", type(a).__name__))
        if a.dtype != np.uint8:
            raise _lib.DfqError("%s[%d] must be uint8, got %s" % (what, i, a.dtype))
        if planes and (a.ndim != 3 or a.shape[2] != planes):
            raise _lib.DfqError("%s[%d] must be HWC with 3 channels, got shape %s" % (what, i, a.shape))
        if not planes and a.ndim != 2:
            raise _lib.DfqError("%s[%d] must be HW, got shape %s" % (what, i, a.shape))
        if a.shape[0] < 1 or a.shape[1] < 1:
            raise _lib.DfqError("%s[%d] is empty: shape %s" % (what, i, a.shape))
        out.append(np.ascontiguousarray(a))
    return out


def _positive(name, v):
    if not isinstance(v, numbers.Integral) or isinstance(v, bool) or v < 1:
        raise _lib.DfqError("%s must be a positive int, got %r" % (name, v))
    return int(v)


def _triple(name, v):
    """A number or 3 numbers (a tuple, a list or a numpy array, as the reference's configs give them) as 3 floats."""
    try:
        a = np.asarray(v, dtype=np.float64).ravel()
    except (TypeError, ValueError):
        raise _lib.DfqError("%s must be a number or 3 numbers, got %r" % (name, v)) from None
    if a.size not in (1, 3) or isinstance(v, (str, bytes)) or not np.isfinite(a).all():
        raise _lib.DfqError("%s must be a finite number or 3 finite numbers, got %r" % (name, v))
    return tuple(float(x) for x in np.broadcast_to(a, 3))


def _stds(std):
    s = _triple("std", std)
    if any(x == 0.0 for x in s) or any(np.float32(x) == 0 for x in s):
        raise _lib.DfqError("std must not be zero, got %r" % (std,))
    return s


def _fits(i, rh, rw, crop_h, crop_w):
    if rh < crop_h or rw < crop_w:
        raise _lib.DfqError("images[%d] resizes to %d x %d, smaller than the %d x %d crop: the reference would pad"
                            % (i, rh, rw, crop_h, crop_w))


# ---- host path -----------------------------------------------------------------------------------------------------------
def _pinned(nbytes):
    return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)


def _device():
    return torch.device("cuda", torch.cuda.current_device())


class _Stage:
    """A batch gathered into one page-locked block: segments placed 64-byte aligned, tables shared by identity (images of
    one size share their tap tables, JPEGs of one encoder their Huffman and quantisation tables)."""

    def __init__(self):
        self.segs, self.offs, self.total, self.tables = [], [], 0, {}

    def place(self, a):
        self.segs.append(a)
        self.offs.append(self.total)
        self.total += (a.nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        return self.offs[-1]

    def table(self, t):
        key = id(t)
        if key not in self.tables:
            self.tables[key] = (self.place(t), t)
        return self.tables[key][0]

    def upload(self, extra=0):
        """Gather into the staging block and move it with one host-to-device copy into a device block `extra` bytes longer
        (room that only the device writes)."""
        lib = _lib.load()
        # A page-locked block of torch's caching host allocator: the non-blocking copy below records its stream on the
        # block, so the block is handed out again (to a later batch of the same or a smaller size) only once that copy has
        # completed, and the host never waits for it.
        buf = _pinned(self.total)
        ptrs = np.array([a.ctypes.data for a in self.segs], np.uintp)
        nbytes = np.array([a.nbytes for a in self.segs], np.uintp)
        offsets = np.array(self.offs, np.uintp)
        _lib.check(lib.dfq_host_copy_segments(C.c_void_p(buf.data_ptr()), _lib.table_ptr(ptrs), _lib.table_ptr(nbytes),
                                              _lib.table_ptr(offsets), len(self.segs), 0, 0), "dfq_host_copy_segments")
        dev = _device()
        if not extra:
            return buf.to(dev, non_blocking=True)
        blob = torch.empty(self.total + extra, dtype=torch.uint8, device=dev)
        blob[:self.total].copy_(buf, non_blocking=True)
        return blob


def _launch(images, labels, xtaps, ytaps, near, filt, norm, out_h, out_w, mean, std):
    """Gather the batch into the staging buffer, one H2D copy, dfq_jpeg_decode when the batch holds JPEG bytes,
    dfq_png_decode when its labels hold PNG bytes, one dfq_pre_resample launch."""
    _lib.require_cuda()
    lib = _lib.load()
    stage = _Stage()
    jpegs, pngs = jpeg._Batch(stage), png._Batch(stage)
    n = len(images)
    desc = np.zeros(n, _lib.PRE_IMAGE_DT)
    coded, coded_labels = {}, {}
    for i, a in enumerate(images):
        d = desc[i]
        d["H"], d["W"] = a.shape[:2]
        if isinstance(a, jpeg._Jpeg):
            coded[i] = jpegs.add(a)
        else:
            d["src"] = stage.place(a)
        d["xtap"], d["ytap"] = stage.table(xtaps[i]), stage.table(ytaps[i])
        d["xk"], d["yk"] = xtaps[i].shape[1], ytaps[i].shape[1]
        if labels is None:
            d["label"] = d["xnear"] = d["ynear"] = -1
        else:
            if isinstance(labels[i], png._Png):
                coded_labels[i] = pngs.add(labels[i])
            else:
                d["label"] = stage.place(labels[i])
            d["xnear"], d["ynear"] = stage.table(near[i][0]), stage.table(near[i][1])
    pngs.base = jpegs.extra                            # the decoded pixels and labels go past every copied byte
    for i, k in coded.items():
        desc[i]["src"] = jpegs.dst(k)
    for i, k in coded_labels.items():
        desc[i]["label"] = pngs.dst(k)
    blob = stage.upload(jpegs.extra + pngs.extra)
    if coded:
        jpegs.launch(blob)
    if coded_labels:
        pngs.launch(blob)
    dev = blob.device
    p = np.zeros(1, _lib.PRE_RESAMPLE_DT)
    p["n"], p["out_h"], p["out_w"], p["filter"], p["norm"], p["blob_bytes"] = n, out_h, out_w, filt, norm, blob.numel()
    p["mean"], p["std"], p["mean64"], p["std64"] = mean, std, mean, std
    out = torch.empty(n, 3, out_h, out_w, dtype=torch.float32, device=dev)
    lab = torch.empty(n, out_h, out_w, dtype=torch.float32, device=dev) if labels is not None else None
    _lib.check(lib.dfq_pre_resample(_lib.table_ptr(p), _lib.table_ptr(desc), C.c_void_p(blob.data_ptr()),
                                    C.c_void_p(out.data_ptr()), C.c_void_p(lab.data_ptr()) if lab is not None else None,
                                    _lib.stream_ptr()), "dfq_pre_resample")
    return out, lab


# ---- public interface ----------------------------------------------------------------------------------------------------
def imagenet(images, resize=256, crop=224, mean=_IMAGENET_MEAN, std=_IMAGENET_STD) -> torch.Tensor:
    """float32 [N, 3, crop, crop] on the current device: torchvision Compose([Resize(resize), CenterCrop(crop), ToTensor(),
    Normalize(mean, std)]) of Image.fromarray(img) for each image, bit for bit (Pillow's antialiased bilinear; x / 255,
    - mean, / std each in fp32).  images: a list of uint8 HWC RGB numpy arrays or CPU tensors, each of its own size.
    mean, std: a number or 3 numbers (a tuple, list or numpy array).
    Items may also be JPEG bytes (jpeg.probe says which are taken), decoded on the device as Pillow decodes them; a
    batch may mix them with arrays.  An image whose resize is smaller than the crop (CenterCrop would pad) is refused.
    Does not synchronise with the host."""
    imgs = _images(images)
    resize, crop = _positive("resize", resize), _positive("crop", crop)
    mean, std = _triple("mean", mean), _stds(std)
    xt, yt = [], []
    for i, a in enumerate(imgs):
        h, w = a.shape[:2]
        if w <= h:
            rw, rh = resize, int(resize * h / w)
        else:
            rh, rw = resize, int(resize * w / h)
        _fits(i, rh, rw, crop, crop)
        top, left = int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0))
        xt.append(_pil_crop(w, rw, left, crop))
        yt.append(_pil_crop(h, rh, top, crop))
    return _launch(imgs, None, xt, yt, None, _lib.PRE_PIL_BILINEAR, _lib.PRE_NORM_F32, crop, crop, mean, std)[0]


def voc_segmentation(images, labels=None, crop_size=513, mean=_IMAGENET_MEAN, std=_IMAGENET_STD):
    """(image float32 [N, 3, crop_size, crop_size], label float32 [N, crop_size, crop_size] or None) on the current device:
    VOCSegmentation.transform_val's sample['image'] and sample['label'], bit for bit.  FixScaleCrop(crop_size) resizes the
    short side to crop_size (Pillow bilinear for the image, nearest for the label) and center-crops; Normalize divides by
    255 in fp32 and applies mean and std in fp64, each rounded back to fp32.  images as for imagenet() (JPEG bytes
    included, EXIF orientation ignored as Pillow ignores it); labels: None or a list of uint8 HW arrays of the images'
    sizes, or of PNG bytes (png.probe says which are taken) decoded on the device as Image.open reads them, mixed with
    arrays if need be; a PNG's size is checked from its header, before any copy.  The label output is what segment.Evaluator.add_logits takes.  Does not synchronise with the host."""
    imgs = _images(images)
    labs = None
    if labels is not None:
        labs = _images(labels, "labels", planes=0)
        if len(labs) != len(imgs):
            raise _lib.DfqError("%d labels for %d images" % (len(labs), len(imgs)))
        for i, (a, l) in enumerate(zip(imgs, labs)):
            if l.shape != a.shape[:2]:
                raise _lib.DfqError("labels[%d] is %s, images[%d] is %s" % (i, l.shape, i, a.shape[:2]))
    crop = _positive("crop_size", crop_size)
    for name, v in (("mean", mean), ("std", std)):
        if isinstance(v, (np.ndarray, np.floating)) and v.dtype.kind == "f" and v.dtype.itemsize < 8:
            raise _lib.DfqError("%s is %s: Normalize would apply it in that precision, not in float64 as it does the "
                                "reference's tuples; pass a tuple or a float64 array" % (name, v.dtype))
    mean, std = _triple("mean", mean), _stds(std)
    xt, yt, near = [], [], []
    for i, a in enumerate(imgs):
        h, w = a.shape[:2]
        if w > h:
            oh, ow = crop, int(1.0 * w * crop / h)
        else:
            ow, oh = crop, int(1.0 * h * crop / w)
        _fits(i, oh, ow, crop, crop)
        x1, y1 = int(round((ow - crop) / 2.)), int(round((oh - crop) / 2.))
        xt.append(_pil_crop(w, ow, x1, crop))
        yt.append(_pil_crop(h, oh, y1, crop))
        if labs is not None:
            near.append((_crop_near(w, ow, x1, crop), _crop_near(h, oh, y1, crop)))
    return _launch(imgs, labs, xt, yt, near, _lib.PRE_PIL_BILINEAR, _lib.PRE_NORM_F64, crop, crop, mean, std)


def ssd(images, size=300, mean=127.0, std=128.0):
    """(float32 [N, 3, size, size], int64 [N, 2] (width, height) of each input) on the current device: the images are
    PredictionTransform(size, mean, std)(img) bit for bit (cv2.resize INTER_LINEAR, float32(x) - float32(mean), / std in
    fp32); the sizes go to detect.postprocess(image_sizes=...).  mean: a number or 3 numbers (a tuple, list or numpy
    array, e.g. the configs' image_mean); std: a Python number (the configs' image_std).  images as for imagenet().
    Given JPEG bytes, decoded as cv2.imread decodes them; bytes with an EXIF orientation other than 1, which cv2.imread
    would rotate, are refused.  Does not synchronise with the host."""
    imgs = _images(images)
    for i, a in enumerate(imgs):
        if isinstance(a, jpeg._Jpeg) and a.orientation != 1:
            raise _lib.DfqError("images[%d] has EXIF orientation %d, which cv2.imread applies and the device decode does not: "
                                "decode it with cv2.imread on the host" % (i, a.orientation))
    size = _positive("size", size)
    if type(std) not in (int, float):
        # a numpy scalar or array would make numpy divide the float32 image in float64 (NEP 50), a Python number in float32
        raise _lib.DfqError("std must be a Python number, as the reference's configs give it, got %r" % (std,))
    mean, std = _triple("mean", mean), _stds(std)
    xt = [_cv_taps(a.shape[1], size, True) for a in imgs]
    yt = [_cv_taps(a.shape[0], size, False) for a in imgs]
    out, _ = _launch(imgs, None, xt, yt, None, _lib.PRE_CV_LINEAR, _lib.PRE_NORM_SUB_DIV, size, size, mean, std)
    sizes = torch.tensor([[a.shape[1], a.shape[0]] for a in imgs], dtype=torch.int64).pin_memory()
    return out, sizes.to(out.device, non_blocking=True)


# The caches keep only the cropped tables, copied out of the whole ones: one entry is at most n * (2 * ceil(in / out) + 1)
# pairs of 8 bytes (70 KB for a 4,000-pixel side cropped to 513), so 512 entries bound the cache well below 100 MB.
@functools.lru_cache(maxsize=512)
def _pil_crop(insz, outsz, lo, n):
    """The taps of the n output coordinates from lo: the crop keeps only these."""
    return _readonly(_pil_taps(insz, outsz)[lo:lo + n].copy())


@functools.lru_cache(maxsize=512)
def _crop_near(insz, outsz, lo, n):
    return _readonly(_nearest_index(insz, outsz)[lo:lo + n].copy())


def _readonly(a):
    a.setflags(write=False)
    return a
