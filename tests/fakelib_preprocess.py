"""tests/fakelib.py's stand-in for libdfq_sm90.so, extended by a host twin of dfq_pre_resample with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.preprocess through it inside a test, so the batch packing (offsets,
shared tables, descriptors, the label tables) runs without a GPU.  The gather is the real library's dfq_host_copy_segments
(a host function), the "device" is the CPU, and the twin applies the blob's tap tables the way k_pre_resample does, so
its output equals the oracle's only if the host path packed the batch right.
"""
import ctypes as C

import numpy as np
import torch

import fakelib
from dfq_b200 import _lib, preprocess
from fakelib import _table, _val

E_ARG = -1
MAX_TAPS = 4096


def _bytes(ptr, n):
    return np.ctypeslib.as_array((C.c_uint8 * int(n)).from_address(int(ptr)))


class FakePreprocessLib(fakelib.FakeLib):
    def __init__(self, real):
        super().__init__()
        self.real = real
        self.refusals = []
        self.descriptors = None     # the last call's DfqPreImage table and DfqPreResample

    def dfq_host_copy_segments(self, *args):
        self.calls.append("dfq_host_copy_segments")
        return self.real.dfq_host_copy_segments(*args)

    def _refuse(self, reason):
        self.refusals.append(reason)
        return E_ARG

    def dfq_pre_resample(self, d_p, im_p, blob_p, out_p, lab_p, stream):
        self.calls.append("dfq_pre_resample")
        d_p, im_p, blob_p, out_p, lab_p = (int(_val(v) or 0) for v in (d_p, im_p, blob_p, out_p, lab_p))
        if not (d_p and im_p and blob_p and out_p):
            return self._refuse("NULL pointer")
        d = _table(d_p, 1, _lib.PRE_RESAMPLE_DT)[0].copy()
        n, oh, ow, filt, norm, B = (int(d[k]) for k in ("n", "out_h", "out_w", "filter", "norm", "blob_bytes"))
        if not (1 <= n <= 65535 and oh >= 1 and ow >= 1 and B >= 1 and filt in (0, 1) and norm in (0, 1, 2)):
            return self._refuse("bad sizes, filter or norm")
        if (d["std64"] == 0).any() if norm == _lib.PRE_NORM_F64 else (d["std"] == 0).any():
            return self._refuse("std is zero")
        ims = _table(im_p, n, _lib.PRE_IMAGE_DT).copy()

        def inside(off, count, elem, align):
            return off >= 0 and off % align == 0 and count >= 0 and count <= (B - off) // elem

        for m in ims:
            H, W, xk, yk = int(m["H"]), int(m["W"]), int(m["xk"]), int(m["yk"])
            ok = H >= 1 and W >= 1 and 1 <= xk <= MAX_TAPS and 1 <= yk <= MAX_TAPS and inside(m["src"], H * W * 3, 1, 1) \
                and inside(m["xtap"], ow * xk, 8, 8) and inside(m["ytap"], oh * yk, 8, 8)
            ok = ok and (m["xnear"] < 0 and m["ynear"] < 0 if m["label"] < 0 else
                         inside(m["label"], H * W, 1, 1) and inside(m["xnear"], ow, 4, 4) and inside(m["ynear"], oh, 4, 4))
            if not ok:
                return self._refuse("image outside the blob or bad taps")
        labelled = int((ims["label"] >= 0).sum())
        if not ((labelled == 0 and not lab_p) or (labelled == n and lab_p)):
            return self._refuse("labels for some images only")
        if blob_p % 8 or out_p % 4 or lab_p % 4:
            return self._refuse("misaligned pointer")
        self.descriptors = (ims, d)
        blob = _bytes(blob_p, B)
        out = np.ctypeslib.as_array((C.c_float * (n * 3 * oh * ow)).from_address(out_p)).reshape(n, 3, oh, ow)
        for i, m in enumerate(ims):
            H, W = int(m["H"]), int(m["W"])
            img = blob[m["src"]:m["src"] + H * W * 3].reshape(H, W, 3).astype(np.int64)
            xt = blob[m["xtap"]:m["xtap"] + ow * m["xk"] * 8].view(np.int32).reshape(ow, m["xk"], 2)
            yt = blob[m["ytap"]:m["ytap"] + oh * m["yk"] * 8].view(np.int32).reshape(oh, m["yk"], 2)
            out[i] = _normalise(_resample(img, xt, yt, filt), norm, d).transpose(2, 0, 1)
            if m["label"] >= 0:
                lab = blob[m["label"]:m["label"] + H * W].reshape(H, W)
                xn = blob[m["xnear"]:m["xnear"] + 4 * ow].view(np.int32)
                yn = blob[m["ynear"]:m["ynear"] + 4 * oh].view(np.int32)
                lo = np.ctypeslib.as_array((C.c_float * (n * oh * ow)).from_address(lab_p)).reshape(n, oh, ow)
                lo[i] = lab[yn][:, xn].astype(np.float32)
        return 0


def _resample(img, xt, yt, filt):
    """The kernel's two passes on whole planes: horizontal sums through the column taps, then the row taps."""
    h = (img[:, xt[:, :, 0]] * xt[:, :, 1][None, :, :, None]).sum(2)          # [H, out_w, 3]
    if filt == _lib.PRE_PIL_BILINEAR:
        h = np.clip((h + (1 << 21)) >> 22, 0, 255)
        v = (h[yt[:, :, 0]] * yt[:, :, 1][:, :, None, None]).sum(1)
        return np.clip((v + (1 << 21)) >> 22, 0, 255)
    v = (((h[yt[:, :, 0]] >> 4) * yt[:, :, 1][:, :, None, None]) >> 16).sum(1)
    return np.clip((v + 2) >> 2, 0, 255)


def _normalise(u, norm, d):
    u = u.astype(np.float32)
    if norm == _lib.PRE_NORM_F32:
        return (u / np.float32(255) - d["mean"]) / d["std"]
    if norm == _lib.PRE_NORM_F64:
        t = (u / np.float32(255)).astype(np.float64)
        return ((t - d["mean64"]).astype(np.float32).astype(np.float64) / d["std64"]).astype(np.float32)
    return (u - d["mean"]) / d["std"]


def install(monkeypatch):
    """fakelib.install() with the preprocessing twin; the CPU stands in for the device while it is active."""
    real = _lib.load()
    fakelib.install(monkeypatch)
    fake = FakePreprocessLib(real)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(_lib, "require_cuda", lambda: None)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(preprocess, "_pinned", lambda nbytes: torch.empty(nbytes, dtype=torch.uint8))
    monkeypatch.setattr(preprocess, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return fake
