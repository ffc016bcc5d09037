"""The seeded JPEG corpus of the decoder's tests and benchmark: Pillow- and cv2-encoded streams over sizes from 1 x 1 to
4000 x 3000, gray and 4:4:4 / 4:2:2 / 4:2:0, qualities 1 to 100, optimized Huffman tables, custom quantisation tables
and restart markers (Pillow 12 writes both restart_marker_blocks and restart_marker_rows)."""
import io

import cv2
import numpy as np
from PIL import Image

SMALL = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 23)]
MID = [(333, 500), (375, 500), (513, 515)]
SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def picture(h, w, seed, noise=0.3):
    """A gradient with a share of noise pixels: every coefficient band in use, and smooth areas that upsampling shows."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), ((xx + yy) * 3) % 256], -1)
    a = np.where(g.random((h, w, 1)) < noise, g.integers(0, 256, (h, w, 3)), base)
    return a.astype(np.uint8)


def pil(a, **kw):
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", **kw)
    return b.getvalue()


def cv(a, quality=95, flags=()):
    extra = [v for kv in flags for v in kv]
    ok, e = cv2.imencode(".jpg", np.ascontiguousarray(a[:, :, ::-1]), [cv2.IMWRITE_JPEG_QUALITY, quality] + extra)
    assert ok
    return e.tobytes()


def corpus(big=True):
    """[(name, bytes)]."""
    out = []
    for h, w in SMALL:
        for q in (1, 50, 90, 95, 100):
            a = picture(h, w, h * 100 + w + q)
            for s, ss in SUBSAMPLING.items():
                out.append(("%dx%d_%s_q%d" % (h, w, s, q), pil(a, quality=q, subsampling=ss)))
            out.append(("%dx%d_gray_q%d" % (h, w, q), pil(a[:, :, 1], quality=q)))
    qt = [list(range(1, 65)), [max(1, 90 - k) for k in range(64)]]
    for h, w in MID:
        a = picture(h, w, h + w)
        for s, ss in SUBSAMPLING.items():
            out.append(("%dx%d_%s_q90" % (h, w, s), pil(a, quality=90, subsampling=ss)))
        out.append(("%dx%d_gray_q50" % (h, w), pil(a[:, :, 0], quality=50)))
        out.append(("%dx%d_420_optimize" % (h, w), pil(a, quality=95, optimize=True)))
        out.append(("%dx%d_422_qtables" % (h, w), pil(a, qtables=qt, subsampling=1)))
        out.append(("%dx%d_420_rst_blocks" % (h, w), pil(a, quality=75, restart_marker_blocks=5)))
        out.append(("%dx%d_444_rst_rows" % (h, w), pil(a, quality=75, subsampling=0, restart_marker_rows=1)))
        out.append(("%dx%d_cv_q95" % (h, w), cv(a)))
        out.append(("%dx%d_cv_422_rst" % (h, w), cv(a, 80, [(cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422),
                                                           (cv2.IMWRITE_JPEG_RST_INTERVAL, 7)])))
    if big:
        out.append(("3000x4000_420_q50", pil(picture(3000, 4000, 7, noise=0.0), quality=50)))
    return out


def pillow(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def opencv(data):
    return cv2.cvtColor(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
