"""Seeded decoded images and labels for the preprocessing tests and tests/golden/ref_preprocess.npz.

Sizes (h, w): the degenerate 1x1, 2x5 and 17x23, 299x301, exactly the crops (224, 513) and the resize targets (256, 300),
VOC- and ImageNet-like long sides of 500 to 2000 in both orientations, and the rounding cases of FixScaleCrop's
int(1.0 * w * oh / h) and round((w - crop) / 2.) (Python rounds halves to even) and of CenterCrop's offsets.
"""
import numpy as np

SIZES = [
    (1, 1), (2, 5), (5, 2), (17, 23), (299, 301), (224, 224), (256, 256), (300, 300), (513, 513),
    (375, 500), (500, 375), (333, 500), (500, 333), (281, 500), (600, 800), (1000, 1500), (2000, 1200),
    (256, 257), (257, 256), (256, 258), (256, 259), (513, 514), (514, 513), (513, 515), (513, 516), (516, 513),
    (337, 500), (500, 337), (287, 431), (401, 599),
]


def image(h, w, seed):
    """uint8 HWC RGB: a smooth field plus noise, so resampling sees both gradients and edges."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 127.5 + 100 * np.sin(xx[..., None] * (0.05 + 0.02 * np.arange(3)) + yy[..., None] * 0.03)
    return np.clip(base + g.normal(0, 25, (h, w, 3)), 0, 255).astype(np.uint8)


def label(h, w, seed):
    """uint8 HW: classes 0..20 in blocks, with 255 borders like VOC's."""
    g = np.random.default_rng(seed + 1000)
    lab = g.integers(0, 21, (max(1, h // 7 + 1), max(1, w // 7 + 1))).repeat(7, 0).repeat(7, 1)[:h, :w].astype(np.uint8)
    lab[g.random((h, w)) < 0.05] = 255
    lab[:, : max(1, w // 50)] = 255
    lab[: max(1, h // 50)] = 255
    return lab


def cases():
    """[(name, image, label)] over SIZES, seeded by position."""
    return [("%dx%d" % hw, image(*hw, seed=i), label(*hw, seed=i)) for i, hw in enumerate(SIZES)]
