"""dfq_b200.png on the H100: png.decode byte-equal to np.array(Image.open(...)) on every stream of the seeded corpus
(Pillow palette labels at every compression level, cv2 gray labels under every deflate strategy, the test writer's
filters, block kinds, long and overlapping matches, 15-bit codes, split IDATs and extreme sizes up to 4000 x 3000), in one
batch and in batches of mixed sizes; every corrupt stream flagged by png.check() with its image, call and reason and the
rest of its batch exact; and voc_segmentation on JPEG and PNG bytes equal to it on arrays and to the reference transform."""
import os
import sys

import numpy as np
import pytest
import torch

from dfq_b200 import _lib, jpeg, png, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus as JC  # noqa: E402
import png_corpus as PC  # noqa: E402
import preprocess_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    return PC.corpus(big=True)


def test_decode_equals_pillow_on_the_whole_corpus(corpus):
    outs = png.decode([d for _, d in corpus])
    for (name, d), o in zip(corpus, outs):
        assert o.is_cuda and o.dtype == torch.uint8
        assert torch.equal(o.cpu(), torch.from_numpy(PC.pillow(d))), name
    png.check()
    for name, d in corpus + PC.accepted_edges():                 # one image per call: no neighbour to lean on
        assert torch.equal(png.decode([d])[0].cpu(), torch.from_numpy(PC.pillow(d))), name
    png.check()


@pytest.mark.parametrize("n,seed", [(8, 1), (32, 2), (256, 3)])
def test_batches_of_voc_like_labels(n, seed):
    g = np.random.default_rng(seed)
    items = []
    for i in range(n):
        a = PC.voc_label(int(g.integers(1, 600)), int(g.integers(1, 600)), seed * 1000 + i)
        items.append(PC.pil_p(a, compress_level=int(g.integers(0, 10))) if i % 3 else PC.cv_gray(a))
    outs = png.decode(items)
    for d, o in zip(items, outs):
        assert torch.equal(o.cpu(), torch.from_numpy(PC.pillow(d)))
    png.check()


def test_each_corrupt_stream_is_flagged_and_the_rest_of_its_batch_is_exact():
    good = [d for _, d in PC.corpus(big=False)[:12]]
    want = [PC.pillow(d) for d in good]
    for call, (name, data, why) in enumerate(PC.corrupt_streams()):
        outs = png.decode(good[:5] + [data] + good[5:])
        for k, (w, o) in enumerate(zip(want, outs[:5] + outs[6:])):
            assert torch.equal(o.cpu(), torch.from_numpy(w)), (name, k)
        with pytest.raises(_lib.DfqError, match="image 5 of decode call 1 of 1 .*" + png._ERRORS[why]):
            png.check()
    png.decode(good[:2])
    bad = PC.corrupt_streams()[0][1]
    png.decode([bad] + good[:2])
    png.decode(good[:3] + [bad])
    with pytest.raises(_lib.DfqError, match="image 0 of decode call 2 of 3"):
        png.check()
    png.check()


@pytest.mark.parametrize("n,seed", [(3, 5), (16, 6)])
def test_segmentation_on_bytes_equals_segmentation_on_arrays_and_the_reference(n, seed):
    g = np.random.default_rng(seed)
    jpgs, labs = [], []
    for i in range(n):
        h, w = int(g.integers(40, 500)), int(g.integers(40, 500))
        jpgs.append(JC.pil(JC.picture(h, w, i), quality=90))
        a = PC.voc_label(h, w, seed * 100 + i)
        labs.append(PC.pil_p(a) if i % 2 else PC.cv_gray(a, [2, 9]))
    imgs = [JC.pillow(d) for d in jpgs]
    arrays = [PC.pillow(d) for d in labs]
    x, y = P.voc_segmentation(imgs, arrays)
    mixed_i = [d if k % 2 else a for k, (d, a) in enumerate(zip(jpgs, imgs))]
    mixed_l = [a if k % 3 == 1 else d for k, (d, a) in enumerate(zip(labs, arrays))]
    for got_i, got_l in ((jpgs, labs), (mixed_i, mixed_l), (imgs, labs)):
        xb, yb = P.voc_segmentation(got_i, got_l)
        assert torch.equal(xb, x) and torch.equal(yb, y)
    for i in range(n):
        want, wlab = O.voc_segmentation(imgs[i], arrays[i])
        assert torch.equal(x[i].cpu(), torch.from_numpy(want)) and torch.equal(y[i].cpu(), torch.from_numpy(wlab))
    png.check()
    jpeg.check()
