"""The crafted JPEG corpus (tests/jpeg_streams.py) on the H100: jpeg.decode of every crafted stream torch.equal to
Pillow, one stream per call; the same streams mixed into batches of 1, 7, 64 and 256 with the Pillow-encoded corpus,
each output still exact; preprocess.imagenet / voc_segmentation / ssd on the crafted bytes equal to the same calls on
Pillow's arrays; and jpeg.check() clean afterwards."""
import os
import sys

import numpy as np
import pytest
import torch

from dfq_b200 import jpeg, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus as JC  # noqa: E402
import jpeg_streams as S  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def crafted():
    return [(n, d, JC.pillow(d)) for n, d in S.streams()]


def test_each_crafted_stream_alone(crafted):
    for name, d, want in crafted:
        (o,) = jpeg.decode([d])
        assert torch.equal(o.cpu(), torch.from_numpy(want)), name
    jpeg.check()


def test_crafted_decodes_match_the_fixture(crafted):
    fx = S.fixture()
    outs = jpeg.decode([d for _, d, _ in crafted])
    for (name, _, _), o in zip(crafted, outs):
        assert S.sha256(o.cpu().numpy()) == fx[name], name
    jpeg.check()


@pytest.mark.parametrize("n,seed", [(1, 1), (7, 2), (64, 3), (256, 4)])
def test_mixed_batches_with_the_pillow_corpus(crafted, n, seed):
    pool = [(d, a) for _, d, a in crafted] + [(d, JC.pillow(d)) for _, d in JC.corpus(big=False)]
    g = np.random.default_rng(seed)
    pick = [pool[k] for k in g.choice(len(pool), n, replace=n > len(pool))]
    if n > 1:
        pick[0] = (crafted[0][1], crafted[0][2])                  # an overshooting stream in every batch
    outs = jpeg.decode([d for d, _ in pick])
    for k, ((d, a), o) in enumerate(zip(pick, outs)):
        assert torch.equal(o.cpu(), torch.from_numpy(a)), k
    jpeg.check()


def test_preprocess_on_crafted_bytes(crafted):
    items = [d for _, d, _ in crafted]
    arrays = [a for _, _, a in crafted]
    labels = [np.full(a.shape[:2], k % 21, np.uint8) for k, a in enumerate(arrays)]
    mixed = [a if k % 3 == 1 else d for k, (d, a) in enumerate(zip(items, arrays))]
    for got in (items, mixed):
        assert torch.equal(P.imagenet(got), P.imagenet(arrays))
        x, y = P.voc_segmentation(got, labels)
        xa, ya = P.voc_segmentation(arrays, labels)
        assert torch.equal(x, xa) and torch.equal(y, ya)
        s, sz = P.ssd(got, mean=np.array([127, 127, 127]), std=128.0)
        sa, sza = P.ssd(arrays, mean=np.array([127, 127, 127]), std=128.0)
        assert torch.equal(s, sa) and torch.equal(sz, sza)
    jpeg.check()
