"""The crafted JPEG corpus on the CPU: the writer writes exactly the blocks it is given under every option; every crafted
stream decodes the same in the oracle, Pillow and OpenCV, and Pillow's decode matches the committed hashes; a Huffman
table that fills a code length is refused before any library call, as libjpeg refuses it; and the host path decodes the
crafted streams through the twin of dfq_jpeg_decode."""
import os
import sys

import numpy as np
import pytest
import torch

from dfq_b200 import _lib, jpeg, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus as JC  # noqa: E402
import jpeg_oracle as O  # noqa: E402
import jpeg_streams as S  # noqa: E402
import jpeg_writer as JW  # noqa: E402


@pytest.fixture(scope="module")
def streams():
    return S.streams()


# ---- the writer ------------------------------------------------------------------------------------------------------------
_OPTIONS = {"plain": {}, "dqt16": dict(qbits=16), "ri1": dict(ri=1), "ri3_fill": dict(ri=3, fill=2),
            "sof1": dict(sof=0xC1), "ids": dict(ids=[0, 1, 2]), "split": dict(group=False),
            "after_sof": dict(tables_after_sof=True), "redefined": dict(redefine=True),
            "extras": dict(extras=True, seed=5), "maxlen9": dict(maxlen=9),
            "explicit": dict(huff={(0, 0): S._DC_EVERY, (1, 0): S._AC_EVERY, (0, 1): S._DC_EVERY, (1, 1): S._AC_EVERY})}


@pytest.mark.parametrize("sampling", ["gray", "444", "422", "420"])
@pytest.mark.parametrize("option", list(_OPTIONS))
def test_writer_round_trip(sampling, option):
    g = np.random.default_rng(len(option) * 10 + len(sampling))
    h, w = 19, 37
    planes = S._random(g, sampling, h, w, dc=900, ac=500, density=0.3)
    if option == "explicit":                                    # only the symbols the explicit tables hold
        for p in planes:
            p[..., 1:] = 0
            p[..., 0] = g.integers(-2000, 2000, p.shape[:2])
            p[..., 1] = 1
    kw = dict(_OPTIONS[option])
    if sampling == "gray" and "ids" in kw:
        kw["ids"] = [0]
    q = [np.arange(64) % 13 + 1, np.arange(64) % 7 + 2]
    wr = JW.write(planes, height=h, width=w, sampling=sampling, qtables=q, **kw)
    (H, W, comps, hm, vm), got = O.coefficients(wr.data, dequantise=False)
    assert (H, W) == (h, w) and len(got) == len(planes)
    for a, b in zip(got, planes):
        assert np.array_equal(a, O.wrap16(b))
    if "maxlen" in kw:
        assert max(max(v) for v in wr.lengths.values()) <= kw["maxlen"]
    assert np.array_equal(JC.pillow(wr.data), O.decode(wr.data))


def test_writer_wraps_dc_and_codes_every_category():
    planes = S._zeros("gray", 8, 8 * 40)
    b = planes[0].reshape(-1, 64)
    b[:, 0] = np.cumsum([(1 if k < 16 else -1) * ((1 << (k % 16)) - 1) for k in range(40)])   # to 65519 and back
    wr = JW.write(planes, height=8, width=8 * 40, qtables=[S._q(1)], huff={(0, 0): S._DC_EVERY})
    assert wr.symbols[(0, 0)] == set(range(16)) and b[:, 0].max() > 32767
    assert np.array_equal(O.coefficients(wr.data, dequantise=False)[1][0], O.wrap16(planes[0]))


# ---- the crafted corpus against the libraries -----------------------------------------------------------------------------
def test_oracle_equals_pillow_and_opencv_on_every_crafted_stream(streams):
    for name, d in streams:
        want = JC.pillow(d)
        assert np.array_equal(O.decode(d), want), name
        assert np.array_equal(JC.opencv(d), want), name
        assert jpeg.probe(d).supported, name


def test_pillow_decodes_match_the_fixture(streams):
    """A libjpeg-turbo whose decode of the crafted streams differs from the one the hashes were taken with fails here,
    not as a decoder bug."""
    fx = S.fixture()
    assert sorted(fx) == sorted(n for n, _ in streams)
    for name, d in streams:
        assert S.sha256(JC.pillow(d)) == fx[name], name


def test_crafted_streams_reach_the_edges(streams):
    """What the corpus is for, over all of it: outputs saturated at both ends, chroma widths 1, 2 and 3."""
    names = dict(streams)
    for s in ("gray", "444", "422", "420"):
        a = JC.pillow(names["overshoot_" + s])
        assert (a == 0).any() and (a == 255).any()
    widths = {-(-jpeg.probe(d).width // 2) for n, d in streams if n.startswith("geo_")}
    assert {1, 2, 3, 8, 9, 16, 17} <= widths


def test_table_builder_on_codes_of_every_length(streams):
    """jpeg._huff's lookahead and maxcode walk give every 16-bit window the symbol libjpeg decodes, for tables with a code
    at each length 1 .. 16 (9- and 10-bit codes on both sides of the lookahead)."""
    for name in ("codes_every_length_gray", "codes_every_length_420", "codes_optimal_max9", "codes_optimal_max10"):
        data = dict(streams)[name]
        j = jpeg._parse(data)
        t = np.frombuffer(j.tables.tobytes(), _lib.JPEG_TABLES_DT)[0]
        (H, W, comps, q), sel, huff, ri, _ = O._segments(data)
        for c, comp in enumerate(comps):
            for kind, h in ((0, t["dc"][c]), (1, t["ac"][c])):
                look = huff[(kind, sel[comp[0]][kind])]
                for bits in range(65536):
                    e = int(h["look"][bits >> 7])
                    got = (e >> 8, e & 255) if e else (0, 0)
                    if not e:
                        for n in range(10, 17):
                            if bits >> (16 - n) <= h["maxcode"][n]:
                                got = (n, int(h["vals"][(bits >> (16 - n)) + h["valoff"][n]]))
                                break
                    assert got == look[bits], (name, c, kind, bits)


# ---- a Huffman table that fills a code length ------------------------------------------------------------------------------
def _full_table(length, full=True):
    """A one-block gray stream whose DC and AC tables have one code at each length below `length` and two at it, the
    last all ones (or, with full=False, one code there)."""
    counts = [0] * 16
    counts[:length - 1] = [1] * (length - 1)
    counts[length - 1] = 2 if full else 1
    n = sum(counts)
    dc = (bytes(counts), bytes(range(n)))
    ac = (bytes(counts), bytes(range(n)))
    planes = S._zeros("gray", 8, 8)                              # DC category 0 and EOB: both tables' first codes
    return JW.write(planes, height=8, width=8, qtables=[S._q(1)], huff={(0, 0): dc, (1, 0): ac}).data


@pytest.mark.parametrize("length", [1, 9, 16])
def test_a_full_code_length_is_refused_as_libjpeg_refuses_it(length, monkeypatch):
    data = _full_table(length)
    with pytest.raises(OSError):
        JC.pillow(data)
    assert JC.cv2.imdecode(np.frombuffer(data, np.uint8), JC.cv2.IMREAD_COLOR) is None
    p = jpeg.probe(data)
    assert not p.supported and p.reason == "bad Huffman table (full at length %d: a code of all ones)" % length
    import fakelib_jpeg
    fake = fakelib_jpeg.install(monkeypatch)
    ok = JC.pil(JC.picture(16, 16, 1))
    calls = [lambda: jpeg.decode([ok, data]), lambda: P.imagenet([ok, data]),
             lambda: P.voc_segmentation([ok, data], [np.zeros((16, 16), np.uint8), np.zeros((8, 8), np.uint8)]),
             lambda: P.ssd([ok, data])]
    for call in calls:
        with pytest.raises(_lib.DfqError, match=r"\[1\]: bad Huffman table \(full at length"):
            call()
    assert fake.calls == []


def test_the_fullest_legal_tables_are_taken():
    """One code short of full: libjpeg takes these tables, and so does the decoder."""
    for length in (1, 9, 16):
        data = _full_table(length, full=False)
        assert jpeg.probe(data).supported, length
        assert np.array_equal(JC.pillow(data), O.decode(data))


# ---- the host path through the twin --------------------------------------------------------------------------------------------
def test_crafted_streams_decode_through_the_twin(streams, monkeypatch):
    import fakelib_jpeg
    fake = fakelib_jpeg.install(monkeypatch)
    items = [d for _, d in streams]
    outs = jpeg.decode(items)
    for (name, d), o in zip(streams, outs):
        assert np.array_equal(o.numpy(), JC.pillow(d)), name
    assert fake.calls.count("dfq_jpeg_decode") == 1
    jpeg.check()


def test_preprocess_on_crafted_bytes_through_the_twin(streams, monkeypatch):
    import fakelib_jpeg
    fakelib_jpeg.install(monkeypatch)
    pick = [d for n, d in streams if not n.startswith("geo_")] + [d for n, d in streams if n.startswith("geo_")][::9]
    arrays = [JC.pillow(d) for d in pick]
    labels = [np.full(a.shape[:2], k % 21, np.uint8) for k, a in enumerate(arrays)]
    assert torch.equal(P.imagenet(pick, resize=36, crop=32), P.imagenet(arrays, resize=36, crop=32))
    x, y = P.voc_segmentation(pick, labels, crop_size=33)
    xa, ya = P.voc_segmentation(arrays, labels, crop_size=33)
    assert torch.equal(x, xa) and torch.equal(y, ya)
    s, sz = P.ssd(pick, size=30)
    sa, sza = P.ssd(arrays, size=30)
    assert torch.equal(s, sa) and torch.equal(sz, sza)
    jpeg.check()
