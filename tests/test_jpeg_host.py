"""JPEG decoding, host side: tests/jpeg_oracle.py byte-equal to Pillow and to OpenCV over the seeded corpus; the header
parser's refusals, each by name; the table builder against libjpeg's rules; and the product's host path (batch packing,
tables, restart-interval segments, decoded images' places, mixed batches, the device error word) through the host twin
of tests/fakelib_jpeg.py."""
import io
import os
import struct
import sys

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from dfq_b200 import _lib, jpeg, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus as JC  # noqa: E402
import jpeg_oracle as O  # noqa: E402


@pytest.fixture(scope="module")
def corpus():
    return JC.corpus()


def test_oracle_equals_pillow_and_opencv_on_the_corpus(corpus):
    names = set()
    for name, data in corpus:
        want = JC.pillow(data)
        assert np.array_equal(JC.opencv(data), want), name
        assert np.array_equal(O.decode(data), want), name
        names.add(name)
    assert len(names) == len(corpus) > 150


def test_product_parser_reads_the_corpus(corpus):
    for name, data in corpus:
        p = jpeg.probe(data)
        assert p.supported, (name, p.reason)
        H, W = JC.pillow(data).shape[:2]
        assert (p.height, p.width) == (H, W), name
        if "gray" in name:
            assert p.sampling == "gray" and p.components == 1
        elif name.split("_")[1] in JC.SUBSAMPLING:
            assert p.sampling == {"444": "4:4:4", "422": "4:2:2", "420": "4:2:0"}[name.split("_")[1]], name
        if "rst" in name:
            assert p.restart_interval > 0, name


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def _base(**kw):
    return JC.pil(JC.picture(24, 40, 3), quality=80, **kw)


def _segments(data):
    """[(marker, start, end)] of the header segments, up to and including SOS."""
    out, pos = [], 2
    while True:
        m = data[pos + 1]
        ln = struct.unpack(">H", data[pos + 2:pos + 4])[0]
        out.append((m, pos, pos + 2 + ln))
        if m == 0xDA:
            return out
        pos += 2 + ln


def _patch(data, marker, offset, value):
    """data with byte `offset` of the first `marker` segment's body (after the length) set to value."""
    for m, s, e in _segments(data):
        if m == marker:
            b = bytearray(data)
            b[s + 4 + offset] = value
            return bytes(b)
    raise AssertionError("no marker 0x%02X" % marker)


def _drop(data, marker):
    for m, s, e in _segments(data):
        if m == marker:
            return data[:s] + data[e:]
    raise AssertionError


def _sof_component(data, k, byte, value):
    return _patch(data, 0xC0, 6 + 3 * k + byte, value)


def _refusals():
    base, gray = _base(), JC.pil(JC.picture(24, 40, 3)[:, :, 0], quality=80)
    b = io.BytesIO()
    Image.fromarray(JC.picture(24, 40, 3)).convert("CMYK").save(b, "JPEG")
    cmyk = b.getvalue()
    no_jfif = _drop(base, 0xE0)
    sos = [s for m, s, e in _segments(base) if m == 0xDA][0]
    adobe = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"   # APP14, transform 0
    at = sos - (len(base) - len(no_jfif))
    two_comp = _patch(gray, 0xC0, 5, 2)
    yield "not a JPEG", b"\x89PNG\r\n\x1a\n" + base[8:], "not a JPEG"
    yield "progressive", _base(progressive=True), "progressive"
    yield "lossless", base.replace(b"\xff\xc0", b"\xff\xc3", 1), "lossless"
    yield "arithmetic", base.replace(b"\xff\xc0", b"\xff\xc9", 1), "arithmetic-coded"
    yield "12-bit", _patch(base, 0xC0, 0, 12), "12-bit"
    yield "2 components", two_comp, "2 components"
    yield "CMYK", cmyk, "4 components"
    yield "Adobe RGB", no_jfif[:at] + adobe + no_jfif[at:], "Adobe transform 0"
    yield "RGB ids", _sof_component(_sof_component(_sof_component(no_jfif, 0, 0, 82), 1, 0, 71), 2, 0, 66), "RGB-coded"
    yield "4:4:0", JC.cv(JC.picture(24, 40, 3), 90, [(cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440)]), "sampling"
    yield "4:1:1", JC.cv(JC.picture(24, 40, 3), 90, [(cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411)]), "sampling"
    yield "odd chroma", _sof_component(base, 1, 1, 0x21), "sampling"
    yield "two scans", base[:-2] + base[sos:sos + 14] + b"\x00" * 4 + b"\xff\xd9", "more than one scan"
    yield "DNL", _patch(_patch(base, 0xC0, 1, 0), 0xC0, 2, 0), "DNL"
    yield "missing DQT", _drop(base, 0xDB), "missing table"
    yield "missing DHT", _drop(base, 0xC4), "missing table"
    yield "truncated", base[:len(base) * 2 // 3], "truncated"
    yield "no EOI", base[:-2], "truncated"


@pytest.mark.parametrize("case", list(_refusals()), ids=lambda c: c[0])
def test_every_unsupported_stream_is_refused_by_name(case, monkeypatch):
    name, data, reason = case
    if name in ("progressive", "CMYK", "4:4:0", "4:1:1"):
        JC.pillow(data)                                # a real stream the libraries read, not a broken one
    p = jpeg.probe(data)
    assert not p.supported and reason in p.reason, (name, p.reason)
    import fakelib_jpeg
    fake = fakelib_jpeg.install(monkeypatch)
    ok = _base()
    for call in (lambda: P.imagenet([ok, data]), lambda: jpeg.decode([ok, data])):
        with pytest.raises(_lib.DfqError, match=r"\[1\]: .*" + reason.split()[0]):
            call()
    assert "dfq_jpeg_decode" not in fake.calls and "dfq_host_copy_segments" not in fake.calls


def test_table_builder_follows_libjpeg():
    data = _base(optimize=True)
    j = jpeg._parse(data)
    t = np.frombuffer(j.tables.tobytes(), _lib.JPEG_TABLES_DT)[0]
    assert j.tables.nbytes == _lib.JPEG_TABLES_DT.itemsize == 9312 and not j.tables.flags.writeable
    (H, W, comps, q), sel, huff, ri, _ = O._segments(data)
    for c, comp in enumerate(comps):
        assert np.array_equal(t["q"][c], q[comp[3]])
        for kind, h in ((0, t["dc"][c]), (1, t["ac"][c])):
            look = huff[(kind, sel[comp[0]][kind])]
            for bits in range(0, 65536, 37):              # every code through lookahead and maxcode walk
                l, sym = look[bits]
                e = int(h["look"][bits >> 7])
                if e:
                    got = (e >> 8, e & 255)
                else:
                    got = (0, 0)
                    for n in range(10, 17):
                        if bits >> (16 - n) <= h["maxcode"][n]:
                            got = (n, int(h["vals"][(bits >> (16 - n)) + h["valoff"][n]]))
                            break
                assert got == (l, sym), (c, kind, bits)
    assert jpeg._parse(_base(optimize=True)).tables is j.tables          # one block per table set


def test_exif_orientation_is_read():
    a = Image.fromarray(JC.picture(24, 40, 3))
    ex = Image.Exif()
    ex[0x0112] = 6
    b = io.BytesIO()
    a.save(b, "JPEG", exif=ex.tobytes())
    assert jpeg.probe(b.getvalue()).orientation == 6 and jpeg.probe(_base()).orientation == 1


# ---- the host path through the twin ------------------------------------------------------------------------------------------
def _mixed_corpus():
    pick = [d for n, d in JC.corpus(big=False) if n.startswith(("7x9", "17x23", "16x16")) and "_q90" in n]
    pick += [JC.pil(JC.picture(61, 90, 1), quality=85, restart_marker_blocks=3),
             JC.pil(JC.picture(44, 70, 2), subsampling=1), JC.cv(JC.picture(50, 48, 5), 70)]
    return pick


def test_decode_through_the_twin(monkeypatch):
    fake = fakelib_jpeg_install(monkeypatch)
    items = _mixed_corpus()
    outs = jpeg.decode(items)
    for d, o in zip(items, outs):
        assert o.dtype == torch.uint8 and np.array_equal(o.numpy(), JC.pillow(d))
    assert fake.calls.count("dfq_host_copy_segments") == 1 and fake.calls.count("dfq_jpeg_decode") == 1
    ims, segs, d = fake.jpeg_descriptors
    assert len(ims) == len(items) and len(segs) > len(items)                # the restart intervals are segments
    assert len(set(ims["tables"].tolist())) < len(items)                     # table blocks are shared
    jpeg.check()


def fakelib_jpeg_install(monkeypatch):
    import fakelib_jpeg
    return fakelib_jpeg.install(monkeypatch)


@pytest.mark.parametrize("order", ["bytes", "mixed"])
def test_preprocess_on_bytes_equals_preprocess_on_arrays(monkeypatch, order):
    fake = fakelib_jpeg_install(monkeypatch)
    items = [JC.pil(JC.picture(h, w, h), quality=90, subsampling=s) for h, w, s in ((40, 55, 2), (33, 47, 1), (52, 39, 0))]
    items.append(JC.pil(JC.picture(45, 45, 9)[:, :, 0], quality=70))
    arrays = [JC.pillow(d) for d in items]
    if order == "mixed":
        items = [items[0], arrays[1], items[2], arrays[3]]
    labels = [np.full(a.shape[:2], k, np.uint8) for k, a in enumerate(arrays)]
    assert torch.equal(P.imagenet(items, resize=36, crop=32), P.imagenet(arrays, resize=36, crop=32))
    x, y = P.voc_segmentation(items, labels, crop_size=33)
    xa, ya = P.voc_segmentation(arrays, labels, crop_size=33)
    assert torch.equal(x, xa) and torch.equal(y, ya)
    s, sz = P.ssd(items, size=30)
    sa, sza = P.ssd(arrays, size=30)
    assert torch.equal(s, sa) and torch.equal(sz, sza)
    # one gather, one decode and one resample per call
    assert fake.calls.count("dfq_jpeg_decode") == 3 and fake.calls.count("dfq_pre_resample") == 6
    jpeg.check()


def test_ssd_refuses_a_rotated_exif_image_and_the_others_ignore_it(monkeypatch):
    fakelib_jpeg_install(monkeypatch)
    ex = Image.Exif()
    ex[0x0112] = 8
    b = io.BytesIO()
    Image.fromarray(JC.picture(40, 50, 4)).save(b, "JPEG", exif=ex.tobytes())
    rot = b.getvalue()
    with pytest.raises(_lib.DfqError, match=r"images\[1\] has EXIF orientation 8"):
        P.ssd([_base(), rot])
    assert torch.equal(P.imagenet([rot], resize=40, crop=32), P.imagenet([JC.pillow(rot)], resize=40, crop=32))


def test_corrupt_scans_are_reported_by_check_and_the_rest_decodes(monkeypatch):
    fakelib_jpeg_install(monkeypatch)
    good = _mixed_corpus()[:3]
    bad = bytearray(JC.pil(JC.picture(64, 64, 8), quality=90))
    sos = _segments(bytes(bad))[-1][2]
    for k in range(sos + 10, len(bad) - 4, 7):
        bad[k] ^= 0x5A
        if bad[k] == 0xFF or bad[k - 1] == 0xFF:      # keep the marker structure: only the entropy-coded bits change
            bad[k] ^= 0x5A
    assert jpeg.probe(bytes(bad)).supported
    outs = jpeg.decode(good + [bytes(bad)])
    for d, o in zip(good, outs):
        assert np.array_equal(o.numpy(), JC.pillow(d))
    with pytest.raises(_lib.DfqError, match="image 3 of decode call 1"):
        jpeg.check()
    jpeg.check()                                           # the word was cleared
    cut = JC.pil(JC.picture(64, 64, 8), quality=90)
    short = cut[:sos + 40] + b"\xff\xd9"                  # EOI long before the last MCU
    assert jpeg.probe(short).supported
    jpeg.decode([short])
    with pytest.raises(_lib.DfqError, match="scan ends before its last MCU|invalid Huffman code"):
        jpeg.check()


def test_struct_mirrors_match_the_library():
    lib = _lib.load()
    for i, (dt, size) in _lib.JPEG_SIZES.items():
        assert lib.dfq_struct_size(i) == dt.itemsize == size, dt
    assert _lib.JPEG_IMAGE_DT.fields["H"][1] == 16 and _lib.JPEG_SEGMENT_DT.fields["image"][1] == 16
    assert _lib.JPEG_TABLES_DT.fields["dc"][1] == 768 and _lib.JPEG_HUFF_DT.fields["look"][1] == 144


def test_library_refuses_bad_descriptors():
    """dfq_jpeg_decode's argument checks run on the host, before any CUDA call."""
    import ctypes as C
    lib = _lib.load()
    err = np.zeros(2, np.int64)
    blob = np.zeros(1 << 16, np.uint8)
    d = np.zeros(1, _lib.JPEG_DECODE_DT)
    d["n"], d["nseg"], d["blob_bytes"] = 1, 1, blob.nbytes
    im = np.zeros(1, _lib.JPEG_IMAGE_DT)
    im["H"], im["W"], im["ncomp"], im["hs"], im["vs"], im["mcux"], im["mcuy"], im["dst"] = 16, 16, 3, 2, 2, 1, 1, 20000
    sg = np.zeros(1, _lib.JPEG_SEGMENT_DT)
    sg["begin"], sg["end"], sg["mcus"] = 10000, 10100, 1

    def call():
        return lib.dfq_jpeg_decode(_lib.table_ptr(d), _lib.table_ptr(im), _lib.table_ptr(sg),
                                   C.c_void_p(blob.ctypes.data + (-blob.ctypes.data % 8)), C.c_void_p(err.ctypes.data), None)

    for field, value, why in ((im, ("vs", 3), "geometry"), (im, ("mcux", 2), "geometry"), (im, ("dst", 1 << 20), "geometry"),
                              (sg, ("end", 1 << 20), "segment 0"), (sg, ("mcus", 2), "segment 0"),
                              (sg, ("image", 1), "segment 0"), (d, ("n", 0), "n must be")):
        old = field[value[0]].copy()
        field[value[0]] = value[1]
        assert call() == -1
        assert why in lib.dfq_last_error().decode(), lib.dfq_last_error()
        field[value[0]] = old
