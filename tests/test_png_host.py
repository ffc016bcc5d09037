"""PNG label decoding, host side: the Pillow behaviour the decoder follows, pinned on crafted streams; tests/png_oracle.py
equal to Pillow over the corpus; the chunk walk's refusals, each by name, through probe, decode and voc_segmentation
before any copy or launch; and the product's host path (joined streams, work rooms and labels placed past the copied
bytes, mixed batches, the device error word) through the host twin of tests/fakelib_png.py."""
import io
import os
import re
import struct
import sys
import zlib

import numpy as np
import pytest
import torch
from PIL import Image, UnidentifiedImageError

from dfq_b200 import _lib, jpeg, png, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_corpus as PC  # noqa: E402
import png_oracle as O  # noqa: E402
import png_writer as W  # noqa: E402


@pytest.fixture(scope="module")
def corpus():
    return PC.corpus(big=False)


# ---- the Pillow contract --------------------------------------------------------------------------------------------------
def _small():
    img = PC._noise(2, 4, 3)
    return img, W.filter_rows(img, (0,))


@pytest.mark.parametrize("size", [(2, 4), (1000, 1000)])
def test_pillow_rejects_a_wrong_adler_when_the_data_ends_at_the_last_row(size):
    img = np.zeros(size, np.uint8)
    raw = W.filter_rows(img, (0,))
    with pytest.raises(OSError, match="broken data stream"):
        PC.pillow(W.png(*size, W.zlib([("dynamic", W.lz77(raw))], raw, adler=b"\0\0\0\1")))


def test_pillow_takes_a_missing_or_partial_trailer_and_bytes_after_it():
    img, raw = _small()
    full = W.zlib([("fixed", list(raw))], raw)
    for s in (full[:-4], full[:-2], full + b"\x01\x02\x03"):
        assert np.array_equal(PC.pillow(W.png(2, 4, s)), img)


def test_pillow_ignores_what_follows_the_last_row():
    img, raw = _small()
    more = W.zlib([("fixed", list(raw) + [9, (3, 1)])], raw, adler=b"\0\0\0\0")
    assert np.array_equal(PC.pillow(W.png(2, 4, more)), img)
    for name, data in PC.accepted_edges():
        assert np.array_equal(PC.pillow(data), O.decode(data)), name


def test_pillow_keeps_the_rows_a_whole_stream_reaches_and_leaves_the_rest_zero():
    for name, data, taken in PC._rows_end():
        if taken is True:
            got = PC.pillow(data)
            rows = int(name.split("_")[2])
            assert (got[rows:] == 0).all() and np.array_equal(got, O.decode(data)), name
        else:
            with pytest.raises(OSError):
                PC.pillow(data)


def test_pillow_rejects_short_data_and_filter_5():
    img, raw = _small()
    with pytest.raises(OSError, match="truncated"):
        PC.pillow(W.png(2, 4, W.zlib([("fixed", list(raw[:-1]))], raw[:-1])))
    bad = bytes([5]) + raw[1:]
    with pytest.raises(OSError):
        PC.pillow(W.png(2, 4, W.zlib([("fixed", list(bad))], bad)))


def test_pillow_checks_header_crcs_not_idat_crcs_and_needs_no_iend():
    img, raw = _small()
    good = W.png(2, 4, W.zlib([("fixed", list(raw))], raw))
    assert np.array_equal(PC.pillow(PC._bad_idat_crc(good)), img)
    assert np.array_equal(PC.pillow(good[:-12]), img)
    bad = bytearray(good)
    bad[8 + 8 + 13] ^= 1
    with pytest.raises(UnidentifiedImageError):
        PC.pillow(bytes(bad))
    assert png.probe(bytes(bad)).reason.startswith("corrupt header chunk (bad CRC in IHDR)")


def test_pillow_returns_palette_indices_and_gray_as_uint8():
    a = PC.voc_label(30, 40, 1)
    for data, mode in ((PC.pil_p(a), "P"), (PC.cv_gray(a), "L")):
        assert Image.open(io.BytesIO(data)).mode == mode
        got = PC.pillow(data)
        assert got.dtype == np.uint8 and np.array_equal(got, a)


def test_every_corrupt_stream_is_one_pillow_rejects():
    for name, data, why in PC.corrupt_streams():
        assert png.probe(data).supported, name
        with pytest.raises(OSError):
            PC.pillow(data)
        H, Wd = png.probe(data).height, png.probe(data).width
        raw, got = O.inflate(png._parse(data).stream, H, Wd)
        if not got:
            got = O.unfilter(raw, H, Wd)[1]
        assert got == why, name


def test_oracle_equals_pillow_on_the_corpus(corpus):
    for name, data in corpus:
        assert np.array_equal(O.decode(data), PC.pillow(data)), name
    assert len(corpus) > 150


def test_product_parser_reads_the_corpus(corpus):
    for name, data in corpus:
        p = png.probe(data)
        assert p.supported, (name, p.reason)
        assert (p.height, p.width) == PC.pillow(data).shape, name
        assert p.colour_type == (3 if name.startswith("pil") or name == "palette_writer" else 0), name


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def _header(data, **kw):
    """data with its IHDR fields replaced (and its CRC recomputed)."""
    W_, H_, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", data[16:29])
    f = dict(W=W_, H=H_, depth=depth, ctype=ctype, comp=comp, filt=filt, inter=inter)
    f.update(kw)
    body = struct.pack(">IIBBBBB", f["W"], f["H"], f["depth"], f["ctype"], f["comp"], f["filt"], f["inter"])
    return data[:8] + W.chunk(b"IHDR", body) + data[33:]


def _refusals():
    a = PC.voc_label(24, 40, 3)
    base = PC.pil_p(a)
    gray = PC.cv_gray(a)
    b = io.BytesIO()
    Image.fromarray(np.dstack([a, a, a])).save(b, "PNG")
    rgb = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(np.dstack([a, a, a, a])).save(b, "PNG")
    rgba = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(np.dstack([a, a])).convert("LA").save(b, "PNG")
    la = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(a.astype(np.uint16) * 200).save(b, "PNG")
    i16 = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(a > 0).save(b, "PNG")
    bilevel = b.getvalue()
    b = io.BytesIO()
    Image.fromarray(a).convert("P").save(b, "PNG", bits=4)
    p4 = b.getvalue()
    stream = zlib.compress(W.filter_rows(a, (0,)))
    idat = [k for k in range(len(gray)) if gray[k:k + 4] == b"IDAT"][0] - 4
    yield "not a PNG", b"\xff\xd8\xff\xe0" + base[4:], "not a PNG"
    yield "truncated", base[:len(base) // 2], "truncated"
    yield "bad IHDR CRC", base[:29] + bytes([base[29] ^ 1]) + base[30:], "bad CRC"
    yield "bad PLTE CRC", _flip_crc(base, b"PLTE"), "bad CRC"
    yield "RGB", rgb, "RGB"
    yield "RGBA", rgba, "RGBA"
    yield "gray+alpha", la, "gray+alpha"
    yield "16-bit", i16, "16-bit"
    yield "1-bit gray", bilevel, "gray below 8 bits"
    yield "4-bit palette", p4, "palette below 8 bits"
    yield "interlaced", _header(gray, inter=1), "interlaced"
    yield "APNG", gray[:33] + W.chunk(b"acTL", b"\0\0\0\1\0\0\0\0") + gray[33:], "APNG"
    yield "compression 1", _header(gray, comp=1), "compression method"
    yield "filter method 1", _header(gray, filt=1), "filter method"
    yield "no IDAT", gray[:idat] + W.chunk(b"IEND", b""), "no IDAT"
    yield "split IDATs", W.SIG + W.ihdr(24, 40) + W.chunk(b"IDAT", stream[:10]) + W.chunk(b"tEXt", b"a\0b") + W.chunk(b"IDAT", stream[10:]) \
        + W.chunk(b"IEND", b""), "not consecutive"
    yield "zlib header", W.png(24, 40, b"\x78\x9d" + stream[2:]), "zlib header"
    yield "zlib method", W.png(24, 40, b"\x79\x9c" + stream[2:]), "zlib header"
    yield "zlib window", W.png(24, 40, bytes([0x88, (31 - (0x88 << 8) % 31) % 31]) + stream[2:]), "zlib header"
    yield "preset dictionary", W.png(24, 40, bytes([0x78, 0x20 + (31 - ((0x78 << 8) + 0x20) % 31) % 31]) + stream[2:]), \
        "preset dictionary"
    yield "bomb", _header(gray, W=20000, H=5000), "decompression-bomb"


def _flip_crc(data, cid):
    i = data.index(cid)
    n = int.from_bytes(data[i - 4:i], "big")
    b = bytearray(data)
    b[i + 4 + n] ^= 0xFF
    return bytes(b)


@pytest.mark.parametrize("case", list(_refusals()), ids=lambda c: c[0])
def test_every_unsupported_stream_is_refused_by_name(case, monkeypatch):
    name, data, reason = case
    if name in ("RGB", "RGBA", "gray+alpha", "16-bit", "1-bit gray", "4-bit palette"):
        PC.pillow(data)                                   # a real stream Pillow reads, not a broken one
    p = png.probe(data)
    assert not p.supported and reason in p.reason, (name, p.reason)
    import fakelib_png
    fake = fakelib_png.install(monkeypatch)
    ok = PC.pil_p(PC.voc_label(24, 40, 3))
    img = np.zeros((24, 40, 3), np.uint8)
    with pytest.raises(_lib.DfqError, match=r"\[1\]: .*" + re.escape(reason.split()[0])):
        png.decode([ok, data])
    with pytest.raises(_lib.DfqError, match=r"labels\[1\]: .*" + re.escape(reason.split()[0])):
        P.voc_segmentation([img, img], [ok, data], crop_size=16)
    assert "dfq_png_decode" not in fake.calls and "dfq_host_copy_segments" not in fake.calls


def test_png_images_stay_refused_and_a_label_of_the_wrong_size_is_refused_before_any_copy(monkeypatch):
    import fakelib_png
    fake = fakelib_png.install(monkeypatch)
    lab = PC.pil_p(PC.voc_label(24, 40, 3))
    with pytest.raises(_lib.DfqError, match=r"images\[0\]: not a JPEG"):
        P.voc_segmentation([lab], [lab])
    with pytest.raises(_lib.DfqError, match=r"labels\[0\] is \(24, 40\), images\[0\] is \(25, 40\)"):
        P.voc_segmentation([np.zeros((25, 40, 3), np.uint8)], [lab], crop_size=16)
    with pytest.raises(_lib.DfqError, match=r"labels\[0\] must be a numpy array, a CPU tensor or PNG bytes, got list"):
        P.voc_segmentation([np.zeros((25, 40, 3), np.uint8)], [[1]], crop_size=16)
    assert fake.calls.count("dfq_host_copy_segments") == 0 and "dfq_png_decode" not in fake.calls
    assert png.probe(42).reason == "not bytes (int)"


# ---- the host path through the twin ------------------------------------------------------------------------------------------
def _labels():
    return [PC.pil_p(PC.voc_label(31, 45, 1)), PC.cv_gray(PC.voc_label(40, 33, 2)),
            PC.pil_p(PC.voc_label(52, 39, 3), compress_level=0), W.image_png(PC._noise(33, 47, 4), filters=(0, 1, 2, 3, 4))]


def test_decode_through_the_twin(monkeypatch, corpus):
    fake = fakelib_png_install(monkeypatch)
    items = [d for _, d in corpus[:40]]
    outs = png.decode(items)
    for d, o in zip(items, outs):
        assert o.dtype == torch.uint8 and np.array_equal(o.numpy(), PC.pillow(d))
    assert fake.calls.count("dfq_host_copy_segments") == 1 and fake.calls.count("dfq_png_decode") == 1
    ims, d = fake.png_descriptors
    assert len(ims) == len(items) and int(d["n"]) == len(items)
    total = int(ims["src_end"].max())
    assert (ims["work"] >= total).all() and (ims["dst"] >= total).all() and (ims["work"] % 64 == 0).all()
    png.check()


def fakelib_png_install(monkeypatch):
    import fakelib_png
    return fakelib_png.install(monkeypatch)


@pytest.mark.parametrize("order", ["bytes", "mixed"])
def test_segmentation_on_png_labels_equals_segmentation_on_arrays(monkeypatch, order):
    import jpeg_corpus as JC
    fake = fakelib_png_install(monkeypatch)
    labels = _labels()
    arrays = [PC.pillow(d) for d in labels]
    jpgs = [JC.pil(JC.picture(a.shape[0], a.shape[1], k), quality=90) for k, a in enumerate(arrays)]
    imgs = [JC.pillow(d) for d in jpgs]
    images = jpgs
    if order == "mixed":
        labels = [labels[0], arrays[1], labels[2], arrays[3]]
        images = [jpgs[0], jpgs[1], imgs[2], imgs[3]]
    x, y = P.voc_segmentation(images, labels, crop_size=29)
    (pre, _), (ims, d), jdesc = fake.descriptors, fake.png_descriptors, fake.jpeg_descriptors[0]
    xa, ya = P.voc_segmentation(imgs, arrays, crop_size=29)
    assert torch.equal(x, xa) and torch.equal(y, ya)
    assert len(ims) == (4 if order == "bytes" else 2)
    coded = [i for i, l in enumerate(labels) if isinstance(l, bytes)]
    assert sorted(pre["label"][coded].tolist()) == sorted(ims["dst"].tolist())   # the resample reads the decoded labels
    ends = [int(j["dst"]) + int(j["H"]) * int(j["W"]) * 3 for j in jdesc]
    assert int(ims["work"].min()) >= max(ends)                                 # the PNG room follows the JPEG room
    assert fake.calls.count("dfq_host_copy_segments") == 2
    png.check()
    jpeg.check()


def test_corrupt_streams_are_reported_by_check_and_the_rest_decodes(monkeypatch):
    fakelib_png_install(monkeypatch)
    good = _labels()
    for name, data, why in PC.corrupt_streams()[:6]:
        outs = png.decode(good[:2] + [data] + good[2:])
        for d, o in zip(good[:2], outs[:2]):
            assert np.array_equal(o.numpy(), PC.pillow(d))
        for d, o in zip(good[2:], outs[3:]):
            assert np.array_equal(o.numpy(), PC.pillow(d))
        with pytest.raises(_lib.DfqError, match="image 2 of decode call 1 of 1 .*" + png._ERRORS[why]):
            png.check()
        png.check()                                        # the word was cleared


def test_struct_mirrors_match_the_library():
    lib = _lib.load()
    for i, (dt, size) in _lib.PNG_SIZES.items():
        assert lib.dfq_struct_size(i) == dt.itemsize == size, dt
    assert _lib.PNG_IMAGE_DT.fields["H"][1] == 32 and _lib.PNG_DECODE_DT.fields["call"][1] == 16


def test_library_refuses_bad_descriptors():
    """dfq_png_decode's argument checks run on the host, before any CUDA call."""
    import ctypes as C
    lib = _lib.load()
    err = np.zeros(2, np.int64)
    blob = np.zeros(1 << 16, np.uint8)
    d = np.zeros(1, _lib.PNG_DECODE_DT)
    d["n"], d["blob_bytes"] = 1, blob.nbytes
    im = np.zeros(1, _lib.PNG_IMAGE_DT)
    im["src"], im["src_end"], im["work"], im["dst"], im["H"], im["W"] = 0, 100, 1024, 4096, 16, 16

    def call():
        return lib.dfq_png_decode(_lib.table_ptr(d), _lib.table_ptr(im), C.c_void_p(blob.ctypes.data),
                                  C.c_void_p(err.ctypes.data), None)

    for field, value, why in ((im, ("H", 0), "image 0"), (im, ("src_end", 1), "image 0"), (im, ("dst", 1 << 20), "image 0"),
                              (im, ("work", 50), "image 0"), (im, ("dst", 1100), "image 0"), (d, ("n", 0), "n must be")):
        old = field[value[0]].copy()
        field[value[0]] = value[1]
        assert call() == -1
        assert why in lib.dfq_last_error().decode(), lib.dfq_last_error()
        field[value[0]] = old
