"""dfq_b200.preprocess on the CPU: the oracle of tests/preprocess_oracle.py byte for byte against Pillow, OpenCV and
torchvision over the size grid, against the fixture tests/golden/ref_preprocess.npz (made by the reference's own transform
classes) and live against those classes where the reference checkout is present; the product's vectorised tap tables
against the oracle's literal ones; the host path (packing, shared tables, descriptors, label tables) through the twin of
tests/fakelib_preprocess.py; and every refusal, which comes before any device work."""
import hashlib
import os
import sys

import cv2
import numpy as np
import pytest
import torch
from PIL import Image
from torchvision import transforms

from dfq_b200 import _lib, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fakelib_preprocess  # noqa: E402
import preprocess_cases as PC  # noqa: E402
import preprocess_oracle as O  # noqa: E402

REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_preprocess.npz")
CASES = PC.cases()
IDS = [c[0] for c in CASES]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


# ---- the resamplers against the libraries ------------------------------------------------------------------------------
RESIZES = [(1, 1, 300, 300), (2, 5, 300, 300), (17, 23, 300, 300), (299, 301, 300, 300), (300, 300, 300, 300),
           (224, 224, 256, 256), (375, 500, 341, 256), (500, 375, 256, 341), (333, 500, 684, 513), (281, 500, 455, 256),
           (2000, 1200, 513, 855), (1000, 1500, 300, 300), (5, 2, 7, 300), (600, 800, 300, 300), (300, 300, 513, 513)]


@pytest.mark.parametrize("h,w,ow,oh", RESIZES)
def test_resamplers_match_pillow_and_opencv(h, w, ow, oh):
    img = PC.image(h, w, seed=h * 7 + w)
    lab = PC.label(h, w, seed=h + w)
    assert np.array_equal(O.pil_bilinear(img, ow, oh), np.asarray(Image.fromarray(img).resize((ow, oh), Image.BILINEAR)))
    assert np.array_equal(O.pil_nearest(lab, ow, oh), np.asarray(Image.fromarray(lab).resize((ow, oh), Image.NEAREST)))
    assert np.array_equal(O.cv_linear(img, ow, oh), cv2.resize(img, (ow, oh)))


def test_opencv_enlargement_keeps_the_border_row_coefficients():
    """Where a row tap reaches past the border, OpenCV reads the border row twice with the unclamped (1 - fy, fy); clamping
    fy to 0 there, as the columns do, differs from cv2 on enlargements."""
    img = PC.image(17, 23, seed=3)
    clamped = O.cv_coeffs(17, 300, True)
    hx = np.stack([img[:, s0].astype(np.int64) * c0 + img[:, s1].astype(np.int64) * c1
                   for s0, s1, c0, c1 in O.cv_coeffs(23, 300, True)], 1)
    wrong = np.clip(np.stack([((((hx[s0] >> 4) * b0) >> 16) + (((hx[s1] >> 4) * b1) >> 16) + 2) >> 2
                              for s0, s1, b0, b1 in clamped]), 0, 255).astype(np.uint8)
    ref = cv2.resize(img, (300, 300))
    assert np.array_equal(O.cv_linear(img, 300, 300), ref) and not np.array_equal(wrong, ref)


@pytest.mark.parametrize("name,img,lab", CASES, ids=IDS)
def test_oracle_matches_torchvision_and_the_libraries(name, img, lab):
    cls = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224), transforms.ToTensor(),
                              transforms.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))])
    assert np.array_equal(O.imagenet(img), cls(Image.fromarray(img)).numpy())
    want = cv2.resize(img, (300, 300)).astype(np.float32) - np.array([127, 127, 127], np.float32)
    assert np.array_equal(O.ssd(img), (want / 128.0).transpose(2, 0, 1))


@pytest.mark.parametrize("name,img,lab", CASES, ids=IDS)
def test_oracle_matches_the_reference_fixture(name, img, lab):
    g = np.load(GOLD)
    assert _sha(O.imagenet(img)) == g["cls_" + name]
    s, l = O.voc_segmentation(img, lab)
    assert _sha(s) == g["seg_" + name] and _sha(l) == g["seglab_" + name]
    assert _sha(O.ssd(img, mean=(127, 127, 127))) == g["ssd_" + name]


def test_fixture_covers_the_grid():
    assert list(np.load(GOLD)["names"]) == IDS


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "dataset", "segmentation", "custom_transforms.py")),
                    reason="reference checkout not present")
@pytest.mark.parametrize("hw", [(17, 23), (375, 500), (500, 337), (513, 515), (2, 5)])
def test_oracle_matches_the_reference_classes_live(hw):
    sys.path.insert(0, REF)
    try:
        import dataset.segmentation.custom_transforms as tr
        from modeling.detection.data_preprocessing import PredictionTransform
    finally:
        sys.path.remove(REF)
    img, lab = PC.image(*hw, seed=99), PC.label(*hw, seed=99)
    seg = transforms.Compose([tr.FixScaleCrop(crop_size=513), tr.Normalize(mean=(0.485, 0.456, 0.406),
                                                                              std=(0.229, 0.224, 0.225)), tr.ToTensor()])
    s = seg({"image": Image.fromarray(img), "label": Image.fromarray(lab)})
    mine, mlab = O.voc_segmentation(img, lab)
    assert np.array_equal(mine, s["image"].numpy()) and np.array_equal(mlab, s["label"].numpy())
    for mean in (127.0, (123.0, 117.0, 104.0)):
        want = PredictionTransform(300, np.array(mean), 128.0)(img).numpy()
        assert np.array_equal(O.ssd(img, mean=mean), want)


def test_each_normalisation_rule_matters():
    """Rounding through fp64 (segmentation) and the fp32 chain (torchvision) differ on some values: the two rules are
    distinct and each is pinned by the fixture."""
    u = np.arange(256, dtype=np.float32) / np.float32(255)
    m, s = 0.456, 0.224
    f32 = (u - np.float32(m)) / np.float32(s)
    f64 = ((u.astype(np.float64) - m).astype(np.float32).astype(np.float64) / s).astype(np.float32)
    assert not np.array_equal(f32, f64)


# ---- the product's host tables against the oracle ----------------------------------------------------------------------
@pytest.mark.parametrize("insz,outsz", [(1, 300), (2, 5), (5, 2), (17, 300), (23, 300), (299, 300), (301, 300),
                                        (300, 300), (375, 256), (500, 341), (2000, 513), (513, 684), (1500, 300)])
def test_tap_tables_match_the_oracle(insz, outsz):
    t = P._pil_taps(insz, outsz)
    for o, (xmin, w) in enumerate(O.pil_coeffs(insz, outsz)):
        k = len(w)
        assert list(t[o, :k, 0]) == list(range(xmin, xmin + k)) and list(t[o, :k, 1]) == w
        assert (t[o, k:, 0] == xmin + k - 1).all() and (t[o, k:, 1] == 0).all()
    for clamp in (True, False):
        assert P._cv_taps(insz, outsz, clamp).reshape(-1, 4)[:, [0, 2, 1, 3]].tolist() == \
            [list(c) for c in O.cv_coeffs(insz, outsz, clamp)]
    assert P._nearest_index(insz, outsz).tolist() == O.pil_nearest_index(insz, outsz)


def test_descriptor_layout_matches_the_library():
    lib = _lib.load(build_if_missing=False)
    assert lib.dfq_struct_size(20) == -1
    for i, (dt, size) in _lib.PRE_SIZES.items():
        assert dt.itemsize == size == lib.dfq_struct_size(i)
    assert _lib.PRE_IMAGE_DT.fields["H"][1] == 48 and _lib.PRE_RESAMPLE_DT.fields["blob_bytes"][1] == 24
    assert _lib.PRE_RESAMPLE_DT.fields["mean64"][1] == 56


# ---- refusals (before any device work) ---------------------------------------------------------------------------------
_OK = np.zeros((4, 5, 3), np.uint8)


@pytest.mark.parametrize("call,msg", [
    (lambda: P.imagenet([]), "empty"),
    (lambda: P.imagenet(_OK), "list"),
    (lambda: P.imagenet([_OK.astype(np.float32)]), "uint8"),
    (lambda: P.imagenet([torch.zeros(4, 5, 3)]), "uint8"),
    (lambda: P.imagenet([_OK[..., 0]]), "3 channels"),
    (lambda: P.imagenet([np.zeros((4, 5, 4), np.uint8)]), "3 channels"),
    (lambda: P.imagenet([np.zeros((0, 5, 3), np.uint8)]), "empty"),
    (lambda: P.imagenet([_OK], resize=0), "resize"),
    (lambda: P.imagenet([_OK], crop=-1), "crop"),
    (lambda: P.imagenet([_OK], std=(0.2, 0.0, 0.2)), "std"),
    (lambda: P.imagenet([_OK], resize=200, crop=224), "pad"),
    (lambda: P.voc_segmentation([_OK], [np.zeros((4, 6), np.uint8)]), "labels\\[0\\]"),
    (lambda: P.voc_segmentation([_OK], [np.zeros((4, 5), np.int64)]), "uint8"),
    (lambda: P.voc_segmentation([_OK], [_OK[..., 0]] * 2), "2 labels"),
    (lambda: P.voc_segmentation([_OK], crop_size=0), "crop_size"),
    (lambda: P.ssd([_OK], size=0), "size"),
    (lambda: P.ssd([_OK], std=0.0), "std"),
    (lambda: P.ssd([_OK], std=(1.0, 2.0, 3.0)), "Python number"),
    (lambda: P.ssd([_OK], mean=(1.0, 2.0)), "mean"),
    (lambda: P.ssd([_OK], mean=np.array([1.0, 2.0])), "mean"),
    (lambda: P.ssd([_OK], mean=None), "mean"),
    (lambda: P.ssd([_OK], mean="abc"), "mean"),
    (lambda: P.ssd([_OK], std=np.float64(128.0)), "Python number"),
    (lambda: P.imagenet([_OK], mean=np.zeros((2, 2))), "mean"),
    (lambda: P.voc_segmentation([_OK], mean=np.array([0.5, 0.4, 0.3], np.float32)), "float64"),
])
def test_refusals(call, msg):
    with pytest.raises(_lib.DfqError, match=msg):
        call()


# ---- the host path through the twin ------------------------------------------------------------------------------------
def _batch(n, seed):
    g = np.random.default_rng(seed)
    hw = [(300, 400), (17, 23), (300, 400)] + [(int(g.integers(40, 700)), int(g.integers(40, 700))) for _ in range(n - 3)]
    return [PC.image(h, w, seed + i) for i, (h, w) in enumerate(hw)], [PC.label(h, w, seed + i) for i, (h, w) in enumerate(hw)]


def test_host_path_packs_the_batch_for_the_kernel(monkeypatch):
    fake = fakelib_preprocess.install(monkeypatch)
    imgs, labs = _batch(6, 5)
    cls = P.imagenet(imgs, resize=160, crop=128)
    assert fake.calls == ["dfq_host_copy_segments", "dfq_pre_resample"]
    ims, d = fake.descriptors
    assert (int(d["n"]), int(d["out_h"]), int(d["out_w"]), int(d["filter"]), int(d["norm"])) == \
        (6, 128, 128, _lib.PRE_PIL_BILINEAR, _lib.PRE_NORM_F32)
    assert [tuple(m) for m in ims[["H", "W"]]] == [a.shape[:2] for a in imgs]
    offs = np.concatenate([ims[k] for k in ("src", "xtap", "ytap")])
    assert (offs % 64 == 0).all() and (ims["label"] == -1).all() and (ims["xnear"] == -1).all()
    assert ims["xtap"][0] == ims["xtap"][2] and ims["ytap"][0] == ims["ytap"][2] != ims["ytap"][1]   # shared by size
    assert len(set(ims["src"])) == 6 and int(d["blob_bytes"]) >= ims["src"].max() + 300 * 400 * 3
    for i, img in enumerate(imgs):
        assert np.array_equal(cls[i].numpy(), O.imagenet(img, 160, 128))


def test_host_path_segmentation_with_labels(monkeypatch):
    fake = fakelib_preprocess.install(monkeypatch)
    imgs, labs = _batch(5, 6)
    seg, lab = P.voc_segmentation(imgs, [torch.from_numpy(l) for l in labs], crop_size=65)
    ims, d = fake.descriptors
    assert int(d["norm"]) == _lib.PRE_NORM_F64 and (ims["label"] >= 0).all() and (ims["label"] % 64 == 0).all()
    assert ims["xnear"][0] == ims["xnear"][2] and ims["ynear"][0] == ims["ynear"][2]
    for i, img in enumerate(imgs):
        want, wlab = O.voc_segmentation(img, labs[i], 65)
        assert np.array_equal(seg[i].numpy(), want) and np.array_equal(lab[i].numpy(), wlab)
    assert (lab == 255).any()


@pytest.mark.parametrize("mean", [127.0, (123.0, 117.0, 104.0), np.array([127, 127, 127]), np.array([123, 117, 104])])
def test_host_path_ssd_with_the_configs_means(monkeypatch, mean):
    """The reference's configs give image_mean as an int64 numpy array and image_std as a float."""
    fakelib_preprocess.install(monkeypatch)
    imgs, _ = _batch(4, 7)
    for std in (128.0, 1.0):
        x, sizes = P.ssd(imgs, mean=mean, std=std)
        assert sizes.tolist() == [[a.shape[1], a.shape[0]] for a in imgs]
        for i, img in enumerate(imgs):
            want = (cv2.resize(img, (300, 300)).astype(np.float32) - np.array(mean, np.float32)) / std
            assert np.array_equal(x[i].numpy(), want.transpose(2, 0, 1)) and np.array_equal(x[i].numpy(), O.ssd(img, 300, mean, std))


def test_numpy_means_and_stds_match_tuples(monkeypatch):
    fakelib_preprocess.install(monkeypatch)
    imgs, labs = _batch(3, 8)
    m, s = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    assert torch.equal(P.imagenet(imgs, mean=np.array(m), std=np.array(s)), P.imagenet(imgs))
    a, la = P.voc_segmentation(imgs, labs, 65, mean=np.array(m), std=np.array(s))
    b, lb = P.voc_segmentation(imgs, labs, 65)
    assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.parametrize("field,value,reason", [
    ("H", 0, "image outside"), ("xk", 0, "bad taps"), ("xk", 4097, "bad taps"), ("src", 10 ** 12, "image outside"),
    ("xtap", 4, "image outside"), ("yk", 0, "bad taps")])
def test_twin_refuses_what_the_library_refuses(monkeypatch, field, value, reason):
    """The descriptor checks of dfq_pre_resample, reached by corrupting one field of a packed batch."""
    fake = fakelib_preprocess.install(monkeypatch)
    imgs, _ = _batch(3, 9)
    call = fake.dfq_pre_resample

    def corrupt(d_p, im_p, *rest):
        ims = _lib_table(im_p, 3)
        ims[1][field] = value
        return call(d_p, im_p, *rest)
    fake.dfq_pre_resample = corrupt
    with pytest.raises(_lib.DfqError, match="dfq_pre_resample"):
        P.imagenet(imgs, resize=64, crop=64)
    assert reason.split()[0] in fake.refusals[-1]


def _lib_table(ptr, n):
    import ctypes as C
    p = int(ptr.value if isinstance(ptr, C.c_void_p) else ptr)
    buf = (C.c_char * (n * _lib.PRE_IMAGE_DT.itemsize)).from_address(p)
    return np.frombuffer(buf, _lib.PRE_IMAGE_DT)
