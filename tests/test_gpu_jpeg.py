"""dfq_b200.jpeg on the H100: jpeg.decode torch.equal to Pillow (and so to OpenCV, which the host tests show equal) on
every entry of the seeded corpus; mixed batches of 1, 7, 64 and 256 streams of mixed sizes and samplings, bytes mixed with
arrays, through all three preprocess functions; one host-to-device copy, one decode and one resample entry and no host synchronisation per call; bit-flipped
and cut-short scans refused on the host or reported by jpeg.check() with the rest of the batch intact; and the chained
affine MobileNetV2, DeepLab-v3+ and SSD-Lite fed from bytes giving what they give fed from decoded arrays."""
import os
import sys

import numpy as np
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from dfq_b200 import _lib, jpeg, preprocess as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_corpus as JC  # noqa: E402

pytestmark = pytest.mark.gpu


def _stream(i, g):
    """A seeded stream of a random size, sampling, quality and encoder."""
    h, w = int(g.integers(40, 700)), int(g.integers(40, 700))
    a = JC.picture(h, w, i)
    kind = i % 6
    if kind == 4:
        return JC.pil(a[:, :, 2], quality=int(g.integers(30, 100)))
    if kind == 5:
        return JC.cv(a, int(g.integers(30, 100)))
    extra = {"restart_marker_blocks": int(g.integers(1, 9))} if i % 4 == 3 else {}
    return JC.pil(a, quality=int(g.integers(30, 100)), subsampling=kind % 3, **extra)


def _batch(n, seed):
    g = np.random.default_rng(seed)
    items = [_stream(seed * 1000 + i, g) for i in range(n)]
    arrays = [JC.pillow(d) for d in items]
    labels = [np.asarray((np.arange(a.shape[1])[None, :] // 9 + np.zeros((a.shape[0], 1), int)) % 21, np.uint8)
              for a in arrays]
    return items, arrays, labels


def test_decode_equals_pillow_on_the_whole_corpus():
    corpus = JC.corpus()
    outs = jpeg.decode([d for _, d in corpus])
    for (name, d), o in zip(corpus, outs):
        assert o.is_cuda and o.dtype == torch.uint8
        assert torch.equal(o.cpu(), torch.from_numpy(JC.pillow(d))), name
    jpeg.check()


@pytest.mark.parametrize("n,seed", [(1, 1), (7, 2), (64, 3), (256, 4)])
def test_mixed_batches_through_every_preprocess(n, seed):
    items, arrays, labels = _batch(n, seed)
    mixed = [a if i % 3 == 1 else d for i, (d, a) in enumerate(zip(items, arrays))]
    for got in (items, mixed):
        assert torch.equal(P.imagenet(got), P.imagenet(arrays))
        x, y = P.voc_segmentation(got, labels)
        xa, ya = P.voc_segmentation(arrays, labels)
        assert torch.equal(x, xa) and torch.equal(y, ya)
        s, sz = P.ssd(got, mean=np.array([127, 127, 127]), std=128.0)
        sa, sza = P.ssd(arrays, mean=np.array([127, 127, 127]), std=128.0)
        assert torch.equal(s, sa) and torch.equal(sz, sza)
    for o, a in zip(jpeg.decode(items), arrays):
        assert torch.equal(o.cpu(), torch.from_numpy(a))
    jpeg.check()


def test_ssd_on_bytes_equals_cv2_imread_decodes():
    items, _, _ = _batch(9, 5)
    arrays = [JC.opencv(d) for d in items]
    assert torch.equal(P.ssd(items)[0], P.ssd(arrays)[0])


class _HostToDevice(TorchDispatchMode):
    """Counts host-to-device copies (aten._to_copy and copy_ from a CPU tensor into a CUDA one) without the profiler, so
    the process's one profiling session stays test_gpu_preprocess.py's."""

    def __init__(self):
        super().__init__()
        self.n = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if func in (torch.ops.aten._to_copy.default, torch.ops.aten.copy_.default):
            src = args[1] if func is torch.ops.aten.copy_.default else args[0]
            self.n += src.device.type == "cpu" and out.device.type == "cuda"
        return out


class _EntryLog:
    """The library, logging the C entries called."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if not name.startswith("dfq_") or name == "dfq_last_error":
            return f

        def logged(*args):
            self.calls.append(name)
            return f(*args)
        return logged


def test_one_copy_and_no_host_synchronisation(monkeypatch):
    items, arrays, labels = _batch(16, 6)
    mixed = [a if i % 4 == 0 else d for i, (d, a) in enumerate(zip(items, arrays))]

    def calls():
        P.imagenet(mixed)
        P.voc_segmentation(mixed, labels)
        P.ssd(mixed)
        jpeg.decode(items)

    calls()
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            calls()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    log = _EntryLog(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: log)
    with _HostToDevice() as h2d:
        calls()
    torch.cuda.synchronize()
    assert h2d.n == 5                                           # one per call, and ssd's sizes
    assert log.calls == ["dfq_host_copy_segments", "dfq_jpeg_decode", "dfq_pre_resample"] * 3 + \
        ["dfq_host_copy_segments", "dfq_jpeg_decode"], log.calls
    monkeypatch.undo()
    jpeg.check()


def test_corrupt_scans_are_reported_and_the_rest_of_the_batch_is_exact():
    items, arrays, _ = _batch(12, 7)
    g = np.random.default_rng(8)
    bad = {}
    for k in (2, 5, 9):
        b = bytearray(items[k])
        start = b.rfind(b"\xff\xda")
        for p in g.integers(start + 20, len(b) - 4, 40):
            if b[p] != 0xFF and b[p - 1] != 0xFF and b[p + 1] != 0xFF:
                b[p] ^= 1 << int(g.integers(0, 8))
                if b[p] == 0xFF:
                    b[p] ^= 1
        bad[k] = bytes(b)
    assert jpeg.probe(items[1]).restart_interval == 0 and jpeg.probe(items[3]).restart_interval > 0
    cut = items[1][:len(items[1]) // 2] + b"\xff\xd9"          # EOI long before the last MCU: found on the device
    cut_rst = items[3][:len(items[3]) // 2] + b"\xff\xd9"      # with restart markers: too few intervals, found on the host
    cut_no_eoi = items[4][:len(items[4]) // 2]
    assert jpeg.probe(cut).supported
    for c in (cut_rst, cut_no_eoi):
        assert not jpeg.probe(c).supported and "truncated" in jpeg.probe(c).reason
    batch = [bad.get(k, cut if k == 1 else d) for k, d in enumerate(items)]
    with pytest.raises(_lib.DfqError, match=r"images\[4\]: truncated"):
        P.imagenet(batch[:4] + [cut_no_eoi])
    outs = jpeg.decode(batch)
    x = P.imagenet(batch)
    xa = P.imagenet(arrays)
    for k, (o, a) in enumerate(zip(outs, arrays)):
        if k not in bad and k != 1:
            assert torch.equal(o.cpu(), torch.from_numpy(a)), k
            assert torch.equal(x[k], xa[k]), k
    with pytest.raises(_lib.DfqError, match=r"image 1 of decode call 1 of 2"):
        jpeg.check()
    jpeg.check()
    assert torch.equal(P.imagenet(items), xa)                   # the decoder is clean after the error
    jpeg.check()


# ---- end to end: the chained networks fed from bytes and from arrays -----------------------------------------------------------
@pytest.fixture
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_chained_networks_fed_from_bytes(_no_tf32):
    import affine_observed_state
    from dfq_b200 import detect, int8, segment
    from test_detect_host import _same, fixture
    items, arrays, labels = _batch(6, 9)
    with affine_observed_state.evaluation_state("mobilenet_v2", size=224) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True)
        with torch.no_grad():
            assert torch.equal(gm(P.imagenet(items)), gm(P.imagenet(arrays)))
    with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        head, ac = segment.split_upsample(int8.chain_affine(model, residual=True, concat=True, fold_pads=True))
        ev, ev_a = segment.Evaluator(21), segment.Evaluator(21)
        with torch.no_grad():
            x, y = P.voc_segmentation(items, labels, crop_size=129)
            ev.add_logits(y, head(x), align_corners=ac)
            x, y = P.voc_segmentation(arrays, labels, crop_size=129)
            ev_a.add_logits(y, head(x), align_corners=ac)
        assert np.array_equal(ev.confusion_matrix, ev_a.confusion_matrix) and ev.confusion_matrix.sum() > 0
    _, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True, heads=True)
        with torch.no_grad():
            x, sizes = P.ssd(items, mean=np.array([127, 127, 127]), std=128.0)
            got = detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
            x, sizes = P.ssd(arrays, mean=np.array([127, 127, 127]), std=128.0)
            want = detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
        assert got.boxes.shape[0] > 0
        for n, (g, w) in enumerate(zip(got.per_image(), want.per_image())):
            assert _same(g, w), n
    jpeg.check()
