"""dfq_b200.preprocess on the H100: every output bit for bit (torch.equal on the float32 tensors) against the CPU
transforms (torchvision, cv2, the oracle of tests/preprocess_oracle.py) and against the reference's own transform classes
through tests/golden/ref_preprocess.npz; mixed-size batches of 1, 7, 30 and 256 images; labels with 255 borders; the configs' numpy means; one
kernel launch and no host synchronisation per call; the refusals; and the chained affine MobileNetV2, DeepLab-v3+ and
SSD-Lite fed by the device path giving what they give fed by the CPU transform."""
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
import preprocess_cases as PC  # noqa: E402
import preprocess_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_preprocess.npz")
CASES = PC.cases()
CLS = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224), transforms.ToTensor(),
                          transforms.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))])


def _sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.cpu().numpy(), np.float32).tobytes()).hexdigest()


def _ssd_cpu(img, mean=(127.0, 127.0, 127.0), std=128.0):
    x = cv2.resize(img, (300, 300)).astype(np.float32) - np.array(mean, np.float32)
    return torch.from_numpy(np.ascontiguousarray((x / std).transpose(2, 0, 1)))


def _mixed(n, seed, lo=120, hi=640):
    g = np.random.default_rng(seed)
    hw = [(int(g.integers(lo, hi)), int(g.integers(lo, hi))) for _ in range(n)]
    return [PC.image(h, w, seed + i) for i, (h, w) in enumerate(hw)], [PC.label(h, w, seed + i) for i, (h, w) in enumerate(hw)]


# ---- the whole size grid in one mixed batch, against the fixture and the libraries ----------------------------------------
def test_grid_matches_the_reference_fixture_and_the_libraries():
    g = np.load(GOLD)
    imgs, labs = [c[1] for c in CASES], [c[2] for c in CASES]
    cls = P.imagenet(imgs)
    seg, seglab = P.voc_segmentation(imgs, labs)
    ssd, sizes = P.ssd(imgs, mean=(127, 127, 127))
    assert cls.shape == (len(imgs), 3, 224, 224) and seg.shape == (len(imgs), 3, 513, 513)
    assert seglab.shape == (len(imgs), 513, 513) and ssd.shape == (len(imgs), 3, 300, 300)
    assert sizes.dtype == torch.int64 and sizes.tolist() == [[a.shape[1], a.shape[0]] for a in imgs]
    for i, (name, img, lab) in enumerate(CASES):
        assert _sha(cls[i]) == g["cls_" + name], name
        assert _sha(seg[i]) == g["seg_" + name] and _sha(seglab[i]) == g["seglab_" + name], name
        assert _sha(ssd[i]) == g["ssd_" + name], name
        assert torch.equal(cls[i].cpu(), CLS(Image.fromarray(img))), name
        assert torch.equal(ssd[i].cpu(), _ssd_cpu(img)), name


@pytest.mark.parametrize("n,seed", [(1, 1), (7, 2)])
def test_segmentation_batches_match_the_oracle(n, seed):
    imgs, labs = _mixed(n, seed)
    labs[0][:, -3:] = 255
    seg, lab = P.voc_segmentation(imgs, labs)
    img_only, none = P.voc_segmentation(imgs)
    assert none is None and torch.equal(img_only, seg)
    for i in range(n):
        want, wlab = O.voc_segmentation(imgs[i], labs[i])
        assert torch.equal(seg[i].cpu(), torch.from_numpy(want)) and torch.equal(lab[i].cpu(), torch.from_numpy(wlab))
    assert (lab == 255).any()


@pytest.mark.parametrize("n,seed", [(1, 11), (7, 12), (256, 13)])
def test_classification_and_ssd_batches_match_the_libraries(n, seed):
    imgs, _ = _mixed(n, seed, lo=60, hi=900)
    cls = P.imagenet(imgs)
    ssd, _ = P.ssd(imgs)
    mean = (123.0, 117.0, 104.0)
    ssd3, _ = P.ssd(imgs, mean=mean, std=1.0)
    ssd_a, _ = P.ssd(imgs, mean=np.array([127, 127, 127]), std=128.0)     # the configs' image_mean / image_std
    ssd_b, _ = P.ssd(imgs, mean=np.array([123, 117, 104]), std=1.0)
    assert torch.equal(ssd_a, ssd) and torch.equal(ssd_b, ssd3)
    for i, img in enumerate(imgs):
        assert torch.equal(cls[i].cpu(), CLS(Image.fromarray(img)))
        assert torch.equal(ssd[i].cpu(), _ssd_cpu(img))
        assert torch.equal(ssd3[i].cpu(), _ssd_cpu(img, mean, 1.0))


def test_off_default_parameters_and_tensor_inputs():
    imgs, labs = _mixed(5, 21)
    got = P.imagenet([torch.from_numpy(a) for a in imgs], resize=160, crop=128, mean=(0.5, 0.4, 0.3), std=(0.2, 0.3, 0.25))
    for i, img in enumerate(imgs):
        want = O.imagenet(img, 160, 128, (0.5, 0.4, 0.3), (0.2, 0.3, 0.25))
        assert torch.equal(got[i].cpu(), torch.from_numpy(want))
    seg, lab = P.voc_segmentation(imgs, labs, crop_size=97)
    for i, img in enumerate(imgs):
        want, wlab = O.voc_segmentation(img, labs[i], 97)
        assert torch.equal(seg[i].cpu(), torch.from_numpy(want)) and torch.equal(lab[i].cpu(), torch.from_numpy(wlab))
    ssd, _ = P.ssd(imgs, size=512, mean=0.0, std=255.0)
    for i, img in enumerate(imgs):
        assert torch.equal(ssd[i].cpu(), torch.from_numpy(O.ssd(img, 512, 0.0, 255.0)))


def test_back_to_back_calls_stay_exact():
    """Calls enqueued without waiting: a staging block is handed out again only after the copy that read it."""
    a, _ = _mixed(9, 31)
    b, _ = _mixed(4, 32)
    outs = [P.imagenet(x) for x in (a, b) * 10]
    for i in range(2, len(outs)):
        assert torch.equal(outs[i], outs[i % 2])


# ---- launches and synchronisation ------------------------------------------------------------------------------------------
def test_one_kernel_launch_and_no_host_synchronisation():
    imgs, labs = _mixed(16, 41)
    P.voc_segmentation(imgs, labs)
    P.imagenet(imgs)
    P.ssd(imgs)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            P.voc_segmentation(imgs, labs)
            P.imagenet(imgs)
            P.ssd(imgs)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        P.imagenet(imgs)
        P.voc_segmentation(imgs, labs)
        P.ssd(imgs)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert sum("k_pre_resample" in n for n in names) == 3, names
    assert sum("Memcpy HtoD" in n for n in names) == 4, names        # one per call, and ssd's sizes


# ---- refusals on the device path ------------------------------------------------------------------------------------------
def test_refusals_on_the_gpu():
    ok = PC.image(20, 30, 0)
    with pytest.raises(_lib.DfqError, match="smaller than the"):
        P.imagenet([ok, ok], resize=100, crop=128)
    with pytest.raises(_lib.DfqError, match="decoded images come from the host"):
        P.imagenet([torch.from_numpy(ok).cuda()])
    with pytest.raises(_lib.DfqError, match="std"):
        P.voc_segmentation([ok], std=0)


# ---- end to end: the chained networks fed by the device path and by the CPU transform -----------------------------------------
@pytest.fixture
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_chained_mobilenet_v2_fed_by_imagenet(_no_tf32):
    import affine_observed_state
    from dfq_b200 import int8
    imgs, _ = _mixed(6, 51, lo=200, hi=700)
    with affine_observed_state.evaluation_state("mobilenet_v2", size=224) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True)
        x = P.imagenet(imgs)
        cpu = torch.stack([CLS(Image.fromarray(a)) for a in imgs]).cuda()
        assert torch.equal(x, cpu)
        with torch.no_grad():
            assert torch.equal(gm(x), gm(cpu))


def test_chained_deeplab_fed_by_voc_segmentation(_no_tf32):
    import affine_observed_state
    from dfq_b200 import int8, segment
    imgs, labs = _mixed(4, 52)
    with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
        head, ac = segment.split_upsample(gm)
        x, y = P.voc_segmentation(imgs, labs, crop_size=129)
        ref = [O.voc_segmentation(a, l, 129) for a, l in zip(imgs, labs)]
        xc = torch.from_numpy(np.ascontiguousarray(np.stack([r[0] for r in ref]))).cuda().contiguous()
        yc = torch.from_numpy(np.ascontiguousarray(np.stack([r[1] for r in ref]))).cuda().contiguous()
        assert x.is_contiguous() and y.is_contiguous()
        assert torch.equal(x, xc) and torch.equal(y, yc) and (y == 255).any()
        ev, ev_cpu = segment.Evaluator(21), segment.Evaluator(21)
        with torch.no_grad():
            ev.add_logits(y, head(x), align_corners=ac)
            ev_cpu.add_logits(yc, head(xc), align_corners=ac)
        assert np.array_equal(ev.confusion_matrix, ev_cpu.confusion_matrix) and ev.confusion_matrix.sum() > 0


def test_chained_ssd_lite_fed_by_ssd(_no_tf32):
    import affine_observed_state
    from dfq_b200 import detect, int8
    from test_detect_host import _same, fixture
    _, t, cv, sv = fixture()
    pri = t["priors"].cuda()
    imgs, _ = _mixed(4, 53)
    with affine_observed_state.evaluation_state("ssd", size=300, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True, heads=True)
        x, sizes = P.ssd(imgs, mean=np.array([127, 127, 127]), std=128.0)      # the configs' image_mean / image_std
        xc = torch.stack([_ssd_cpu(a) for a in imgs]).cuda()
        sc = torch.tensor([[a.shape[1], a.shape[0]] for a in imgs], device="cuda")
        assert torch.equal(x, xc) and torch.equal(sizes, sc)
        with torch.no_grad():
            got = detect.postprocess(*gm(x), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sizes)
            want = detect.postprocess(*gm(xc), priors=pri, center_variance=cv, size_variance=sv, image_sizes=sc)
        assert got.boxes.shape[0] > 0
        for n, (g, w) in enumerate(zip(got.per_image(), want.per_image())):
            assert _same(g, w), n
