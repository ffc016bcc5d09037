"""dfq_b200.segment on the GPU: predict against torch's resize + max bit for bit over sizes, class counts and special
values; the Evaluator's counts against torch.bincount for every label type; refusals that leave the counts alone; no host
synchronisation; an evaluation past 2^31 output pixels; and split_upsample + Evaluator on the padded DeepLab, fp32 and
chained under both int8 schemes, before and after save / load."""
import numpy as np
import pytest
import torch
import torch.fx as fx
import torch.nn.functional as F

from dfq_b200 import _lib

pytestmark = pytest.mark.gpu

RESIZES = [((129, 129), (513, 513), True), ((129, 129), (513, 513), False), ((65, 97), (257, 385), True),
           ((65, 97), (257, 385), False), ((7, 9), (1, 1), False), ((1, 1), (33, 17), True), ((1, 1), (33, 17), False),
           ((513, 513), (129, 129), False), ((33, 47), (33, 47), None)]


def _logits(N, C, H, W, kind, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "constant":
        return torch.full((N, C, H, W), 0.25, device="cuda")
    x = torch.randn(N, C, H, W, device="cuda", generator=g)
    if C >= 2:
        x[:, 1, ::3] = x[:, 0, ::3]                                  # ties between classes 0 and 1
        x[:, :, 1::4, ::5] = -0.0                                    # -0.0 against +0.0
        x[:, 1, 1::4, ::5] = 0.0
        x[:, :, 1::4, 1::5] = -1.
    if C >= 3:
        x[:, 2, ::7, ::3] = float("inf")
        x[:, C - 1, 2::7, ::3] = -float("inf")
        x[:, C // 2, ::11] = float("nan")                           # NaN in some classes
        x[:, C - 1, ::13, 1::2] = float("nan")
    return x


def _torch_pred(x, size, ac):
    y = x if size is None or tuple(size) == tuple(x.shape[2:]) else F.interpolate(x, size, mode="bilinear",
                                                                                    align_corners=ac)
    return torch.max(y, 1)[1]


@pytest.mark.parametrize("src,dst,ac", RESIZES)
@pytest.mark.parametrize("C", [1, 2, 21, 150, 160])
@pytest.mark.parametrize("N", [1, 3])
def test_predict_equals_torch_bit_for_bit(src, dst, ac, C, N):
    from dfq_b200 import segment
    for kind in ("random", "constant"):
        x = _logits(N, C, *src, kind, seed=C + N)
        got = segment.predict(x, dst, ac)
        want = _torch_pred(x, dst, ac)
        assert got.dtype == torch.int64 and got.shape == want.shape
        assert torch.equal(got, want), (kind, int((got != want).sum()))
    assert torch.equal(segment.predict(x), torch.max(x, 1)[1])


def _torch_counts(labels, pred, C):
    if labels.dtype == torch.float32:
        ok = (labels > -1) & (labels < 256)
        gt = torch.where(ok, labels, torch.zeros_like(labels)).trunc().long()
        gt = torch.where(ok, gt, torch.full_like(gt, -1))
    else:
        gt = labels.long()
    keep = (gt >= 0) & (gt < C)
    return torch.bincount((C * gt + pred)[keep], minlength=C * C).view(C, C)


def _labels(N, H, W, C, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.randint(-3, C + 3, (N, H, W), device="cuda", generator=g)
    lab[torch.rand(N, H, W, device="cuda", generator=g) < 0.5] = 0
    lab[:, :2] = 255
    if dtype == torch.uint8:
        return lab.clamp(0, 255).to(torch.uint8)
    if dtype == torch.int64:
        return lab
    f = lab.float() + torch.rand(N, H, W, device="cuda", generator=g) * 0.99
    f[:, 2, :4] = -0.5
    f[:, 2, 4:8] = float("nan")
    f[:, 2, 8:12] = 300.
    f[:, 2, 12:16] = -1.
    f[:, 2, 16:20] = 255.9
    return f


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int64, torch.float32])
@pytest.mark.parametrize("C", [2, 21, 160])
def test_counts_equal_bincount_and_accumulate(dtype, C):
    from dfq_b200 import segment
    ev = segment.Evaluator(C)
    want = torch.zeros(C, C, dtype=torch.int64, device="cuda")
    for i, (N, (h, w), (H, W), ac) in enumerate((
            (2, (33, 33), (129, 129), True), (1, (20, 30), (77, 61), False), (3, (40, 40), (40, 40), None))):
        x = _logits(N, C, h, w, "random", seed=i)
        lab = _labels(N, H, W, C, dtype, seed=10 + i)
        ev.add_logits(lab, x, align_corners=ac)
        want += _torch_counts(lab, _torch_pred(x, (H, W), ac), C)
        assert torch.equal(ev.counts, want), i
    assert np.array_equal(ev.confusion_matrix, want.cpu().numpy().astype(np.float64))
    ev.reset()
    assert not ev.counts.any()


@pytest.mark.parametrize("case", ["C161", "fp16", "logits_nc", "labels_nc", "labels_cpu", "logits_cpu", "no_ac"])
def test_refusals_leave_the_counts(case):
    from dfq_b200 import segment
    ev = segment.Evaluator(21)
    x = _logits(2, 21, 17, 17, "random")
    lab = _labels(2, 65, 65, 21, torch.uint8, 1)
    ev.add_logits(lab, x, align_corners=True)
    before = ev.counts.clone()
    if case == "C161":
        d = np.zeros(1, _lib.SEG_ARGMAX_DT)
        d[0] = (2, 161, 17, 17, 65, 65, 1, _lib.SEG_LABEL_U8)
        x = _logits(2, 161, 17, 17, "random")
        rc = _lib.load().dfq_seg_argmax(x.data_ptr(), lab.data_ptr(), None, ev.counts.data_ptr(), _lib.table_ptr(d),
                                        _lib.stream_ptr())
        assert rc == -2                                        # DFQ_E_UNSUPPORTED
    with pytest.raises(_lib.DfqError):
        if case == "C161":
            segment.predict(x, (65, 65), True)
        elif case == "fp16":
            ev.add_logits(lab, x.half(), align_corners=True)
        elif case == "logits_nc":
            ev.add_logits(lab, x.transpose(2, 3), align_corners=True)
        elif case == "labels_nc":
            ev.add_logits(lab.transpose(1, 2), x, align_corners=True)
        elif case == "labels_cpu":
            ev.add_logits(lab.cpu(), x, align_corners=True)
        elif case == "logits_cpu":
            ev.add_logits(lab, x.cpu(), align_corners=True)
        elif case == "no_ac":
            ev.add_logits(lab, x)
    torch.cuda.synchronize()
    assert torch.equal(ev.counts, before)


def test_cross_device_evaluator_is_refused():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    from dfq_b200 import segment
    ev = segment.Evaluator(3)
    ev.add_logits(torch.zeros(1, 4, 4, dtype=torch.uint8, device="cuda:0"), torch.randn(1, 3, 4, 4, device="cuda:0"))
    with torch.cuda.device(1), pytest.raises(_lib.DfqError, match="counts on cuda:0"):
        ev.add_logits(torch.zeros(1, 4, 4, dtype=torch.uint8, device="cuda:1"), torch.randn(1, 3, 4, 4, device="cuda:1"))


def test_no_host_synchronisation():
    from dfq_b200 import segment
    x = _logits(2, 21, 33, 33, "random")
    lab = _labels(2, 129, 129, 21, torch.float32, 3)
    ev = segment.Evaluator(21)
    ev.add_logits(lab, x, align_corners=True)             # first call: allocation and library load
    segment.predict(x, (129, 129), True)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            ev.add_logits(lab, x, align_corners=True)
            p = segment.predict(x, (129, 129), True)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert torch.equal(p, _torch_pred(x, (129, 129), True))
    assert torch.equal(ev.counts, 4 * _torch_counts(lab, p, 21))


@pytest.mark.parametrize("ac", [True, False])
def test_past_2_31_output_pixels(ac):
    """Two 33,000 x 33,000 label maps (2.18e9 pixels) from 1 x 1 logits, counting only: each image's prediction is its
    logits' argmax everywhere (the classes are far apart), so the matrix has a closed form."""
    from dfq_b200 import segment
    N, S, C = 2, 33000, 5
    assert N * S * S > 2 ** 31
    x = torch.tensor([[0., 9., 1., 2., 3.], [4., 0., 1., 20., 3.]], device="cuda").view(N, C, 1, 1)
    lab = torch.full((N, S, S), 3, dtype=torch.uint8, device="cuda")
    lab[0, 0] = 255
    lab[1] = 1
    lab[1, -1, -7:] = 4
    ev = segment.Evaluator(C)
    ev.add_logits(lab, x, align_corners=ac)
    want = np.zeros((C, C))
    want[3, 1] = S * S - S
    want[1, 3] = S * S - 7
    want[4, 3] = 7
    assert np.array_equal(ev.confusion_matrix, want)
    del lab


# ---- DeepLab end to end -------------------------------------------------------------------------------------------------
def _end_to_end(gm, x, label_seed=0):
    from dfq_b200 import segment
    head, ac = segment.split_upsample(gm)
    assert ac is True
    with torch.no_grad():
        full, low = gm(x), head(x)
    size = tuple(x.shape[2:])
    assert torch.equal(F.interpolate(low, size, mode="bilinear", align_corners=ac).view(torch.int32),
                       full.view(torch.int32))
    pred = torch.max(full, 1)[1]
    assert torch.equal(segment.predict(low, size, ac), pred)
    lab = _labels(x.shape[0], *size, 21, torch.uint8, label_seed)
    ev = segment.Evaluator(21)
    ev.add_logits(lab, low, align_corners=ac)
    assert torch.equal(ev.counts, _torch_counts(lab, pred, 21))
    return head


SIZES = [(129, 129), (97, 129)]


def test_deeplab_fp32_traced():
    from deeplab_mobilenet_padded import DeepLabMobileNetPadded
    torch.manual_seed(0)
    gm = fx.symbolic_trace(DeepLabMobileNetPadded().cuda().eval())
    for s in SIZES:
        x = torch.randn(2, 3, *s, device="cuda")
        head = _end_to_end(gm, x)
    # the input's size query fed only the final resize; the inner resizes keep theirs
    assert not [n for n in head.graph.nodes if n.op == "call_method" and n.target == "size" and n.args[0].op == "placeholder"]
    assert [n for n in gm.graph.nodes if n.op == "call_method" and n.target == "size" and n.args[0].op == "placeholder"]


def test_deeplab_ncnn_chain_and_loaded(tmp_path):
    from dfq_b200 import int8
    import test_gpu_int8_layout as GL
    model, _ = GL._net("deeplab", 2, 129)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
    for s in SIZES:
        _end_to_end(gm, torch.randn(2, 3, *s, device="cuda"))
    int8.save(gm, tmp_path / "deeplab.pt")
    loaded = int8.load(tmp_path / "deeplab.pt")
    for s in SIZES:
        _end_to_end(loaded, torch.randn(2, 3, *s, device="cuda"), 1)


def test_deeplab_affine_chain_and_loaded(tmp_path):
    import affine_observed_state
    from dfq_b200 import int8
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
            g = torch.Generator(device="cuda").manual_seed(2)
            xs = [torch.randn(2, 3, *s, device="cuda", generator=g).clamp_(-2.5, 2.5) for s in SIZES]
            for x in xs:
                head = _end_to_end(gm, x)
            assert head.graph.output_node().args[0].op == "call_module"       # the observer in front of the resize
            int8.save(gm, tmp_path / "deeplab_affine.pt")
        loaded = int8.load(tmp_path / "deeplab_affine.pt")
        for x in xs:
            _end_to_end(loaded, x, 1)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
