"""dfq_b200.classify on the GPU: predict and the Evaluator's count against torch.max(logits, 1)[1] and (pred == label).sum()
on the GPU, bit for bit, over class counts from 1 to ImageNet-21k's 21,843 and batches past the kernel's grid; rows of
ties, NaN in every place, +-inf, -0.0 against +0.0 and subnormals, which pin torch's CUDA argmax rule (DESIGN.md section
4); labels out of range, on the CPU and on the GPU; and no host synchronisation per add_logits."""
import numpy as np
import pytest
import torch

from dfq_b200 import _lib

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


def _logits(N, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, C, device="cuda", generator=g)
    if C >= 2:
        x[::3, C - 1] = x[::3].max(1)[0]                          # ties with the row's maximum, at the far end
        x[1::5] = 0.0
        x[1::5, ::2] = -0.0                                       # -0.0 against +0.0
    if C >= 3:
        x[2::7, C // 2] = NAN
        x[2::14, C - 1] = NAN                                     # two NaN in a row
        x[3::7, 1] = INF
        x[3::7, C - 2] = INF
        x[4::9] = -INF
        x[5::11] = torch.finfo(torch.float32).tiny / 4            # subnormals, tied
        x[5::11, C // 3] = torch.finfo(torch.float32).tiny / 2
    return x


def _labels(N, C, seed, pred):
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(-3, C + 3, (N,), generator=g)              # some outside 0 .. C-1
    y[::2] = pred[::2].cpu()
    return y


@pytest.mark.parametrize("C", [1, 2, 31, 1000, 21843])
@pytest.mark.parametrize("N", [1, 7, 256])
def test_count_and_predict_equal_torch(C, N):
    from dfq_b200 import classify
    x = _logits(N, C, seed=C + N)
    want = torch.max(x, 1)[1]
    got = classify.predict(x)
    assert got.dtype == torch.int64 and got.shape == (N,) and torch.equal(got, want)
    y = _labels(N, C, C * N, want)
    ev = classify.Evaluator(C)
    ev.add_logits(x, y)                                           # CPU labels
    ev.add_logits(x, y.cuda())                                    # GPU labels
    main_correct = np.sum(want.cpu().numpy() == y.numpy())       # main_cls.py inference_all
    assert ev.num_correct == 2 * main_correct == 2 * int((want.cpu() == y).sum())
    assert ev.num_total == 2 * N
    assert ev.accuracy() == (0 + main_correct + main_correct) / (0 + N + N)


def test_special_rows_pin_torch_rule():
    from dfq_b200 import classify
    tiny = torch.finfo(torch.float32).tiny
    rows = [[NAN, 1., 2., 3.], [1., NAN, 3., NAN], [1., 2., 3., NAN], [NAN] * 4, [INF, INF, 1., NAN],
            [-INF, -INF, -INF, -INF], [-0., 0., -0., 0.], [0., -0., 0., -0.], [tiny / 8, tiny / 4, tiny / 4, -tiny],
            [-1., -1., -2., -1.], [3., 3., 3., 3.], [1., INF, INF, -INF], [-INF, -1e38, -INF, -1e38]]
    for C in (4, 37, 1000):                                        # the same rows spread over more lanes and columns
        x = torch.full((len(rows), C), -INF, device="cuda")
        for i, r in enumerate(rows):
            x[i, torch.arange(4) * (C // 4)] = torch.tensor(r, device="cuda")
        assert torch.equal(classify.predict(x), torch.max(x, 1)[1]), C
        want = (torch.max(x, 1)[1] // (C // 4)).cpu().tolist()
        # the rule as DESIGN.md section 4 states it: the first NaN, else the first of the largest values, -0.0 == +0.0
        assert want == [0, 1, 3, 0, 3, 0, 0, 0, 1, 0, 0, 1, 1], (C, want)


def test_past_the_grid_stride_limit():
    from dfq_b200 import classify
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 8 * 8 * sms * 3 + 5                                        # more rows than warps in the grid
    x = _logits(N, 31, seed=3)
    want = torch.max(x, 1)[1]
    y = _labels(N, 31, 4, want).cuda()
    ev = classify.Evaluator(31)
    ev.add_logits(x, y)
    assert torch.equal(classify.predict(x), want)
    assert ev.num_correct == int((want == y).sum()) and ev.num_total == N


def test_refusals_leave_the_count():
    from dfq_b200 import classify
    ev = classify.Evaluator(10)
    x = _logits(4, 10, 0)
    y = torch.tensor([1, 2, 3, 4])
    ev.add_logits(x, y)
    before = int(ev.num_correct)
    for args, msg in [((x.cpu(), y), "on the GPU"), ((x[:, :5].contiguous(), y), "5 classes"),
                      ((x, y.cuda().int()), "int64"), ((x, y[:3]), r"shape \[4\]")]:
        with pytest.raises(_lib.DfqError, match=msg):
            ev.add_logits(*args)
    assert ev.num_correct == before and ev.num_total == 4


def test_no_host_synchronisation():
    from dfq_b200 import classify
    x = _logits(256, 1000, 5)
    y = _labels(256, 1000, 6, torch.max(x, 1)[1])
    yd = y.cuda()
    ev = classify.Evaluator(1000)
    ev.add_logits(x, y)                                            # first call: allocation, library load, pinned pool
    classify.predict(x)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            ev.add_logits(x, y)
            ev.add_logits(x, yd)
            p = classify.predict(x)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert torch.equal(p, torch.max(x, 1)[1])
    assert ev.num_correct == 7 * int((p.cpu() == y).sum()) and ev.num_total == 7 * 256
