"""CPU side of the activation fake-quantization, observer and distillation-loss kernels.

* The oracle statements the GPU tests of tests/test_gpu_activation.py compare against: the tensor-range prologue against
  PyTorch-CPU eager, the NaN rules, and the float64 BN-statistics loss against float64 autograd (zero-std rule included).
* The host wrappers through tests/fakelib.py: the EMA momentum, the refusal of a batch that does not divide the tensor, and
  the checks on caller-supplied statistics tensors.
"""
import numpy as np
import pytest
import torch

import fakelib
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


def _same(a, b):
    """Bit-equal, or both NaN."""
    a = np.asarray(a, f32); b = np.asarray(b, f32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("symmetric", [False, True])
@pytest.mark.parametrize("bits", [2, 4, 8, 16])
def test_tensor_range_prologue_matches_torch_cpu(bits, symmetric):
    """quantize(x, bits) with no range (quantize.py:24-74 on 0-d fp32 tensors, the bias path) in PyTorch-CPU eager
    against oracle.quantize_tensor_range(prologue=1)."""
    g = torch.Generator().manual_seed(bits)
    x = torch.randn(997, generator=g) * 2.3 + (0.4 if not symmetric else -0.9)
    y = x.view(1, -1)
    mn, mx = y.min(-1)[0].mean(-1), y.max(-1)[0].mean(-1)
    if symmetric:
        qmin, qmax = -2. ** (bits - 1), 2 ** (bits - 1) - 1
        max_value, min_value = abs(mx), abs(mn)
        if max_value < min_value:
            max_value = min_value
        scale, min_value = max_value / qmax, 0.
    else:
        qmin, qmax = 0., 2. ** bits - 1.
        scale, min_value = (mx - mn) / (qmax - qmin), mn
    scale = max(scale, 1e-8)
    want = x.clone().add_(-min_value).div_(scale).clamp_(qmin, qmax).round_().mul_(scale).add_(min_value)
    assert _same(O.quantize_tensor_range(x.numpy(), bits, float(mn), float(mx), symmetric, prologue=1), want.numpy())


def test_clamp_keeps_nan_in_torch_and_in_the_oracle():
    """The premise of the NaN rule: torch's clamp_ keeps a NaN, and so do the oracle's quantizers and clip_weight."""
    t = torch.tensor([float("nan"), 1.0, -3.0])
    assert torch.isnan(t.clone().add_(.5).div_(.01).clamp_(0, 255).round_()[0])
    x = np.array([np.nan, 0.3, -np.inf, np.inf, -0.0], f32)
    for y in (O.quantize(x, 8, -1.0, 1.0), O.quantize(x, 8, -1.0, 1.0, div_mode="recip"),
              O.quantize_tensor_range(x, 8, -1.0, 1.0, prologue=2), O.clip_weight(x)):
        assert np.isnan(y[0]) and not np.isnan(y[1:]).any()


def test_statistics_skip_nan():
    """DESIGN.md section 4: the min/max reductions skip NaN; an all-NaN sample contributes (+inf, -inf)."""
    x = np.array([[1.0, np.nan, -2.0], [np.nan, np.nan, np.nan], [0.5, 4.0, np.nan]], f32)
    assert O.flat_minmax(x) == (f32(-2.0), f32(4.0))
    assert O.flat_minmax(x[1]) == (f32(np.inf), f32(-np.inf))
    assert O.per_sample_minmax_mean(x[[0, 2]]) == (f32(-0.75), f32(2.5))
    assert O.per_sample_minmax_mean(x) == (f32(np.inf), f32(-np.inf))


# ---------------------------------------------------------------------------------------------------------------------
def _reference_formula(x, bn_mean, bn_std, eps=1e-6):
    """distill_data.py:171-185."""
    n, c = x.size(0), x.size(1)
    flat = x.view(n, c, -1)
    own = lambda a, b: (a - b).norm() ** 2 / a.size(0)
    return own(bn_mean, torch.mean(flat, dim=2)), own(bn_std, torch.std(flat + eps, dim=2))


@pytest.mark.parametrize("shape", [(2, 3, 4, 5), (3, 2, 7), (1, 1, 2, 1), (4, 5, 3, 3)])
def test_bn_stat_loss_oracle_matches_float64_autograd(shape):
    """oracle.bn_stat_loss against float64 autograd of the reference formula, with a constant zero row, a constant
    non-zero row and a row with |mean|/std = 1e4: a constant row gets no std gradient."""
    g = torch.Generator().manual_seed(len(shape) * 7 + shape[0])
    x = torch.randn(*shape, generator=g, dtype=torch.float64) * 1.3 + 0.2
    x[0, 0] = 0.0
    x[-1, -1] = 2.75
    if shape[0] * shape[1] > 2:
        x[0, -1] = 1e4 + torch.randn(x[0, -1].shape, generator=g, dtype=torch.float64)
    mu = torch.randn(shape[1], generator=g, dtype=torch.float64) * 0.3
    sd = torch.rand(shape[1], generator=g, dtype=torch.float64) + 0.5
    lm, ls, gm, gs = O.bn_stat_loss(x.numpy(), mu.numpy(), sd.numpy())
    for k, want_l, want_g in ((0, lm, gm), (1, ls, gs)):
        xr = x.clone().requires_grad_(True)
        loss = _reference_formula(xr, mu, sd)[k]
        loss.backward()
        assert abs(float(loss) - want_l) <= 1e-12 * abs(want_l), (k, float(loss), want_l)
        assert np.allclose(xr.grad.numpy(), want_g, rtol=1e-9, atol=1e-12), k
    assert not gs[0, 0].any() and not gs[-1, -1].any()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("momentum", [0.1, 0.9, 0.99])
def test_observer_ema_momentum_twin(monkeypatch, momentum):
    """QuantMeasure in training mode: running*(1-m) + stat*m with 1-m formed from the Python float (quantize.py:112-113),
    not from m rounded to fp32 first.  The two factors differ by an ulp for m = 0.9 and 0.99; over 16 seeded starting
    values that changes some running values."""
    fakelib.install(monkeypatch)
    from dfq_b200.utils.quantize import QuantMeasure
    x = torch.randn(8, 3, 5, 5, generator=torch.Generator().manual_seed(17)) * 1.9 + 0.3
    st_min, st_max = O.per_sample_minmax_mean(x.numpy())
    m32 = f32(momentum)
    old_om = f32(1.0 - float(m32))
    differs = 0
    for a, b in np.random.default_rng(3).uniform(-200, 200, (16, 2)).astype(f32):
        qm = QuantMeasure(False, momentum=momentum).train()
        qm.running_min.fill_(float(a)); qm.running_max.fill_(float(b))
        qm(x)
        rmin, rmax, _, _ = O.observer_ema(a, b, x.numpy(), momentum)
        assert _same(qm.running_min.numpy(), [rmin]) and _same(qm.running_max.numpy(), [rmax]), (a, b)
        differs += (a * old_om + st_min * m32 != rmin) + (b * old_om + st_max * m32 != rmax)
    assert (differs > 0) == (momentum != 0.1), differs


def test_momentum_binding_takes_python_and_ctypes_numbers():
    """The momentum is a C double: a Python float reaches the kernel unchanged, a c_float (an ABI 1 caller) widened exactly."""
    import ctypes as C
    for v, want in ((0.9, 0.9), (0.99, 0.99), (C.c_double(0.01), 0.01), (C.c_float(0.9), float(f32(0.9))), (1, 1.0)):
        got = _lib._Momentum.from_param(v)
        assert isinstance(got, C.c_double) and got.value == want, (v, got)
    assert [_lib._Momentum in _lib.SIGNATURES[n] for n in ("dfq_observer_update", "dfq_observe_quant")] == [True, True]


def test_a_batch_that_does_not_divide_the_tensor_is_refused(monkeypatch):
    """quantize(x, num_chunks=k) views x as [B // k, -1]; the reference's view raises when that does not divide x, and so
    do both wrappers instead of leaving the tail of the output unwritten."""
    fakelib.install(monkeypatch)
    from dfq_b200.utils.quantize import quantize
    x = torch.randn(5, 3)
    with pytest.raises(RuntimeError):
        x.view(5 // 2, -1)
    with pytest.raises(_lib.DfqError, match="cannot view"):
        quantize(x, 8, num_chunks=2)
    with pytest.raises(_lib.DfqError, match="cannot view"):
        quantize(x, 8, min_value=-1.0, num_chunks=2)
    x6 = torch.randn(6, 3)
    assert _same(quantize(x6, 8, num_chunks=2).numpy(),
                 O.quantize_tensor_range(x6.numpy(), 8, *O.per_sample_minmax_mean(x6.numpy().reshape(3, -1)), prologue=1))


def test_running_buffers_are_checked_and_converted(monkeypatch):
    """observe_and_quant: float64 running buffers are updated through an fp32 copy; a buffer of the wrong length or on
    another device is refused before the kernel runs."""
    fakelib.install(monkeypatch)
    from dfq_b200.utils.quantize import OBS_UPDATE, observe_and_quant
    x = torch.randn(4, 10, generator=torch.Generator().manual_seed(2))
    rmin = torch.zeros(1, dtype=torch.float64); rmax = torch.zeros(1, dtype=torch.float64)
    observe_and_quant(x, 8, OBS_UPDATE, rmin, rmax)
    want = O.observer_update(0.0, 0.0, x.numpy())
    assert rmin.dtype == torch.float64 and (float(rmin), float(rmax)) == (float(want[0]), float(want[1]))
    with pytest.raises(_lib.DfqError, match="one element"):
        observe_and_quant(x, 8, OBS_UPDATE, torch.zeros(2), torch.zeros(1))
    with pytest.raises(_lib.DfqError, match="is on meta"):
        observe_and_quant(x, 8, OBS_UPDATE, torch.zeros(1), torch.zeros(1, device="meta"))


def test_bn_statistics_are_checked(monkeypatch):
    """The fused BN-statistics loss refuses a statistic of the wrong length or on another device before any launch."""
    fakelib.install(monkeypatch)
    from dfq_b200.distill import _BNStatLoss
    x = torch.randn(2, 3, 4, 4)
    with pytest.raises(_lib.DfqError, match="2 elements for 3 channels"):
        _BNStatLoss.apply(x, torch.zeros(2), torch.ones(3), 1e-6)
    with pytest.raises(_lib.DfqError, match="is on meta"):
        _BNStatLoss.apply(x, torch.zeros(3), torch.ones(3, device="meta"), 1e-6)
