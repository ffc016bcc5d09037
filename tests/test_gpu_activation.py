"""-m gpu: every entry point of csrc/tensor_ops.cu (activation fake quantization, observer, statistics, ranges, clamp) and
csrc/distill.cu (the BN-statistics loss of the distilled-data generation) against an independent reference.

* Quantizer, statistics, EMA and ranges: bit-exact against oracle/dfq_oracle.py (NaN equal to NaN).
* BN-statistics loss and gradient: float64 autograd of distill_data.py:171-185.  The kernel's error against it may be at
  most twice the error of the same formula evaluated by PyTorch in fp32 on the same input, plus 4 fp32 ulps.

Shapes are derived from the SM count and the launch formulas (constants pinned in tests/test_boundary_guards.py), so each
case lands on its intended side of every grid-stride loop, split and alignment branch on any H100.
"""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import dfq_oracle as O
from test_boundary_guards import CONSTANTS

pytestmark = pytest.mark.gpu
f32 = np.float32
K = {k: v[1] for k, v in CONSTANTS.items()}
THREADS, ITEM, RANGE_CTA, DTHREADS, BN_CTA = (K[k] for k in ("kThreads", "kItemFloats", "kRangeCtaRow", "kDThreads",
                                                              "kBnstatCtaRow"))
OBS_BLOCKS_PER_SM = 4        # dfq_observe_quant: at most 4 CTAs per SM (k_observe_quant fits more)
EPS = 1e-6


def _lib():
    from dfq_b200 import _lib as L
    return L, L.load()


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _sms():
    L, lib = _lib()
    sm = C.c_int(); ctas = C.c_int()
    L.check(lib.dfq_device_info(C.byref(sm), C.byref(ctas)), "dfq_device_info")
    return sm.value


def _same(got, want):
    """Bit-equal fp32 arrays, NaN equal to NaN (payloads may differ); -0.0 differs from +0.0."""
    a = np.ascontiguousarray(got, f32).reshape(-1); b = np.ascontiguousarray(want, f32).reshape(-1)
    bad = (a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))
    return a.shape == b.shape and not bad.any(), (int(bad.sum()), a[bad][:4], b[bad][:4])


def _rand(n, seed, scale=1.7, shift=0.1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, device="cuda", generator=g) * scale + shift


def _unaligned(x):
    """The same values one float past a 16-byte boundary."""
    buf = torch.empty(x.numel() + 1, device="cuda")
    buf[1:].copy_(x.reshape(-1))
    out = buf[1:]
    assert out.data_ptr() % 16 == 4
    return out


# ---------------------------------------------------------------------------------------------------------------------
# dfq_observe_quant: statistic, running update and quantization in one cooperative launch
# ---------------------------------------------------------------------------------------------------------------------
def _observer_oracle(x, batch, flags, rmin, rmax, m, bits, sym, div_mode, prologue):
    st = O.per_sample_minmax_mean(x.reshape(batch, -1))
    rmin, rmax = f32(rmin), f32(rmax)
    if flags & 4:
        q = st
    else:
        if flags & 1:
            rmin, rmax = np.fmin(rmin, st[0]), np.fmax(rmax, st[1])
        if flags & 2:
            om, mf = f32(1.0 - m), f32(m)
            rmin, rmax = f32(rmin * om) + f32(st[0] * mf), f32(rmax * om) + f32(st[1] * mf)
            q = st
        else:
            q = (rmin, rmax)
    if prologue == 0:
        y = O.quantize(x, bits, float(q[0]), float(q[1]), sym, div_mode="recip" if div_mode else "div")
    else:
        y = O.quantize_tensor_range(x, bits, q[0], q[1], sym, prologue)
    return y, f32(rmin), f32(rmax), st


def _run_observer(x, batch, flags, m=0.1, bits=8, sym=False, div_mode=1, prologue=0, r0=(-0.5, 0.7)):
    L, lib = _lib()
    per = x.numel() // batch
    y = torch.full_like(x, float("nan"))
    stat = torch.full((2,), float("nan"), device="cuda")
    rmin = torch.tensor([r0[0]], device="cuda"); rmax = torch.tensor([r0[1]], device="cuda")
    own = bool(flags & 4)
    L.check(lib.dfq_observe_quant(P(x), P(y), batch, per, None if own else P(rmin), None if own else P(rmax), P(stat), flags,
                                  C.c_double(m), bits, int(sym), div_mode, prologue, L.stream_ptr()), "dfq_observe_quant")
    want_y, want_rmin, want_rmax, want_st = _observer_oracle(x.cpu().numpy(), batch, flags, r0[0], r0[1], m, bits, sym,
                                                             div_mode, prologue)
    case = (batch, per, flags, m, bits, sym, div_mode, prologue)
    assert _same(stat.cpu().numpy(), want_st)[0], (case, stat, want_st)
    if not own:
        assert _same(rmin.cpu().numpy(), [want_rmin])[0] and _same(rmax.cpu().numpy(), [want_rmax])[0], \
            (case, float(rmin), float(want_rmin), float(rmax), float(want_rmax))
    ok, info = _same(y.cpu().numpy(), want_y)
    assert ok, (case, info)


def _observer_geometries(sms):
    grid = sms * OBS_BLOCKS_PER_SM
    big_per = 2359296                             # one sample of 64 x 192 x 192: a 4469-float chunk on 132 SMs
    splits = min(-(-big_per // (THREADS * ITEM)), grid)
    chunk = -(-big_per // splits)
    assert chunk % 4 != 0, "every split after the first should start unaligned"
    items_batch = 4096
    assert items_batch > grid, "more (sample, split) items than CTAs"
    return [("one-sample-unaligned-splits", 1, big_per), ("items-exceed-grid", items_batch, 48), ("per1", 37, 1),
            ("per3", 29, 3), ("per675", 16, 675), ("n3", 1, 3), ("n2-per1", 2, 1)]


SMALL = ["items-exceed-grid", "per1", "per3", "per675", "n3", "n2-per1"]


@pytest.mark.parametrize("geometry", SMALL + ["one-sample-unaligned-splits"])
def test_observer_geometry_every_mode(geometry):
    """Flags UPDATE, EMA, UPDATE|EMA and OWN x prologue 0/1/2 x symmetric x both division modes on the small geometries;
    the 2.36 M-element sample with a subset of them."""
    geo = {g[0]: g[1:] for g in _observer_geometries(_sms())}
    batch, per = geo[geometry]
    x = _rand(batch * per, batch + per)
    big = batch * per > 1 << 20
    combos = [(f, p, s, d) for f in (1, 2, 3, 4) for p in (0, 1, 2) for s in (False, True) for d in (0, 1)]
    if big:
        combos = [(f, 0, False, 1) for f in (1, 2, 3, 4)] + [(4, 2, True, 1), (3, 1, False, 0)]
    moms = [0.1, 0.01, 0.5, 0.9, 0.99]
    for i, (flags, prologue, sym, div_mode) in enumerate(combos):
        _run_observer(x, batch, flags, moms[i % len(moms)], (8, 4, 16, 2)[i % 4], sym, div_mode, prologue)


def test_observer_unaligned_input_and_resnet_sized_activation():
    """x one float past alignment (scalar paths of both phases), and the 64 x 64 x 56 x 56 ResNet-18 conv input."""
    x = _unaligned(_rand(7 * 3001, 3))
    for flags in (1, 2, 4):
        _run_observer(x, 7, flags, 0.9, prologue=0)
        _run_observer(x, 7, flags, 0.99, prologue=2, sym=True)
    xa = _rand(64 * 64 * 56 * 56, 5)
    for flags in (1, 2, 3):
        _run_observer(xa, 64, flags, 0.1)
    _run_observer(xa, 64, 4, prologue=2, sym=True)


def test_observer_momentum_seeded():
    """EMA at momentum 0.1, 0.01, 0.5, 0.9, 0.99 and 64 seeded values, through dfq_observe_quant and dfq_observer_update."""
    L, lib = _lib()
    rng = np.random.default_rng(64)
    x = _rand(8 * 4000, 9)
    moms = [0.1, 0.01, 0.5, 0.9, 0.99] + list(rng.uniform(0, 1, 64))
    for m in moms:
        _run_observer(x, 8, 2, float(m), r0=(-0.37, 0.61))
    stat = torch.tensor([-1.2345678, 2.3456789], device="cuda")
    for m in moms:
        rmin = torch.tensor([-0.37], device="cuda"); rmax = torch.tensor([0.61], device="cuda")
        L.check(lib.dfq_observer_update(P(rmin), P(rmax), P(stat), 2, C.c_double(float(m)), L.stream_ptr()), "ema")
        om, mf = f32(1.0 - float(m)), f32(m)
        want = (f32(f32(-0.37) * om) + f32(f32(-1.2345678) * mf), f32(f32(0.61) * om) + f32(f32(2.3456789) * mf))
        assert _same([float(rmin), float(rmax)], want)[0], (m, float(rmin), want)


def test_observer_through_quantize_and_quantmeasure_inplace():
    """quantize(x) with no range on CUDA (prologue 2, a tensor divisor: true division), num_chunks, in place; and
    QuantMeasure with float64 running buffers."""
    from dfq_b200.utils import quantize as Q
    x = _rand(64 * 3 * 17 * 5, 4).view(64, 3, 17, 5)
    for num_chunks, sym in ((None, False), (16, True), (64, False)):
        batch = 64 // (num_chunks or 64)
        want = O.quantize_tensor_range(x.cpu().numpy(), 8, *O.per_sample_minmax_mean(x.cpu().numpy().reshape(batch, -1)),
                                       symmetric=sym, prologue=2)
        xi = x.clone()
        got = Q.quantize(xi, 8, symmetric=sym, num_chunks=num_chunks, inplace=True)
        assert got.data_ptr() == xi.data_ptr() and _same(xi.cpu().numpy(), want)[0], (num_chunks, sym)
    qm = Q.QuantMeasure(True).eval()
    qm.running_min = torch.zeros(1, device="cuda", dtype=torch.float64)
    qm.running_max = torch.zeros(1, device="cuda", dtype=torch.float64)
    y = qm(x)
    rmin, rmax = O.observer_update(0.0, 0.0, x.cpu().numpy())
    assert qm.running_min.dtype == torch.float64 and (float(qm.running_min), float(qm.running_max)) == (float(rmin), float(rmax))
    assert _same(y.cpu().numpy(), O.quantize(x.cpu().numpy(), 8, float(rmin), float(rmax), div_mode="recip"))[0]


def test_observer_refuses_bad_caller_tensors():
    """Running buffers on the wrong device or of the wrong length, BN statistics likewise: refused on the host."""
    from dfq_b200 import _lib as L
    from dfq_b200.distill import bn_stat_loss
    from dfq_b200.utils import quantize as Q
    x = _rand(4 * 10, 1).view(4, 10)
    with pytest.raises(L.DfqError, match="is on cpu"):
        Q.observe_and_quant(x, 8, 1, torch.zeros(1), torch.zeros(1, device="cuda"))
    with pytest.raises(L.DfqError, match="one element"):
        Q.observe_and_quant(x, 8, 1, torch.zeros(3, device="cuda"), torch.zeros(1, device="cuda"))
    with pytest.raises(L.DfqError, match="cannot view"):
        Q.quantize(_rand(5 * 3, 2).view(5, 3), 8, num_chunks=2)
    xb = _rand(2 * 3 * 16, 3).view(2, 3, 4, 4)
    with pytest.raises(L.DfqError, match="is on cpu"):
        bn_stat_loss(xb, torch.zeros(3), torch.ones(3, device="cuda"))
    with pytest.raises(L.DfqError, match="elements for 3 channels"):
        bn_stat_loss(xb, torch.zeros(4, device="cuda"), torch.ones(3, device="cuda"))
    # float64 statistics are converted, not reinterpreted
    mu, sd = torch.randn(3, device="cuda", dtype=torch.float64), torch.rand(3, device="cuda", dtype=torch.float64) + 0.5
    lm, ls = bn_stat_loss(xb, mu, sd)
    rl, rs, _, _ = O.bn_stat_loss(xb.cpu().numpy(), mu.float().cpu().numpy(), sd.float().cpu().numpy())
    assert abs(float(lm) - rl) <= 1e-5 * rl and abs(float(ls) - rs) <= 1e-5 * rs


def test_per_sample_statistic_batch_limit():
    """dfq_act_minmax_per_sample: batch 65535 is accepted and exact, 65536 is refused with a message."""
    L, lib = _lib()
    for batch in (65535, 65536):
        x = _rand(batch * 3, 6)
        out = torch.empty(2, device="cuda"); scratch = torch.empty(2 * batch, device="cuda")
        rc = lib.dfq_act_minmax_per_sample(P(x), batch, 3, P(out), P(scratch), L.stream_ptr())
        if batch == 65535:
            L.check(rc, "dfq_act_minmax_per_sample")
            assert _same(out.cpu().numpy(), O.per_sample_minmax_mean(x.cpu().numpy().reshape(batch, 3)))[0]
        else:
            assert rc != 0 and b"batch too large" in lib.dfq_last_error()


def test_statistics_skip_nan():
    """DESIGN.md section 4: NaN elements are skipped by every min/max reduction; an all-NaN sample gives (+inf, -inf)."""
    from dfq_b200.utils import quantize as Q
    x = _rand(6 * 5000, 8).view(6, 5000)
    x[0, 17] = float("nan"); x[2, ::3] = float("nan"); x[3] = float("nan")
    xn = x.cpu().numpy()
    assert _same(Q.tensor_minmax(x).cpu().numpy(), O.flat_minmax(xn))[0]
    assert _same(Q.tensor_minmax(x[3]).cpu().numpy(), [np.inf, -np.inf])[0]
    assert _same(Q.per_sample_minmax_mean(x).cpu().numpy(), O.per_sample_minmax_mean(xn))[0]
    keep = [0, 1, 2, 4, 5]
    _run_observer(x[keep].contiguous(), 5, 1)
    _run_observer(x.contiguous(), 6, 4)


# ---------------------------------------------------------------------------------------------------------------------
# element-wise quantizer and clamp: values
# ---------------------------------------------------------------------------------------------------------------------
def _value_vector(lo, hi, bits, sym):
    """Grid points, every rounding boundary and 1-3 ulps around it, NaN, +-inf, +-0, subnormals, the range ends."""
    if sym:
        a = max(abs(lo), abs(hi)); qmin, qmax, base = -2.0 ** (bits - 1), 2.0 ** (bits - 1) - 1, 0.0
        s = max(a / qmax, 1e-8)
    else:
        qmin, qmax, base = 0.0, 2.0 ** bits - 1, lo
        s = max((hi - lo) / qmax, 1e-8)
    k = np.arange(qmin, min(qmax, qmin + 600) + 1)
    pts = [f32(base) + (k * s).astype(f32), f32(base) + ((k + 0.5) * s).astype(f32)]
    ties = pts[1]
    for d in (1, 2, 3):
        up, dn = ties.copy(), ties.copy()
        for _ in range(d):
            up, dn = np.nextafter(up, f32(np.inf)), np.nextafter(dn, f32(-np.inf))
        pts += [up, dn]
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-45, -1e-45, 1e-39, -3e-39, 1.17e-38, lo, hi,
                        np.nextafter(f32(lo), f32(-np.inf)), np.nextafter(f32(hi), f32(np.inf)), 3e38, -3e38], f32)
    return np.concatenate(pts + [special]).astype(f32)


RANGES = [(-1.3, 2.1, False), (0.0, 6.0, False), (-3.0, 1.0, True), (0.5, 0.5, False), (0.0, 0.0, True)]


@pytest.mark.parametrize("bits", [2, 4, 8, 16])
@pytest.mark.parametrize("lo,hi,sym", RANGES)
def test_quantizer_values(lo, hi, sym, bits):
    """dfq_quant_dequant (both division modes), dfq_quant_dequant_dev (prologue 0/1/2), dfq_quant_error and dfq_clamp on
    NaN, +-inf, -0.0, subnormals and every rounding boundary of the grid, bit-exact against the oracle."""
    L, lib = _lib()
    from dfq_b200.utils import quantize as Q
    xn = _value_vector(lo, hi, bits, sym)
    x = torch.from_numpy(xn).cuda()
    for div_mode in (0, 1):
        got = Q.fake_quant_explicit(x, bits, lo, hi, sym, div_mode=div_mode)
        ok, info = _same(got.cpu().numpy(), O.quantize(xn, bits, lo, hi, sym, div_mode="recip" if div_mode else "div"))
        assert ok, ("explicit", div_mode, info)
    mn, mx = torch.tensor([lo], device="cuda"), torch.tensor([hi], device="cuda")
    for prologue in (0, 1, 2):
        for div_mode in (0, 1):
            got = Q.fake_quant_device_range(x, bits, mn, mx, sym, prologue=prologue, div_mode=div_mode)
            want = (O.quantize(xn, bits, float(f32(lo)), float(f32(hi)), sym, div_mode="recip" if div_mode else "div")
                    if prologue == 0 else O.quantize_tensor_range(xn, bits, lo, hi, sym, prologue))
            ok, info = _same(got.cpu().numpy(), want)
            assert ok, ("device range", prologue, div_mode, info)
    mm = torch.tensor([lo, hi], device="cuda")
    eps = torch.empty_like(x)
    L.check(lib.dfq_quant_error(P(x), P(eps), x.numel(), P(mm), bits, int(sym), L.stream_ptr()), "dfq_quant_error")
    with np.errstate(invalid="ignore"):
        want = O.quantize(xn, bits, float(f32(lo)), float(f32(hi)), sym) - xn
    assert _same(eps.cpu().numpy(), want)[0]
    c = x.clone()
    L.check(lib.dfq_clamp(P(c), c.numel(), C.c_float(lo), C.c_float(hi), L.stream_ptr()), "dfq_clamp")
    # np.clip leaves the sign of a zero at a zero bound open: +-0 compare equal here
    assert np.array_equal(c.cpu().numpy(), np.clip(xn, f32(lo), f32(hi)), equal_nan=True)


def test_nan_survives_the_observer_quantizer():
    """A NaN activation stays NaN through QuantMeasure (torch's clamp_ keeps it); its neighbours are quantized as usual."""
    from dfq_b200.utils import quantize as Q
    x = _rand(4 * 999, 12).view(4, 999)
    x[1, 5] = float("nan")
    qm = Q.QuantMeasure(True).eval()
    y = qm(x)
    rmin, rmax = O.observer_update(0.0, 0.0, x.cpu().numpy())
    assert _same(y.cpu().numpy(), O.quantize(x.cpu().numpy(), 8, float(rmin), float(rmax), div_mode="recip"))[0]
    assert torch.isnan(y[1, 5]) and int(torch.isnan(y).sum()) == 1


# ---------------------------------------------------------------------------------------------------------------------
# element-wise quantizer, minmax and ranges: geometry
# ---------------------------------------------------------------------------------------------------------------------
def test_flat_kernels_grid_stride_tails_and_alignment():
    """n past the grid-stride limits of k_quant (flat_grid(n, 8)) and k_minmax (flat_grid(n, kItemFloats), far enough for
    its four-load loop), tails n % 4 in {1, 2, 3}, a misaligned `codes` beside an aligned x, and an unaligned x."""
    L, lib = _lib()
    from dfq_b200.utils import quantize as Q
    cap = _sms() * 8 * THREADS
    sizes = [5 * cap * ITEM + 3, 3 * cap * 8 + 1, 1000001, 1000002, 1000003, 1, 2, 3]
    for i, n in enumerate(sizes):
        x = _rand(n, 20 + i, 2.0, -0.3)
        xn = x.cpu().numpy()
        assert _same(Q.tensor_minmax(x).cpu().numpy(), O.flat_minmax(xn))[0], n
        lo, hi = float(xn.min()), float(xn.max())
        want, codes_want = O.quantize(xn, 8, lo, hi, div_mode="recip", return_codes=True)
        y = torch.empty_like(x)
        codes = torch.empty(n + 1, device="cuda")[1:]
        qmin, qmax, mn, scale = O.quant_scalars(8, lo, hi)
        L.check(lib.dfq_quant_dequant(P(x), P(y), n, C.c_float(mn), C.c_double(scale), C.c_float(qmin), C.c_float(qmax), 1,
                                      P(codes), L.stream_ptr()), "dfq_quant_dequant")
        assert _same(y.cpu().numpy(), want)[0] and _same(codes.cpu().numpy(), codes_want)[0], n
        mm = torch.tensor([lo, hi], device="cuda")
        codes2 = torch.empty(n + 1, device="cuda")[1:]
        L.check(lib.dfq_quant_dequant_dev(P(x), P(y), n, P(mm[0:1]), P(mm[1:2]), 8, 0, 0, 1, P(codes2), L.stream_ptr()), "dev")
        assert _same(y.cpu().numpy(), O.quantize_tensor_range(xn, 8, lo, hi, prologue=1))[0], n
        L.check(lib.dfq_quant_error(P(x), P(y), n, P(mm), 8, 1, L.stream_ptr()), "dfq_quant_error")
        assert _same(y.cpu().numpy(), O.quantize(xn, 8, lo, hi, True) - xn)[0], n
        if n < cap:
            xu = _unaligned(x)
            assert _same(Q.tensor_minmax(xu).cpu().numpy(), O.flat_minmax(xn))[0], n
            yu = Q.fake_quant_explicit(xu, 8, lo, hi)
            assert _same(yu.cpu().numpy(), want)[0], n
            xi = x.clone()
            Q.quantize(xi, 8, lo, hi, inplace=True)
            assert _same(xi.cpu().numpy(), want)[0], n


def test_range_rows_both_paths_and_grid_stride():
    """dfq_range_rows: row_len 2048 (warp per row), 2049 and 4608 (CTA per row), with more rows than the grid holds."""
    L, lib = _lib()
    sms = _sms()
    assert RANGE_CTA == 2048
    for rows, row_len in ((sms * 8 * (THREADS // 32) + 5, 2048), (sms * 8 + 3, 2049), (sms * 8 + 3, 4608), (3, 2049), (5, 7)):
        w = _rand(rows * row_len, rows + row_len)
        for src in (w, _unaligned(w) if row_len % 4 else w):
            mn = torch.empty(rows, device="cuda"); mx = torch.empty(rows, device="cuda")
            L.check(lib.dfq_range_rows(P(src), rows, row_len, P(mn), P(mx), L.stream_ptr()), "dfq_range_rows")
            wn = w.cpu().numpy().reshape(rows, row_len)
            assert _same(mn.cpu().numpy(), wn.min(1))[0] and _same(mx.cpu().numpy(), wn.max(1))[0], (rows, row_len)


# ---------------------------------------------------------------------------------------------------------------------
# BN-statistics loss of the distilled-data generation
# ---------------------------------------------------------------------------------------------------------------------
def _reference_formula(x, bn_mean, bn_std, eps=EPS):
    """distill_data.py:171-185."""
    n, c = x.size(0), x.size(1)
    flat = x.view(n, c, -1)
    own = lambda a, b: (a - b).norm() ** 2 / a.size(0)
    return own(bn_mean, torch.mean(flat, dim=2)), own(bn_std, torch.std(flat + eps, dim=2))


def _reference_formula_f64(x, bn_mean, bn_std, eps=EPS):
    """The same formula evaluated in float64 inside an fp32 network."""
    lm, ls = _reference_formula(x.double(), bn_mean.double(), bn_std.double(), eps)
    return lm.float(), ls.float()


def _ref_loss_grad(x, mu, sd, gm, gs, dtype):
    xr = x.detach().to(dtype).requires_grad_(True)
    lm, ls = _reference_formula(xr, mu.to(dtype), sd.to(dtype))
    (gm * lm + gs * ls).backward()
    return np.array([float(lm), float(ls)]), xr.grad.double()


def _ulps(v):
    return 4.0 * float(np.spacing(f32(abs(v))))


def _check_bnstat(x, mu, sd, gm=1.7, gs=0.6, accumulate=False, what=""):
    """The kernels through the C ABI (x may be unaligned), against float64 autograd with the fp32 yardstick."""
    L, lib = _lib()
    n, c = x.shape[0], x.shape[1]
    hw = x.numel() // (n * c)
    m = torch.empty(n * c, device="cuda"); s = torch.empty(n * c, device="cuda")
    loss = torch.empty(2, device="cuda", dtype=torch.float64)
    L.check(lib.dfq_bnstat_loss_fwd(P(x), n, c, hw, P(mu), P(sd), C.c_float(EPS), P(m), P(s), P(loss), L.stream_ptr()), "fwd")
    base = torch.randn(x.shape, device="cuda") if accumulate else torch.zeros(x.shape, device="cuda")
    gx = base.clone()
    g2 = torch.tensor([gm, gs], device="cuda")
    L.check(lib.dfq_bnstat_loss_bwd(P(x), P(gx), n, c, hw, P(mu), P(sd), C.c_float(EPS), P(m), P(s), P(g2), int(accumulate),
                                    L.stream_ptr()), "bwd")
    l64, g64 = _ref_loss_grad(x, mu, sd, gm, gs, torch.float64)
    l32, g32 = _ref_loss_grad(x, mu, sd, gm, gs, torch.float32)
    got = loss.cpu().numpy()
    for k in range(2):
        err, yard = abs(got[k] - l64[k]), 2 * abs(l32[k] - l64[k]) + _ulps(l64[k])
        assert err <= yard, (what, k, got[k], l64[k], err, yard)
    assert torch.isfinite(gx).all(), what
    gerr = float((gx.double() - base.double() - g64).abs().max())
    yard = 2 * float((g32 - g64).abs().max()) + _ulps(float(g64.abs().max()))
    if accumulate:
        yard += float(np.spacing(f32((base.double() + g64).abs().max().item())))
    assert gerr <= yard, (what, gerr, yard)


HW = [2, 3, 5, 7, 49, 2047, 2048, 2049, 2050]


@pytest.mark.parametrize("hw", HW)
def test_bnstat_spatial_sizes_with_constant_and_offset_rows(hw):
    """Both fwd paths (warp per row below kBnstatCtaRow, CTA per row from it), vector and scalar loops, rows straddling a
    four-element group in the backward pass; with a constant zero row, a constant non-zero row and |mean|/std = 1e4."""
    assert BN_CTA == 2048
    g = torch.Generator(device="cuda").manual_seed(hw)
    n, c = 3, 5
    x = torch.randn(n, c, hw, device="cuda", generator=g) * 1.3 + 0.2
    x[0, 0] = 0.0
    x[1, 2] = 2.75
    x[2, 1] = 1e4 + torch.randn(hw, device="cuda", generator=g)
    x[2, 3] = -3e3 + 0.3 * torch.randn(hw, device="cuda", generator=g)
    mu = torch.randn(c, device="cuda", generator=g) * 0.3
    sd = torch.rand(c, device="cuda", generator=g) + 0.5
    _check_bnstat(x, mu, sd, what=("hw", hw))
    _check_bnstat(_unaligned(x).view(x.shape), mu, sd, what=("unaligned", hw))
    _check_bnstat(x, mu, sd, accumulate=True, what=("accumulate", hw))


def test_bnstat_grid_stride_loops_and_degenerate_shapes():
    """Rows above the warp-path grid (SMs x 8 CTAs x 8 warps) and the CTA-path grid (SMs x 8), totals above the backward
    grid (SMs x 16 x 1024 elements per pass); N = 1, C = 1."""
    sms = _sms()
    warp_rows = sms * 8 * (DTHREADS // 32) + 9
    cta_rows = sms * 9
    assert cta_rows * 2049 > sms * 16 * DTHREADS * 4
    g = torch.Generator(device="cuda").manual_seed(1)
    for what, shape in (("warp grid", (1, warp_rows, 7)), ("warp grid N", (warp_rows, 1, 6)),
                        ("cta grid", (3, cta_rows // 3, 2049)), ("N=1", (1, 4, 33)), ("C=1", (6, 1, 2050))):
        x = torch.randn(*shape, device="cuda", generator=g) * 0.9 - 0.1
        mu = torch.randn(shape[1], device="cuda", generator=g) * 0.3
        sd = torch.rand(shape[1], device="cuda", generator=g) + 0.5
        _check_bnstat(x, mu, sd, what=what)


def test_bnstat_wrapper_channels_last_and_hw1_fallback():
    """bn_stat_loss on a channels_last input, and a 1x1 input, which takes the reference's own view(C, -1) formula."""
    from dfq_b200.distill import bn_stat_loss
    g = torch.Generator(device="cuda").manual_seed(2)
    x = (torch.randn(4, 6, 9, 7, device="cuda", generator=g)).to(memory_format=torch.channels_last).requires_grad_(True)
    mu = torch.randn(6, device="cuda", generator=g) * 0.3
    sd = torch.rand(6, device="cuda", generator=g) + 0.5
    lm, ls = bn_stat_loss(x, mu, sd)
    (1.7 * lm + 0.6 * ls).backward()
    l64, g64 = _ref_loss_grad(x.contiguous(), mu, sd, 1.7, 0.6, torch.float64)
    l32, g32 = _ref_loss_grad(x.contiguous(), mu, sd, 1.7, 0.6, torch.float32)
    for k, v in enumerate((lm, ls)):
        assert abs(float(v) - l64[k]) <= 2 * abs(l32[k] - l64[k]) + _ulps(l64[k]) + float(np.spacing(f32(l64[k])))
    assert float((x.grad.double() - g64).abs().max()) <= 2 * float((g32 - g64).abs().max()) + _ulps(float(g64.abs().max()))
    # 1x1: distill_data.py:181-182 takes the std over x.view(C, -1), a reinterpretation of the memory, not per channel
    x1 = torch.randn(5, 8, 1, 1, device="cuda", generator=g)
    mu1, sd1 = torch.randn(8, device="cuda", generator=g), torch.rand(8, device="cuda", generator=g) + 0.5
    lm1, ls1 = bn_stat_loss(x1, mu1, sd1)
    x64 = x1.double()
    own = lambda a, b: (a - b).norm() ** 2 / a.size(0)
    want_m = float(own(mu1.double(), x64.view(5, 8, -1).mean(2)))
    want_s = float(own(sd1.double(), torch.std(x64.view(8, -1) + EPS, dim=1)))
    assert abs(float(lm1) - want_m) <= 1e-6 * want_m and abs(float(ls1) - want_s) <= 1e-6 * want_s


def _bn_inputs(model, batch=32, seed=0):
    torch.manual_seed(seed)
    acts = []
    hooks = [m.register_forward_hook(lambda mod, i, o: acts.append((mod, i[0].detach())))
             for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        model(torch.randn(batch, 3, 224, 224, device="cuda"))
    for h in hooks:
        h.remove()
    return acts


def _seeded(name):
    import torchvision
    torch.manual_seed(0)
    model = getattr(torchvision.models, name)(weights=None).cuda().eval()
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.3); m.running_var.uniform_(0.5, 1.5)
    return model


@pytest.mark.parametrize("name", ["resnet18", "mobilenet_v2"])
def test_bnstat_every_bn_input_of_real_models(name):
    """Every BatchNorm input of seeded ResNet-18 / MobileNetV2 at batch 32, 224x224 (rows of 12544 down to 49, dead ReLU
    channels included): the kernels' loss and gradient against float64 autograd."""
    model = _seeded(name)
    for k, (bn, x) in enumerate(_bn_inputs(model)):
        mu = bn.running_mean.detach().float().contiguous()
        sd = torch.sqrt(bn.running_var + EPS).detach().float().contiguous()
        _check_bnstat(x.contiguous(), mu, sd, what=(name, k, tuple(x.shape)))


def test_get_distil_data_iteration_zero_against_the_reference_formula(monkeypatch):
    """getDistilData(gpu=True) on seeded ResNet-18: the first iteration's loss and pixel gradient with the fused kernels
    against the same call with bn_stat_loss replaced by the reference formula evaluated in float64 (same noise,
    deterministic cuDNN).  The loss agrees to 1e-5.  The pixel gradient sums the backward passes of all 20 layers' losses
    through the network and is far more sensitive: on an H100 the reference formula in fp32 sits 5.5e-4 (normwise) from
    the float64 one, the fused kernels 5.9e-4.  So the gradient gets the yardstick of the other distillation tests: at most
    twice the fp32 formula's error."""
    from dfq_b200 import distill
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    model = _seeded("resnet18")

    def run(patch):
        seen = {}

        class Adam(torch.optim.Adam):
            def step(self, closure=None):
                seen["grad"] = self.param_groups[0]["params"][0].grad.detach().double().clone()
                return super().step(closure)

        class Plateau(torch.optim.lr_scheduler.ReduceLROnPlateau):
            def step(self, metrics, *a, **k):
                seen["loss"] = float(metrics)
                return super().step(metrics, *a, **k)

        with monkeypatch.context() as mp:
            mp.setattr(distill, "optim", types.SimpleNamespace(Adam=Adam, lr_scheduler=types.SimpleNamespace(ReduceLROnPlateau=Plateau)))
            if patch:
                mp.setattr(distill, "bn_stat_loss", patch)
            torch.manual_seed(11)
            distill.getDistilData(model, "imagenet", 4, num_batch=1, gpu=True, iterations=1)
        return seen

    fused, ref, ref32 = run(None), run(_reference_formula_f64), run(_reference_formula)
    err = lambda a: (abs(a["loss"] - ref["loss"]) / abs(ref["loss"]),
                     float((a["grad"] - ref["grad"]).abs().max() / ref["grad"].abs().max()))
    print("iteration 0 against the float64 formula: fused loss %.3g grad %.3g, fp32 formula loss %.3g grad %.3g"
          % (err(fused) + err(ref32)))
    assert err(fused)[0] <= 1e-5, err(fused)
    assert err(fused)[1] <= 2 * err(ref32)[1] + 1e-6, (err(fused), err(ref32))


def test_every_quantmeasure_input_of_mobilenet_v2():
    """The input of every Conv2d / Linear of seeded MobileNetV2 at batch 32 (what QuantMeasure sees): update_stat in eval
    mode, then one training (EMA) step, bit-exact against the oracle."""
    from dfq_b200.utils import quantize as Q
    import torchvision
    torch.manual_seed(0)
    model = torchvision.models.mobilenet_v2(weights=None).cuda().eval()
    acts = []
    hooks = [m.register_forward_hook(lambda mod, i, o: acts.append(i[0].detach()))
             for m in model.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear))]
    with torch.no_grad():
        model(torch.randn(32, 3, 224, 224, device="cuda"))
    for h in hooks:
        h.remove()
    assert len(acts) == 53
    for k, x in enumerate(acts):
        xn = x.cpu().numpy()
        qm = Q.QuantMeasure(True).cuda().eval()
        y = qm(x)
        rmin, rmax = O.observer_update(0.0, 0.0, xn)
        assert (float(qm.running_min), float(qm.running_max)) == (float(rmin), float(rmax)), k
        assert _same(y.cpu().numpy(), O.quantize(xn, 8, float(rmin), float(rmax), div_mode="recip"))[0], k
        qm.train()
        y = qm(x)
        er_min, er_max, st_min, st_max = O.observer_ema(rmin, rmax, xn)
        er_min, er_max = O.observer_ema(f32(np.fmin(rmin, st_min)), f32(np.fmax(rmax, st_max)), xn)[:2]
        assert (float(qm.running_min), float(qm.running_max)) == (float(er_min), float(er_max)), k
        assert _same(y.cpu().numpy(), O.quantize(xn, 8, float(st_min), float(st_max), div_mode="recip"))[0], k
