"""CPU oracle for the DFQ calibration hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
leg may import this module.  The product package ``dfq_b200`` never does: it runs the sm_90a CUDA
kernels behind ``libdfq_sm90.so`` and raises when that library is missing.

What it is: a numpy (IEEE fp32, explicit op order) restatement of the arithmetic of the reference
jakc4103/DFQ (commit 6f15805c) for the path SURVEY.md section 8 names.  Each function cites the
reference ``file:line`` it follows.  The reference's arithmetic lives in PyTorch's CPU kernels;
every op used here (+, -, *, /, sqrt, rint, min, max on float32) is a correctly rounded IEEE op in
both numpy and ATen, which is why results can be compared bit for bit.

Parity pinning (see ``tests/test_oracle_pins.py`` and ``tools/make_golden.py``):
  * the reference's only checked-in numeric artefact, ``modeling/ncnn/model_quant_relu_equal.table``,
    is reproduced by this oracle (BN fold + signed equalization + activation ranges) when the
    reference tree is present;
  * fixtures under ``tests/golden/`` were produced by importing and running the reference itself in
    the build container (``tools/make_golden.py``) and are compared bit-exactly (equalization,
    fake-quant codes, BN fold) or to 1e-5 normwise (bias correction, whose fp32 BLAS mat-vec has no
    defined summation order).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

f32 = np.float32


# --------------------------------------------------------------------------------------------
# fake quantization: utils/quantize.py:23-76 (UniformQuantize.forward), explicit-range path
# --------------------------------------------------------------------------------------------
def quant_scalars(num_bits: int, min_value: float, max_value: float, symmetric: bool = False):
    """Python-double scalar prologue of UniformQuantize.forward (quantize.py:49-66).

    Returns (qmin, qmax, min_value, scale) as Python floats (doubles), exactly as the reference forms
    them before they are rounded to fp32 by the in-place tensor ops.
    """
    min_value = float(min_value)
    max_value = float(max_value)
    if symmetric:
        qmin = -2.0 ** (num_bits - 1)
        qmax = float(2 ** (num_bits - 1) - 1)
        max_value = abs(max_value)
        min_value = abs(min_value)
        if max_value < min_value:
            max_value = min_value
        scale = max_value / qmax
        min_value = 0.0
    else:
        qmin = 0.0
        qmax = 2.0 ** num_bits - 1.0
        scale = (max_value - min_value) / (qmax - qmin)
    scale = max(scale, 1e-8)
    return qmin, qmax, min_value, scale


def quantize(x: np.ndarray, num_bits: int = 8, min_value: Optional[float] = None,
             max_value: Optional[float] = None, symmetric: bool = False,
             div_mode: str = "div", return_codes: bool = False):
    """Fake-quantize ``x`` (fp32) on the reference grid.  quantize.py:70-74:
    ``add_(-min).div_(scale).clamp_(qmin, qmax).round_().mul_(scale).add_(min)``  -  four separately
    rounded fp32 ops around a clamp and a round-half-even.

    div_mode "div"   : true IEEE division  (PyTorch CPU, ``div_(python_float)``)
    div_mode "recip" : ``t * fp32(1.0 / scale)`` with the reciprocal formed in double from the Python scalar - what PyTorch
                       CUDA eager computes for ``div_(python_float)`` [probed with torch 2.11]
    """
    x = np.ascontiguousarray(x, dtype=f32)
    if min_value is None:
        min_value = float(x.min())
    if max_value is None:
        max_value = float(x.max())
    qmin, qmax, mn, scale = quant_scalars(num_bits, min_value, max_value, symmetric)
    s32 = f32(scale)
    t = x + f32(-mn)
    if div_mode == "div":
        t = t / s32
    elif div_mode == "recip":
        t = t * f32(1.0 / scale)
    else:
        raise ValueError(div_mode)
    t = np.minimum(np.maximum(t, f32(qmin)), f32(qmax))
    codes = np.rint(t)
    y = codes * s32
    y = y + f32(mn)
    if return_codes:
        return y.astype(f32), codes.astype(f32)
    return y.astype(f32)


def tensor_range_scalars(num_bits: int, min_value, max_value, symmetric: bool, prologue: int):
    """Scalar prologue when min/max are fp32 0-d TENSORS (quantize.py:24-35, then :49-66 on tensors): every step an fp32
    op.  ``prologue`` 1: ``/ qmax`` is a true division (CPU tensors); 2: a multiply by the fp32 reciprocal of qmax (a CUDA
    tensor divided by a Python scalar).  Returns (qmin, qmax, min_value, scale) as fp32."""
    mn, mx = f32(min_value), f32(max_value)
    with np.errstate(over="ignore", invalid="ignore"):
        if symmetric:
            qmin, qmax = f32(-2.0 ** (num_bits - 1)), f32(2 ** (num_bits - 1) - 1)
            mx, mn = abs(mx), abs(mn)
            if mx < mn:
                mx = mn
            d, mn = mx, f32(0)
        else:
            qmin, qmax = f32(0), f32(2.0 ** num_bits - 1)
            d = f32(mx - mn)
        scale = f32(d * (f32(1) / qmax)) if prologue == 2 else f32(d / qmax)
    if f32(1e-8) > scale:
        scale = f32(1e-8)
    return qmin, qmax, mn, scale


def quantize_tensor_range(x: np.ndarray, num_bits: int, min_value, max_value, symmetric: bool = False, prologue: int = 1):
    """quantize.py:70-74 with the range of ``tensor_range_scalars``.  The element-wise ``div_(scale)`` is by a tensor and
    therefore a true division on both devices."""
    qmin, qmax, mn, scale = tensor_range_scalars(num_bits, min_value, max_value, symmetric, prologue)
    x = np.ascontiguousarray(x, dtype=f32)
    with np.errstate(over="ignore", invalid="ignore"):
        t = (x + (-mn)) / scale
        return (np.rint(np.minimum(np.maximum(t, qmin), qmax)) * scale + mn).astype(f32)


def quantize_error(w: np.ndarray, num_bits: int = 8, signed: bool = False) -> np.ndarray:
    """dfq.py:8-25 with ``reduction=None``: Q(W) - W using the tensor's own min/max."""
    w = np.ascontiguousarray(w, dtype=f32)
    q = quantize(w, num_bits, float(w.min()), float(w.max()), symmetric=signed)
    return (q - w).astype(f32)


# --------------------------------------------------------------------------------------------
# BN fold: utils/layer_transform.py:246-272
# --------------------------------------------------------------------------------------------
def bn_fold(w: np.ndarray, b: Optional[np.ndarray], gamma, beta, mean, var, eps: float, sqrt_fn=None):
    """Returns (W', b', fake_weight, fake_bias).  Op order follows layer_transform.py:251,260-261.
    `sqrt_fn`: None = correctly rounded IEEE root (numpy; what the GPU computes); tests that compare with numbers a
    particular HOST produced with the reference inject that host's torch.sqrt (MKL VML: faithful, not correctly rounded)."""
    w = np.ascontiguousarray(w, dtype=f32)
    O = w.shape[0]
    gamma = np.asarray(gamma, f32); beta = np.asarray(beta, f32)
    mean = np.asarray(mean, f32); var = np.asarray(var, f32)
    if b is None:
        b = np.zeros(O, f32)
    den = (np.sqrt if sqrt_fn is None else sqrt_fn)(var + f32(eps)).astype(f32)
    f = gamma / den                                   # [O]   (:251 quotient formed first)
    w2 = w * f.reshape((O,) + (1,) * (w.ndim - 1))
    b2 = b * f + (beta - (gamma * mean) / den)         # (:260-261 grouping)
    return w2.astype(f32), b2.astype(f32), np.abs(gamma).astype(f32), beta.copy()


# --------------------------------------------------------------------------------------------
# cross-layer equalization, one relation: dfq.py:28-75
# --------------------------------------------------------------------------------------------
def _view3(w: np.ndarray) -> np.ndarray:
    """[O, J, kk] view of a conv ([O,J,k,k]) or linear ([O,J]) weight."""
    return w.reshape(w.shape[0], w.shape[1], -1)


def group_count(c_first: int, j_second: int) -> int:
    """dfq.py:29-32."""
    return 1 if c_first == j_second else c_first // j_second


def channel_ranges(w1: np.ndarray, w2: np.ndarray, signed: bool):
    """Per-channel (r1, r2) of dfq.py:48-55 for all channels at once.

    r1[c]  : range of output row c of W1;  r2[c] : range of input column (g, ii) of W2 where
    c = g*gi + ii.  Computing all ranges first is bit-identical to the reference's channel loop
    because rows/columns of different channels are disjoint (SURVEY.md appendix A.2).
    """
    C1 = w1.shape[0]
    J2 = w2.shape[1]
    G = group_count(C1, J2)
    gi = C1 // G
    go = w2.shape[0] // G
    w1r = w1.reshape(C1, -1)
    w2v = _view3(w2)
    if signed:
        r1 = np.abs(w1r).max(axis=1)
    else:
        r1 = w1r.max(axis=1) - w1r.min(axis=1)
    r2 = np.zeros(C1, f32)
    covered = np.zeros(C1, bool)
    for g in range(G):
        blk = w2v[g * go:(g + 1) * go]               # [go, J2, kk]
        if signed:
            rr = np.abs(blk).max(axis=(0, 2))
        else:
            rr = blk.max(axis=(0, 2)) - blk.min(axis=(0, 2))
        r2[g * gi:g * gi + J2] = rr
        covered[g * gi:g * gi + J2] = True
    return r1.astype(f32), r2.astype(f32), covered, (G, gi, go)


def solve_scale(r1: np.ndarray, r2: np.ndarray, s_range=(1e-8, 1e8), eps=0, sqrt_fn=None):
    """dfq.py:58-59.  Returns (s, inv_s) as fp32 arrays.

    ``sqrt_fn``: the square root to use.  Default ``np.sqrt`` = IEEE correctly rounded, which is what
    the CUDA path computes (``sqrt.rn.f32``).  The reference's ``torch.sqrt`` on an x86 host goes
    through MKL VML and is only faithful (<=1 ulp): on the build container it differs from the
    correctly rounded root for ~0.7 % of inputs [probed].  The pin tests therefore pass
    ``torch.sqrt`` here to show bit-equality with the reference, and use the default elsewhere.

    ``s = (1/(r1+eps)) * sqrt(r1*r2+eps)`` in fp32, then Python ``max(lo, min(hi, s))``:
    NaN -> hi (``nan < hi`` is False), comparisons are made against the fp32-rounded bounds, and a
    clamped value is the Python float bound, whose reciprocal ``1/s`` (dfq.py:73) is a double
    division rounded to fp32 instead of an fp32 reciprocal.
    """
    lo, hi = float(s_range[0]), float(s_range[1])
    e = f32(eps)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        root = (sqrt_fn or np.sqrt)(r1 * r2 + e)
        s = (f32(1.0) / (r1 + e)) * np.asarray(root, f32)
        take_s = s < f32(hi)                          # False for NaN
        m_is_hi = ~take_s
        # max(lo, m): m if m > lo else lo
        keep = np.where(m_is_hi, hi > lo, s > f32(lo))
        out = np.where(keep, np.where(m_is_hi, f32(hi), s), f32(lo)).astype(f32)
        clamped_hi = keep & m_is_hi
        clamped_lo = ~keep
        inv = (f32(1.0) / out).astype(f32)
        if hi != 0:
            inv = np.where(clamped_hi, f32(1.0 / hi), inv)
        if lo != 0:
            inv = np.where(clamped_lo, f32(1.0 / lo), inv)
    return out.astype(f32), inv.astype(f32)


def layer_equalization(w1, w2, b1=None, bn_w=None, bn_b=None, s_range=(1e-8, 1e8), signed=False, eps=0,
                       sqrt_fn=None):
    """In-place equalization of one relation (numpy arrays are modified).  Returns S[C1].

    dfq.py:28-75.  Channels not covered by the loop (none for well-formed conv pairs) keep S=0 and
    are left untouched, as in the reference where ``S = torch.zeros(C1)`` (:37).
    """
    r1, r2, covered, (G, gi, go) = channel_ranges(w1, w2, signed)
    s, inv = solve_scale(r1, r2, s_range, eps, sqrt_fn)
    S = np.where(covered, s, f32(0)).astype(f32)
    mult = np.where(covered, s, f32(1)).astype(f32)
    C1 = w1.shape[0]
    w1 *= mult.reshape((C1,) + (1,) * (w1.ndim - 1))
    for v in (bn_w, bn_b, b1):
        if v is not None:
            v *= mult
    w2v = _view3(w2)
    J2 = w2.shape[1]
    for g in range(G):
        w2v[g * go:(g + 1) * go] *= inv[g * gi:g * gi + J2].reshape(1, J2, 1)
    return S


# --------------------------------------------------------------------------------------------
# sweep driver: dfq.py:78-117
# --------------------------------------------------------------------------------------------
@dataclass
class OLayer:
    """One target layer (Conv/Linear) of the oracle-side model."""
    w: np.ndarray
    b: Optional[np.ndarray] = None


@dataclass
class ORelation:
    first: int
    second: int
    bn: int                      # index into the list of (fake_weight, fake_bias) pairs
    S: Optional[np.ndarray] = None


def mean_abs_diff(a: np.ndarray, b: np.ndarray) -> float:
    """dfq.py:108 ``float(torch.mean(torch.abs(W - W_prev)))``: fp32 subtract/abs, mean accumulated
    here in float64 (the reference's fp32 reduction order is an ATen implementation detail; its
    result agrees to ~1e-7 relative, far inside the 1 % margin of the exit test, SURVEY.md H2)."""
    d = np.abs(a.astype(f32) - b.astype(f32))
    return float(d.sum(dtype=np.float64) / d.size)


def cross_layer_equalization(layers: List[OLayer], bns: List[Tuple[np.ndarray, np.ndarray]],
                             relations: List[ORelation], s_range=(1e-8, 1e8), converge_thres=2e-7,
                             converge_count=20, signed=False, eps=0, max_sweeps=None, sqrt_fn=None):
    """Gauss-Seidel sweeps over ``relations`` until the reference's exit rule fires (dfq.py:81-115).

    Returns (n_sweeps, [diff per sweep]).  ``layers`` are modified in place.
    """
    diff = 10
    count = 0
    diffs = []
    n = 0
    while diff > converge_thres and count < converge_count:
        prev = [l.w.copy() for l in layers]
        for rr in relations:
            l1, l2 = layers[rr.first], layers[rr.second]
            if l1.b is None:
                l1.b = np.zeros(l1.w.shape[0], f32)         # dfq.py:91-92
            bw, bb = bns[rr.bn]
            S = layer_equalization(l1.w, l2.w, l1.b, bw, bb, s_range=s_range, signed=signed, eps=eps,
                                   sqrt_fn=sqrt_fn)
            rr.S = S if rr.S is None else (rr.S * S).astype(f32)   # relation.py:20-24
        diff_tmp = 0.0
        for l, p in zip(layers, prev):
            diff_tmp += mean_abs_diff(l.w, p)
        diffs.append(diff_tmp)
        n += 1
        if abs(diff - diff_tmp) > 1e-9:
            count = 0
            diff = diff_tmp
        else:
            count += 1
        if max_sweeps is not None and n >= max_sweeps:
            break
    return n, diffs


# --------------------------------------------------------------------------------------------
# bias correction numerics: dfq.py:173-293
# --------------------------------------------------------------------------------------------
def std_normal_pdf(x32: np.ndarray) -> np.ndarray:
    """dfq.py:182 ``torch.from_numpy(norm(0,1).pdf(x)).float()``: float64 evaluation on the fp32
    argument, result rounded to fp32.  scipy: exp(-x**2/2)/sqrt(2*pi)."""
    x = np.asarray(x32, f32).astype(np.float64)
    return (np.exp(-x * x / 2.0) / math.sqrt(2.0 * math.pi)).astype(f32)


def std_normal_cdf(x32: np.ndarray) -> np.ndarray:
    """dfq.py:183 ``norm.cdf`` = scipy.special.ndtr in float64 -> fp32."""
    from scipy.special import ndtr
    return ndtr(np.asarray(x32, f32).astype(np.float64)).astype(f32)


def relu_expectation(fake_weight: np.ndarray, fake_bias: np.ndarray) -> np.ndarray:
    """E[ReLU(N(beta, gamma^2))] as the reference forms it (dfq.py:184, 239-240):
    ``gamma*pdf(-beta/gamma) + beta*(1 - cdf(-beta/gamma))`` in fp32, negatives set to 0."""
    g = np.asarray(fake_weight, f32); b = np.asarray(fake_bias, f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (-b) / g
        e = g * std_normal_pdf(q) + b * (f32(1.0) - std_normal_cdf(q))
    e = e.astype(f32)
    e[e < 0] = 0                                       # NaN stays NaN, as ``expect[expect < 0] = 0``
    return e


def bias_delta(w: np.ndarray, expect: np.ndarray, signed: bool = False, num_bits: int = 8) -> np.ndarray:
    """dfq.py:216-219, 281-287: per-output-channel expected quantization error.

    eps = Q8(W) - W; E = sum over k*k (fp32); per group g: E[g-th rows] @ expect[g-th slice].
    The reference's mat-vec is an fp32 BLAS call; the dot is accumulated in float64 here and
    compared normwise (1e-5) - SURVEY.md section 8(d) config 2.
    """
    w = np.ascontiguousarray(w, f32)
    eps = quantize_error(w, num_bits, signed)
    O, J = w.shape[0], w.shape[1]
    E = eps.reshape(O, J, -1).sum(axis=-1, dtype=f32)
    G = expect.shape[0] // J
    so = O // G
    si = expect.shape[0] // G
    out = np.zeros(O, f32)
    for g in range(G):
        out[g * so:(g + 1) * so] = (E[g * so:(g + 1) * so].astype(np.float64)
                                    @ expect[g * si:(g + 1) * si].astype(np.float64)).astype(f32)
    return out


def bias_delta_bound(w: np.ndarray, expect: np.ndarray, signed: bool = False, num_bits: int = 8, raw: bool = False):
    """Per-row acceptance bound for a bias-correction kernel: returns (exact, bound), both float64 [O].

    ``exact[o]`` = sum over (c, t) of eps[o, c, t] * E[c] in float64 from the bit-exact per-element errors
    eps = Q(W) - W (``raw``: the bias-absorption form, W itself in place of eps).  The documented arithmetic (fp32 sum over the
    kk taps of one column, float64 dot with E[x], one rounding to fp32) stays within

        (kk - 1) * 2^-24 * sum_c |E_c| * sum_t |eps_oct|      fp32 sum of the taps, any order
      + n * 2^-53 * sum_c |E_c * sum_t eps_oct|               float64 dot over the n = cols columns
      + 2^-24 * |exact[o]|                                     final rounding to fp32

    of ``exact[o]``.  Unlike a normwise gate over the whole layer this sees an error confined to one row, column or tap.
    """
    w = np.ascontiguousarray(w, f32)
    eps = w if raw else quantize_error(w, num_bits, signed)
    O, J = w.shape[0], w.shape[1]
    e3 = eps.reshape(O, J, -1).astype(np.float64)
    kk = e3.shape[2]
    expect = np.asarray(expect, f32).astype(np.float64)
    G = expect.shape[0] // J
    so = O // G
    ex = expect.reshape(G, J)[np.arange(O) // so]                  # [O, J]: the E[x] slice each row reads
    colsum = e3.sum(axis=2)                                         # float64: its rounding is far below the bound
    exact = (colsum * ex).sum(axis=1)
    bound = ((kk - 1) * 2.0 ** -24 * (np.abs(ex) * np.abs(e3).sum(axis=2)).sum(axis=1)
             + J * 2.0 ** -53 * np.abs(colsum * ex).sum(axis=1)
             + 2.0 ** -24 * np.abs(exact))
    return exact, bound


def rows_outside_bound(got: np.ndarray, exact: np.ndarray, bound: np.ndarray) -> np.ndarray:
    """Indices of the rows where a kernel's delta ``got`` leaves the bias_delta_bound interval."""
    err = np.abs(np.asarray(got, np.float64) - exact)
    return np.nonzero(~(err <= bound))[0]


# --------------------------------------------------------------------------------------------
# activation observer: utils/quantize.py:102-119
# --------------------------------------------------------------------------------------------
def flat_minmax(x: np.ndarray) -> Tuple[np.float32, np.float32]:
    """(min, max) of a tensor as the library's reductions form them: NaN elements are skipped (DESIGN.md section 4), so a
    tensor of NaN alone gives (+inf, -inf).  Without NaN this is ``x.min()``, ``x.max()``."""
    x = np.ascontiguousarray(x, f32).reshape(-1)
    return f32(np.fmin.reduce(x, initial=np.inf)), f32(np.fmax.reduce(x, initial=-np.inf))


def per_sample_minmax_mean(x: np.ndarray) -> Tuple[np.float32, np.float32]:
    """``x.view(B,-1).min(-1)[0].mean()`` / ``.max(...)`` (quantize.py:106-107): exact per-sample
    extrema, fp32 mean over the batch (accumulated in float64, rounded once).  NaN elements are skipped as in
    ``flat_minmax``: an all-NaN sample contributes +inf to the minimum and -inf to the maximum."""
    x = np.ascontiguousarray(x, f32).reshape(x.shape[0], -1)
    with np.errstate(invalid="ignore"):
        mn = np.fmin.reduce(x, axis=1, initial=np.inf).astype(np.float64).mean()
        mx = np.fmax.reduce(x, axis=1, initial=-np.inf).astype(np.float64).mean()
    return f32(mn), f32(mx)


def observer_update(running_min: float, running_max: float, x: np.ndarray):
    """update_stat branch of QuantMeasure.forward (quantize.py:103-107)."""
    mn, mx = per_sample_minmax_mean(x)
    return f32(min(f32(running_min), mn)), f32(max(f32(running_max), mx))


def observer_ema(running_min: float, running_max: float, x: np.ndarray, momentum: float = 0.1):
    """training branch (quantize.py:109-113): ``running.mul_(1-m).add_(value*m)`` in fp32."""
    mn, mx = per_sample_minmax_mean(x)
    rmin = f32(running_min) * f32(1 - momentum) + mn * f32(momentum)
    rmax = f32(running_max) * f32(1 - momentum) + mx * f32(momentum)
    return f32(rmin), f32(rmax), mn, mx


# --------------------------------------------------------------------------------------------
# distilled data: the BN-statistics loss of ZeroQ/distill_data.py:171-185
# --------------------------------------------------------------------------------------------
def bn_stat_loss(x: np.ndarray, bn_mean: np.ndarray, bn_std: np.ndarray, eps: float = 1e-6):
    """float64 (L_mean, L_std, dL_mean/dx, dL_std/dx) of one BatchNorm input x [N, C, ...] with more than one element per
    (n, c) row:  m = mean_hw x,  s = std_hw(x + eps) (unbiased),  L_mean = sum (mu_c - m)^2 / C,  L_std = sum (sigma_c - s)^2 / C.
    A row with s == 0 has no std gradient, as torch's std backward masks a zero result."""
    x64 = np.asarray(x, np.float64)
    n, c = x64.shape[0], x64.shape[1]
    flat = x64.reshape(n, c, -1)
    hw = flat.shape[2]
    assert hw > 1, "hw == 1 takes the reference's view(C, -1) path"
    mu = np.asarray(bn_mean, np.float64).reshape(1, c)
    sigma = np.asarray(bn_std, np.float64).reshape(1, c)
    y = flat + eps
    m = flat.mean(axis=2)
    dev = y - y.mean(axis=2, keepdims=True)
    dev[y.min(axis=2) == y.max(axis=2)] = 0.0          # a constant row: its rounded mean must not leave a residue
    s = np.sqrt((dev * dev).sum(axis=2) / (hw - 1))
    l_mean = ((mu - m) ** 2).sum() / c
    l_std = ((sigma - s) ** 2).sum() / c
    g_mean = np.broadcast_to((2.0 * (m - mu) / (c * hw))[:, :, None], flat.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(s > 0, 2.0 * (s - sigma) / (c * (hw - 1) * s), 0.0)
    g_std = k[:, :, None] * dev
    return l_mean, l_std, g_mean.reshape(x64.shape).copy(), g_std.reshape(x64.shape)


# --------------------------------------------------------------------------------------------
# misc helpers of the path
# --------------------------------------------------------------------------------------------
def clip_weight(w: np.ndarray, lo: float = -15, hi: float = 15) -> np.ndarray:
    """dfq.py:167-170."""
    return np.clip(w, f32(lo), f32(hi)).astype(f32)


def bias_absorb_c(fake_weight, fake_bias, N=3):
    """dfq.py:143-144: c = clamp(beta - N*gamma, 0)."""
    c = np.asarray(fake_bias, f32) - f32(N) * np.asarray(fake_weight, f32)
    return np.maximum(c, f32(0)).astype(f32)


def bias_absorb_wc(w2: np.ndarray, c: np.ndarray, c_first: int) -> np.ndarray:
    """dfq.py:139-153: wc[g-th rows] = (sum_k W2)[rows] @ c[g-th slice], G = C1 // W2.shape[1]."""
    O, J = w2.shape[0], w2.shape[1]
    G = c_first // J
    so = O // G
    si = c_first // G
    Wk = _view3(w2).sum(axis=-1, dtype=f32)
    out = np.zeros(O, f32)
    for g in range(G):
        out[g * so:(g + 1) * so] = (Wk[g * so:(g + 1) * so].astype(np.float64)
                                    @ c[g * si:(g + 1) * si].astype(np.float64)).astype(f32)
    return out
