"""Edge cases of dfq_bias_correct_absorb_clip (bias absorption and weight clipping inside the bias correction), as data: what
tests/test_gpu_absorb_clip_edges.py runs on the GPU against the oracle and tests/test_absorb_clip_edges_host.py checks on the
CPU with the oracle alone (that every case reaches what its claims name).  No GPU code is imported here.

A case is a set of chains drawn as tests/stack_cases.py draws them (chain_layers, the same edits), each layer folded with its
own BN on the host (O.bn_fold).  In a chain, layer k and layer k + 1 form an absorbing relation whose BN vectors are layer
k's fake_weight / fake_bias; every layer but the first has a correction entry whose E[x] is ReLU of that BN.  The first layer
of a chain therefore has no entry: its bias loses c directly (k_absorb_vectors' first_bias) and only k_clip_tensors clips it.
The middle layer of a three-layer chain adds the (sum_k W) . c of its input relation and subtracts the c of its output
relation (AcSlot.sub_c_off)."""
import numpy as np

import stack_cases as SC
from oracle import dfq_oracle as O

f32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)
SUBNORMAL = SC.SUBNORMAL

# (shapes per layer); the comments name the branch of the two correction kernels the chain's corrected layers take
CHAINS = [
    [(48, 16, 3, 3), (40, 48, 3, 3)],                   # 432-float rows: 10 rows per tile (k_bc_engine: a warp per row)
    [(512, 4, 1, 1), (8, 512, 3, 3)],                   # 4608 floats = kStageFloats: one row per tile; 512 columns = kBcExCols
    [(576, 8, 1, 1), (24, 576, 1, 1)],                  # 576 columns > kBcExCols: k_bc_stream reads E[x] from global memory
    [(1200, 4), (6, 1200, 2, 2)],                       # 4800-float rows > kStageFloats: TK_DIRECT, processed in the arena
    [(64, 8, 1, 1), (64, 1, 3, 3)],                     # depthwise second layer: 64 groups, one c per row (wc_so 1)
    [(64, 8, 1, 1), (24, 32, 3, 3)],                    # grouped second layer: 2 groups of 12 rows (wc_so 12)
    [(3, 4, 1, 1), (16, 3, 3, 3)],                      # 27-float rows: tiles the TMA unit cannot move (TK_PLAIN)
    [(32, 8, 3, 3), (48, 32, 1, 1), (20, 48, 3, 3)],    # middle layer: its own entry adds wc and subtracts c (sub_c_off)
]


def _compose(*edits):
    def edit(ci, k, d):
        for e in edits:
            e(ci, k, d)
    return edit


def _where_shape(edit, ok):
    """edit only the layers whose weight shape passes ok(shape) (the others keep their data: chain_layers edits after every
    draw)"""
    def e(ci, k, d):
        if ok(tuple(d["w"].shape)):
            edit(ci, k, d)
    e.__doc__ = edit.__doc__
    return e


# stack_cases' degenerate rows and columns need 8 rows (first layer) and 3 columns (second layer)
edit_degenerate = _where_shape(SC.edit_degenerate, lambda s: s[0] >= 8 and s[1] >= 3)


def edit_signed_zeros(ci, k, d):
    """every 53rd tap -0.0 (after the fold: -0.0 or +0.0 by the sign of the factor)"""
    d["w"].view(-1)[1::53] = -0.0


def edit_nonfinite(ci, k, d):
    """every corrected layer: a NaN, a +inf and a -inf tap; chain 0's first BN: a NaN beta (fake_bias NaN -> c NaN)"""
    if k >= 1:
        w = d["w"].view(-1)
        n = w.numel()
        w[n // 3] = float("nan")
        w[n // 2] = float("inf")
        w[(2 * n) // 3] = float("-inf")
    if ci == 0 and k == 0:
        d["beta"][1] = float("nan")


def edit_inf_taps(ci, k, d):
    """every corrected layer: one +inf and one -inf tap (clamped to the bounds of a wide range)"""
    if k >= 1:
        w = d["w"].view(-1)
        w[w.numel() // 2] = float("inf")
        w[w.numel() // 5] = float("-inf")


def edit_c_boundary(N):
    def edit(ci, k, d):
        """per BN, channels with beta == fl(N * |gamma|) (c = +0.0 exactly), one ulp above (c > 0, tiny) and one ulp below
        (c < 0 before the clamp)"""
        n = d["gamma"].numel()
        t = max(1, n // 8)
        idx = np.random.default_rng(1000 + 10 * ci + k).permutation(n)[:3 * t]
        nfw = (f32(N) * np.abs(d["gamma"].numpy())).astype(f32)
        beta = d["beta"].numpy()          # shares the tensor's memory
        beta[idx[:t]] = nfw[idx[:t]]
        beta[idx[t:2 * t]] = np.nextafter(nfw[idx[t:2 * t]], f32(np.inf))
        beta[idx[2 * t:]] = np.nextafter(nfw[idx[2 * t:]], f32(-np.inf))
    return edit


def clip_at_weights(folded):
    """bounds equal to weight values of chain 0's second layer (its 20th and 80th percentile taps)"""
    w = np.sort(folded[0][1][0].ravel())
    return float(w[len(w) // 5]), float(w[4 * len(w) // 5])


def all_ones_scale():
    """(0, hi) with fl((hi - 0) / 255) = a scale whose mantissa is all ones: the one divisor bc_fast_quant refuses inside
    its exponent window (test_gpu_engine.py's w_ones)"""
    s = np.uint32((f32(1e-3).view(np.uint32) & np.uint32(0xff800000)) | np.uint32(0x7fffff)).view(np.float32)
    return 0.0, float(f32(float(s) * 255.0))


def _case(name, N, clip, edits=(), chains=None, seed=71, **claims):
    return dict(name=name, N=N, clip=clip, edit=_compose(*edits) if edits else None, chains=chains or CHAINS, seed=seed,
                claims=claims)


CASES = [
    # stack_cases' degenerate rows and columns; bounds that are weight values and bite on both sides; N = -0.25
    _case("degenerate_bounds_at_weights", -0.25, clip_at_weights, [edit_degenerate], zero_rows=True, subnormal_taps=True,
          bound_is_weight=True, bites_lo=True, bites_hi=True, c_positive=True),
    # negative gammas (negative fold factors); a range only the upper bound bites; N = 0
    _case("negative_gamma_one_side", 0.0, (-1e30, 0.02), [SC.edit_negative_gamma], negative_factors=True, bites_hi=True,
          bites_lo=False, c_positive=True),
    # zero gammas (zero rows, fake_weight 0, E[x] of 0 / 0 is NaN where beta - c is 0) and signed zeros; lo = hi = 0: range 0
    _case("zero_gamma_range_zero", 0.0, (0.0, 0.0), [SC.edit_zero_gamma(26), edit_signed_zeros], zero_fake_weight=True,
          range_zero=True, negative_zero_taps=True, c_positive=True),
    # zero variances with bn_eps 1e-3; lo = hi != 0: every weight becomes 0.01
    _case("zero_var_range_constant", -0.25, (0.01, 0.01), [SC.edit_zero_var], zero_var=True, range_constant=True,
          c_positive=True),
    # a range no weight lies in: every tap clamps to lo
    _case("no_weight_in_range", 0.0, (1e3, 2e3), no_weight_inside=True, c_positive=True),
    # +-FLT_MAX: accepted, clips nothing; N = 3 with fake_bias == 3 * fake_weight exactly (c = +0.0) and one ulp either side
    _case("flt_max_c_boundary", 3.0, (-FLT_MAX, FLT_MAX), [edit_c_boundary(3.0)], clip_noop=True, c_exact_zero=True,
          c_positive=True),
    # subnormal bounds (a flush-to-zero build would clamp to 0) and subnormal taps
    _case("subnormal_bounds", 0.0, (-SUBNORMAL, SUBNORMAL), [edit_degenerate], subnormal_bounds=True, bites_lo=True,
          bites_hi=True, c_positive=True),
    # NaN / +inf / -inf taps and a NaN fake_bias (c NaN: k_absorb_vectors' clamp keeps it)
    _case("nonfinite", -0.25, (-0.05, 0.05), [edit_nonfinite], nan_taps=True, inf_taps=True, c_nan=True, bites_lo=True,
          bites_hi=True),
    # N so large that N * fake_weight overflows: c = inf on some channels
    _case("c_overflow", -3e38, (-0.05, 0.05), c_inf=True, bites_lo=True, bites_hi=True),
    # the clamped range gives a scale with an all-ones mantissa: bc_fast_quant refuses it, k_bc_stream takes the IEEE chain
    _case("ieee_chain_all_ones_scale", 0.0, all_ones_scale(), ieee_chain=True, c_positive=True),
    # +-inf taps clamped to +-1e25: a quantization step above bc_fast_quant's exponent window, the IEEE chain again
    _case("ieee_chain_wide_range", 0.0, (-1e25, 1e25), [edit_inf_taps], inf_taps=True, ieee_chain=True, c_positive=True),
    # absorption without a clip
    _case("no_clip", -0.25, None, c_positive=True),
]


def clip_of(case, folded):
    c = case["clip"]
    return c(folded) if callable(c) else c


def folded_chains(case):
    """Per chain, per layer (w, bias, fake_weight, fake_bias) as numpy fp32 arrays: the drawn layers folded with their BN."""
    lay = SC.chain_layers(case["chains"], case["seed"], case["edit"])
    out = []
    with np.errstate(all="ignore"):
        for cl in lay:
            out.append([O.bn_fold(d["w"].numpy(), d["bias"].numpy(), d["gamma"].numpy(), d["beta"].numpy(), d["mean"].numpy(),
                                  d["var"].numpy(), d["bn_eps"]) for d in cl])
    return out


def absorb_vectors(folded, N):
    """Per chain, per relation k (layers k, k + 1): c = clamp(fake_bias - N * fake_weight, 0) and fake_bias - c
    (dfq.py:143-144,163)."""
    out = []
    with np.errstate(all="ignore"):
        for cl in folded:
            rel = []
            for k in range(len(cl) - 1):
                fw, fb = cl[k][2], cl[k][3]
                c = O.bias_absorb_c(fw, fb, N)
                rel.append((c, (fb - c).astype(f32)))
            out.append(rel)
    return out


def clipped(w, clip):
    return w.copy() if clip is None else O.clip_weight(w, clip[0], clip[1])


def fast_quant_refuses(mn, mx, num_bits=8):
    """bc_fast_quant's guard (bc_stream.cuh) on an unsigned per-tensor range: True where k_bc_stream takes the IEEE chain."""
    scale = (float(mx) - float(mn)) / (2.0 ** num_bits - 1.0)
    if 1e-8 > scale:
        scale = 1e-8
    with np.errstate(over="ignore"):
        s = f32(scale)
    bits = int(s.view(np.uint32))
    e = (bits >> 23) & 0xff
    return not (40 <= e <= 200 and (bits & 0x7fffff) != 0x7fffff and s == s)
