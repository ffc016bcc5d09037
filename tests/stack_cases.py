"""Edge cases of k_cle_stack (the streaming equalization of stacks of two-layer chains) and of the BN fold deferred into its
first sweep, as data: what tests/test_gpu_stack_edges.py runs on the GPU and tests/test_stack_cases_host.py checks on the CPU
with the oracle alone (that every case still reaches the branch its comment names).  No GPU code is imported here.

The layers of a case are drawn exactly as tests/test_gpu_engine.py::_chains_session always drew them; a case may then edit
each layer dict (w, bias, gamma, beta, mean, var, bn_eps) before it is bound, and may pass equalization parameters other than
the defaults."""
import numpy as np
import torch

from oracle import dfq_oracle as O

STACK_BLOCKS = [
    ((128, 64, 3, 3), (256, 128, 3, 3)),   # non-square 3x3 block
    ((96, 64, 3, 3), (200, 96, 1, 1)),     # 3x3 next to 1x1
    ((512, 256, 1, 1), (64, 512, 3, 3)),   # second layer at kBcExCols 512 columns and kStageFloats 4608 floats
    ((44, 16, 3, 3), (37, 44, 3, 3)),      # 396-float rows: 11 per tile, 37 rows = partial tiles, not a multiple of 32
    ((100, 4, 3, 3), (24, 100, 1, 1)),     # 36-float rows: 4608 / 36 = 128, capped at 32 rows per tile
]

# the equalization parameters of dfq.py (run_cle_plan / O.cross_layer_equalization keyword names)
DEFAULT_PARAMS = dict(signed=False, s_range=(1e-8, 1e8), eps=0, converge_thres=2e-7, converge_count=20, max_sweeps=0)
VECTORS = ("w", "bias", "gamma", "beta", "mean", "var")


def mk(shape, seed, gain=True):
    """randn weights; gain: rows scaled by 10^U(-1, 1)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(*shape, generator=g)
    if gain:
        w = w * (10 ** torch.empty(shape[0]).uniform_(-1, 1, generator=g)).view(-1, *([1] * (len(shape) - 1)))
    return w.contiguous()


def chain_layers(chains, seed=61, edit=None):
    """The layer dicts of _chains_session: per chain, per layer dict(w, bias, gamma, beta, mean, var, bn_eps) of CPU tensors.
    edit(ci, k, d): changes layer k of chain ci in place (after every draw, so that the other layers keep their data)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for ci, shapes in enumerate(chains):
        cl = []
        for k, s in enumerate(shapes):
            d = dict(w=mk(s, seed + 7 * ci + k, gain=(k % 2 == 0)) * 0.1, bias=torch.randn(s[0], generator=g) * 0.1,
                     gamma=torch.rand(s[0], generator=g) + 0.5, beta=torch.randn(s[0], generator=g) * 0.2,
                     mean=torch.randn(s[0], generator=g) * 0.1, var=torch.rand(s[0], generator=g) + 0.5, bn_eps=1e-5)
            if edit is not None:
                edit(ci, k, d)
                for n in VECTORS:
                    d[n] = d[n].contiguous()
            cl.append(d)
        out.append(cl)
    return out


def oracle_params(params):
    """run_cle_plan keywords -> O.cross_layer_equalization keywords (max_sweeps 0 = no limit)."""
    p = dict(DEFAULT_PARAMS, **(params or {}))
    return dict(signed=p["signed"], s_range=p["s_range"], eps=p["eps"], converge_thres=p["converge_thres"],
                converge_count=p["converge_count"], max_sweeps=p["max_sweeps"] or None)


def oracle_chains(before, one_group, params=None):
    """The oracle of _chains_session: BN fold, equalization (per chain, or one call over all chains).  `before`: per chain
    lists of layer dicts of numpy arrays (w, bias, gamma, beta, mean, var, bn_eps).  Returns (layers, bns, sweeps per group,
    diffs per group, S per relation)."""
    kw = oracle_params(params)
    out, diffs, done = [], [], []
    layers, bns, rels = [], [], []
    for cl in before:
        base = len(layers)
        for d in cl:
            with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
                w2, b2, fw, fb = O.bn_fold(d["w"], d["bias"], d["gamma"], d["beta"], d["mean"], d["var"], d.get("bn_eps", 1e-5))
            layers.append(O.OLayer(w2, b2)); bns.append([fw, fb])
        crel = [O.ORelation(base + k, base + k + 1, base + k) for k in range(len(cl) - 1)]
        if not one_group:
            crel_local = [O.ORelation(k, k + 1, k) for k in range(len(cl) - 1)]
            with np.errstate(over="ignore", invalid="ignore"):
                n, df = O.cross_layer_equalization(layers[base:], [tuple(x) for x in bns[base:]], crel_local, **kw)
            out.append(n); diffs.append(df); done += crel_local
        rels += crel
    if one_group:
        with np.errstate(over="ignore", invalid="ignore"):
            n, df = O.cross_layer_equalization(layers, [tuple(x) for x in bns], rels, **kw)
        out, diffs, done = [n], [df], rels
    return layers, bns, out, diffs, [r.S for r in done]


def exit_trace(diffs, params=None):
    """Replays the exit rule of dfq.py:105-115 on one group's diffs.  Returns (converged, [(d_move, d_thres)] per sweep):
    converged - the rule, not max_sweeps, ended the run; d_move = | |diff - diff_tmp| - 1e-9 | / 1e-9 and
    d_thres = |diff_tmp - converge_thres| / converge_thres (inf when the threshold is 0) - how far each comparison was from
    going the other way, relative to the constant it compares with."""
    p = dict(DEFAULT_PARAMS, **(params or {}))
    thres, cc = p["converge_thres"], p["converge_count"]
    diff, count, margins = 10.0, 0, []
    for t in diffs:
        margins.append((abs(abs(diff - t) - 1e-9) / 1e-9, abs(t - thres) / thres if thres > 0 else np.inf))
        if abs(diff - t) > 1e-9:
            count, diff = 0, t
        else:
            count += 1
    return not (diff > thres and count < cc), margins


def _gen(case_seed, ci, k):
    return torch.Generator().manual_seed(1000 * case_seed + 10 * ci + k)


# ---- edits ---------------------------------------------------------------------------------------------------------
def edit_wide_gains(ci, k, d):
    """first layer: rows over six decades (10^U(-3, 3))"""
    if k == 0:
        g = _gen(2, ci, k)
        d["w"] = d["w"] * (10 ** torch.empty(d["w"].shape[0]).uniform_(-3, 3, generator=g)).view(-1, *([1] * (d["w"].dim() - 1)))


SUBNORMAL = 1e-40          # below FLT_MIN 1.18e-38: a flush-to-zero build would turn it into 0


def edit_degenerate(ci, k, d):
    """first layer: a zero row (range 0 -> s NaN -> s_hi), a constant row (range 0 -> s_hi), a row of -0.0 and a row of
    subnormals; second layer: a zero input column (r2 = 0 -> s = 0 -> s_lo) and scattered subnormal entries"""
    w = d["w"]
    if k == 0:
        w[1] = 0.0
        w[3] = 0.5
        w[5] = -0.0
        g = _gen(5, ci, k)
        w[7] = torch.randn(w[7].shape, generator=g) * SUBNORMAL
    else:
        w.view(w.shape[0], w.shape[1], -1)[:, 2] = 0.0
        w.view(-1)[::97] = SUBNORMAL


def edit_negative_gamma(ci, k, d):
    """about 30 % negative gammas in both BNs: the fold factor flips the sign of a row and swaps its extrema"""
    g = _gen(6, ci, k)
    flip = torch.rand(d["gamma"].shape, generator=g) < 0.3
    d["gamma"] = torch.where(flip, -d["gamma"], d["gamma"])


def edit_zero_gamma(seed):
    def edit(ci, k, d):
        """a few zero gammas in each BN: folded rows of +-0.0 (range 0 -> s_hi every sweep); fake weight 0"""
        g = _gen(seed, ci, k)
        idx = torch.randperm(d["gamma"].numel(), generator=g)[:max(2, d["gamma"].numel() // 16)]
        d["gamma"][idx] = 0.0
    return edit


def edit_zero_var(ci, k, d):
    """some channels with var = 0 (factor gamma / sqrt(bn_eps)) and bn_eps = 1e-3; a few negative gammas"""
    g = _gen(8, ci, k)
    idx = torch.randperm(d["var"].numel(), generator=g)[:max(2, d["var"].numel() // 8)]
    d["var"][idx] = 0.0
    d["gamma"][idx[:1]] = -d["gamma"][idx[:1]]
    d["bn_eps"] = 1e-3


def _case(name, chains, one_group=False, params=None, edit=None, seed=61, correct=True, nonfinite=False, **claims):
    return dict(name=name, chains=chains, one_group=one_group, params=dict(params or {}), edit=edit, seed=seed, correct=correct,
                nonfinite=nonfinite, claims=claims)


COUNT3 = dict(converge_thres=0.0, converge_count=3)
COUNT6 = dict(converge_thres=0.0, converge_count=6)
PAST64 = [[(64, 16, 3, 3), (48, 64, 3, 3)], [(64, 16, 1, 1), (48, 64, 1, 1)]]

CASES = [
    # 1. count branch of the exit rule (converge_thres 0: diff never reaches it), one group per block: the groups stop at
    #    different sweeps past the third (GroupState.acc[2], slot recycling); converge_count 3 ends every block after an odd
    #    number of sweeps (the correction's hints come from column-extrema buffer 1), 6 after an even number (buffer 0)
    _case("count3_groups", STACK_BLOCKS, params=COUNT3, distinct_stops=3, parities={1}),
    _case("count6_groups", STACK_BLOCKS, params=COUNT6, distinct_stops=3, parities={0}),
    # ... and the same data as one group
    _case("count3_one_group", STACK_BLOCKS, one_group=True, params=COUNT3, min_sweeps=3),
    # 2. past the 64 sweeps CleResult.diffs records, through the threshold branch: rows over six decades and s_range
    #    (0.95, 1.05) - most channels sit at a clamp in every sweep; 3x3 and 1x1 as two groups
    _case("past64_clamped", PAST64, params=dict(s_range=(0.95, 1.05)), edit=edit_wide_gains, min_sweeps=65,
          distinct_stops=2, clamp_hi=True, clamp_lo=True),
    # 3. max_sweeps: the run ends on the cap, not on the rule (converged False); after 1 sweep the hints are buffer 1
    _case("max_sweeps_1", STACK_BLOCKS, params=dict(max_sweeps=1), capped=True),
    _case("max_sweeps_3", STACK_BLOCKS, params=dict(COUNT3, max_sweeps=3), capped=True),
    # 4. other parameters: signed ranges (range_of), both clamps of solve_scale (inv_lo / inv_hi formed in double), eps
    _case("signed", STACK_BLOCKS, params=dict(signed=True), signed_ranges=True),
    _case("s_range_half_double", STACK_BLOCKS, params=dict(s_range=(0.5, 2.0)), min_sweeps=3, clamp_hi=True, clamp_lo=True),
    _case("s_range_third_triple", STACK_BLOCKS, params=dict(s_range=(1 / 3.0, 3.0)), clamp_hi=True, clamp_lo=True),
    _case("eps", STACK_BLOCKS, params=dict(eps=1e-3), min_sweeps=3),
    # 5. degenerate weights: zero / constant / -0.0 / subnormal rows and a zero column
    #    - the zero rows take s_hi = 1e8 in all 25 sweeps: their biases and BN vectors overflow to inf (no correction)
    _case("degenerate_weights", STACK_BLOCKS, edit=edit_degenerate, correct=False, nonfinite=True, clamp_hi=True, clamp_lo=True,
          zero_rows=True, subnormal=True, inf_bias=True, min_sweeps=3),
    # 6. BN statistics through the deferred fold
    _case("negative_gamma", STACK_BLOCKS, edit=edit_negative_gamma, negative_factors=True),
    _case("zero_gamma", STACK_BLOCKS, edit=edit_zero_gamma(26), zero_rows=True, clamp_hi=True),
    _case("zero_var_bn_eps", STACK_BLOCKS, edit=edit_zero_var, negative_factors=True),
    # ... zero gammas over many sweeps: s_hi every sweep overflows the first-layer biases and BN vectors to inf while the
    #     second layer's columns shrink through the subnormals (inf / NaN in the results: compared with equal_nan)
    #     (edit seed 26: every exit comparison at least 10 % away from its constant; seed 7 came within 1.2e-4)
    _case("zero_gamma_count3", STACK_BLOCKS, params=COUNT3, edit=edit_zero_gamma(26), correct=False, nonfinite=True,
          zero_rows=True, clamp_hi=True, inf_bias=True, subnormal=True, min_sweeps=4),
]


def case_data(case):
    """(chain layer dicts of CPU tensors, numpy copy of them) of a case."""
    lay = chain_layers(case["chains"], case["seed"], case["edit"])
    before = [[dict((n, d[n].numpy().copy()) for n in VECTORS) for d in cl] for cl in lay]
    for cl, bl in zip(lay, before):
        for d, b in zip(cl, bl):
            b["bn_eps"] = d["bn_eps"]
    return lay, before
