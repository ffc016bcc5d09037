"""-m gpu: k_cle_stack and the BN fold deferred into its first sweep, off the two-sweep default problem (tests/stack_cases.py,
whose claims tests/test_stack_cases_host.py checks on the CPU): groups that stop at different sweeps past the third and past
64, the count branch of the exit rule, max_sweeps, signed ranges, both clamps, eps, degenerate rows and columns, subnormals,
negative / zero BN scales and var = 0 - and torchvision ResNet-18 / ResNet-34 with trained-like BN statistics.

Every case runs three times on identical input bits: (a) k_cle_stack with the fold deferred into it, (b) k_cle_stack after the
undeferred fold (with its column scan), (c) k_cle_engine.  All three and the oracle agree bit for bit."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import stack_cases as SC
from oracle import dfq_oracle as O
from test_gpu_engine import _bind_chains, _chains_session, _oracle_chains

pytestmark = pytest.mark.gpu


def _eq(a, b, nan):
    return np.array_equal(a, b, equal_nan=nan)


def _second_col_extrema(w):
    w = w.reshape(w.shape[0], w.shape[1], -1)
    return w.min(axis=(0, 2)), w.max(axis=(0, 2))


@pytest.mark.parametrize("case", SC.CASES, ids=[c["name"] for c in SC.CASES])
def test_stack_kernel_edge_case_equals_engine_and_oracle(case, monkeypatch):
    # equal_nan only where the case produces inf / NaN (case["nonfinite"]: degenerate_weights and zero_gamma_count3, whose
    # s_hi rows overflow their biases and BN vectors; the host test pins which cases those are)
    nan = case["nonfinite"]
    kw = dict(seed=case["seed"], params=case["params"], edit=case["edit"], correct=case["correct"])
    ex_a, ex_b = {}, {}
    runs = dict(a=_chains_session(case["chains"], case["one_group"], "1", "stream", True, monkeypatch, extra=ex_a, **kw),
                b=_chains_session(case["chains"], case["one_group"], "1", "stream", True, monkeypatch, plan_stack="0", extra=ex_b, **kw),
                c=_chains_session(case["chains"], case["one_group"], "0", "stream", False, monkeypatch, **kw))
    assert ex_a["fold"]["deferred"] and not ex_b["fold"]["deferred"]
    before = runs["a"][0]
    for k in ("b", "c"):
        assert np.array_equal(runs[k][0][0][0]["w"], before[0][0]["w"])                      # identical input bits
    # ---- (a) = (b) = (c), bit for bit ----
    _, a_after, a_res, a_d, a_e, a_s = runs["a"]
    for k in ("b", "c"):
        _, after, res, d, e, s = runs[k]
        assert (res.n_sweeps, res.converged) == (a_res.n_sweeps, a_res.converged), (k, res.n_sweeps, a_res.n_sweeps)
        assert np.array_equal(res.group_sweeps, a_res.group_sweeps), (k, res.group_sweeps, a_res.group_sweeps)
        for ci, (x, y) in enumerate(zip(after, a_after)):
            for li, (p, q) in enumerate(zip(x, y)):
                for key in p:
                    assert _eq(p[key], q[key], nan), (k, ci, li, key)
        for i, (x, y) in enumerate(zip(s, a_s)):
            assert _eq(x, y, nan), (k, "S", i)
        for i, (x, y) in enumerate(zip(d + e, a_d + a_e)):        # (a) corrects with the column hints, (c) streams the weights
            assert _eq(x, y, nan), (k, "correction", i)
    # ---- the oracle ----
    layers, bns, sweeps, diffs, S_ref = _oracle_chains(before, case["one_group"], case["params"])
    assert list(a_res.group_sweeps) == sweeps, (list(a_res.group_sweeps), sweeps)
    assert a_res.n_sweeps == max(sweeps)
    assert a_res.converged == all(SC.exit_trace(df, case["params"])[0] for df in diffs)
    n0 = min(sweeps[0], 64)
    np.testing.assert_allclose(a_res.diffs[:n0], diffs[0][:n0], rtol=1e-6, atol=1e-12)
    for i, (x, y) in enumerate(zip(a_s, S_ref)):
        assert _eq(x, y, nan), ("S", i)
    signed = SC.DEFAULT_PARAMS["signed"] if "signed" not in case["params"] else case["params"]["signed"]
    for b, cl in enumerate(a_after):
        l0, l1 = layers[2 * b], layers[2 * b + 1]
        assert _eq(cl[0]["w"], l0.w, nan) and _eq(cl[1]["w"], l1.w.reshape(cl[1]["w"].shape), nan), b
        assert _eq(cl[0]["bias"], l0.b, nan) and _eq(cl[0]["fake_w"], bns[2 * b][0], nan) and _eq(cl[0]["fake_b"], bns[2 * b][1], nan), b
        assert _eq(cl[1]["fake_w"], bns[2 * b + 1][0], nan), b
        if case["correct"]:
            np.testing.assert_array_max_ulp(a_e[b], O.relu_expectation(*bns[2 * b]), maxulp=1)
            exact, bound = O.bias_delta_bound(l1.w, a_e[b], signed=signed)
            assert O.rows_outside_bound(a_d[b], exact, bound).size == 0, b
            assert np.array_equal(cl[1]["bias"], l1.b + (-a_d[b])) and np.array_equal(cl[1]["fake_b"], bns[2 * b + 1][1] + (-a_d[b])), b
        else:
            assert _eq(cl[1]["bias"], l1.b, nan) and _eq(cl[1]["fake_b"], bns[2 * b + 1][1], nan), b
    # ---- (a): the deferred fold's read-only scan left the true column extrema of the folded second layers in buffer 0 ----
    for b, (cl, (cmn, cmx)) in enumerate(zip(before, ex_a["cols0"])):
        d = cl[1]
        w2 = O.bn_fold(d["w"], d["bias"], d["gamma"], d["beta"], d["mean"], d["var"], d["bn_eps"])[0]
        mn, mx = _second_col_extrema(w2)
        assert np.array_equal(cmn, mn) and np.array_equal(cmx, mx), b


def test_negative_zero_does_not_clobber_the_min_max_reductions():
    """Elements of -0.0 around one -1 and one +1 (as a zero BN scale leaves a row): the per-tensor range the fake-quant takes
    is [-1, 1], whichever block's partial extremum (-0.0 for all but two) reaches the atomic min / max first."""
    from dfq_b200.engine import Session
    x = torch.full((1 << 20,), -0.0)
    x[0], x[-1] = -1.0, 1.0
    ref = O.quantize(x.numpy(), 8, -1.0, 1.0)
    sess = Session()
    off = sess.bind(x)
    sess.upload()
    sess.run_quantize([(off, x.numel(), 8, False)])
    sess.download()
    assert np.array_equal(x.numpy(), ref), (float(x[0]), float(x[-1]))


# ---- calls between a deferred fold and its equalization ---------------------------------------------------------------
PENDING_CALLS = ["download", "upload", "quantize", "fold_again", "other_plan", "grow_arena"]


def _pending_session(monkeypatch, defer):
    """STACK_BLOCKS with ~30 % negative gammas (a skipped fold or a wrong sign changes every result), one group per block, the
    fold run and - when `defer` - pending."""
    from dfq_b200.engine import Session
    monkeypatch.setenv("DFQ_CLE_STACK", "1" if defer else "0")
    sess = Session()
    lay = SC.chain_layers(SC.STACK_BLOCKS, 61, SC.edit_negative_gamma)
    rels, groups, folds, _ = _bind_chains(sess, lay, False)
    cle = sess.plan_cle(rels, groups=groups)
    fold = sess.plan_bn_fold(folds, cle_plan=cle)
    assert bool(fold["deferred"]) == defer
    monkeypatch.setenv("DFQ_CLE_STACK", "1")
    sess.upload()
    sess.run_bn_fold(fold)
    assert sess.fold_pending == defer
    return sess, lay, rels, groups, cle, fold


def _session_state(sess, lay, cle):
    v = lambda off, n: sess.view(int(off), int(n)).cpu().numpy().copy()
    out = []
    for cl in lay:
        for d in cl:
            l = sess.layer(d["li"])
            n = d["w"].shape[0]
            out += [v(l["w_off"], d["w"].numel()), v(l["bias_off"], n), v(d["fake_w_off"], n), v(d["fake_b_off"], n)]
        lt = cle["lt"][cl[1]["li"]]
        out += [v(lt["cmin_off"], 2 * cl[0]["w"].shape[0]), v(lt["cmax_off"], 2 * cl[0]["w"].shape[0])]
    return out + [v(o, sess.layer(r[0])["rows"]) for o, r in zip(cle["s_offs"], cle["relations"])]


def _call(call, sess, lay, rels, groups, cle, fold, monkeypatch):
    if call == "download":
        sess.download()
    elif call == "upload":
        sess.upload()
    elif call == "quantize":
        l = sess.layer(lay[0][0]["li"])
        sess.run_quantize([(l["w_off"], lay[0][0]["w"].numel(), 8, False)])
    elif call == "fold_again":
        sess.run_bn_fold(fold)
    elif call == "other_plan":
        monkeypatch.setenv("DFQ_CLE_STACK", "0")
        sess.run_cle_plan(sess.plan_cle(rels, groups=groups), max_sweeps=1)
        monkeypatch.setenv("DFQ_CLE_STACK", "1")
    elif call == "grow_arena":
        n0 = sess.arena.numel()
        sess.plan_cle(rels, groups=groups)            # its scratch does not fit the arena: the next call copies it into a larger one
        assert sess._n > n0


@pytest.mark.parametrize("call", PENDING_CALLS)
def test_calls_between_a_deferred_fold_and_its_equalization(call, monkeypatch):
    """Each call completes the pending fold first (or, for a second deferred fold and an arena that grows, hands it on to the
    equalization intact): the state after the call and after the equalization equals the undeferred fold's, bit for bit."""
    states, host, res = [], [], []
    for defer in (True, False):
        sess, lay, rels, groups, cle, fold = _pending_session(monkeypatch, defer)
        n0 = sess.arena.numel()
        _call(call, sess, lay, rels, groups, cle, fold, monkeypatch)
        pending_after = call in ("fold_again", "grow_arena")
        assert sess.fold_pending == (defer and pending_after), call
        mid = None if pending_after else _session_state(sess, lay, cle)
        host.append([d[k].clone() for cl in lay for d in cl for k in ("w", "bias")])
        # the equalization: on the stack kernel where the fold's column extrema still describe the weights, else on the engine
        ready = call in ("download", "fold_again", "grow_arena")
        monkeypatch.setenv("DFQ_CLE_STACK", "1" if ready else "0")
        r = sess.run_cle_plan(cle, cols_ready=fold["scanned"] if ready else None)
        assert not sess.fold_pending
        if call == "grow_arena":
            assert sess.arena.numel() > n0
        res.append(r)
        states.append((mid, _session_state(sess, lay, cle)))
    (mid_d, end_d), (mid_u, end_u) = states
    if mid_d is not None:
        assert all(np.array_equal(x, y) for x, y in zip(mid_d, mid_u)), "state right after the call"
    assert all(torch.equal(x, y) for x, y in zip(*host)), "host tensors"
    assert np.array_equal(res[0].group_sweeps, res[1].group_sweeps) and res[0].n_sweeps == res[1].n_sweeps
    for i, (x, y) in enumerate(zip(end_d, end_u)):
        assert np.array_equal(x, y), ("state after the equalization", i)


# ---- torchvision ResNets -------------------------------------------------------------------------------------------
TARG = [nn.Conv2d, nn.Linear]


def _resnet(name, zero_init, seed):
    """weights=None, trained-like BN statistics: gamma ~ N(0.8, 0.5) with ~5 % exactly 0, beta ~ N(0, 0.2), mean ~ N(0, 0.1),
    var ~ U(0.2, 2) with ~2 % exactly 0.  zero_init_residual: every block's bn2 keeps gamma = beta = 0."""
    tv = pytest.importorskip("torchvision")
    torch.manual_seed(seed)
    model = getattr(tv.models, name)(weights=None, zero_init_residual=zero_init).eval()
    g = torch.Generator().manual_seed(seed)
    keep = {id(m.bn2) for m in model.modules() if zero_init and hasattr(m, "bn2")}
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                n = m.num_features
                m.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
                var = torch.empty(n).uniform_(0.2, 2.0, generator=g)
                var[torch.rand(n, generator=g) < 0.02] = 0.0
                m.running_var.copy_(var)
                if id(m) in keep:
                    continue
                gamma = torch.randn(n, generator=g) * 0.5 + 0.8
                gamma[torch.rand(n, generator=g) < 0.05] = 0.0
                m.weight.copy_(gamma); m.bias.copy_(torch.randn(n, generator=g) * 0.2)
    return model


def _graph_state(graph, rels):
    """Weights, biases, fake_weight / fake_bias and S, keyed by graph position (the traced keys differ between model copies)."""
    out = {}
    for i, m in enumerate(graph.values()):
        if type(m) in TARG:
            out["w%d" % i] = m.weight.detach().cpu().numpy().copy()
            out["b%d" % i] = m.bias.detach().cpu().numpy().copy()
        elif hasattr(m, "fake_bias") and not isinstance(m, str):
            out["fw%d" % i] = m.fake_weight.cpu().numpy().copy(); out["fb%d" % i] = m.fake_bias.cpu().numpy().copy()
    for i, r in enumerate(rels):
        out["S%d" % i] = r.S.cpu().numpy().copy()
    return out


def _calibrate(model, stack, signed, correction, monkeypatch):
    from dfq_b200.calibrate import GraphCalibration
    from dfq_b200.trace import trace_graph
    monkeypatch.setenv("DFQ_CLE_STACK", stack)
    graph, bottoms = trace_graph(copy.deepcopy(model))
    cal = GraphCalibration(graph, bottoms, TARG)          # the fold plan is made here
    assert bool(cal._fold_plan_scan["deferred"]) == (stack == "1")
    res = cal.run(equalize=True, correction=correction, signed=signed)
    return _graph_state(graph, cal.relations), res


def _assert_states_equal(a, b, what, nan=False):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=nan), (what, k)


@pytest.mark.parametrize("name,zero_init", [("resnet18", False), ("resnet34", False), ("resnet18", True)])
@pytest.mark.parametrize("signed", [False, True])
def test_resnets_on_the_stack_kernel_equal_the_engine_and_the_oracle(name, zero_init, signed, monkeypatch):
    """Every basic block's conv1 -> conv2 is a two-layer chain the stack kernel takes (layer4's conv2: 512 columns = kBcExCols,
    4608-float rows = kStageFloats).  GraphCalibration with the fold deferred into k_cle_stack equals the undeferred fold on
    k_cle_engine (modules, BN vectors, S, sweeps), and both equal the drop-in calls run by the oracle executor."""
    import fakelib
    from dfq_b200 import dfq
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    model = _resnet(name, zero_init, seed=4)
    st, rs = _calibrate(model, "1", signed, False, monkeypatch)
    en, re = _calibrate(model, "0", signed, False, monkeypatch)
    assert rs.n_sweeps == re.n_sweeps and rs.converged and re.converged
    _assert_states_equal(st, en, "stack vs engine")
    # the oracle executor: merge_batchnorm -> create_relation -> cross_layer_equalization on the oracle
    with monkeypatch.context() as mp:
        fakelib.install(mp)
        m = copy.deepcopy(model)
        graph, bottoms = trace_graph(m)
        LT.merge_batchnorm(m, graph, bottoms, TARG)
        rels = create_relation(graph, bottoms, TARG)
        assert sum(1 for _ in rels) == {"resnet18": 8, "resnet34": 16}[name]
        dfq.cross_layer_equalization(graph, rels, TARG, signed=signed)
        n_ref = dfq.cross_layer_equalization.last_result.n_sweeps
        ref = _graph_state(graph, rels)
    assert rs.n_sweeps == n_ref
    _assert_states_equal(st, ref, "stack vs oracle")
    print("%s%s %s: %d sweeps" % (name, " zero_init_residual" if zero_init else "", "signed" if signed else "unsigned", n_ref))
    if zero_init:
        return      # gamma = beta = 0 after every block's bn2: the reference's E[x] is 0/0 there
    # equal_nan: for ResNet-34 unsigned, corrected biases downstream of zero-scale BN channels (whose BN shift is multiplied by
    # s_hi = 1e8 in every sweep) come out NaN - on both kernels alike
    st, _ = _calibrate(model, "1", signed, True, monkeypatch)
    en, _ = _calibrate(model, "0", signed, True, monkeypatch)
    _assert_states_equal(st, en, "corrected: stack (column hints) vs engine", nan=True)
