"""-m gpu: dfq_bias_correct_absorb_clip against the oracle, row by row, on the edge data of tests/absorb_clip_edges.py and on
both correction kernels (DFQ_BC_STREAM=0 / 1, and the size rule's own choice).  The session holds exactly the case's folded
layers and BN vectors, so every input is known:
  * c, fake_bias - c and the bias of each chain's first layer: bit for bit (O.bias_absorb_c);
  * every weight: O.clip_weight bit for bit - taps the clip leaves alone keep their bits, NaN and -0.0 included;
  * the kernel's E[x] scratch: within 1 ulp of O.relu_expectation on the absorbed fake vectors;
  * delta: within O.bias_delta_bound on the CLIPPED weights; wc (the raw-sum runs, where it is the delta scratch): within the
    raw bound on the UNCLIPPED weights with c as the expectation; the final bias fl(fl(fl(b + wc) - c) - delta) within the
    sum of both bounds and its three fp32 roundings;
  * the per-tensor range: the unclipped min / max, whose clamp is the clipped tensor's range.
Where the oracle's value is NaN or inf, the kernel's must be the same.  Also: host-side refusals of the C entry leave the arena
bit-identical, a 512-channel GraphCalibration takes k_bc_stream<true> by size, and re-running one GraphCalibration with other
flags equals a fresh one."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import absorb_clip_edges as AE
from oracle import dfq_oracle as O

pytestmark = pytest.mark.gpu
f32 = np.float32
U24 = 2.0 ** -24
TARG = [nn.Conv2d, nn.Linear]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _force(monkeypatch, variant):
    if variant == "default":
        monkeypatch.delenv("DFQ_BC_STREAM", raising=False)
    else:
        monkeypatch.setenv("DFQ_BC_STREAM", "1" if variant == "stream" else "0")


def _build(case, raw):
    """One session with the case's folded chains: per chain, layer ids, BN offsets; the DfqAbsorb table; the plan."""
    from dfq_b200.engine import Session
    folded = AE.folded_chains(case)
    sess = Session()
    chains = []
    for cl in folded:
        ids = [sess.add_layer(torch.from_numpy(w.copy()), torch.from_numpy(b.copy())) for w, b, _, _ in cl]
        bns = [(sess.bind(torch.from_numpy(fw.copy())), sess.bind(torch.from_numpy(fb.copy()))) for _, _, fw, fb in cl[:-1]]
        chains.append((ids, bns))
    at = sess.plan_absorb([(ids[k], ids[k + 1], bw, bb) for ids, bns in chains for k, (bw, bb) in enumerate(bns)])
    c_off = {(int(a["first"]), int(a["second"])): int(a["c_off"]) for a in at}
    items = []
    for ids, bns in chains:
        for k in range(1, len(ids)):
            n = sess.layer(ids[k - 1])["rows"]
            if raw:            # the absorption alone, as GraphCalibration.plan_absorption plans it
                co = c_off[(ids[k - 1], ids[k])]
                items.append(dict(layer=ids[k], signed=False, level=0, next_bn_b_off=-1, raw_sum=True, add=True,
                                  terms=[dict(bn_w_off=co, bn_b_off=co, n=n, relu=False, op="set")]))
            else:
                items.append(dict(layer=ids[k], signed=False, level=0, next_bn_b_off=-1,
                                  terms=[dict(bn_w_off=bns[k - 1][0], bn_b_off=bns[k - 1][1], n=n, relu=True, op="set")]))
    plan = sess.plan_bias_correct(items)
    sess.upload()
    return sess, folded, chains, at, c_off, plan


def _bits_equal(a, b):
    """bit for bit, except that any NaN equals any NaN"""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def _within_ulp(got, want, ulps=1):
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    gi, wi = got.view(np.int32).astype(np.int64), want.view(np.int32).astype(np.int64)
    close = np.isfinite(got) & np.isfinite(want) & (np.sign(got) == np.sign(want)) & (np.abs(gi - wi) <= ulps)
    return np.nonzero(~(same | close))[0]


def _rows_outside(got, exact, bound):
    """Rows where the kernel's fp32 result leaves [exact - bound, exact + bound]; where fl(exact) is inf or NaN the kernel's
    must be the same."""
    with np.errstate(all="ignore"):
        ex32 = exact.astype(f32)
        fin = np.isfinite(ex32)
        bad = fin & ~(np.abs(np.asarray(got, np.float64) - exact) <= bound)
    bad |= ~fin & ~((got == ex32) | (np.isnan(got) & np.isnan(ex32)))
    return np.nonzero(bad)[0]


def _check(sess, folded, chains, at, c_off, plan, N, clip, raw):
    view = lambda off, n: sess.view(int(off), int(n)).cpu().numpy().copy()
    vec = AE.absorb_vectors(folded, N)
    slot = {int(b["layer"]): b for b in plan["bt"]}
    for ci, ((ids, bns), cl, rel) in enumerate(zip(chains, folded, vec)):
        where = lambda k, what: (ci, k, what)
        # ---- c, fake_bias - c ----
        for k, (c, fb_after) in enumerate(rel):
            n = c.size
            assert _bits_equal(view(c_off[(ids[k], ids[k + 1])], n), c), where(k, "c")
            assert _bits_equal(view(bns[k][1], n), fb_after), where(k, "fake_bias")
            assert _bits_equal(view(bns[k][0], n), cl[k][2]), where(k, "fake_weight")
        for k, li in enumerate(ids):
            w0, b0 = cl[k][0], cl[k][1]
            L = sess.layer(li)
            rows = L["rows"]
            # ---- the weights: clipped bit for bit, untouched taps keep their bits ----
            got_w = view(L["w_off"], w0.size).reshape(w0.shape)
            want_w = AE.clipped(w0, clip)
            bad = np.nonzero(got_w.view(np.uint32).ravel() != want_w.view(np.uint32).ravel())[0]
            assert bad.size == 0, (where(k, "weights"), bad[:6], got_w.ravel()[bad[:6]], w0.ravel()[bad[:6]])
            got_b = view(L["bias_off"], rows)
            csub = rel[k][0] if k < len(rel) else None
            if k == 0:          # no correction entry: k_absorb_vectors' first.bias -= c
                with np.errstate(all="ignore"):
                    assert _bits_equal(got_b, (b0 - csub).astype(f32)), where(k, "first bias")
                continue
            b = slot[li]
            c_in = rel[k - 1][0]
            # ---- the per-tensor range: the unclipped min / max (NaN skipped); its clamp is the clipped tensor's ----
            mm = view(b["minmax_off"], 2)
            if not raw:
                assert _bits_equal(mm, np.array(O.flat_minmax(w0), f32)), (where(k, "range"), mm, O.flat_minmax(w0))
            rng = O.flat_minmax(want_w)
            if clip is not None and not raw:
                assert _bits_equal(np.clip(mm, f32(clip[0]), f32(clip[1])), np.array(rng, f32)), where(k, "clamped range")
            # ---- E[x] scratch ----
            got_ex = view(b["expect_off"], b["expect_len"])
            with np.errstate(all="ignore"):
                want_ex = c_in if raw else O.relu_expectation(cl[k - 1][2], rel[k - 1][1])
            bad = _within_ulp(got_ex, want_ex, 0 if raw else 1)
            assert bad.size == 0, (where(k, "E[x]"), bad[:6], got_ex[bad[:6]], want_ex[bad[:6]])
            got_d = view(b["delta_off"], rows)
            with np.errstate(all="ignore"):
                wc_ex, wc_bd = O.bias_delta_bound(w0, c_in, raw=True)                 # on the unclipped weights
                if raw:
                    bad = _rows_outside(got_d, wc_ex, wc_bd)
                    assert bad.size == 0, (where(k, "wc"), bad[:6], got_d[bad[:6]], wc_ex[bad[:6]], wc_bd[bad[:6]])
                    want_b = (b0 + got_d).astype(f32)
                    if csub is not None:
                        want_b = (want_b - csub).astype(f32)
                    assert _bits_equal(got_b, want_b), where(k, "raw bias")
                    continue
                d_ex, d_bd = O.bias_delta_bound(want_w, got_ex, value_range=rng)       # on the clipped weights
            bad = _rows_outside(got_d, d_ex, d_bd)
            assert bad.size == 0, (where(k, "delta"), bad[:6], got_d[bad[:6]], d_ex[bad[:6]], d_bd[bad[:6]])
            # ---- the final bias: fl(fl(fl(b + wc) - c) - delta) ----
            cs = np.zeros(rows) if csub is None else csub.astype(np.float64)
            with np.errstate(all="ignore"):
                ideal = b0.astype(np.float64) + wc_ex - cs - d_ex
                m1 = np.abs(b0) + np.abs(wc_ex) + wc_bd
                m2 = m1 + np.abs(cs)
                m3 = m2 + np.abs(d_ex) + d_bd
                tol = wc_bd + d_bd + U24 * (m1 + m2 + m3) * (1 + 2.0 ** -20)
                ideal32 = (b0 + wc_ex.astype(f32)).astype(f32)
                if csub is not None:
                    ideal32 = (ideal32 - csub).astype(f32)
                ideal32 = (ideal32 - d_ex.astype(f32)).astype(f32)
                fin = np.isfinite(ideal32) & np.isfinite(ideal)
                bad = fin & ~(np.abs(got_b.astype(np.float64) - ideal) <= tol)
                bad |= ~fin & ~((got_b == ideal32) | (np.isnan(got_b) & np.isnan(ideal32)))
            bad = np.nonzero(bad)[0]
            assert bad.size == 0, (where(k, "bias"), bad[:6], got_b[bad[:6]], ideal[bad[:6]], tol[bad[:6]])


@pytest.mark.parametrize("variant", ["engine", "stream", "default"])
@pytest.mark.parametrize("case", AE.CASES, ids=[c["name"] for c in AE.CASES])
def test_fused_correction_row_by_row(case, variant, monkeypatch):
    _force(monkeypatch, variant)
    sess, folded, chains, at, c_off, plan = _build(case, raw=False)
    clip = AE.clip_of(case, folded)
    sess.run_bias_correct_absorb_clip(plan, 8, absorb=at, absorb_n=case["N"], clip=clip)
    _check(sess, folded, chains, at, c_off, plan, case["N"], clip, raw=False)


@pytest.mark.parametrize("variant", ["engine", "stream"])
@pytest.mark.parametrize("case", AE.CASES, ids=[c["name"] for c in AE.CASES])
def test_absorb_only_raw_sums_row_by_row(case, variant, monkeypatch):
    """correction=False, absorption=True: raw-sum entries whose delta is wc itself, clamping as they go."""
    _force(monkeypatch, variant)
    sess, folded, chains, at, c_off, plan = _build(case, raw=True)
    clip = AE.clip_of(case, folded)
    sess.run_bias_correct_absorb_clip(plan, 8, absorb=at, absorb_n=case["N"], clip=clip)
    _check(sess, folded, chains, at, c_off, plan, case["N"], clip, raw=True)


def test_refusals_leave_the_arena_untouched():
    """Argument refusals on the host return nonzero before anything is enqueued: the arena stays bit-identical.  The same
    call without the violation then succeeds."""
    from dfq_b200 import _lib
    case = AE.CASES[0]
    sess, folded, chains, at, c_off, plan = _build(case, raw=False)
    lib = sess.lib
    lt, bt, tt, lp = plan["lt"], plan["bt"], plan["tt"], plan["level_ptr"]

    def call(bt=bt, lp=lp, at=at, lo=-0.05, hi=0.05):
        return lib.dfq_bias_correct_absorb_clip(sess._ptr(), sess.arena.numel(), _lib.table_ptr(lt), len(lt), _lib.table_ptr(bt),
                                                len(bt), _lib.table_ptr(tt), plan["n_terms"], _lib.table_ptr(lp), len(lp) - 1, 8,
                                                _lib.table_ptr(at), len(at), C.c_float(0.0), 1, C.c_float(lo), C.c_float(hi),
                                                _lib.stream_ptr())
    prepared = bt.copy()
    prepared["flags"][1] |= _lib.BC_PREPARED
    twice = np.ascontiguousarray(np.concatenate([bt, bt[:1]]))
    lp_twice = lp.copy()
    lp_twice[-1] += 1
    out_of_range = at.copy()
    out_of_range["first"][2] = len(lt)
    torch.cuda.synchronize()
    before = sess.arena.clone()
    for what, kw in [("prepared", dict(bt=prepared)), ("two entries", dict(bt=twice, lp=lp_twice)),
                     ("absorption index", dict(at=out_of_range)), ("lo > hi", dict(lo=0.05, hi=-0.05))]:
        rc = call(**kw)
        torch.cuda.synchronize()
        assert rc != 0, what
        assert torch.equal(sess.arena.view(torch.int32), before.view(torch.int32)), what
    assert call() == 0
    torch.cuda.synchronize()
    assert not torch.equal(sess.arena.view(torch.int32), before.view(torch.int32))


def test_stack_of_512_channels_takes_the_stream_kernel_by_size(monkeypatch):
    """GraphCalibration on independent 512-channel 3x3 blocks: enough one-row tiles in the correction's one level that the
    size rule of bc_launch picks k_bc_stream<true>; the result equals the separate calls bit for bit."""
    from dfq_b200 import workload
    from test_gpu_calibrate_absorb_clip import _compare
    monkeypatch.delenv("DFQ_BC_STREAM", raising=False)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_blocks = -(-16 * sms // 512)                   # tiles of the one level: 512 per block (4608-float rows)
    assert n_blocks * 512 >= 16 * sms and n_blocks <= 6      # at most ~130 MB of weights per graph
    cal = _compare(workload.stack_topology(n_blocks, channels=512), 12, absorption=True, absorption_n=0.0,
                   clip_weight=(-0.02, 0.02))
    assert cal._bc_plan["n_levels"] == 1


def _fresh(topo, seed, **kw):
    from dfq_b200 import workload
    from dfq_b200.calibrate import GraphCalibration
    g, b, _ = workload.build_graph(topo, seed=seed)
    GraphCalibration(g, b, TARG).run(**kw)
    return g


@pytest.mark.parametrize("first,second", [
    (dict(signed=True), dict(signed=False)),
    (dict(signed=False), dict(signed=True)),
    (dict(absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05)), dict()),
    (dict(), dict(absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05))),
    (dict(signed=True, absorption=True, absorption_n=0.0, clip_weight=(-0.05, 0.05)), dict(quantize_bits=(8, 16))),
], ids=["signed_then_unsigned", "unsigned_then_signed", "flags_then_none", "none_then_flags", "all_then_plain"])
def test_rerunning_one_calibration_equals_a_fresh_one(first, second):
    """upload(); run_device(**first); upload(); run_device(**second); download() equals a fresh run(**second)."""
    from dfq_b200 import workload
    from dfq_b200.calibrate import GraphCalibration
    topo = workload.load_topology(os.path.join(GOLD, "topology_resnet18.json"))
    g, b, _ = workload.build_graph(topo, seed=21)
    cal = GraphCalibration(g, b, TARG)
    cal.plan_absorption()
    cal.upload()
    cal.run_device(**first)
    cal.upload()
    cal.run_device(**second)
    cal.download()
    want = _fresh(topo, 21, **second)
    for (k, m), mw in zip(g.items(), want.values()):
        if type(m) in TARG:
            assert torch.equal(m.weight, mw.weight), ("weight", k)
            assert torch.equal(m.bias, mw.bias), ("bias", k)
        if isinstance(m, nn.BatchNorm2d) and hasattr(m, "fake_bias"):
            assert torch.equal(m.fake_weight, mw.fake_weight) and torch.equal(m.fake_bias, mw.fake_bias), ("bn", k)
