"""A stand-in for libdfq_sm90.so that EXECUTES THE SAME DESCRIPTOR TABLES WITH THE NUMPY ORACLE on host memory.

Test infrastructure only (it lives under tests/ and imports oracle/).  It lets the `-m "not gpu"` suite drive
the product's host logic - graph walks, arena planning, descriptor construction, write-back - end to end on a
machine without a GPU, and compare the outcome with fixtures produced by the reference.  The product never
sees it: `install()` monkeypatches `dfq_b200._lib` inside a test, and the real library is what the `-m gpu`
tests, smoke() and bench.py load.
"""
import ctypes as C

import numpy as np
import torch

from dfq_b200 import _lib, engine
from oracle import dfq_oracle as O

f32 = np.float32


def _floats(ptr, n):
    ptr = ptr.value if isinstance(ptr, C.c_void_p) else ptr
    return np.ctypeslib.as_array((C.c_float * int(n)).from_address(int(ptr)))


def _table(ptr, count, dt):
    ptr = ptr.value if isinstance(ptr, C.c_void_p) else ptr
    if count == 0:
        return np.zeros(0, dt)
    buf = (C.c_char * (int(count) * dt.itemsize)).from_address(int(ptr))
    return np.frombuffer(buf, dtype=dt)


def _val(x):
    return x.value if hasattr(x, "value") else x


class FakeLib:
    def __init__(self, sqrt_fn=None):
        self.calls = []
        self.stats = {}     # protocol counters: "cols_ready" (layers that arrived pre-scanned), "hinted" (ranges taken from hints)
        # None = IEEE sqrt (what the GPU computes); tests comparing with reference fixtures inject the HOST's
        # torch.sqrt (MKL VML, faithful but not correctly rounded) to reproduce the reference bit for bit
        self.sqrt_fn = sqrt_fn

    # ---- plumbing ---------------------------------------------------------------------------------
    def dfq_abi_version(self):
        return _lib.ABI_VERSION

    def dfq_last_error(self):
        return b"fake"

    # ---- arena passes -----------------------------------------------------------------------------
    def _wview(self, arena, l):
        n = int(l["rows"]) * int(l["cols"]) * int(l["kk"])
        return arena[int(l["w_off"]): int(l["w_off"]) + n].reshape(int(l["rows"]), int(l["cols"]), int(l["kk"]))

    @staticmethod
    def _col_extrema(w, go, gi):
        """[C] column minima / maxima of a `second` layer (rows in groups of `go`, gi columns per group)."""
        rows = w.shape[0]
        G = rows // go
        v = w.reshape(G, go, gi, -1)
        return v.min(axis=(1, 3)).reshape(-1).astype(f32), v.max(axis=(1, 3)).reshape(-1).astype(f32)

    def dfq_cle_run(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream):
        self.calls.append("dfq_cle_run")
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        R = _table(rt_p, nR, _lib.RELATION_DT)
        sp = np.ctypeslib.as_array((C.c_int32 * (n_steps + 1)).from_address(int(_val(sp_p))))
        sl = np.ctypeslib.as_array((C.c_int32 * int(sp[n_steps])).from_address(int(_val(sl_p))))
        P = _table(P_p, 1, _lib.CLE_PARAMS_DT)[0]
        res = _table(R_p, 1, _lib.CLE_RESULT_DT)
        # protocol check: a layer flagged COLS_READY must arrive with buffer 0 = the column extrema of its current weights
        for r in R:
            l2 = L[int(r["second"])]
            if int(l2["flags"]) & _lib.LAYER_COLS_READY:
                Cn = int(r["channels"])
                cmn, cmx = self._col_extrema(self._wview(arena, l2), int(r["go"]), int(r["gi"]))
                assert np.array_equal(arena[int(l2["cmin_off"]): int(l2["cmin_off"]) + Cn], cmn), "COLS_READY but stale column minima"
                assert np.array_equal(arena[int(l2["cmax_off"]): int(l2["cmax_off"]) + Cn], cmx), "COLS_READY but stale column maxima"
                self.stats["cols_ready"] = self.stats.get("cols_ready", 0) + 1
        used = sorted(set(int(x) for x in sl))
        remap = {li: k for k, li in enumerate(used)}
        layers = []
        for li in used:
            l = L[li]
            layers.append(O.OLayer(self._wview(arena, l), arena[int(l["bias_off"]): int(l["bias_off"]) + int(l["rows"])]))
        bns, rels = [], []
        for r in R:
            Cn = int(r["channels"])
            bw = arena[int(r["bn_w_off"]): int(r["bn_w_off"]) + Cn] if r["bn_w_off"] >= 0 else None
            bb = arena[int(r["bn_b_off"]): int(r["bn_b_off"]) + Cn] if r["bn_b_off"] >= 0 else None
            bns.append((bw, bb))
            rels.append(O.ORelation(remap[int(r["first"])], remap[int(r["second"])], len(bns) - 1))
        if int(P["apply_only"]):
            for r, rel in zip(R, rels):
                S = arena[int(r["s_acc_off"]): int(r["s_acc_off"]) + int(r["channels"])].copy()
                l1, l2 = layers[rel.first], layers[rel.second]
                l1.w *= S.reshape(-1, 1, 1); l1.b *= S
                for v in bns[rel.bn]:
                    if v is not None:
                        v *= S
                G, gi, go = int(r["groups"]), int(r["gi"]), int(r["go"])
                inv = (f32(1) / S).astype(f32)
                for g in range(G):
                    l2.w[g * go:(g + 1) * go] *= inv[g * gi:(g + 1) * gi].reshape(1, -1, 1)
            res[0]["n_sweeps"] = 1; res[0]["converged"] = 1
            return 0
        lo, hi = float(P["s_lo"]), float(P["s_hi"])
        # the product passes fp32-rounded bounds and their reciprocals; hand the oracle doubles that round to the same
        gs = np.ctypeslib.as_array((C.c_int32 * int(n_groups)).from_address(int(_val(gs_p)))) if _val(gs_p) else None
        n, diffs = 0, []
        for g in range(int(n_groups)):       # one oracle call per convergence group (= per model)
            sel = [k for k, r in enumerate(R) if int(L[int(r["first"])]["group"]) == g]
            if not sel:
                continue
            used_g = sorted({rels[k].first for k in sel} | {rels[k].second for k in sel})
            rm = {li: j for j, li in enumerate(used_g)}
            sub = [O.ORelation(rm[rels[k].first], rm[rels[k].second], rels[k].bn) for k in sel]
            ng, dg = O.cross_layer_equalization(
                [layers[li] for li in used_g], bns, sub,
                s_range=(_unround(lo, float(P["inv_lo"])), _unround(hi, float(P["inv_hi"]))),
                converge_thres=float(P["converge_thres"]), converge_count=int(P["converge_count"]),
                signed=bool(P["signed_mode"]), eps=float(P["eps"]), max_sweeps=int(P["max_sweeps"]) or None,
                sqrt_fn=self.sqrt_fn)
            for k, sr in zip(sel, sub):
                rels[k].S = sr.S
            if gs is not None:
                gs[g] = ng
            if g == 0:
                diffs = dg
            n = max(n, ng)
        for r, rel in zip(R, rels):
            arena[int(r["s_acc_off"]): int(r["s_acc_off"]) + int(r["channels"])] = rel.S
            # like the device: the column extrema of the final weights sit in buffer (sweeps of the group & 1); poison the other
            l2 = L[int(r["second"])]
            Cn = int(r["channels"])
            ng = int(gs[int(l2["group"])]) if gs is not None else n
            cmn, cmx = self._col_extrema(self._wview(arena, l2), int(r["go"]), int(r["gi"]))
            for off, val in ((int(l2["cmin_off"]), cmn), (int(l2["cmax_off"]), cmx)):
                arena[off + (ng & 1) * Cn: off + (ng & 1) * Cn + Cn] = val
                arena[off + ((ng & 1) ^ 1) * Cn: off + ((ng & 1) ^ 1) * Cn + Cn] = np.nan
        res[0]["n_sweeps"] = n
        res[0]["converged"] = 0 if (int(P["max_sweeps"]) and n >= int(P["max_sweeps"]) and diffs and diffs[-1] > float(P["converge_thres"])) else 1
        res[0]["last_diff"] = diffs[-1] if diffs else 10.0
        for i, d in enumerate(diffs[:64]):
            res[0]["diffs"][i] = d
        return 0

    def dfq_bn_fold(self, arena_p, n_arena, lt_p, nL, ft_p, nF, stream):
        self.calls.append("dfq_bn_fold")
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        Ft = _table(ft_p, nF, _lib.FOLD_DT)
        for f in Ft:
            l = L[int(f["layer"])]
            rows = int(l["rows"])
            v = lambda off: arena[int(off): int(off) + rows]
            w = self._wview(arena, l)
            b = arena[int(l["bias_off"]): int(l["bias_off"]) + rows]
            w2, b2, fw, fb = O.bn_fold(w.copy(), b.copy(), v(f["gamma_off"]), v(f["beta_off"]), v(f["mean_off"]),
                                       v(f["var_off"]), float(f["bn_eps"]), sqrt_fn=self.sqrt_fn)
            w[...] = w2; b[...] = b2
            v(f["fake_w_off"])[...] = fw; v(f["fake_b_off"])[...] = fb
            if int(f["scan_go"]) > 0:     # column extrema of the folded weights -> buffer 0
                cmn, cmx = self._col_extrema(w, int(f["scan_go"]), int(f["scan_gi"]))
                arena[int(l["cmin_off"]): int(l["cmin_off"]) + cmn.size] = cmn
                arena[int(l["cmax_off"]): int(l["cmax_off"]) + cmx.size] = cmx
        return 0

    def dfq_bias_correct(self, arena_p, n_arena, lt_p, nL, bt_p, nB, tt_p, nT, lp_p, n_levels, num_bits, stream):
        self.calls.append("dfq_bias_correct")
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        B = _table(bt_p, nB, _lib.BC_LAYER_DT)
        T = _table(tt_p, max(nT, 1), _lib.TERM_DT)
        lp = np.ctypeslib.as_array((C.c_int32 * (n_levels + 1)).from_address(int(_val(lp_p))))
        for lev in range(n_levels):
            expects = {}
            for bi in range(int(lp[lev]), int(lp[lev + 1])):       # phase E of the whole level first
                b = B[bi]
                ex = np.zeros(int(b["expect_len"]), f32)
                for ti in range(int(b["term_begin"]), int(b["term_end"])):
                    t = T[ti]
                    n = int(t["n"])
                    fb = arena[int(t["bn_b_off"]): int(t["bn_b_off"]) + n]
                    v = O.relu_expectation(arena[int(t["bn_w_off"]): int(t["bn_w_off"]) + n], fb) if t["relu"] else fb.copy()
                    d = int(t["dst_off"])
                    ex[d: d + n] = (ex[d: d + n] + v) if t["accumulate"] else v
                expects[bi] = ex
            for bi in range(int(lp[lev]), int(lp[lev + 1])):
                b = B[bi]
                l = L[int(b["layer"])]
                rows = int(l["rows"])
                w = self._wview(arena, l)
                if int(b["n_col"]) > 0:   # the caller vouches for these column extrema: they must give the tensor's range
                    hmn = arena[int(b["colmin_off"]): int(b["colmin_off"]) + int(b["n_col"])]
                    hmx = arena[int(b["colmax_off"]): int(b["colmax_off"]) + int(b["n_col"])]
                    assert hmn.min() == w.min() and hmx.max() == w.max(), "column-extrema hint does not match the weights"
                    self.stats["hinted"] = self.stats.get("hinted", 0) + 1
                if int(b["flags"]) & 1:
                    d = O.bias_absorb_wc(w, expects[bi], expects[bi].shape[0])
                else:
                    d = O.bias_delta(w, expects[bi], signed=bool(b["signed_mode"]), num_bits=int(num_bits))
                arena[int(b["delta_off"]): int(b["delta_off"]) + rows] = d
                bias = arena[int(l["bias_off"]): int(l["bias_off"]) + rows]
                bias[...] = bias + (d if int(b["flags"]) & 2 else -d)
                if b["next_bn_b_off"] >= 0:
                    nb = arena[int(b["next_bn_b_off"]): int(b["next_bn_b_off"]) + rows]
                    nb[...] = nb + (-d)
        return 0

    def dfq_quantize_tensors(self, arena_p, n_arena, qt_p, nQ, div_mode, stream):
        self.calls.append("dfq_quantize_tensors")
        arena = _floats(arena_p, n_arena)
        for q in _table(qt_p, nQ, _lib.QUANT_TASK_DT):
            x = arena[int(q["off"]): int(q["off"]) + int(q["n"])]
            x[...] = O.quantize(x.copy(), int(q["num_bits"]), float(x.min()), float(x.max()), bool(q["symmetric"]),
                                div_mode="recip" if div_mode else "div")
        return 0

    # ---- stand-alone tensor ops -------------------------------------------------------------------------
    def dfq_minmax(self, x_p, n, out_p, stream):
        x = _floats(x_p, n); out = _floats(out_p, 2)
        out[0] = x.min(); out[1] = x.max()
        return 0

    def dfq_quant_dequant(self, x_p, y_p, n, mn, scale, qmin, qmax, div_mode, codes_p, stream):
        x = _floats(x_p, n); y = _floats(y_p, n)
        scale_d = float(_val(scale))
        mn, scale, qmin, qmax = (f32(_val(v)) for v in (mn, scale, qmin, qmax))
        t = x + (-mn)
        t = t * f32(1.0 / scale_d) if div_mode else t / scale
        t = np.rint(np.minimum(np.maximum(t, qmin), qmax))
        y[...] = t * scale + mn
        return 0

    def dfq_quant_dequant_dev(self, x_p, y_p, n, mn_p, mx_p, bits, sym, div_mode, prologue, codes_p, stream):
        x = _floats(x_p, n); y = _floats(y_p, n)
        mn, mx = float(_floats(mn_p, 1)[0]), float(_floats(mx_p, 1)[0])
        if prologue == 0:
            y[...] = O.quantize(x.copy(), bits, mn, mx, bool(sym), div_mode="recip" if div_mode else "div")
        else:
            mn32, mx32 = f32(mn), f32(mx)
            if sym:
                qmin, qmax = f32(-2.0 ** (bits - 1)), f32(2 ** (bits - 1) - 1)
                a = max(abs(mx32), abs(mn32))
                scale = a * (f32(1) / qmax) if prologue == 2 else a / qmax
                mn32 = f32(0)
            else:
                qmin, qmax = f32(0), f32(2.0 ** bits - 1)
                d = mx32 - mn32
                scale = d * (f32(1) / qmax) if prologue == 2 else d / qmax
            scale = f32(max(scale, f32(1e-8)))
            t = (x + (-mn32)) / scale
            y[...] = np.rint(np.minimum(np.maximum(t, qmin), qmax)) * scale + mn32
        return 0

    def dfq_quant_error(self, w_p, e_p, n, mm_p, bits, sym, stream):
        w = _floats(w_p, n); e = _floats(e_p, n); mm = _floats(mm_p, 2)
        e[...] = O.quantize(w.copy(), bits, float(mm[0]), float(mm[1]), bool(sym)) - w
        return 0

    def dfq_act_minmax_per_sample(self, x_p, batch, per, out_p, scratch_p, stream):
        x = _floats(x_p, batch * per).reshape(batch, per); out = _floats(out_p, 2)
        out[0], out[1] = O.per_sample_minmax_mean(x)
        return 0

    def dfq_observe_quant(self, x_p, y_p, batch, per, rmin_p, rmax_p, stat_p, flags, momentum, bits, sym, div_mode, prologue, stream):
        self.calls.append("dfq_observe_quant")
        x = _floats(x_p, batch * per); y = _floats(y_p, batch * per)
        st_min, st_max = O.per_sample_minmax_mean(x.reshape(batch, per))
        if flags & 4:
            q_min, q_max = st_min, st_max
        else:
            rmin = _floats(rmin_p, 1); rmax = _floats(rmax_p, 1)
            if flags & 1:
                rmin[0] = min(rmin[0], st_min); rmax[0] = max(rmax[0], st_max)
            if flags & 2:
                m = f32(_val(momentum)); om = f32(1.0 - float(m))
                rmin[0] = rmin[0] * om + st_min * m; rmax[0] = rmax[0] * om + st_max * m
                q_min, q_max = st_min, st_max
            else:
                q_min, q_max = rmin[0], rmax[0]
        if _val(stat_p):
            st = _floats(stat_p, 2); st[0] = st_min; st[1] = st_max
        tmp = np.array([q_min, q_max], f32)
        return self.dfq_quant_dequant_dev(x_p, y_p, batch * per, tmp[0:1].ctypes.data, tmp[1:2].ctypes.data, bits, sym, div_mode,
                                          prologue, None, stream)

    def dfq_observer_update(self, rmin_p, rmax_p, stat_p, mode, momentum, stream):
        rmin = _floats(rmin_p, 1); rmax = _floats(rmax_p, 1); st = _floats(stat_p, 2)
        m = f32(_val(momentum))
        if mode == 1:
            rmin[0] = min(rmin[0], st[0]); rmax[0] = max(rmax[0], st[1])
        else:
            om = f32(1.0 - float(m))
            rmin[0] = rmin[0] * om + st[0] * m; rmax[0] = rmax[0] * om + st[1] * m
        return 0

    def dfq_clamp(self, x_p, n, lo, hi, stream):
        x = _floats(x_p, n)
        x[...] = np.clip(x, f32(_val(lo)), f32(_val(hi)))
        return 0


def _unround(v32: float, inv32: float) -> float:
    """A double whose fp32 rounding is v32 and whose double reciprocal rounds to inv32 (the oracle re-derives both)."""
    for cand in (v32, 1.0 / inv32 if inv32 not in (0.0, float("inf")) else v32):
        if f32(cand) == f32(v32) and (cand == 0 or f32(1.0 / cand) == f32(inv32)):
            return cand
    return v32


def torch_sqrt(x):
    return torch.sqrt(torch.from_numpy(np.ascontiguousarray(x))).numpy()


def install(monkeypatch, sqrt_fn=None):
    """Route dfq_b200 through the oracle-backed fake on the CPU for the duration of a test."""
    fake = FakeLib(sqrt_fn)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(_lib, "require_cuda", lambda: None)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(_lib, "check", lambda rc, what: None if rc == 0 else (_ for _ in ()).throw(_lib.DfqError(what)))
    monkeypatch.setattr(engine, "_default_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(engine, "_PIN", False)
    import dfq_b200.utils.quantize as q
    monkeypatch.setattr(q, "_dev_f32", lambda x: (x.contiguous(), True))
    return fake


def install_plain(sqrt_fn=None):
    """install() without pytest (spawned worker processes): returns the fake; patches stay for the process lifetime."""
    class _MP:
        def setattr(self, obj, name, value):
            setattr(obj, name, value)
    return install(_MP(), sqrt_fn)
