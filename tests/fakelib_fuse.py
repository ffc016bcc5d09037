"""tests/fakelib_defer.py's stand-in, extended with the first two equalization sweeps in one pass (ABI 8): DfqFold.scan_rows,
DfqLayer DFQ_LAYER_ROWS_READY and DfqCleResult.fused_sweeps.  Test infrastructure only, like fakelib itself.

The fused pass computes the same bits as two sweeps, so the stand-in keeps the oracle's one equalization path and only
evaluates the device's guard (fuse_guard) to report fused_sweeps.  fuse_guard is also what tests/test_gpu_cle_fuse.py predicts
the device's choice with."""
import numpy as np

import fakelib
import fakelib_defer
from fakelib import _floats, _table
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


def row_extrema(w):
    """Row minima / maxima of a [rows, ...] weight as the device reduces them: NaN ignored, (+inf, -inf) for a row of NaN."""
    r = w.reshape(w.shape[0], -1)
    return np.where(np.isnan(r), np.inf, r).min(1).astype(f32), np.where(np.isnan(r), -np.inf, r).max(1).astype(f32)


def _term_bound(mn, mx, s):
    m = np.maximum(np.abs(mn.astype(np.float64)), np.abs(mx.astype(np.float64)))
    sd = s.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        t = m * (np.abs(sd - 1.0) - 2.0 ** -24 * sd) - 2.0 ** -149
    return np.where((t > 0) & (t < 1e300), t, 0.0)


def fuse_guard(blocks, s_range=(1e-8, 1e8), eps=0, signed=False, converge_thres=2e-7, converge_count=20, max_sweeps=0,
               sqrt_fn=None):
    """Whether k_cle_stack applies the first two sweeps in one pass (include/dfq_b200.h DFQ_LAYER_ROWS_READY; the guard of
    dfq_b200/csrc/cle_engine.cu): `blocks` = (group, w1, w2) per two-layer chain with the FOLDED weights, w2 [rows, C, kk].
    Per group: the lower bound of sweep 1's metric exceeds 2 x converge_thres, or s2 = inv2 = 1 on every channel; every s1
    finite and > 0; converge_count >= 2 and max_sweeps != 1."""
    if converge_count < 2 or max_sweeps == 1:
        return False
    rng = (lambda mn, mx: np.maximum(np.abs(mn), np.abs(mx))) if signed else (lambda mn, mx: (mx - mn).astype(f32))
    lb, moves = {}, {}
    for g, w1, w2 in blocks:
        rmn, rmx = row_extrema(w1)
        cmn, cmx = row_extrema(np.ascontiguousarray(np.swapaxes(w2.reshape(w2.shape[0], w2.shape[1], -1), 0, 1)))
        s1, inv1 = O.solve_scale(rng(rmn, rmx), rng(cmn, cmx), s_range=s_range, eps=eps, sqrt_fn=sqrt_fn)
        if not np.all((s1 > 0) & (s1 < np.inf)):
            return False
        with np.errstate(over="ignore", invalid="ignore"):
            r1 = rng((rmn * s1).astype(f32), (rmx * s1).astype(f32))
            c1 = rng((cmn * inv1).astype(f32), (cmx * inv1).astype(f32))
        s2, inv2 = O.solve_scale(r1, c1, s_range=s_range, eps=eps, sqrt_fn=sqrt_fn)
        moves[g] = moves.get(g, False) or bool(np.any((s2 != 1) | (inv2 != 1)))
        lb[g] = lb.get(g, 0.0) + _term_bound(rmn, rmx, s1).sum() / w1.size + _term_bound(cmn, cmx, inv1).sum() / w2.size
    return all(lb[g] > 2.0 * converge_thres or not moves[g] for g in lb)


class FuseFakeLib(fakelib_defer.DeferFakeLib):
    def dfq_bn_fold(self, arena_p, n_arena, lt_p, nL, ft_p, nF, stream):
        rc = super().dfq_bn_fold(arena_p, n_arena, lt_p, nL, ft_p, nF, stream)
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        for f in _table(ft_p, nF, _lib.FOLD_DT):
            if int(f["scan_rows"]):          # (DFQ_FOLD_DEFER only: the factors are stored, the weights not yet folded)
                l = L[int(f["layer"])]
                rows, off = int(l["rows"]), int(l["rext_off"])
                fac = arena[int(f["fac_off"]): int(f["fac_off"]) + rows]
                rmn, rmx = row_extrema((self._wview(arena, l) * fac.reshape(-1, 1, 1)).astype(f32))
                arena[off: off + rows] = rmn
                arena[off + rows: off + 2 * rows] = rmx
        return rc

    def dfq_cle_run(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream):
        fused = self._fuses(_floats(arena_p, n_arena), _table(lt_p, nL, _lib.LAYER_DT), rt_p, nR, sp_p, sl_p, n_steps, P_p)
        rc = super().dfq_cle_run(arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream)
        _table(R_p, 1, _lib.CLE_RESULT_DT)[0]["fused_sweeps"] = 2 if fused else 0
        return rc

    def _folded(self, arena, l):
        """The layer's weights as the equalization sees them: a pending fold applied (arena untouched)."""
        w = self._wview(arena, l)
        if int(l["flags"]) & _lib.LAYER_FOLD_PENDING:
            fac = arena[int(l["fold_off"]): int(l["fold_off"]) + int(l["rows"])]
            w = (w * fac.reshape(-1, 1, 1)).astype(f32)
        return w

    def _fuses(self, arena, L, rt_p, nR, sp_p, sl_p, n_steps, P_p):
        """The fused pass runs when every first layer arrives ROWS_READY (whose row extrema must then be those of its
        folded weights) and the guard accepts."""
        R = _table(rt_p, nR, _lib.RELATION_DT)
        P = _table(P_p, 1, _lib.CLE_PARAMS_DT)[0]
        sp = np.ctypeslib.as_array((fakelib.C.c_int32 * (int(n_steps) + 1)).from_address(int(fakelib._val(sp_p))))
        sl = np.ctypeslib.as_array((fakelib.C.c_int32 * int(sp[int(n_steps)])).from_address(int(fakelib._val(sl_p))))
        first = [int(x) for x in sl[int(sp[0]): int(sp[1])]]
        if int(n_steps) != 2 or int(P["apply_only"]) or not all(int(L[i]["flags"]) & _lib.LAYER_ROWS_READY for i in first):
            return False
        blocks = []
        for i in first:
            l = L[i]
            rows, off = int(l["rows"]), int(l["rext_off"])
            w1 = self._folded(arena, l)
            rmn, rmx = row_extrema(w1)
            assert np.array_equal(arena[off: off + rows], rmn) and np.array_equal(arena[off + rows: off + 2 * rows], rmx), \
                "ROWS_READY but stale row extrema"
            blocks.append((int(l["group"]), w1, self._folded(arena, L[int(R[int(l["rel_out"])]["second"])])))
        lo, hi = float(P["s_lo"]), float(P["s_hi"])
        return fuse_guard(blocks, s_range=(fakelib._unround(lo, float(P["inv_lo"])), fakelib._unround(hi, float(P["inv_hi"]))),
                          eps=float(P["eps"]), signed=bool(P["signed_mode"]), converge_thres=float(P["converge_thres"]),
                          converge_count=int(P["converge_count"]), max_sweeps=int(P["max_sweeps"]), sqrt_fn=self.sqrt_fn)


def install(monkeypatch, sqrt_fn=None, takes=True):
    """fakelib.install() with the fusing stand-in."""
    fakelib.install(monkeypatch, sqrt_fn)
    d = FuseFakeLib(sqrt_fn, takes)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: d)
    return d
