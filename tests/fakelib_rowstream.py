"""tests/fakelib_fuse.py's stand-in, extended with the deferred fold's row PREFIX (ABI 11): DfqFold.row_prefix, DfqLayer.rext_rows
and DfqCleResult.rows_streamed.  Test infrastructure only, like fakelib itself.

The fold writes the row extrema of the prefix only (the other rows of the scratch get NaN, which no guard could use), and the
equalization reports which way the device goes (prefix_guard): the prefix decides, it leaves a group undecided, or the host
does not let the guard use it.  Either way the stand-in completes the scratch first and then evaluates fuse_guard on every
row, as the device does."""
import numpy as np

import fakelib
import fakelib_fuse
from fakelib import _floats, _table
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


def prefix_rows(rows, prefix):
    """DfqLayer.rext_rows / DfqFold.row_prefix: rows whose extrema the fold scans (0 or >= rows: all)."""
    return rows if prefix <= 0 or prefix >= rows else prefix


def prefix_guard(blocks, prefix, s_range=(1e-8, 1e8), eps=0, signed=False, converge_thres=2e-7, sqrt_fn=None):
    """Whether k_cle_stack's guard decides from the first `prefix` rows of every first conv (cle_engine.cu
    fuse_guard_scan<true> / fuse_prefix_groups): per group, the sum of fuse_term_bound over the prefix's rows and the matching
    columns of the second conv exceeds 2 x converge_thres.  `blocks` as fakelib_fuse.fuse_guard takes them."""
    rng = (lambda mn, mx: np.maximum(np.abs(mn), np.abs(mx))) if signed else (lambda mn, mx: (mx - mn).astype(f32))
    lb = {}
    for g, w1, w2 in blocks:
        p = prefix_rows(w1.shape[0], prefix)
        rmn, rmx = fakelib_fuse.row_extrema(w1)
        cmn, cmx = fakelib_fuse.row_extrema(np.ascontiguousarray(np.swapaxes(w2.reshape(w2.shape[0], w2.shape[1], -1), 0, 1)))
        rmn, rmx, cmn, cmx = rmn[:p], rmx[:p], cmn[:p], cmx[:p]
        s1, inv1 = O.solve_scale(rng(rmn, rmx), rng(cmn, cmx), s_range=s_range, eps=eps, sqrt_fn=sqrt_fn)
        lb[g] = lb.get(g, 0.0) + (fakelib_fuse._term_bound(rmn, rmx, s1).sum() / w1.size
                                  + fakelib_fuse._term_bound(cmn, cmx, inv1).sum() / w2.size)
    return all(v > 2.0 * converge_thres for v in lb.values())


class RowStreamFakeLib(fakelib_fuse.FuseFakeLib):
    def dfq_bn_fold(self, arena_p, n_arena, lt_p, nL, ft_p, nF, stream):
        rc = super().dfq_bn_fold(arena_p, n_arena, lt_p, nL, ft_p, nF, stream)
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        for f in _table(ft_p, nF, _lib.FOLD_DT):
            if int(f["scan_rows"]):
                l = L[int(f["layer"])]
                rows, off = int(l["rows"]), int(l["rext_off"])
                p = prefix_rows(rows, int(f["row_prefix"]))
                arena[off + p: off + rows] = np.nan
                arena[off + rows + p: off + 2 * rows] = np.nan
        return rc

    def dfq_cle_run(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream):
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        R = _table(rt_p, nR, _lib.RELATION_DT)
        P = _table(P_p, 1, _lib.CLE_PARAMS_DT)[0]
        sp = np.ctypeslib.as_array((fakelib.C.c_int32 * (int(n_steps) + 1)).from_address(int(fakelib._val(sp_p))))
        sl = np.ctypeslib.as_array((fakelib.C.c_int32 * int(sp[int(n_steps)])).from_address(int(fakelib._val(sl_p))))
        first = [int(x) for x in sl[int(sp[0]): int(sp[1])]] if int(n_steps) >= 1 else []
        ready = [i for i in first if int(L[i]["flags"]) & _lib.LAYER_ROWS_READY]
        prefixed = [i for i in ready if prefix_rows(int(L[i]["rows"]), int(L[i]["rext_rows"])) < int(L[i]["rows"])]
        streamed = _lib.ROWS_FULL
        if prefixed:
            lo, hi = float(P["s_lo"]), float(P["s_hi"])
            fuse = (int(n_steps) == 2 and not int(P["apply_only"]) and len(ready) == len(first)
                    and int(P["converge_count"]) >= 2 and int(P["max_sweeps"]) != 1)
            if fuse and lo > 0 and np.isfinite(lo) and np.isfinite(hi):
                blocks = [(int(L[i]["group"]), self._folded(arena, L[i]), self._folded(arena, L[int(R[int(L[i]["rel_out"])]["second"])]))
                          for i in prefixed]
                ok = prefix_guard(blocks, int(L[prefixed[0]]["rext_rows"]),
                                  s_range=(fakelib._unround(lo, float(P["inv_lo"])), fakelib._unround(hi, float(P["inv_hi"]))),
                                  eps=float(P["eps"]), signed=bool(P["signed_mode"]), converge_thres=float(P["converge_thres"]),
                                  sqrt_fn=self.sqrt_fn)
                streamed = _lib.ROWS_STREAMED if ok else _lib.ROWS_UNDECIDED
            else:
                streamed = _lib.ROWS_HOST_FULL
            for i in prefixed:          # the device's own scan of the remaining rows (or, streamed, the fused pass)
                l = L[i]
                rows, off = int(l["rows"]), int(l["rext_off"])
                rmn, rmx = fakelib_fuse.row_extrema(self._folded(arena, l))
                arena[off: off + rows] = rmn
                arena[off + rows: off + 2 * rows] = rmx
        rc = super().dfq_cle_run(arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream)
        _table(R_p, 1, _lib.CLE_RESULT_DT)[0]["rows_streamed"] = streamed
        return rc


def install(monkeypatch, sqrt_fn=None, takes=True):
    """fakelib.install() with the row-prefix stand-in."""
    fakelib.install(monkeypatch, sqrt_fn)
    d = RowStreamFakeLib(sqrt_fn, takes)
    monkeypatch.setattr(fakelib_fuse._lib, "load", lambda build_if_missing=True: d)
    return d
