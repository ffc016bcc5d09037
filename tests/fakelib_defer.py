"""fakelib's oracle-backed stand-in, extended with the deferred BN fold (ABI 6): dfq_cle_takes_stack, DfqFold.mode
(DFQ_FOLD_DEFER / DFQ_FOLD_APPLY) and DfqLayer DFQ_LAYER_FOLD_PENDING.  Test infrastructure only, like fakelib itself.

`takes`: what dfq_cle_takes_stack reports (the host code defers exactly when it says 1).  The stand-in has one equalization
path, so a pending fold is applied to the weights on entry of dfq_cle_run - the device's engine path."""
import numpy as np

import fakelib
from fakelib import FakeLib, _floats, _table
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


class DeferFakeLib(FakeLib):
    def __init__(self, sqrt_fn=None, takes=True):
        super().__init__(sqrt_fn)
        self.takes = takes
        self.pending_seen = []      # per dfq_cle_run call: the layers that arrived with FOLD_PENDING
        self.fold_modes = []        # per dfq_bn_fold call: the modes of its folds

    def dfq_cle_takes_stack(self, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, apply_only, takes_p):
        self.calls.append("dfq_cle_takes_stack")
        t = np.ctypeslib.as_array((fakelib.C.c_int32 * 1).from_address(int(fakelib._val(takes_p))))
        t[0] = 1 if (self.takes and not apply_only) else 0
        return 0

    def _factors(self, arena, f, rows):
        """gamma / sqrt(var + eps) per row: the oracle's fold of a column of ones."""
        v = lambda off: arena[int(off): int(off) + rows]
        w2, _, _, _ = O.bn_fold(np.ones((rows, 1), f32), None, v(f["gamma_off"]), v(f["beta_off"]), v(f["mean_off"]),
                                v(f["var_off"]), float(f["bn_eps"]), sqrt_fn=self.sqrt_fn)
        return w2[:, 0].copy()

    def dfq_bn_fold(self, arena_p, n_arena, lt_p, nL, ft_p, nF, stream):
        Ft = _table(ft_p, nF, _lib.FOLD_DT)
        self.fold_modes.append([int(f["mode"]) for f in Ft])
        if all(int(f["mode"]) == _lib.FOLD_FULL for f in Ft):
            return super().dfq_bn_fold(arena_p, n_arena, lt_p, nL, ft_p, nF, stream)
        self.calls.append("dfq_bn_fold")
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        for f in Ft:
            l = L[int(f["layer"])]
            rows = int(l["rows"])
            w = self._wview(arena, l)
            mode = int(f["mode"])
            if mode == _lib.FOLD_FULL:
                one = np.array([f], dtype=_lib.FOLD_DT)
                super().dfq_bn_fold(arena_p, n_arena, lt_p, nL, one.ctypes.data, 1, stream)
                continue
            fac = arena[int(f["fac_off"]): int(f["fac_off"]) + rows]
            if mode == _lib.FOLD_APPLY:
                w[...] = (w * fac.reshape(-1, 1, 1)).astype(f32)
                continue
            # DFQ_FOLD_DEFER: vectors + factors; the scan sees the folded values, the weights stay as they are
            v = lambda off: arena[int(off): int(off) + rows]
            b = arena[int(l["bias_off"]): int(l["bias_off"]) + rows]
            _, b2, fw, fb = O.bn_fold(w.copy(), b.copy(), v(f["gamma_off"]), v(f["beta_off"]), v(f["mean_off"]),
                                      v(f["var_off"]), float(f["bn_eps"]), sqrt_fn=self.sqrt_fn)
            fac[...] = self._factors(arena, f, rows)
            b[...] = b2
            v(f["fake_w_off"])[...] = fw; v(f["fake_b_off"])[...] = fb
            if int(f["scan_go"]) > 0:
                cmn, cmx = self._col_extrema((w * fac.reshape(-1, 1, 1)).astype(f32), int(f["scan_go"]), int(f["scan_gi"]))
                arena[int(l["cmin_off"]): int(l["cmin_off"]) + cmn.size] = cmn
                arena[int(l["cmax_off"]): int(l["cmax_off"]) + cmx.size] = cmx
        return 0

    def dfq_cle_run(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream):
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        pend = [i for i in range(int(nL)) if int(L[i]["flags"]) & _lib.LAYER_FOLD_PENDING]
        self.pending_seen.append(pend)
        for i in pend:
            l = L[i]
            w = self._wview(arena, l)
            fac = arena[int(l["fold_off"]): int(l["fold_off"]) + int(l["rows"])]
            w[...] = (w * fac.reshape(-1, 1, 1)).astype(f32)
        return super().dfq_cle_run(arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream)


def install(monkeypatch, sqrt_fn=None, takes=True):
    """fakelib.install() with the deferring stand-in."""
    fakelib.install(monkeypatch, sqrt_fn)
    d = DeferFakeLib(sqrt_fn, takes)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: d)
    return d
