"""tests/fakelib_fuse.py's stand-in, extended with the bias correction attached to the equalization (ABI 9): dfq_cle_run_bc,
DfqCleResult.bc_prepared and DfqBcLayer DFQ_BC_PREPARED.  Test infrastructure only, like fakelib itself.

The attached correction is computed by the oracle from the final weights, as a later dfq_bias_correct would, and reported
prepared exactly when the device reports it: the fused pass ran and every group stopped after sweep 2.  A DFQ_BC_PREPARED
table is checked against a fresh oracle correction of the current weights (a stale prepared delta fails the test) and
then only retired."""
import numpy as np

import fakelib
import fakelib_fuse
from fakelib import _floats, _table
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


class BcFakeLib(fakelib_fuse.FuseFakeLib):
    def __init__(self, sqrt_fn=None, takes=True):
        super().__init__(sqrt_fn, takes)
        self.attached = []          # per equalization call: entries of the attached correction (0: none)
        self.retired = 0            # dfq_bias_correct calls that only retired prepared deltas

    def _expect(self, arena, b, T):
        ex = np.zeros(int(b["expect_len"]), f32)
        for ti in range(int(b["term_begin"]), int(b["term_end"])):
            t = T[ti]
            n = int(t["n"])
            fb = arena[int(t["bn_b_off"]): int(t["bn_b_off"]) + n]
            v = O.relu_expectation(arena[int(t["bn_w_off"]): int(t["bn_w_off"]) + n], fb) if t["relu"] else fb.copy()
            d = int(t["dst_off"])
            ex[d: d + n] = (ex[d: d + n] + v) if t["accumulate"] else v
        return ex

    def _delta(self, arena, L, b, T, num_bits):
        w = self._wview(arena, L[int(b["layer"])])
        return O.bias_delta(w, self._expect(arena, b, T), signed=bool(b["signed_mode"]), num_bits=int(num_bits))

    def dfq_cle_run(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream):
        self.attached.append(0)
        return super().dfq_cle_run(arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream)

    def dfq_cle_run_bc(self, arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, bc_p, n_bc,
                       bct_p, n_bct, bc_bits, stream):
        rc = super().dfq_cle_run(arena_p, n_arena, lt_p, nL, rt_p, nR, sp_p, sl_p, n_steps, P_p, R_p, n_groups, gs_p, stream)
        res = _table(R_p, 1, _lib.CLE_RESULT_DT)[0]
        n_bc = int(n_bc) if fakelib._val(bc_p) else 0
        self.attached.append(n_bc)
        if n_bc == 0:
            return rc
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        B = _table(bc_p, n_bc, _lib.BC_LAYER_DT)
        T = _table(bct_p, max(int(n_bct), 1), _lib.TERM_DT)
        for b in B:       # dfq_cle_run_bc's conditions on an attached correction
            l = L[int(b["layer"])]
            assert int(l["rel_in"]) >= 0 and int(l["rel_out"]) < 0 and int(b["flags"]) == 0 and int(b["expect_len"]) == int(l["cols"])
        gs = np.ctypeslib.as_array((fakelib.C.c_int32 * int(n_groups)).from_address(int(fakelib._val(gs_p))))
        res["bc_prepared"] = 1 if (int(res["fused_sweeps"]) == 2 and np.all(gs == 2)) else 0
        if res["bc_prepared"]:
            for b in B:
                w = self._wview(arena, L[int(b["layer"])])
                rows = w.shape[0]
                arena[int(b["delta_off"]): int(b["delta_off"]) + rows] = self._delta(arena, L, b, T, bc_bits)
                arena[int(b["expect_off"]): int(b["expect_off"]) + int(b["expect_len"])] = self._expect(arena, b, T)
                arena[int(b["minmax_off"])], arena[int(b["minmax_off"]) + 1] = w.min(), w.max()
        return rc

    def dfq_bias_correct(self, arena_p, n_arena, lt_p, nL, bt_p, nB, tt_p, nT, lp_p, n_levels, num_bits, stream):
        B = _table(bt_p, nB, _lib.BC_LAYER_DT)
        prep = (B["flags"] & _lib.BC_PREPARED) != 0
        if not prep.any():
            return super().dfq_bias_correct(arena_p, n_arena, lt_p, nL, bt_p, nB, tt_p, nT, lp_p, n_levels, num_bits, stream)
        assert prep.all(), "a table that mixes prepared and unprepared entries"
        self.calls.append("dfq_bias_correct")
        self.retired += 1
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        T = _table(tt_p, max(int(nT), 1), _lib.TERM_DT)
        for b in B:
            l = L[int(b["layer"])]
            rows = int(l["rows"])
            d = arena[int(b["delta_off"]): int(b["delta_off"]) + rows].copy()
            assert np.array_equal(d, self._delta(arena, L, b, T, num_bits)), "DFQ_BC_PREPARED but the delta is stale"
            bias = arena[int(l["bias_off"]): int(l["bias_off"]) + rows]
            bias[...] = bias - d
            if b["next_bn_b_off"] >= 0:
                nb = arena[int(b["next_bn_b_off"]): int(b["next_bn_b_off"]) + rows]
                nb[...] = nb + (-d)
        return 0


def install(monkeypatch, sqrt_fn=None, takes=True):
    """fakelib.install() with the correcting stand-in."""
    fakelib.install(monkeypatch, sqrt_fn)
    d = BcFakeLib(sqrt_fn, takes)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: d)
    return d
