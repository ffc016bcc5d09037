"""tests/fakelib_bc.py's stand-in, extended with dfq_bias_correct_absorb_clip (bias absorption and weight clipping inside the
correction): the library's refusals, the absorption vectors (oracle bias_absorb_c), first.bias -= c where `first` has no
correction entry, the clip-only layers, and per entry the absorption dot over the UNCLIPPED weights (bias_absorb_wc, grouped),
the clamp (clip_weight) and the correction of the clamped weights, with the bias rounded as fl(fl(fl(b + wc) - c) - delta).
Test infrastructure only, like fakelib itself."""
import math

import numpy as np

import fakelib
import fakelib_bc
from fakelib import C, _floats, _table, _val
from dfq_b200 import _lib
from oracle import dfq_oracle as O

f32 = np.float32


class AbsorbClipFakeLib(fakelib_bc.BcFakeLib):
    def __init__(self, sqrt_fn=None, takes=True):
        super().__init__(sqrt_fn, takes)
        self.absorb_clip = []      # per call: (absorbing relations, clip-only layers, correction entries)

    def dfq_bias_correct_absorb_clip(self, arena_p, n_arena, lt_p, nL, bt_p, nB, tt_p, nT, lp_p, n_levels, num_bits, at_p, nA,
                                     absorb_n, clip, lo, hi, stream):
        self.calls.append("dfq_bias_correct_absorb_clip")
        N, lo, hi = f32(_val(absorb_n)), f32(_val(lo)), f32(_val(hi))
        nB, nA = max(int(nB), 0), max(int(nA), 0)
        if nA and not math.isfinite(float(N)):
            return 1
        if clip and not (math.isfinite(float(lo)) and math.isfinite(float(hi)) and lo <= hi):
            return 1
        arena = _floats(arena_p, n_arena)
        L = _table(lt_p, nL, _lib.LAYER_DT)
        B = _table(bt_p, nB, _lib.BC_LAYER_DT) if nB else np.zeros(0, _lib.BC_LAYER_DT)
        A = _table(at_p, nA, _lib.ABSORB_DT) if nA else np.zeros(0, _lib.ABSORB_DT)
        if (B["flags"] & _lib.BC_PREPARED).any():
            return 1
        slot = {int(b["layer"]): i for i, b in enumerate(B)}
        if len(slot) != len(B):
            return 1
        vec = lambda off, n: arena[int(off): int(off) + int(n)]
        wc_c, sub_c = {}, {}            # entry -> c of its absorption dot / of the c it subtracts
        # ---- k_absorb_vectors -------------------------------------------------------------------------------------
        for a in A:
            n, l1 = int(a["n"]), L[int(a["first"])]
            if int(a["second"]) not in slot:
                return 1
            c = O.bias_absorb_c(vec(a["bn_w_off"], n), vec(a["bn_b_off"], n), N)
            vec(a["c_off"], n)[...] = c
            fb = vec(a["bn_b_off"], n)
            fb[...] = fb - c
            s2 = slot[int(a["second"])]
            if not int(B[s2]["flags"]) & 1:
                wc_c[s2] = (c, n)
            if int(a["first"]) in slot:
                sub_c[slot[int(a["first"])]] = c
            else:
                b1 = vec(l1["bias_off"], l1["rows"])
                b1[...] = b1 - c
        # ---- k_clip_tensors: the layers no entry reads ----------------------------------------------------------------
        clip_only = [li for li in range(int(nL)) if li not in slot] if clip else []
        for li in clip_only:
            w = self._wview(arena, L[li])
            w[...] = O.clip_weight(w, lo, hi)
        self.absorb_clip.append((len(A), clip_only, len(B)))
        if not nB:
            return 0
        # ---- the correction in its AC mode ----------------------------------------------------------------------------
        T = _table(tt_p, max(int(nT), 1), _lib.TERM_DT)
        lp = np.ctypeslib.as_array((C.c_int32 * (int(n_levels) + 1)).from_address(int(_val(lp_p))))
        for lev in range(int(n_levels)):
            expects = {bi: self._expect(arena, B[bi], T) for bi in range(int(lp[lev]), int(lp[lev + 1]))}
            for bi in range(int(lp[lev]), int(lp[lev + 1])):
                b = B[bi]
                l = L[int(b["layer"])]
                rows = int(l["rows"])
                w = self._wview(arena, l)
                raw = bool(int(b["flags"]) & 1)
                if raw:                                      # the absorption alone: its sums before the clip
                    d = O.bias_absorb_wc(w, expects[bi], expects[bi].shape[0])
                wc = O.bias_absorb_wc(w, wc_c[bi][0], wc_c[bi][1]) if bi in wc_c else None
                if clip:
                    w[...] = O.clip_weight(w, lo, hi)
                if not raw:
                    d = O.bias_delta(w, expects[bi], signed=bool(b["signed_mode"]), num_bits=int(num_bits))
                vec(b["delta_off"], rows)[...] = d
                sd = d if int(b["flags"]) & 2 else -d
                bias = vec(l["bias_off"], rows)
                nbias = bias.copy()
                if raw:
                    nbias = nbias + sd
                elif wc is not None:
                    nbias = nbias + wc
                if bi in sub_c:
                    nbias = nbias - sub_c[bi]
                if not raw:
                    nbias = nbias + sd
                bias[...] = nbias
                if b["next_bn_b_off"] >= 0:
                    nb = vec(b["next_bn_b_off"], rows)
                    nb[...] = nb + (-d)
        return 0


def install(monkeypatch, sqrt_fn=None, takes=True):
    """fakelib.install() with the absorbing and clipping stand-in."""
    fakelib.install(monkeypatch, sqrt_fn)
    d = AbsorbClipFakeLib(sqrt_fn, takes)
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: d)
    return d
