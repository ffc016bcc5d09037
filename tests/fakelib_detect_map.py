"""tests/fakelib_detect.py's stand-in for libdfq_sm90.so, extended by host twins of dfq_map_match and dfq_map_curve: the
verdicts computed by tests/ssd_map_oracle.py, the keys, counts, error bits and curve outputs in the library's layout, and
the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.detect.Evaluator through it inside a test, so its argument checks,
buffer plumbing, growth and the host's last sums run without a GPU.
"""
import ctypes as C

import numpy as np
import torch

import fakelib_detect
import ssd_map_oracle as O
from dfq_b200 import _lib
from fakelib import _floats, _val
from fakelib_int8 import E_UNSUPPORTED, _array

E_ARG = -1
MAX_CLASSES = 4096


def _doubles(ptr, n):
    return np.ctypeslib.as_array((C.c_double * int(n)).from_address(int(_val(ptr))))


def score_desc(p):
    """The lower 32 bits of a key: the score's descending rank bits (-0.0 as +0.0, NaN last)."""
    u = np.asarray(p, np.float32).view(np.uint32).copy()
    u[u == 0x80000000] = 0
    d = np.where(u & 0x80000000, u, ~(u | 0x80000000)).astype(np.uint32)
    d[np.isnan(np.asarray(p, np.float32))] = 0xffffffff
    return d.astype(np.uint64)


class FakeDetectMapLib(fakelib_detect.FakeDetectLib):
    def _classes(self, C_, who):
        if C_ < 2:
            return self._refuse(who, E_ARG, "C must be at least 2")
        if C_ > MAX_CLASSES:
            return self._refuse(who, E_UNSUPPORTED, "C is above the limit")
        return 0

    def dfq_map_match(self, db, dl, dp, do, T, gb, gl, gd, go, G, N, C_, thr, keys, flags, cnt, err, stream):
        who = "dfq_map_match"
        self.calls.append(who)
        if rc := self._classes(C_, who):
            return rc
        if N < 1 or T < 0 or G < 0:
            return self._refuse(who, E_ARG, "N must be positive and T, G non-negative")
        if not all(_val(p) for p in (do, go, cnt, err)):
            return self._refuse(who, E_ARG, "NULL pointer")
        if T > 0 and (not all(_val(p) for p in (dl, dp, keys, flags)) or not self._aligned(db)):
            return self._refuse(who, E_ARG, "NULL or misaligned detection pointer")
        if G > 0 and (not all(_val(p) for p in (gl, gd)) or not self._aligned(gb)):
            return self._refuse(who, E_ARG, "NULL or misaligned ground-truth pointer")
        if T > 2 ** 31 - 1:
            return self._refuse(who, E_UNSUPPORTED, "T above the limit")
        d_off, g_off = _array(do, N + 1, np.int64), _array(go, N + 1, np.int64)
        boxes = _floats(db, 4 * T).reshape(T, 4) if T else np.zeros((0, 4), np.float32)
        labels = _array(dl, T, np.int64) if T else np.zeros(0, np.int64)
        probs = _floats(dp, T) if T else np.zeros(0, np.float32)
        g_boxes = _floats(gb, 4 * G).reshape(G, 4) if G else np.zeros((0, 4), np.float32)
        g_labels = _array(gl, G, np.int64) if G else np.zeros(0, np.int64)
        g_diff = _array(gd, G, np.uint8) if G else np.zeros(0, np.uint8)
        error = _array(err, 1, np.int32)
        bad = 0
        if not (d_off[0] == 0 and d_off[-1] == T and (np.diff(d_off) >= 0).all()):
            bad |= _lib.MAP_ERR_DET_OFFSETS
        if not (g_off[0] == 0 and g_off[-1] == G and (np.diff(g_off) >= 0).all()):
            bad |= _lib.MAP_ERR_GT_OFFSETS
        if bad:                               # the device skips the images whose offsets are wrong; here all of them
            error[0] |= bad
            return 0
        if ((g_labels < 0) | (g_labels >= C_)).any():
            error[0] |= _lib.MAP_ERR_GT_LABEL
        if ((labels < 1) | (labels >= C_)).any():
            error[0] |= _lib.MAP_ERR_DET_LABEL
        ok = (g_labels >= 0) & (g_labels < C_) & (g_diff == 0)
        _array(cnt, C_, np.int64)[...] += np.bincount(g_labels[ok], minlength=C_)[:C_]
        if T:
            dets = [(torch.from_numpy(boxes[a:b].copy()), torch.from_numpy(labels[a:b].copy()),
                     torch.from_numpy(probs[a:b].copy())) for a, b in zip(d_off[:-1], d_off[1:])]
            gts = [(g_boxes[a:b], g_labels[a:b], g_diff[a:b]) for a, b in zip(g_off[:-1], g_off[1:])]
            _, verdicts = O.average_precision(dets, gts, C_, thr)
            valid = (labels >= 1) & (labels < C_)
            _array(flags, T, np.uint8)[...] = np.where(valid, verdicts, _lib.MAP_FP)
            _array(keys, T, np.uint64)[...] = (np.where(valid, labels, 0).astype(np.uint64) << np.uint64(32)) | \
                score_desc(probs)
        return 0

    def dfq_map_curve(self, keys, flags, D, C_, cnt, use_2007, out, out_len, term_count, stream):
        who = "dfq_map_curve"
        self.calls.append(who)
        if rc := self._classes(C_, who):
            return rc
        if D < 0:
            return self._refuse(who, E_ARG, "D must be non-negative")
        if use_2007 not in (0, 1):
            return self._refuse(who, E_ARG, "use_2007 must be 0 or 1")
        if not all(_val(p) for p in (cnt, out, term_count)) or (D > 0 and not (_val(keys) and _val(flags))):
            return self._refuse(who, E_ARG, "NULL pointer")
        if out_len < (11 * (C_ - 1) if use_2007 else C_):
            return self._refuse(who, E_ARG, "out too small")
        if D > 2 ** 31 - 1:
            return self._refuse(who, E_UNSUPPORTED, "D above the limit")
        k = _array(keys, D, np.uint64) if D else np.zeros(0, np.uint64)
        f = _array(flags, D, np.uint8) if D else np.zeros(0, np.uint8)
        gt_count = _array(cnt, C_, np.int64)
        res, counts = _doubles(out, out_len), _array(term_count, C_, np.int64)
        order = np.argsort(k, kind="stable")
        k, f = k[order], f[order]
        cls = (k >> np.uint64(32)).astype(np.int64)
        base = 0
        for c in range(1, C_):
            sel = f[cls == c]
            tp, fp = np.cumsum(sel == _lib.MAP_TP).astype(np.float64), np.cumsum(sel == _lib.MAP_FP).astype(np.float64)
            with np.errstate(all="ignore"):
                precision, recall = tp / (tp + fp), tp / float(gt_count[c])
                if use_2007:
                    for j in range(11):
                        s = precision[recall >= j * 0.1]
                        res[11 * (c - 1) + j] = s.max() if s.size else 0.0
                    counts[c] = sel.size
                else:
                    p = np.maximum.accumulate(np.concatenate([[0.0], precision, [0.0]])[::-1])[::-1]
                    r = np.concatenate([[0.0], recall, [1.0]])
                    cp = np.nonzero(r[1:] != r[:-1])[0]
                    terms = (r[cp + 1] - r[cp]) * p[cp + 1]
                    res[base:base + terms.size] = terms
                    counts[c] = terms.size
                    base += int(gt_count[c]) + 1
        return 0


def install(monkeypatch):
    """fakelib_detect.install() with the evaluation twins."""
    fakelib_detect.install(monkeypatch)
    fake = FakeDetectMapLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    return fake
