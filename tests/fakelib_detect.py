"""tests/fakelib.py's stand-in for libdfq_sm90.so, extended by host twins of dfq_ssd_decode, dfq_ssd_nms and
dfq_ssd_compact computed by tests/ssd_postprocess_oracle.py, with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.detect through it inside a test, so its argument checks, buffer
plumbing and output assembly run without a GPU.
"""
import numpy as np
import torch

import fakelib
import ssd_postprocess_oracle as SO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_int8 import E_UNSUPPORTED, _array

E_ARG = -1
MAX_CANDIDATES = 1024


class FakeDetectLib(fakelib.FakeLib):
    def __init__(self, sqrt_fn=None):
        super().__init__(sqrt_fn)
        self.refusals = []          # (entry, code, reason) of every refused call

    def _refuse(self, who, code, reason):
        self.refusals.append((who, code, reason))
        return code

    def _desc(self, d_p, who, nms):
        if not _val(d_p):
            return None, self._refuse(who, E_ARG, "descriptor is NULL")
        d = _table(d_p, 1, _lib.SSD_NMS_DT)[0]
        d = {k: d[k].item() for k in _lib.SSD_NMS_DT.names}
        if d["N"] < 1 or d["P"] < 1:
            return None, self._refuse(who, E_ARG, "N and P must be positive")
        if d["prior_batch"] not in (1, d["N"]):
            return None, self._refuse(who, E_ARG, "prior_batch must be 1 or N")
        if nms:
            if d["C"] < 2:
                return None, self._refuse(who, E_ARG, "C must be at least 2")
            if d["candidate_size"] < 1:
                return None, self._refuse(who, E_ARG, "candidate_size must be at least 1")
            if d["candidate_size"] > MAX_CANDIDATES:
                return None, self._refuse(who, E_UNSUPPORTED, "candidate_size is above the limit")
        return d, 0

    @staticmethod
    def _aligned(*ps):
        return all(_val(p) and int(_val(p)) % 16 == 0 for p in ps)

    def dfq_ssd_decode(self, loc_p, pri_p, box_p, d_p, stream):
        self.calls.append("dfq_ssd_decode")
        d, rc = self._desc(d_p, "dfq_ssd_decode", False)
        if rc:
            return rc
        if not self._aligned(loc_p, pri_p, box_p):
            return self._refuse("dfq_ssd_decode", E_ARG, "NULL or misaligned pointer")
        N, P, B = d["N"], d["P"], d["prior_batch"]
        loc = torch.from_numpy(_floats(loc_p, N * P * 4).reshape(N, P, 4))
        pri = torch.from_numpy(_floats(pri_p, B * P * 4).reshape(B, P, 4))
        cv, sv = np.float32(d["center_variance"]).item(), np.float32(d["size_variance"]).item()
        _floats(box_p, N * P * 4)[...] = SO.decode(loc, pri, cv, sv).numpy().reshape(-1)
        return 0

    def dfq_ssd_nms(self, sc_p, box_p, sb_p, sp_p, cnt_p, off_p, d_p, stream):
        self.calls.append("dfq_ssd_nms")
        d, rc = self._desc(d_p, "dfq_ssd_nms", True)
        if rc:
            return rc
        if not all(_val(p) for p in (sc_p, sp_p, cnt_p, off_p)) or not self._aligned(box_p, sb_p):
            return self._refuse("dfq_ssd_nms", E_ARG, "NULL or misaligned pointer")
        N, P, C, K = d["N"], d["P"], d["C"], d["candidate_size"]
        S = N * (C - 1)
        scores = torch.from_numpy(_floats(sc_p, N * P * C).reshape(N, P, C))
        boxes = torch.from_numpy(_floats(box_p, N * P * 4).reshape(N, P, 4))
        slot_boxes = _floats(sb_p, S * K * 4).reshape(S, K, 4)
        slot_probs = _floats(sp_p, S * K).reshape(S, K)
        counts = _array(cnt_p, S, np.int32)
        thr, iou_thr = np.float32(d["prob_threshold"]).item(), np.float32(d["iou_threshold"]).item()
        for n in range(N):
            for c in range(1, C):
                s = n * (C - 1) + c - 1
                keep = scores[n, :, c] > thr
                probs, cand = scores[n, keep, c], boxes[n, keep]
                picks = SO.hard_nms(cand, probs, iou_thr, d["top_k"], K) if probs.numel() else torch.zeros(0, dtype=torch.int64)
                counts[s] = picks.numel()
                slot_boxes[s, :picks.numel()] = cand[picks].numpy()
                slot_probs[s, :picks.numel()] = probs[picks].numpy()
        _array(off_p, S + 1, np.int64)[...] = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
        return 0

    def dfq_ssd_compact(self, sb_p, sp_p, cnt_p, off_p, sizes_p, ob_p, ol_p, op_p, d_p, stream):
        self.calls.append("dfq_ssd_compact")
        d, rc = self._desc(d_p, "dfq_ssd_compact", True)
        if rc:
            return rc
        if not all(_val(p) for p in (sp_p, cnt_p, off_p, ol_p, op_p)) or not self._aligned(sb_p, ob_p):
            return self._refuse("dfq_ssd_compact", E_ARG, "NULL or misaligned pointer")
        N, C, K = d["N"], d["C"], d["candidate_size"]
        S = N * (C - 1)
        counts, offs = _array(cnt_p, S, np.int32), _array(off_p, S + 1, np.int64)
        T = int(offs[S])
        slot_boxes, slot_probs = _floats(sb_p, S * K * 4).reshape(S, K, 4), _floats(sp_p, S * K).reshape(S, K)
        sizes = _floats(sizes_p, 2 * N).reshape(N, 2) if _val(sizes_p) else None
        out_b, out_l, out_p = _floats(ob_p, 4 * T).reshape(T, 4), _array(ol_p, T, np.int64), _floats(op_p, T)
        for s in range(S):
            n, k, o = s // (C - 1), int(counts[s]), int(offs[s])
            b = slot_boxes[s, :k].copy()
            if sizes is not None:
                b *= np.array([sizes[n, 0], sizes[n, 1], sizes[n, 0], sizes[n, 1]], np.float32)
            out_b[o:o + k], out_l[o:o + k], out_p[o:o + k] = b, s % (C - 1) + 1, slot_probs[s, :k]
        return 0


def install(monkeypatch):
    """fakelib.install() with the detection twins; every tensor counts as a CUDA tensor while it is active."""
    fakelib.install(monkeypatch)
    fake = FakeDetectLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return fake
