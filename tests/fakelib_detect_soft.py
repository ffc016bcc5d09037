"""tests/fakelib_detect.py's stand-in extended by host twins of dfq_ssd_soft_nms and dfq_ssd_soft_compact computed by
the soft NMS of tests/ssd_soft_nms_oracle.py, with the library's refusals.

Test infrastructure only: `install()` routes dfq_b200.detect through it inside a test, so the soft path's argument
checks, buffer plumbing and output assembly run without a GPU.
"""
import math

import numpy as np
import torch

import fakelib
import fakelib_detect
import ssd_soft_nms_oracle as SO
from dfq_b200 import _lib
from fakelib import _floats, _table, _val
from fakelib_detect import E_ARG
from fakelib_int8 import _array


class FakeSoftDetectLib(fakelib_detect.FakeDetectLib):
    def _soft_desc(self, d_p, sigma, who):
        if not _val(d_p):
            return None, self._refuse(who, E_ARG, "descriptor is NULL")
        d = _table(d_p, 1, _lib.SSD_NMS_DT)[0]
        d = {k: d[k].item() for k in _lib.SSD_NMS_DT.names}
        if d["N"] < 1 or d["P"] < 1:
            return None, self._refuse(who, E_ARG, "N and P must be positive")
        if d["prior_batch"] not in (1, d["N"]):
            return None, self._refuse(who, E_ARG, "prior_batch must be 1 or N")
        if d["C"] < 2:
            return None, self._refuse(who, E_ARG, "C must be at least 2")
        sigma = float(np.float32(sigma))
        if not (sigma > 0 and math.isfinite(sigma)):
            return None, self._refuse(who, E_ARG, "sigma must be a finite positive number")
        return d, 0

    def _picks(self, sc_p, box_p, d, sigma):
        """[(segment, rows [K, 5])] of every segment, and the candidate counts."""
        N, P, C = d["N"], d["P"], d["C"]
        scores = torch.from_numpy(_floats(sc_p, N * P * C).reshape(N, P, C))
        boxes = torch.from_numpy(_floats(box_p, N * P * 4).reshape(N, P, 4))
        thr = np.float32(d["prob_threshold"]).item()
        out, cands = [], []
        for n in range(N):
            for c in range(1, C):
                keep = scores[n, :, c] > thr
                cands.append(int(keep.sum()))
                rows = SO.soft_nms(boxes[n, keep], scores[n, keep, c], thr, float(np.float32(sigma)), d["top_k"]) \
                    if cands[-1] else torch.zeros(0, 5)
                out.append(rows)
        return out, np.array(cands, np.int32)

    def dfq_ssd_soft_nms(self, sc_p, box_p, cand_p, cnt_p, off_p, d_p, sigma, stream):
        who = "dfq_ssd_soft_nms"
        self.calls.append(who)
        d, rc = self._soft_desc(d_p, sigma, who)
        if rc:
            return rc
        if not all(_val(p) for p in (sc_p, cand_p, cnt_p, off_p)) or not self._aligned(box_p):
            return self._refuse(who, E_ARG, "NULL or misaligned pointer")
        S = d["N"] * (d["C"] - 1)
        rows, cands = self._picks(sc_p, box_p, d, sigma)
        counts = np.array([r.shape[0] for r in rows], np.int32)
        _array(cand_p, S, np.int32)[...] = cands
        _array(cnt_p, S, np.int32)[...] = counts
        _array(off_p, S + 1, np.int64)[...] = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
        return 0

    def dfq_ssd_soft_compact(self, sc_p, box_p, cand_p, off_p, sizes_p, ob_p, ol_p, op_p, d_p, sigma, stream):
        who = "dfq_ssd_soft_compact"
        self.calls.append(who)
        d, rc = self._soft_desc(d_p, sigma, who)
        if rc:
            return rc
        if not all(_val(p) for p in (sc_p, cand_p, off_p, ol_p, op_p)) or not self._aligned(box_p, ob_p):
            return self._refuse(who, E_ARG, "NULL or misaligned pointer")
        N, C = d["N"], d["C"]
        S = N * (C - 1)
        offs = _array(off_p, S + 1, np.int64)
        T = int(offs[S])
        sizes = _floats(sizes_p, 2 * N).reshape(N, 2) if _val(sizes_p) else None
        out_b, out_l, out_p = _floats(ob_p, 4 * T).reshape(T, 4), _array(ol_p, T, np.int64), _floats(op_p, T)
        rows, _ = self._picks(sc_p, box_p, d, sigma)
        for s, r in enumerate(rows):
            n, k, o = s // (C - 1), r.shape[0], int(offs[s])
            b = r[:, :4].numpy().copy()
            if sizes is not None:
                b *= np.array([sizes[n, 0], sizes[n, 1], sizes[n, 0], sizes[n, 1]], np.float32)
            out_b[o:o + k], out_l[o:o + k], out_p[o:o + k] = b, s % (C - 1) + 1, r[:, 4].numpy()
        return 0


def install(monkeypatch):
    """fakelib.install() with the detection twins, soft NMS included; every tensor counts as a CUDA tensor while it is
    active."""
    fakelib.install(monkeypatch)
    fake = FakeSoftDetectLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: fake)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return fake
