"""Host side of the calibration engine: arena planning, descriptor tables, C-ABI calls.

A :class:`Session` owns one fp32 device *arena* holding every weight, bias and per-channel vector of
the layers being calibrated, plus the scratch the kernels need.  Host logic (graph walks, which layer
pairs with which) produces small descriptor tables; all arithmetic happens in libdfq_sm90.so.

The session is the object behind the drop-in functions of :mod:`dfq_b200.dfq` and
:mod:`dfq_b200.utils.layer_transform`; it can also be driven directly (bench.py, tests) with tensors
that already live on the GPU.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import DfqError

# threads of the host gather/scatter (dfq_host_copy_segments); 0 = the library's default
_HOST_COPY_THREADS = int(os.environ.get("DFQ_HOST_COPY_THREADS", "0"))
# parts the upload of a model is cut into (gather of part i+1 overlaps the H2D copy of part i).  The H2D copy of a
# MobileNetV2 is short next to a library call, not worth hiding behind extra calls, so one part is the default.
_UPLOAD_PARTS = int(os.environ.get("DFQ_UPLOAD_PARTS", "1"))


_PIN = True       # page-locked staging buffers (tests that run the host logic without a GPU turn this off)


def _default_device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


@dataclass
class CleResult:
    n_sweeps: int            # max over convergence groups
    converged: bool
    last_diff: float
    diffs: List[float]       # diff_tmp per sweep of group 0
    group_sweeps: Optional[np.ndarray] = None
    apply_only: bool = False


@dataclass
class _Bound:
    off: int
    n: int
    tensor: Optional[torch.Tensor]   # host/device tensor mirrored at [off, off+n); None = scratch
    writeback: bool = True
    upload: bool = True              # False: an output-only mirror (results land in it at download; nothing to send)


class Session:
    """One arena + its descriptor tables.  Not thread-safe; one CUDA device."""

    def __init__(self, device: Optional[torch.device] = None):
        _lib.require_cuda()
        self.lib = _lib.load()
        self.device = torch.device(device) if device is not None else _default_device()
        self._n = 0
        self._bound: List[_Bound] = []
        self._by_storage: Dict[tuple, _Bound] = {}     # (data_ptr, numel, device) -> its one mirror in the arena
        self._xfer = None                               # cached copy lists of upload()/download(), dropped by bind()
        self._layers: List[dict] = []
        self.arena: Optional[torch.Tensor] = None
        self._staging: Optional[torch.Tensor] = None
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    # ---- arena planning ---------------------------------------------------------------------------
    def alloc(self, n: int, align: int = 4) -> int:
        """Reserve n floats of scratch; returns the float offset."""
        off = _round_up(self._n, align)
        self._n = off + int(n)
        return off

    def bind(self, t: torch.Tensor, writeback: bool = True, upload: bool = True) -> int:
        """Mirror tensor `t` (fp32, any device) in the arena; returns its offset.  A tensor that is bound twice (one
        module reached from two places of a graph, a conv feeding two BNs, ...) gets ONE mirror: the passes then update it one
        after the other like the reference updates the one parameter, instead of two copies racing at write-back."""
        if t.dtype != torch.float32:
            raise DfqError("calibration tensors must be float32, got %s" % t.dtype)
        key = (t.data_ptr(), t.numel(), str(t.device)) if t.numel() else None
        hit = self._by_storage.get(key) if key is not None else None
        if hit is not None and hit.tensor is not None and hit.tensor.shape == t.shape and hit.tensor.stride() == t.stride():
            if (writeback and not hit.writeback) or (upload and not hit.upload):
                hit.writeback = hit.writeback or writeback
                hit.upload = hit.upload or upload
                self._xfer = None
            return hit.off
        off = self.alloc(t.numel())
        b = _Bound(off, t.numel(), t, writeback, upload)
        self._bound.append(b)
        if key is not None:
            self._by_storage[key] = b
        self._xfer = None
        return off

    def mirror(self, off: int, t: torch.Tensor):
        """Make host/device tensor `t` an output-only mirror of the already planned arena range [off, off+numel): the
        range's contents are written into `t` at download() (e.g. scratch that holds a result, like Relation.S)."""
        self._bound.append(_Bound(int(off), t.numel(), t, True, False))
        self._xfer = None

    def add_layer(self, weight: torch.Tensor, bias: Optional[torch.Tensor], weight_writeback: bool = True) -> int:
        """Register a Conv2d ([O,J,k,k]) or Linear ([O,J]) weight and its bias (None -> zeros scratch)."""
        if weight.dim() not in (2, 4):
            raise DfqError("target layer weight must be 2-D or 4-D, got %s" % (tuple(weight.shape),))
        rows, cols = int(weight.shape[0]), int(weight.shape[1])
        kk = int(weight.numel() // (rows * cols))
        w_off = self.bind(weight, weight_writeback)
        if bias is not None:
            b_off = self.bind(bias)
        else:
            b_off = self.alloc(rows)
        self._layers.append(dict(w_off=w_off, bias_off=b_off, rows=rows, cols=cols, kk=kk, has_bias=bias is not None))
        return len(self._layers) - 1

    def alloc_layer(self, rows: int, cols: int, kk: int, bias_off: Optional[int] = None) -> int:
        """Reserve an (uninitialised, device-only) layer: weight [rows, cols*kk] and bias [rows] (`bias_off`: a range the
        caller reserved elsewhere, e.g. one block holding the biases of a whole stack)."""
        w_off = self.alloc(rows * cols * kk)
        b_off = self.alloc(rows) if bias_off is None else int(bias_off)
        self._layers.append(dict(w_off=w_off, bias_off=b_off, rows=rows, cols=cols, kk=kk, has_bias=False))
        return len(self._layers) - 1

    def layer(self, li: int) -> dict:
        return self._layers[li]

    def attach_bias(self, li: int, bias: torch.Tensor):
        """Bind a (new, zero) bias tensor to the scratch bias of layer li so it is written back."""
        l = self._layers[li]
        assert not l["has_bias"] and bias.numel() == l["rows"]
        self._bound.append(_Bound(l["bias_off"], l["rows"], bias, True))
        self._xfer = None
        l["has_bias"] = True

    # ---- materialise / move data --------------------------------------------------------------------
    def materialize(self, extra_floats: int = 0):
        """Allocate the device arena (zero-filled) sized for everything planned so far (+extra)."""
        if self.arena is not None:
            return
        total = _round_up(self._n + extra_floats + 4, 4)
        self.arena = torch.zeros(total, dtype=torch.float32, device=self.device)

    def _ensure_room(self):
        if self.arena is None:
            self.materialize()
        elif self._n > self.arena.numel():
            grown = torch.zeros(_round_up(self._n + 4, 4), dtype=torch.float32, device=self.device)
            grown[: self.arena.numel()].copy_(self.arena)
            self.arena = grown

    @staticmethod
    def _runs(bounds):
        """Coalesce [off, off+n) of `bounds` (sorted by offset) into copy runs; only alignment padding (< 4 floats) between
        two mirrors may be swallowed by a run - anything wider is scratch that must keep its device value."""
        runs = []
        for b in bounds:
            if runs and b.off - runs[-1][1] < 4:
                runs[-1][1] = max(runs[-1][1], b.off + b.n)
            else:
                runs.append([b.off, b.off + b.n])
        return runs

    def _transfer_lists(self):
        """(span_lo, h2d runs, h2d staging views, h2d sources, d2h runs, d2h staging views, d2h destinations, non-contiguous
        d2h, device-resident uploads, device-resident write-backs) - built once per binding set: upload()/download() of a
        whole model are then a handful of calls (torch._foreach_copy_ + one copy per run) instead of a Python loop per tensor."""
        if self._xfer is not None:
            return self._xfer
        host = sorted((b for b in self._bound if b.tensor is not None and not b.tensor.is_cuda and b.n), key=lambda b: b.off)
        up = [b for b in host if b.upload]
        down = [b for b in host if b.writeback]
        lo = min((b.off for b in host), default=0)
        hi = max((b.off + b.n for b in host), default=0)
        if host and (self._staging is None or self._staging.numel() < hi - lo):
            self._staging = torch.empty(hi - lo, dtype=torch.float32, pin_memory=_PIN)
        st = self._staging
        x = dict(lo=lo, hi=hi,
                 h2d_runs=self._runs(up), h2d_dst=[st[b.off - lo: b.off - lo + b.n] for b in up],
                 h2d_bounds=up,
                 d2h_runs=self._runs(down),
                 d2h_src=[st[b.off - lo: b.off - lo + b.n] for b in down], d2h_bounds=down,
                 dev_up=[b for b in self._bound if b.tensor is not None and b.tensor.is_cuda and b.upload and b.n],
                 dev_down=[b for b in self._bound if b.tensor is not None and b.tensor.is_cuda and b.writeback and b.n])
        self._xfer = x
        return x

    def _host_copy(self, x: dict, which: str, direction: int, i0: int = 0, i1: Optional[int] = None) -> bool:
        """Gather (0) / scatter (1) between the bound host tensors [i0, i1) and the staging image with the library's
        memcpy loop (dfq_host_copy_segments; faster for a MobileNetV2 than the per-tensor copy
        dispatch).  The addresses are read per call (a caller may have re-pointed a parameter's .data); returns False -
        the caller then takes the tensor-library path - when a tensor is not a contiguous fp32 host tensor of the bound size."""
        fn = getattr(self.lib, "dfq_host_copy_segments", None)
        bounds = x[which + "_bounds"]
        if fn is None or not bounds or self._staging is None:
            return False
        seg = x.get(which + "_seg")
        if seg is None:
            lo = x["lo"]
            seg = x[which + "_seg"] = (np.array([4 * b.n for b in bounds], dtype=np.uint64),
                                       np.array([4 * (b.off - lo) for b in bounds], dtype=np.uint64),
                                       np.empty(len(bounds), dtype=np.uint64))
        nbytes, offs, ptrs = seg
        i1 = len(bounds) if i1 is None else i1
        for i in range(i0, i1):
            b = bounds[i]
            t = b.tensor
            if t.dtype != torch.float32 or t.numel() != b.n or not t.is_contiguous() or t.is_cuda:
                return False
            ptrs[i] = t.data_ptr()
        _lib.check(fn(C.c_void_p(self._staging.data_ptr()), _lib.table_ptr(ptrs[i0:i1]), _lib.table_ptr(nbytes[i0:i1]),
                      _lib.table_ptr(offs[i0:i1]), i1 - i0, direction, _HOST_COPY_THREADS), "dfq_host_copy_segments")
        return True

    def _upload_parts(self, x: dict):
        """[(i0, i1, runs)]: the upload mirrors cut into a few parts of equal bytes - the H2D copy of one part crosses PCIe
        while the host gathers the next one (a 14 MB model: 4 parts)."""
        parts = x.get("h2d_parts")
        if parts is None:
            up = x["h2d_bounds"]
            total = sum(b.n for b in up)
            k = max(1, min(_UPLOAD_PARTS, (4 * total) >> 21))            # >= 2 MB per part
            parts, i0, acc = [], 0, 0
            for i, b in enumerate(up):
                acc += b.n
                if acc * k >= total * (len(parts) + 1) or i + 1 == len(up):
                    parts.append((i0, i + 1, self._runs(up[i0:i + 1])))
                    i0 = i + 1
            x["h2d_parts"] = parts
        return parts

    def upload(self):
        """Copy every bound tensor into the arena: host tensors through ONE pinned staging buffer and one H2D copy per
        run of adjacent mirrors, device tensors with device-to-device copies."""
        self._ensure_room()
        x = self._transfer_lists()
        with torch.no_grad():
            if x["h2d_bounds"]:
                lo, st = x["lo"], self._staging
                # (the sources are looked up per call: a caller may have re-pointed a parameter's .data since the last one)
                for i0, i1, runs in self._upload_parts(x):
                    if not self._host_copy(x, "h2d", 0, i0, i1):
                        torch._foreach_copy_(x["h2d_dst"][i0:i1], [b.tensor.detach().reshape(-1) for b in x["h2d_bounds"][i0:i1]])
                    for a, e in runs:
                        self.arena[a:e].copy_(st[a - lo: e - lo], non_blocking=True)
                        self.h2d_bytes += 4 * (e - a)
            for b in x["dev_up"]:
                self.arena[b.off: b.off + b.n].copy_(b.tensor.detach().reshape(-1))

    def download_begin(self):
        """Enqueue the device-to-host copies of every write-back run (asynchronous; host work that does not read the results
        can overlap them).  download_end() waits and writes the tensors."""
        x = self._transfer_lists()
        with torch.no_grad():
            lo, st = x["lo"], self._staging
            for a, e in x["d2h_runs"]:
                st[a - lo: e - lo].copy_(self.arena[a:e], non_blocking=True)
                self.d2h_bytes += 4 * (e - a)

    def download_end(self):
        x = self._transfer_lists()
        with torch.no_grad():
            if x["d2h_runs"]:
                if self.arena.is_cuda:
                    torch.cuda.current_stream().synchronize()
                dst, src = [], []
                for b, v in (() if self._host_copy(x, "d2h", 1) else zip(x["d2h_bounds"], x["d2h_src"])):
                    t = b.tensor.detach()
                    if t.is_contiguous():
                        dst.append(t.view(-1)); src.append(v)
                    else:
                        t.copy_(v.reshape(t.shape))
                if dst:
                    torch._foreach_copy_(dst, src)
            for b in x["dev_down"]:
                b.tensor.detach().copy_(self.arena[b.off: b.off + b.n].reshape(b.tensor.shape))

    def download(self):
        """Write every bound tensor (writeback=True) back into its original storage, in place.  Only the runs that hold
        write-back mirrors cross PCIe (a pass that leaves the weights alone does not fetch them)."""
        self.download_begin()
        self.download_end()

    def view(self, off: int, n: int) -> torch.Tensor:
        self._ensure_room()
        return self.arena[off: off + n]

    # ---- tables ------------------------------------------------------------------------------------
    def _layer_table(self, roles: Optional[Dict[int, dict]] = None) -> np.ndarray:
        t = np.zeros(len(self._layers), dtype=_lib.LAYER_DT)
        for i, l in enumerate(self._layers):
            t[i]["w_off"] = l["w_off"]; t[i]["bias_off"] = l["bias_off"]
            t[i]["rows"] = l["rows"]; t[i]["cols"] = l["cols"]; t[i]["kk"] = l["kk"]
            t[i]["rel_in"] = -1; t[i]["rel_out"] = -1; t[i]["col_mode"] = 0; t[i]["group"] = 0
            t[i]["cmin_off"] = -1; t[i]["cmax_off"] = -1
            if roles and i in roles:
                for k, v in roles[i].items():
                    t[i][k] = v
        return t

    def _ptr(self):
        return C.c_void_p(self.arena.data_ptr())

    # ---- BN fold --------------------------------------------------------------------------------------
    def plan_bn_fold(self, folds: Sequence[dict], cle_plan: Optional[dict] = None) -> dict:
        """cle_plan: the equalization plan that will run right after this fold.  The fold then also writes the column
        extrema of every folded `second` layer (it has each tile in shared memory anyway) and `plan["scanned"]` lists those
        layers: pass it to run_cle_plan(cols_ready=...) so that the equalization skips its initial 4 B/weight scan."""
        ft = np.zeros(len(folds), dtype=_lib.FOLD_DT)
        scanned = []
        for i, f in enumerate(folds):
            for k in ft.dtype.names:
                ft[i][k] = f.get(k, 0)
            if cle_plan is not None:
                ri = int(cle_plan["lt"][f["layer"]]["rel_in"])
                if ri >= 0:
                    ft[i]["scan_go"] = cle_plan["rt"][ri]["go"]; ft[i]["scan_gi"] = cle_plan["rt"][ri]["gi"]
                    scanned.append(int(f["layer"]))
        return dict(ft=ft, lt=cle_plan["lt"] if cle_plan is not None else self._layer_table(), scanned=scanned)

    def run_bn_fold(self, folds):
        """folds: dicts(layer, bn_eps, gamma_off, beta_off, mean_off, var_off, fake_w_off, fake_b_off), or a plan."""
        plan = folds if isinstance(folds, dict) else (self.plan_bn_fold(folds) if len(folds) else None)
        if plan is None:
            return
        self._ensure_room()
        ft, lt = plan["ft"], plan["lt"]
        _lib.check(self.lib.dfq_bn_fold(self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt),
                                        _lib.table_ptr(ft), len(ft), _lib.stream_ptr()), "dfq_bn_fold")

    # ---- cross-layer equalization -----------------------------------------------------------------
    def plan_cle(self, relations: Sequence[Tuple[int, int, int, int]], groups: Optional[Sequence[int]] = None) -> dict:
        """Build the descriptor tables + scratch for a list of relations
        (first_layer, second_layer, bn_w_off | -1, bn_b_off | -1) in processing order (dfq.py:85-86).

        groups[i] = convergence group (independent model) of relation i; default: one group, i.e. the reference's
        single-model exit rule.  All relations of a chain must share a group."""
        nR = len(relations)
        if groups is None:
            groups = [0] * nR
        n_groups = max(groups) + 1
        rel_in: Dict[int, int] = {}
        rel_out: Dict[int, int] = {}
        for i, (a, b, _, _) in enumerate(relations):
            if a in rel_out or b in rel_in:
                raise DfqError("a layer may be `first` of one relation and `second` of one relation only")
            rel_out[a] = i
            rel_in[b] = i
        for l in set(rel_in) & set(rel_out):
            if rel_in[l] > rel_out[l]:
                raise DfqError("relations must be in forward chain order (as utils.relation.create_relation emits)")
        rt = np.zeros(nR, dtype=_lib.RELATION_DT)
        # the accumulated scale vectors (Relation.S, the result a multi-GPU step exchanges) sit in ONE contiguous block
        s_offs = [self.alloc(self._layers[a]["rows"]) for (a, _, _, _) in relations]
        roles: Dict[int, dict] = {}
        for i, (a, b, bnw, bnb) in enumerate(relations):
            la, lb = self._layers[a], self._layers[b]
            C1, J2 = la["rows"], lb["cols"]
            G = 1 if C1 == J2 else C1 // max(J2, 1)              # dfq.py:29-32
            if G < 1 or G * J2 != C1 or lb["rows"] % G != 0:
                raise DfqError("unsupported relation shapes: first rows %d, second [%d, %d]" % (C1, lb["rows"], J2))
            r = rt[i]
            r["first"] = a; r["second"] = b; r["channels"] = C1; r["groups"] = G
            r["gi"] = C1 // G; r["go"] = lb["rows"] // G
            r["bn_w_off"] = bnw; r["bn_b_off"] = bnb
            r["s_acc_off"] = s_offs[i]; r["s_step_off"] = self.alloc(C1); r["inv_off"] = self.alloc(C1)
            roles.setdefault(a, {})["rel_out"] = i
            roles[a]["group"] = int(groups[i])
            rb = roles.setdefault(b, {})
            rb["rel_in"] = i
            rb["group"] = int(groups[i])
            rb["cmin_off"] = self.alloc(2 * C1); rb["cmax_off"] = self.alloc(2 * C1)
        for l, ro in roles.items():
            if "rel_in" in ro:
                if "rel_out" not in ro:
                    ro["col_mode"] = 0
                elif self._layers[l]["cols"] == 1 and rt[ro["rel_in"]]["go"] == 1:
                    ro["col_mode"] = 1
                else:
                    ro["col_mode"] = 2
        # chain position of every layer -> steps (forward order guarantees pos[first] is known)
        pos: Dict[int, int] = {}
        for a, b, _, _ in relations:
            if a not in pos:
                pos[a] = 0
            pos[b] = pos[a] + 1
        n_steps = max(pos.values()) + 1
        buckets: List[List[int]] = [[] for _ in range(n_steps)]
        for l in sorted(pos):
            buckets[pos[l]].append(l)
        step_ptr = np.zeros(n_steps + 1, dtype=np.int32)
        for p in range(n_steps):
            step_ptr[p + 1] = step_ptr[p] + len(buckets[p])
        step_layers = np.array([l for bk in buckets for l in bk], dtype=np.int32)
        return dict(rt=rt, lt=self._layer_table(roles), step_ptr=step_ptr, step_layers=step_layers, n_steps=n_steps,
                    s_offs=s_offs, relations=list(relations), n_groups=n_groups)

    def run_cle_plan(self, plan: dict, s_range=(1e-8, 1e8), converge_thres=2e-7, converge_count=20, signed=False,
                     eps=0, max_sweeps=0, apply_only=False, cols_ready: Optional[Sequence[int]] = None) -> CleResult:
        """Run dfq.py:78-117 on a planned relation list; see include/dfq_b200.h dfq_cle_run.
        cols_ready: layers whose column extrema (buffer 0) a fold planned with cle_plan=plan has JUST written."""
        self._ensure_room()
        lo, hi = float(s_range[0]), float(s_range[1])
        P = np.zeros(1, dtype=_lib.CLE_PARAMS_DT)
        P[0]["s_lo"] = np.float32(lo); P[0]["s_hi"] = np.float32(hi)
        with np.errstate(divide="ignore"):
            P[0]["inv_lo"] = np.float32(np.float64(1.0) / np.float64(lo)) if lo != 0 else np.float32(np.inf)
            P[0]["inv_hi"] = np.float32(np.float64(1.0) / np.float64(hi)) if hi != 0 else np.float32(np.inf)
        P[0]["eps"] = np.float32(eps); P[0]["signed_mode"] = 1 if signed else 0
        P[0]["converge_thres"] = float(converge_thres); P[0]["converge_count"] = int(converge_count)
        P[0]["max_sweeps"] = 1 if apply_only else int(max_sweeps)
        P[0]["apply_only"] = 1 if apply_only else 0
        R = np.zeros(1, dtype=_lib.CLE_RESULT_DT)
        lt, rt = plan["lt"], plan["rt"]
        if cols_ready:
            key = tuple(cols_ready)
            if plan.get("_ready_key") != key:
                lt2 = lt.copy()
                lt2["flags"][list(cols_ready)] |= _lib.LAYER_COLS_READY
                plan["_ready_key"], plan["_ready_lt"] = key, lt2
            lt = plan["_ready_lt"]
        gs = np.zeros(plan["n_groups"], dtype=np.int32)
        _lib.check(self.lib.dfq_cle_run(self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt),
                                        _lib.table_ptr(rt), len(rt), _lib.table_ptr(plan["step_ptr"]),
                                        _lib.table_ptr(plan["step_layers"]), plan["n_steps"], _lib.table_ptr(P),
                                        _lib.table_ptr(R), plan["n_groups"], _lib.table_ptr(gs), _lib.stream_ptr()),
                   "dfq_cle_run")
        n = int(R[0]["n_sweeps"])
        res = CleResult(n, bool(R[0]["converged"]), float(R[0]["last_diff"]), [float(x) for x in R[0]["diffs"][:min(n, 64)]])
        res.group_sweeps = gs
        res.apply_only = bool(apply_only)
        return res

    def cle_col_hints(self, plan: dict, res: CleResult) -> Optional[Dict[str, np.ndarray]]:
        """The column extrema dfq_cle_run left for every `second` layer of `plan` (the buffer of parity
        sweeps-of-its-group & 1), as parallel arrays dict(layer, colmin_off, colmax_off, n_col).  Valid until the weights
        change again; hand it to run_bias_correct_plan(col_hints=...) so that the per-tensor range of dfq.py:14 is reduced
        from C values instead of streaming the weights a second time."""
        if res is None or res.n_sweeps <= 0 or res.apply_only or res.group_sweeps is None:
            return None
        lt, rt = plan["lt"], plan["rt"]
        second = rt["second"].astype(np.int64)
        Cn = rt["channels"].astype(np.int64)
        par = (np.asarray(res.group_sweeps, dtype=np.int64)[lt["group"][second]] & 1)
        return dict(layer=second, colmin_off=lt["cmin_off"][second] + par * Cn, colmax_off=lt["cmax_off"][second] + par * Cn,
                    n_col=Cn)

    def run_cle(self, relations: Sequence[Tuple[int, int, int, int]], s_range=(1e-8, 1e8), converge_thres=2e-7,
                converge_count=20, signed=False, eps=0, max_sweeps=0) -> Tuple[CleResult, List[int]]:
        """plan_cle + run_cle_plan.  Returns (result, [s_acc offsets]); s_acc[i] holds Relation.S of relation i."""
        if len(relations) == 0:
            return CleResult(0, True, 10.0, []), []
        plan = self.plan_cle(relations)
        res = self.run_cle_plan(plan, s_range, converge_thres, converge_count, signed, eps, max_sweeps)
        return res, plan["s_offs"]

    # ---- bias correction ----------------------------------------------------------------------------
    def plan_bias_correct(self, items: Sequence[dict]) -> dict:
        """items (in graph order): dict(layer, signed, terms=[dict(bn_w_off, bn_b_off, n, relu, op)], next_bn_b_off,
        level[, raw_sum, add]) with op in {'set', 'cat', 'add'}."""
        bt = np.zeros(len(items), dtype=_lib.BC_LAYER_DT)
        terms = []
        order = sorted(range(len(items)), key=lambda i: (items[i]["level"], i))
        delta_offs = [0] * len(items)
        levels = []
        for slot, i in enumerate(order):
            it = items[i]
            l = self._layers[it["layer"]]
            b = bt[slot]
            b["layer"] = it["layer"]; b["signed_mode"] = 1 if it.get("signed") else 0
            b["flags"] = (1 if it.get("raw_sum") else 0) | (2 if it.get("add") else 0)
            b["term_begin"] = len(terms)
            length = 0
            for k, t in enumerate(it["terms"]):
                op = t["op"] if k else "set"
                if op in ("set", "cat"):
                    dst, acc = length, 0
                    length += t["n"]
                else:
                    if t["n"] != length:
                        raise DfqError("bias correction: summed expectations differ in length (%d vs %d)" % (t["n"], length))
                    dst, acc = 0, 1
                terms.append((t["bn_w_off"], t["bn_b_off"], t["n"], 1 if t["relu"] else 0, dst, acc))
            b["term_end"] = len(terms)
            if length == 0 or length % l["cols"] != 0:
                raise DfqError("bias correction: expectation length %d incompatible with %d input channels" % (length, l["cols"]))
            b["expect_len"] = length
            b["expect_off"] = self.alloc(length)
            b["delta_off"] = self.alloc(l["rows"])
            b["minmax_off"] = self.alloc(2)
            b["next_bn_b_off"] = it.get("next_bn_b_off", -1)
            delta_offs[i] = int(b["delta_off"])
            levels.append(it["level"])
        tt = np.zeros(max(1, len(terms)), dtype=_lib.TERM_DT)
        for k, t in enumerate(terms):
            tt[k] = t
        uniq = sorted(set(levels))
        level_ptr = np.zeros(len(uniq) + 1, dtype=np.int32)
        for k, lv in enumerate(uniq):
            level_ptr[k + 1] = level_ptr[k] + sum(1 for x in levels if x == lv)
        return dict(bt=bt, tt=tt, n_terms=len(terms), level_ptr=level_ptr, n_levels=len(uniq), delta_offs=delta_offs,
                    lt=self._layer_table())

    def run_bias_correct_plan(self, plan: dict, num_bits: int = 8, col_hints: Optional[Dict[str, np.ndarray]] = None):
        """col_hints: see cle_col_hints (only meaningful for the layers' CURRENT weights)."""
        self._ensure_room()
        lt, bt, tt = plan["lt"], plan["bt"], plan["tt"]
        if col_hints is not None and len(col_hints["layer"]):
            bt = bt.copy()
            lut = np.full(len(lt), -1, dtype=np.int64)
            lut[col_hints["layer"]] = np.arange(len(col_hints["layer"]))
            k = lut[bt["layer"]]
            m = (k >= 0) & ((bt["flags"] & 1) == 0)          # bias absorption (raw sums) needs no range at all
            for name in ("colmin_off", "colmax_off", "n_col"):
                col = bt[name]
                col[m] = col_hints[name][k[m]]
        _lib.check(self.lib.dfq_bias_correct(self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt),
                                             _lib.table_ptr(bt), len(bt), _lib.table_ptr(tt), plan["n_terms"],
                                             _lib.table_ptr(plan["level_ptr"]), plan["n_levels"], int(num_bits),
                                             _lib.stream_ptr()), "dfq_bias_correct")

    def run_bias_correct(self, items: Sequence[dict], num_bits: int = 8):
        """plan + run; returns the list of delta offsets ([rows] each), in the order of `items`."""
        if not items:
            return []
        plan = self.plan_bias_correct(items)
        self.run_bias_correct_plan(plan, num_bits)
        return plan["delta_offs"]

    # ---- weight / bias fake quantization ---------------------------------------------------------
    def plan_quantize(self, tasks: Sequence[Tuple[int, int, int, bool]]) -> dict:
        qt = np.zeros(len(tasks), dtype=_lib.QUANT_TASK_DT)
        for i, (off, n, bits, sym) in enumerate(tasks):
            qt[i]["off"] = off; qt[i]["n"] = n; qt[i]["num_bits"] = bits; qt[i]["symmetric"] = 1 if sym else 0
            qt[i]["minmax_off"] = self.alloc(2)
        return dict(qt=qt)

    def run_quantize(self, tasks: Sequence[Tuple[int, int, int, bool]], div_mode: int = 0):
        """tasks: (offset, n, num_bits, symmetric); per-tensor min/max then in-place fake-quant.
        div_mode 0 = true division (what the reference computes on CPU-resident parameters), 1 = multiply by
        the fp32 reciprocal (what PyTorch CUDA eager computes)."""
        if isinstance(tasks, dict):
            qt = tasks["qt"]
        else:
            if not tasks:
                return
            qt = self.plan_quantize(tasks)["qt"]
        self._ensure_room()
        _lib.check(self.lib.dfq_quantize_tensors(self._ptr(), self.arena.numel(), _lib.table_ptr(qt), len(qt),
                                                 int(div_mode), _lib.stream_ptr()), "dfq_quantize_tensors")
