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

_PIN = True       # page-locked staging buffers (tests that run the host logic without a GPU turn this off)


def _default_device() -> torch.device:
    return torch.device("cuda", torch.cuda.current_device())


# Rows of each `first` layer whose extrema a deferred fold scans (plan_bn_fold); DFQ_ROW_PREFIX overrides it, 0 = every row.
ROW_PREFIX = 16


def row_prefix() -> int:
    return max(0, int(os.environ.get("DFQ_ROW_PREFIX", ROW_PREFIX)))


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
    fused_sweeps: int = 0    # 2: k_cle_stack applied the first two sweeps in one pass (plan_bn_fold's row scan), else 0
    bc_prepared: bool = False  # the correction attached to the plan (plan_bias_correct(cle_plan=...)) was computed in that pass
    rows_streamed: int = 0   # _lib.ROWS_*: how k_cle_stack completed the row extrema of a prefix scan (plan_bn_fold)


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
        self._pending = None        # a fold plan whose weight pass was deferred into the equalization (plan_bn_fold)
        self._bc_ready = None       # (correction plan, num_bits) whose deltas the last equalization computed (plan_bias_correct)

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

    def _host_copy(self, x: dict, which: str, direction: int) -> bool:
        """Gather (0) / scatter (1) between the bound host tensors and the staging image with the library's
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
        for i, b in enumerate(bounds):
            t = b.tensor
            if t.dtype != torch.float32 or t.numel() != b.n or not t.is_contiguous() or t.is_cuda:
                return False
            ptrs[i] = t.data_ptr()
        # (last argument 0: the library's default number of copy threads)
        _lib.check(fn(C.c_void_p(self._staging.data_ptr()), _lib.table_ptr(ptrs), _lib.table_ptr(nbytes), _lib.table_ptr(offs),
                      len(bounds), direction, 0), "dfq_host_copy_segments")
        return True

    def upload(self):
        """Copy every bound tensor into the arena: host tensors through ONE pinned staging buffer and one H2D copy per
        run of adjacent mirrors, device tensors with device-to-device copies."""
        self._ensure_room()
        self.finish_fold()
        x = self._transfer_lists()
        with torch.no_grad():
            if x["h2d_bounds"]:
                lo, st = x["lo"], self._staging
                # (the sources are looked up per call: a caller may have re-pointed a parameter's .data since the last one)
                if not self._host_copy(x, "h2d", 0):
                    torch._foreach_copy_(x["h2d_dst"], [b.tensor.detach().reshape(-1) for b in x["h2d_bounds"]])
                for a, e in x["h2d_runs"]:
                    self.arena[a:e].copy_(st[a - lo: e - lo], non_blocking=True)
                    self.h2d_bytes += 4 * (e - a)
            for b in x["dev_up"]:
                self.arena[b.off: b.off + b.n].copy_(b.tensor.detach().reshape(-1))

    def download_begin(self):
        """Enqueue the device-to-host copies of every write-back run (asynchronous; host work that does not read the results
        can overlap them).  download_end() waits and writes the tensors."""
        self.finish_fold()
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
        self.finish_fold()
        return self.arena[off: off + n]

    # ---- tables ------------------------------------------------------------------------------------
    def _layer_table(self, roles: Optional[Dict[int, dict]] = None) -> np.ndarray:
        t = np.zeros(len(self._layers), dtype=_lib.LAYER_DT)
        for i, l in enumerate(self._layers):
            t[i]["w_off"] = l["w_off"]; t[i]["bias_off"] = l["bias_off"]
            t[i]["rows"] = l["rows"]; t[i]["cols"] = l["cols"]; t[i]["kk"] = l["kk"]
            t[i]["rel_in"] = -1; t[i]["rel_out"] = -1; t[i]["col_mode"] = 0; t[i]["group"] = 0
            t[i]["cmin_off"] = -1; t[i]["cmax_off"] = -1; t[i]["fold_off"] = -1; t[i]["rext_off"] = -1
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
        layers: pass it to run_cle_plan(cols_ready=...) so that the equalization skips its initial 4 B/weight scan.

        When the library reports that cle_plan runs on the stack kernel (dfq_cle_takes_stack), the fold of the plan's layers
        is DEFERRED: run_bn_fold does the [rows]-vector work and a read-only scan of the `second` layers, and the
        equalization's first sweep multiplies every row by its fold factor as it reads it - one read-write pass over the
        weights fewer.  Until run_cle_plan(cle_plan) has run, every other call of this session that touches the arena
        completes the fold first (finish_fold), so nothing ever sees unfolded weights.

        A deferred fold also reads the plan's `first` layers and writes their row extrema (`plan["rows_scanned"]`: pairs
        (layer, offset of its [2][rows] scratch)).  With those and the column extrema, the stack kernel knows the scales of
        the first two sweeps before it reads a weight and, where its guard allows, applies both in one pass.

        Only the first row_prefix() rows of each first layer are scanned (`plan["row_prefix"]`, 0 = all): their bound on
        the first sweep's metric is enough for the stack kernel's guard on ordinary weights, and the fused pass finds the
        other rows' extrema in the rows it holds anyway.  Where the prefix does not decide, the kernel scans the rest
        itself; either way the scratch and the results are those of a full scan."""
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
        deferred, rows_scanned = [], []
        prefix = row_prefix()
        lt = cle_plan["lt"] if cle_plan is not None else self._layer_table()
        if cle_plan is not None and self._takes_stack(cle_plan, scanned):
            in_plan = set(int(x) for x in cle_plan["step_layers"])
            for i, f in enumerate(folds):
                li = int(f["layer"])
                if li in in_plan:
                    ft[i]["mode"] = _lib.FOLD_DEFER
                    ft[i]["fac_off"] = self.alloc(self._layers[li]["rows"])
                    deferred.append((li, int(ft[i]["fac_off"])))
                    if lt[li]["rel_out"] >= 0 and lt[li]["rel_in"] < 0:
                        ft[i]["scan_rows"] = 1
                        ft[i]["row_prefix"] = prefix
                        rows_scanned.append((li, self.alloc(2 * self._layers[li]["rows"])))
            if rows_scanned:
                lt = lt.copy()
                lt["rext_off"][[r[0] for r in rows_scanned]] = [r[1] for r in rows_scanned]
        return dict(ft=ft, lt=lt, scanned=scanned, deferred=deferred, rows_scanned=rows_scanned, row_prefix=prefix,
                    cle_plan=cle_plan)

    def _takes_stack(self, cle_plan: dict, cols_ready: Sequence[int]) -> bool:
        """Whether dfq_cle_run will take `cle_plan` (with these layers' column extrema ready) on the stack kernel - the
        library's own decision.  A library without the query (a test stand-in) never defers."""
        fn = getattr(self.lib, "dfq_cle_takes_stack", None)
        if fn is None:
            return False
        lt = cle_plan["lt"].copy()
        if cols_ready:
            lt["flags"][list(cols_ready)] |= _lib.LAYER_COLS_READY
        return self._takes_stack_lt(cle_plan, lt)

    def _takes_stack_lt(self, cle_plan: dict, lt: np.ndarray) -> bool:
        fn = getattr(self.lib, "dfq_cle_takes_stack", None)
        if fn is None:
            return False
        takes = np.zeros(1, dtype=np.int32)
        _lib.check(fn(_lib.table_ptr(lt), len(lt), _lib.table_ptr(cle_plan["rt"]), len(cle_plan["rt"]),
                      _lib.table_ptr(cle_plan["step_ptr"]), _lib.table_ptr(cle_plan["step_layers"]), cle_plan["n_steps"], 0,
                      _lib.table_ptr(takes)), "dfq_cle_takes_stack")
        return bool(takes[0])

    def run_bn_fold(self, folds):
        """folds: dicts(layer, bn_eps, gamma_off, beta_off, mean_off, var_off, fake_w_off, fake_b_off), or a plan."""
        plan = folds if isinstance(folds, dict) else (self.plan_bn_fold(folds) if len(folds) else None)
        if plan is None:
            return
        self._ensure_room()
        self.finish_fold()
        ft, lt = plan["ft"], plan["lt"]
        _lib.check(self.lib.dfq_bn_fold(self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt),
                                        _lib.table_ptr(ft), len(ft), _lib.stream_ptr()), "dfq_bn_fold")
        if plan.get("deferred"):
            self._pending = plan

    @property
    def fold_pending(self) -> bool:
        """A deferred fold's weight pass is still outstanding (see plan_bn_fold)."""
        return self._pending is not None

    def finish_fold(self):
        """Complete a deferred fold now: W[o,:] *= its stored factor (one read-write pass over the deferred layers).
        Every session call that touches the arena runs this first; it also forgets a prepared correction (plan_bias_correct),
        whose deltas may no longer be those of the weights."""
        self._bc_ready = None
        plan, self._pending = self._pending, None
        if plan is None:
            return
        ft = np.zeros(len(plan["deferred"]), dtype=_lib.FOLD_DT)
        for k, (li, fac_off) in enumerate(plan["deferred"]):
            ft[k]["layer"] = li; ft[k]["mode"] = _lib.FOLD_APPLY; ft[k]["fac_off"] = fac_off
        lt = plan["lt"]
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
        cols_ready: layers whose column extrema (buffer 0) a fold planned with cle_plan=plan has JUST written.
        A fold planned with cle_plan=plan and deferred (plan_bn_fold) is completed by this call.
        A bias correction attached to plan (plan_bias_correct(cle_plan=plan)) is computed in the same pass when the stack
        kernel runs it; CleResult.bc_prepared says whether its deltas are those of the final weights."""
        self._ensure_room()
        self._bc_ready = None
        pending = self._pending
        if pending is not None and pending["cle_plan"] is not plan:
            self.finish_fold()
            pending = None
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
        if pending is not None:
            # the deferred layers are marked FOLD_PENDING: the stack kernel folds them in its first sweep, any other path of
            # dfq_cle_run applies the fold before it starts
            # the first layers whose row extrema the fold scanned are marked ROWS_READY
            key = (id(lt), tuple(pending["deferred"]), tuple(pending["rows_scanned"]))
            if pending.get("_pending_key") != key:
                lt2 = lt.copy()
                li = [d[0] for d in pending["deferred"]]
                lt2["flags"][li] |= _lib.LAYER_FOLD_PENDING
                lt2["fold_off"][li] = [d[1] for d in pending["deferred"]]
                if pending["rows_scanned"]:
                    li = [d[0] for d in pending["rows_scanned"]]
                    lt2["flags"][li] |= _lib.LAYER_ROWS_READY
                    lt2["rext_off"][li] = [d[1] for d in pending["rows_scanned"]]
                    lt2["rext_rows"][li] = pending.get("row_prefix", 0)
                pending["_pending_key"], pending["_pending_lt"], pending["_pending_base"] = key, lt2, lt
            lt = pending["_pending_lt"]
        gs = np.zeros(plan["n_groups"], dtype=np.int32)
        # the attached correction goes along only where the library accepts it: on the stack kernel (a library without
        # dfq_cle_run_bc - a test stand-in - never gets it)
        att = plan.get("bc")
        run_bc = getattr(self.lib, "dfq_cle_run_bc", None)
        if att is not None and (run_bc is None or apply_only or not self._takes_stack_lt(plan, lt)):
            att = None
        args = (self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt), _lib.table_ptr(rt), len(rt),
                _lib.table_ptr(plan["step_ptr"]), _lib.table_ptr(plan["step_layers"]), plan["n_steps"], _lib.table_ptr(P),
                _lib.table_ptr(R), plan["n_groups"], _lib.table_ptr(gs))
        if att is not None:
            _lib.check(run_bc(*args, _lib.table_ptr(att["plan"]["bt"]), len(att["plan"]["bt"]), _lib.table_ptr(att["plan"]["tt"]),
                              att["plan"]["n_terms"], int(att["num_bits"]), _lib.stream_ptr()), "dfq_cle_run_bc")
        else:
            _lib.check(self.lib.dfq_cle_run(*args, _lib.stream_ptr()), "dfq_cle_run")
        if pending is not None:
            self._pending = None
        n = int(R[0]["n_sweeps"])
        res = CleResult(n, bool(R[0]["converged"]), float(R[0]["last_diff"]), [float(x) for x in R[0]["diffs"][:min(n, 64)]])
        res.group_sweeps = gs
        res.apply_only = bool(apply_only)
        res.fused_sweeps = int(R[0]["fused_sweeps"])
        res.rows_streamed = int(R[0]["rows_streamed"])
        res.bc_prepared = att is not None and bool(R[0]["bc_prepared"])
        if res.bc_prepared:
            self._bc_ready = (att["plan"], int(att["num_bits"]))
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
    def plan_bias_correct(self, items: Sequence[dict], cle_plan: Optional[dict] = None, num_bits: int = 8) -> dict:
        """items (in graph order): dict(layer, signed, terms=[dict(bn_w_off, bn_b_off, n, relu, op)], next_bn_b_off,
        level[, raw_sum, add]) with op in {'set', 'cat', 'add'}.

        cle_plan: the equalization plan that runs right before this correction.  When the correction is one the stack
        kernel can compute in its fused pass (one level; every item the `second` layer of one of cle_plan's relations, once;
        no raw sums or added deltas; an expectation as long as the layer's input), it is attached to cle_plan
        (`plan["attached"]`): run_cle_plan(cle_plan) then computes the deltas from the rows it holds anyway, and a
        run_bias_correct_plan(plan, num_bits, col_hints=...) right after it only retires them - no second read of the
        weights.  Anything else in between (any session call that touches the arena), another num_bits, no col_hints or an
        equalization that did not stop after two fused sweeps: the full correction runs, as without cle_plan."""
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
        plan = dict(bt=bt, tt=tt, n_terms=len(terms), level_ptr=level_ptr, n_levels=len(uniq), delta_offs=delta_offs,
                    lt=self._layer_table(), attached=False)
        if cle_plan is not None and self._bc_attachable(bt, len(uniq), cle_plan):
            cle_plan["bc"] = dict(plan=plan, num_bits=int(num_bits))
            plan["attached"] = True
        return plan

    def _bc_attachable(self, bt: np.ndarray, n_levels: int, cle_plan: dict) -> bool:
        """dfq_cle_run's conditions on an attached correction (include/dfq_b200.h), checked on the host."""
        lt = cle_plan["lt"]
        layers = bt["layer"].astype(np.int64)
        return (n_levels == 1 and len(bt) > 0 and not bt["flags"].any() and len(set(layers.tolist())) == len(layers)
                and bool(np.all(lt["rel_in"][layers] >= 0)) and bool(np.all(lt["rel_out"][layers] < 0))
                and bool(np.all(bt["expect_len"] == lt["cols"][layers])))

    def run_bias_correct_plan(self, plan: dict, num_bits: int = 8, col_hints: Optional[Dict[str, np.ndarray]] = None):
        """col_hints: see cle_col_hints (only meaningful for the layers' CURRENT weights).
        Right after the run_cle_plan that computed this plan's correction (plan_bias_correct(cle_plan=...)) at this
        num_bits, with col_hints (the range that run reduced), only the deltas are retired."""
        self._ensure_room()
        ready = self._bc_ready
        self.finish_fold()
        lt, bt, tt = plan["lt"], plan["bt"], plan["tt"]
        if ready is not None and ready[0] is plan and ready[1] == int(num_bits) and col_hints is not None:
            bt = bt.copy()
            bt["flags"] |= _lib.BC_PREPARED
        else:
            bt = self._with_col_hints(lt, bt, col_hints)
        _lib.check(self.lib.dfq_bias_correct(self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt),
                                             _lib.table_ptr(bt), len(bt), _lib.table_ptr(tt), plan["n_terms"],
                                             _lib.table_ptr(plan["level_ptr"]), plan["n_levels"], int(num_bits),
                                             _lib.stream_ptr()), "dfq_bias_correct")

    @staticmethod
    def _with_col_hints(lt: np.ndarray, bt: np.ndarray, col_hints: Optional[Dict[str, np.ndarray]]) -> np.ndarray:
        if col_hints is None or not len(col_hints["layer"]):
            return bt
        bt = bt.copy()
        lut = np.full(len(lt), -1, dtype=np.int64)
        lut[col_hints["layer"]] = np.arange(len(col_hints["layer"]))
        k = lut[bt["layer"]]
        m = (k >= 0) & ((bt["flags"] & 1) == 0)          # bias absorption (raw sums) needs no range at all
        for name in ("colmin_off", "colmax_off", "n_col"):
            col = bt[name]
            col[m] = col_hints[name][k[m]]
        return bt

    # ---- bias absorption and weight clipping inside the correction --------------------------------------------------
    def plan_absorb(self, relations: Sequence[Tuple[int, int, int, int]]) -> np.ndarray:
        """relations: (first_layer, second_layer, bn_w_off, bn_b_off) of every relation that absorbs (dfq.py:121-164), in
        the order of the relation list.  Reserves each one's c vector; returns the DfqAbsorb table."""
        at = np.zeros(len(relations), dtype=_lib.ABSORB_DT)
        for i, (a, b, bnw, bnb) in enumerate(relations):
            n = self._layers[a]["rows"]
            at[i]["first"] = a; at[i]["second"] = b; at[i]["n"] = n
            at[i]["bn_w_off"] = bnw; at[i]["bn_b_off"] = bnb; at[i]["c_off"] = self.alloc(n)
        return at

    def run_bias_correct_absorb_clip(self, plan: Optional[dict], num_bits: int = 8,
                                     col_hints: Optional[Dict[str, np.ndarray]] = None, absorb: Optional[np.ndarray] = None,
                                     absorb_n: float = 3, clip: Optional[Tuple[float, float]] = None):
        """dfq_bias_correct_absorb_clip: bias absorption (absorb: plan_absorb's table, factor absorb_n) and weight clipping
        (clip: (lo, hi), every layer of the session) inside the correction `plan` (plan_bias_correct; None: no correction -
        the clip alone, or a plan of raw-sum entries that is the absorption itself).  The weights of `plan` are read once."""
        self._ensure_room()
        self.finish_fold()
        lt = plan["lt"] if plan is not None else self._layer_table()
        at = absorb if absorb is not None and len(absorb) else np.zeros(1, dtype=_lib.ABSORB_DT)
        n_abs = len(absorb) if absorb is not None else 0
        if plan is not None:
            bt, tt, n_terms, lp, n_levels = self._with_col_hints(lt, plan["bt"], col_hints), plan["tt"], plan["n_terms"], \
                plan["level_ptr"], plan["n_levels"]
        else:
            bt, tt, n_terms = np.zeros(1, dtype=_lib.BC_LAYER_DT), np.zeros(1, dtype=_lib.TERM_DT), 0
            lp, n_levels = np.zeros(1, dtype=np.int32), 0
        lo, hi = (float(clip[0]), float(clip[1])) if clip is not None else (0.0, 0.0)
        _lib.check(self.lib.dfq_bias_correct_absorb_clip(
            self._ptr(), self.arena.numel(), _lib.table_ptr(lt), len(lt), _lib.table_ptr(bt), len(plan["bt"]) if plan else 0,
            _lib.table_ptr(tt), n_terms, _lib.table_ptr(lp), n_levels, int(num_bits), _lib.table_ptr(at), n_abs,
            float(absorb_n), 1 if clip is not None else 0, lo, hi, _lib.stream_ptr()), "dfq_bias_correct_absorb_clip")

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
        self.finish_fold()
        _lib.check(self.lib.dfq_quantize_tensors(self._ptr(), self.arena.numel(), _lib.table_ptr(qt), len(qt),
                                                 int(div_mode), _lib.stream_ptr()), "dfq_quantize_tensors")
