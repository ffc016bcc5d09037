"""Whole-model calibration in ONE arena residency: the GPU-native way to run the path.

The reference's drivers call merge_batchnorm / cross_layer_equalization / bias_correction / quantize_targ_layer one
after the other on CPU-resident parameters (main_cls.py:144-180); the drop-in functions of this package mirror that and
therefore stage the model to the GPU and back once per call.  `GraphCalibration` plans all requested passes over a
graph once, stages the model ONCE (one pinned H2D copy), runs 3-4 kernel launches and writes everything back ONCE:

    cal = GraphCalibration(graph, bottoms, [nn.Conv2d, nn.Linear])      # BN fold + create_relation + recipes
    cal.run(equalize=True, correction=True, quantize_bits=(8, 16))      # same results as the four separate calls
    cal.relations                                                        # utils.relation.Relation objects with .S set

Semantics are those of the separate calls in the reference's order (fold -> equalize -> absorb -> clip -> correct ->
quantize, main_cls.py:149-181); it is exercised against them in tests/test_gpu_pipeline.py and
tests/test_gpu_calibrate_absorb_clip.py.  The mains' --absorption and --clip_weight flags:

    cal.run(equalize=True, absorption=True, clip_weight=(-15, 15), correction=True, quantize_bits=(8, 16))

run inside the same residency: the absorption vectors are formed on the device, and the correction reads each weight row
once to add its absorption dot, clamp it and take its quantization error (dfq_bias_correct_absorb_clip).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn

from ._lib import DfqError
from .engine import CleResult, Session
from .graphwalk import bias_correction_recipe, relu_between
from .utils.layer_transform import _identity_bn_eps
from .utils.relation import create_relation


class GraphCalibration:
    def __init__(self, graph, bottoms, targ_type, bn_type=nn.BatchNorm2d, delete_single: bool = False, fold: bool = True,
                 device=None):
        self.graph, self.bottoms, self.targ_type, self.bn_type = graph, bottoms, list(targ_type), bn_type
        self.sess = Session(device)
        sess = self.sess
        self._layer = {}          # graph key -> session layer index
        self._bn = {}             # graph key -> dict of vector offsets
        self.fold_pairs: List[Tuple[object, object]] = []
        with torch.no_grad():
            # ---- layers and BN vectors --------------------------------------------------------------------------
            for key in graph:
                mod = graph[key]
                if type(mod) in self.targ_type:
                    if mod.bias is None:          # every pass of the path may create it (dfq.py:91-92, layer_transform.py:253)
                        mod.bias = nn.Parameter(torch.zeros(mod.weight.size(0), dtype=torch.float32, device=mod.weight.device),
                                                requires_grad=False)
                    self._layer[key] = sess.add_layer(mod.weight, mod.bias)
            folds = []
            if fold:
                for key in graph:
                    if bottoms[key] is None or type(graph[key]) != nn.BatchNorm2d:
                        continue
                    for src in bottoms[key]:
                        if type(graph[src]) in self.targ_type:
                            bn = graph[key]
                            n = bn.num_features
                            # fake_weight / fake_bias: output-only mirrors of buffers registered on the BN right here, so
                            # that they come back inside the ONE device-to-host copy of download()
                            if not hasattr(bn, "fake_weight"):
                                bn.register_buffer("fake_weight", torch.zeros(n, device=bn.weight.device))
                                bn.register_buffer("fake_bias", torch.zeros(n, device=bn.weight.device))
                            v = dict(gamma=sess.bind(bn.weight.detach(), False), beta=sess.bind(bn.bias.detach(), False),
                                     mean=sess.bind(bn.running_mean, False), var=sess.bind(bn.running_var, False),
                                     fake_w=sess.bind(bn.fake_weight, True, upload=False),
                                     fake_b=sess.bind(bn.fake_bias, True, upload=False), n=n, folded=True)
                            self._bn[key] = v
                            self.fold_pairs.append((key, src))
                            folds.append(dict(layer=self._layer[src], bn_eps=bn.eps, gamma_off=v["gamma"], beta_off=v["beta"],
                                              mean_off=v["mean"], var_off=v["var"], fake_w_off=v["fake_w"], fake_b_off=v["fake_b"]))
                            break
            else:
                for key in graph:
                    bn = graph[key]
                    if type(bn) == bn_type and hasattr(bn, "fake_weight"):
                        self._bn[key] = dict(fake_w=sess.bind(bn.fake_weight), fake_b=sess.bind(bn.fake_bias), n=bn.fake_bias.numel())
            self._fold_plan = sess.plan_bn_fold(folds) if folds else None
            # ---- equalization plan ---------------------------------------------------------------------------------
            self.relations = create_relation(graph, bottoms, self.targ_type, delete_single=delete_single)
            table = []
            for rr in self.relations:
                a, b, bn_key = rr.get_idxs()
                v = self._bn[bn_key]
                table.append((self._layer[a], self._layer[b], v["fake_w"], v["fake_b"]))
            self._cle_plan = sess.plan_cle(table) if table else None
            # Relation.S comes back the same way: the accumulated scale vectors are mirrored into host tensors
            self._S_host = []
            if self._cle_plan is not None:
                for off, t in zip(self._cle_plan["s_offs"], table):
                    n = sess.layer(t[0])["rows"]
                    first = self.relations[len(self._S_host)].get_idxs()[0]
                    h = torch.zeros(n, dtype=torch.float32, device=graph[first].weight.device)
                    sess.mirror(off, h)
                    self._S_host.append(h)
            # the fold that precedes an equalization also fills the column extrema the equalization starts from
            self._fold_plan_scan = sess.plan_bn_fold(folds, cle_plan=self._cle_plan) if (folds and self._cle_plan) else None
            # ---- bias correction plan ----------------------------------------------------------------------------------
            items = []
            for step in bias_correction_recipe(graph, bottoms, self.targ_type, bn_type):
                terms = [dict(bn_w_off=self._bn[t["bn"]]["fake_w"], bn_b_off=self._bn[t["bn"]]["fake_b"], n=self._bn[t["bn"]]["n"],
                              relu=t["relu"], op=t["op"]) for t in step["terms"]]
                nxt = self._bn[step["next_bn"]]["fake_b"] if step["next_bn"] is not None else -1
                items.append(dict(layer=self._layer[step["layer"]], signed=False, level=step["level"], next_bn_b_off=nxt, terms=terms))
            self._bc_items = items
            self._bc_plan = sess.plan_bias_correct(items) if items else None
            self._quant_plan = None
            self._quant_bits = None
            self._absorb = None       # plan_absorb's table, planned on the first run that absorbs
            self._absorb_raw = None   # the absorption alone as raw-sum correction entries (runs without the correction)
        self.last_cle: Optional[CleResult] = None

    @staticmethod
    def _check_flags(absorption_n, clip_weight):
        """The refusals of absorption_n and clip_weight, before anything is planned or launched."""
        try:
            n = float(absorption_n)
        except (TypeError, ValueError):
            raise DfqError("absorption_n must be a number, got %r" % (absorption_n,)) from None
        with np.errstate(over="ignore"):             # the library takes N as a float32: beyond its range it is inf
            if not (math.isfinite(n) and np.isfinite(np.float32(n))):
                raise DfqError("absorption_n must be finite in float32, got %r" % (absorption_n,))
        if clip_weight is not None:
            try:
                lo, hi = (float(v) for v in clip_weight)
            except (TypeError, ValueError):
                raise DfqError("clip_weight must be a (lo, hi) pair of numbers, got %r" % (clip_weight,)) from None
            with np.errstate(over="ignore"):         # a bound beyond float32 becomes inf: refused like inf itself
                lo, hi = np.float32(lo), np.float32(hi)
            if not (np.isfinite(lo) and np.isfinite(hi) and lo <= hi):
                raise DfqError("clip_weight must be two finite numbers with lo <= hi, got %r" % (clip_weight,))

    def plan_absorption(self):
        """Plan the absorption: which relations absorb (a torch.nn.ReLU between the layers, dfq.py:123-130) and their c
        vectors.  run() does it before its upload.  A caller that drives upload() / run_device() / download() itself calls it
        before upload(): planned later, the first run_device(absorption=True) grows the arena on the device."""
        if self._absorb is not None:
            return
        table, items = [], []
        for rr in self.relations:
            a, b, bn_key = rr.get_idxs()
            if relu_between(self.graph, self.bottoms, b, a):
                v = self._bn[bn_key]
                table.append((self._layer[a], self._layer[b], v["fake_w"], v["fake_b"]))
        self._absorb = self.sess.plan_absorb(table)
        for t in self._absorb:        # without the correction: (sum_k W) . c added to the bias (dfq.py:150-153,164)
            c = int(t["c_off"])
            items.append(dict(layer=int(t["second"]), signed=False, level=0, next_bn_b_off=-1, raw_sum=True, add=True,
                              terms=[dict(bn_w_off=c, bn_b_off=c, n=int(t["n"]), relu=False, op="set")]))
        self._absorb_raw = self.sess.plan_bias_correct(items) if items else None

    # -- device-resident pieces (bench: time them separately) -----------------------------------------------------------
    def upload(self):
        """Stage the model in the arena (one H2D copy).  To absorb in the runs that follow, plan_absorption() first."""
        self.sess.upload()

    def run_device(self, equalize=True, correction=True, quantize_bits: Optional[Tuple[int, int]] = None, signed=False,
                   s_range=(1e-8, 1e8), converge_thres=2e-7, converge_count=20, eps=0, absorption=False, absorption_n=3,
                   clip_weight: Optional[Tuple[float, float]] = None):
        """absorption: bias_absorption(relations, bottoms, absorption_n) after the equalization (dfq.py:121-164);
        clip_weight: (lo, hi), clip_weight(graph, [lo, hi], targ) after it (dfq.py:167-170).  Both run inside the
        correction's pass over the weights; neither adds a transfer or a host synchronisation."""
        self._check_flags(absorption_n, clip_weight)
        if absorption:
            self.plan_absorption()
        sess = self.sess
        run_cle = equalize and self._cle_plan is not None
        scan = run_cle and self._fold_plan_scan is not None
        if self._fold_plan is not None:
            sess.run_bn_fold(self._fold_plan_scan if scan else self._fold_plan)
        hints = None
        if run_cle:
            self.last_cle = sess.run_cle_plan(self._cle_plan, s_range, converge_thres, converge_count, signed, eps,
                                              cols_ready=self._fold_plan_scan["scanned"] if scan else None)
            hints = sess.cle_col_hints(self._cle_plan, self.last_cle)   # weights stay untouched until the correction
        absorb = self._absorb if absorption and len(self._absorb) else None
        clip = tuple(clip_weight) if clip_weight is not None else None
        if correction and self._bc_plan is not None:
            if any(it["signed"] != bool(signed) for it in self._bc_items):    # every run sets the mode: replan on a change
                for it in self._bc_items:
                    it["signed"] = bool(signed)
                self._bc_plan = sess.plan_bias_correct(self._bc_items)
            if absorb is not None or clip is not None:
                sess.run_bias_correct_absorb_clip(self._bc_plan, 8, col_hints=hints, absorb=absorb, absorb_n=absorption_n,
                                                  clip=clip)
            else:
                sess.run_bias_correct_plan(self._bc_plan, 8, col_hints=hints)      # quirk Q2: always 8 bits (dfq.py:218)
        elif absorb is not None or clip is not None:
            sess.run_bias_correct_absorb_clip(self._absorb_raw if absorb is not None else None, 8, absorb=absorb,
                                              absorb_n=absorption_n, clip=clip)
        if quantize_bits is not None:
            if self._quant_plan is None or self._quant_bits != tuple(quantize_bits):
                bw, bb = quantize_bits
                tasks = []
                for key, li in self._layer.items():
                    l = sess.layer(li)
                    tasks.append((l["w_off"], l["rows"] * l["cols"] * l["kk"], bw, False))
                    if bb < 32:
                        tasks.append((l["bias_off"], l["rows"], bb, False))
                self._quant_plan = sess.plan_quantize(tasks)
                self._quant_bits = tuple(quantize_bits)
            on_cuda = next(iter(self._layer)) is not None and self.graph[next(iter(self._layer))].weight.is_cuda
            sess.run_quantize(self._quant_plan, div_mode=1 if on_cuda else 0)

    def download(self):
        sess = self.sess
        with torch.no_grad():
            sess.download_begin()    # weights, biases, fake_weight / fake_bias and the scale vectors: one D2H copy ...
            eps = _identity_bn_eps()
            folded = [self.graph[key] for key, v in self._bn.items() if v.get("folded")]
            if folded:      # identity BN (layer_transform.py:268-272): four batched fills instead of four per layer
                ones = [bn.weight.detach() for bn in folded] + [bn.running_var for bn in folded]
                torch._foreach_zero_(ones + [bn.bias.detach() for bn in folded] + [bn.running_mean for bn in folded])
                torch._foreach_add_(ones, 1.0)
                for bn in folded:
                    bn.eps = eps
            sess.download_end()      # ... that crosses PCIe while the identity fills above run on the host
            if self._cle_plan is not None and self.last_cle is not None:
                for rr, s in zip(self.relations, self._S_host):
                    rr.S = None
                    rr.set_scale_vec(s.clone())

    def run(self, **kw):
        """upload -> fold/equalize/[absorb/clip]/correct/quantize on the device -> download (results in place in the modules).
        Keywords: those of run_device."""
        self._check_flags(kw.get("absorption_n", 3), kw.get("clip_weight"))
        if kw.get("absorption"):
            self.plan_absorption()
        self.upload()
        self.run_device(**kw)
        self.download()
        return self.last_cle
