"""Synthetic workloads of the calibration path: Conv/BN stacks and graph/bottoms dictionaries.

The reference's entry points take a traced model: ``graph`` (OrderedDict key -> nn.Module | op-name string, in
trace order) and ``bottoms`` (key -> list of input keys), SURVEY.md section 8(b).  On the GPU box neither the
reference's tracer nor its model files exist, so workloads are described by small *topology* records (node types,
layer hyper-parameters, edges - facts about the architectures, produced once by ``tools/make_golden.py`` from the
reference's own trace and committed under ``tests/golden/``) and materialised here with seeded random weights
("synthetic random Conv/BN weight stacks of the named shapes", BASELINE.json).

Also here: the synthetic stack of BASELINE.json config 5 (independent Conv[C,C,k,k]+BN+ReLU -> Conv[C,C,k,k]+BN
blocks), generated directly inside a device arena.
"""
from __future__ import annotations

import json
import math
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

# ----------------------------------------------------------------------------------------------------
# topology <-> graph
# ----------------------------------------------------------------------------------------------------
_SIMPLE = {"ReLU": nn.ReLU, "ReLU6": nn.ReLU6, "Dropout": nn.Dropout, "Dropout2d": nn.Dropout2d,
           "Identity": nn.Identity}


def describe_module(m) -> Optional[dict]:
    """Topology record of one traced module (used by tools/make_golden.py)."""
    t = type(m).__name__
    if isinstance(m, nn.Conv2d):
        return dict(type="Conv2d", args=dict(in_channels=m.in_channels, out_channels=m.out_channels,
                                             kernel_size=list(m.kernel_size), stride=list(m.stride),
                                             padding=list(m.padding), dilation=list(m.dilation), groups=m.groups,
                                             bias=m.bias is not None))
    if isinstance(m, nn.Linear):
        return dict(type="Linear", args=dict(in_features=m.in_features, out_features=m.out_features, bias=m.bias is not None))
    if isinstance(m, nn.BatchNorm2d):
        return dict(type="BatchNorm2d", args=dict(num_features=m.num_features, eps=m.eps))
    if isinstance(m, nn.AvgPool2d):
        return dict(type="AvgPool2d", args=dict(kernel_size=m.kernel_size, stride=m.stride, padding=m.padding))
    if isinstance(m, nn.MaxPool2d):
        return dict(type="MaxPool2d", args=dict(kernel_size=m.kernel_size, stride=m.stride, padding=m.padding))
    if isinstance(m, nn.AdaptiveAvgPool2d):
        return dict(type="AdaptiveAvgPool2d", args=dict(output_size=m.output_size))
    if t in _SIMPLE:
        return dict(type=t, args={})
    return dict(type="Opaque", args=dict(name=t))


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(int(seed))


def init_conv_(conv: nn.Conv2d, seed: int, gain_decades: float = 1.0):
    """He-normal weights (as the reference model files initialise them) times a per-output-channel gain
    10^U(-g, g) so the channel ranges are imbalanced; bias (if any) ~ N(0, 0.1)."""
    g = _gen(seed)
    k = conv.kernel_size[0] * conv.kernel_size[1]
    std = math.sqrt(2.0 / (k * conv.out_channels))
    with torch.no_grad():
        w = torch.randn(conv.weight.shape, generator=g) * std
        if gain_decades:
            gain = 10 ** torch.empty(conv.out_channels).uniform_(-gain_decades, gain_decades, generator=g)
            w = w * gain.view(-1, 1, 1, 1)
        conv.weight.copy_(w)
        if conv.bias is not None:
            conv.bias.copy_(torch.randn(conv.out_channels, generator=g) * 0.1)


def init_linear_(lin: nn.Linear, seed: int):
    g = _gen(seed)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) * 0.01)
        if lin.bias is not None:
            lin.bias.copy_(torch.randn(lin.out_features, generator=g) * 0.01)


def init_bn_(bn: nn.BatchNorm2d, seed: int):
    """gamma ~ U(0.5, 1.5), beta ~ N(0, 0.2), mean ~ N(0, 0.1), var ~ U(0.5, 1.5)  (SURVEY.md 8d, config 1)."""
    g = _gen(seed)
    n = bn.num_features
    with torch.no_grad():
        bn.weight.copy_(torch.empty(n).uniform_(0.5, 1.5, generator=g))
        bn.bias.copy_(torch.randn(n, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(n, generator=g) * 0.1)
        bn.running_var.copy_(torch.empty(n).uniform_(0.5, 1.5, generator=g))


def build_graph(topology: dict, seed: int = 0, conv_cls=nn.Conv2d, linear_cls=nn.Linear,
                gain_decades: float = 1.0) -> Tuple[OrderedDict, OrderedDict, List[nn.Module]]:
    """Materialise a topology as (graph, bottoms, modules) with seeded random parameters.

    Module nodes are keyed by ``id(module)`` and functional nodes by their op-name string, exactly like the
    reference tracer's output; `conv_cls` / `linear_cls` choose the target layer classes (nn.Conv2d or one of the
    Quant* flavours).
    """
    graph, bottoms = OrderedDict(), OrderedDict()
    key_of: Dict[str, object] = {}
    modules: List[nn.Module] = []
    for i, node in enumerate(topology["nodes"]):
        t, args = node["type"], node.get("args", {})
        name = node["key"]
        if t == "Data":
            key, obj = "Data", "Data"
        elif t == "Func":
            key, obj = name, name
        else:
            if t == "Conv2d":
                a = dict(args)
                for k in ("kernel_size", "stride", "padding", "dilation"):
                    a[k] = tuple(a[k])
                obj = conv_cls(**a)
                init_conv_(obj, seed * 100003 + i, gain_decades)
            elif t == "Linear":
                obj = linear_cls(**args)
                init_linear_(obj, seed * 100003 + i)
            elif t == "BatchNorm2d":
                obj = nn.BatchNorm2d(args["num_features"], eps=args.get("eps", 1e-5))
                init_bn_(obj, seed * 100003 + i)
            elif t == "AvgPool2d":
                obj = nn.AvgPool2d(**args)
            elif t == "MaxPool2d":
                obj = nn.MaxPool2d(**args)
            elif t == "AdaptiveAvgPool2d":
                obj = nn.AdaptiveAvgPool2d(args["output_size"])
            elif t in _SIMPLE:
                obj = _SIMPLE[t]()
            else:
                obj = nn.Identity()
            obj.eval()
            key = id(obj)
            modules.append(obj)
        key_of[name] = key
        graph[key] = obj
        b = node.get("bottoms")
        bottoms[key] = None if b is None else [key_of[x] for x in b]
    return graph, bottoms, modules


def load_topology(path: str) -> dict:
    with open(path) as f:
        return json.load(f)


def stack_topology(n_blocks: int, channels: int = 512, k: int = 3, in_channels: Optional[int] = None) -> dict:
    """BASELINE.json config 5 as a topology: independent blocks Data -> Conv+BN+ReLU -> Conv+BN (chains of length 1,
    like ResNet basic blocks).  Every block hangs off 'Data', so the first conv of a block is not bias-corrected
    (dfq.py:197-198) and the second one is."""
    ic = in_channels or channels
    nodes = [dict(key="Data", type="Data", bottoms=None)]
    for b in range(n_blocks):
        conv = lambda i, o: dict(in_channels=i, out_channels=o, kernel_size=[k, k], stride=[1, 1], padding=[k // 2, k // 2],
                                 dilation=[1, 1], groups=1, bias=False)
        nodes += [
            dict(key="b%d_conv1" % b, type="Conv2d", args=conv(ic, channels), bottoms=["Data"]),
            dict(key="b%d_bn1" % b, type="BatchNorm2d", args=dict(num_features=channels, eps=1e-5), bottoms=["b%d_conv1" % b]),
            dict(key="b%d_relu" % b, type="ReLU", args={}, bottoms=["b%d_bn1" % b]),
            dict(key="b%d_conv2" % b, type="Conv2d", args=conv(channels, channels), bottoms=["b%d_relu" % b]),
            dict(key="b%d_bn2" % b, type="BatchNorm2d", args=dict(num_features=channels, eps=1e-5), bottoms=["b%d_conv2" % b]),
        ]
    return dict(name="stack_%dx%d_k%d" % (2 * n_blocks, channels, k), input=[1, ic, 8, 8], nodes=nodes)


# ----------------------------------------------------------------------------------------------------
# config 5 directly inside a device arena
# ----------------------------------------------------------------------------------------------------
class DeviceStack:
    """`n_blocks` independent Conv[C,C,k,k]+BN+ReLU -> Conv[C,C,k,k]+BN blocks living only in a Session arena.

    Pipeline per calibration step (the BASELINE metric's unit of work, per Conv/BN pair), N weights per conv:
      BN fold: the per-channel vectors and a read-only scan of both convs (column extrema of the second, row extrema of
      the first: 4N B per conv; the weight pass itself is deferred into the first sweep, see Session.plan_bn_fold) ->
      equalization to convergence (2 sweeps, applied in ONE pass of 8N B that also folds and computes the second conv's
      bias correction from the rows it holds; a later sweep would be 8N B more) -> the correction's retirement, [C]-sized
      vectors only [-> 8-bit weight fake-quant (8N+4N B)].  12N B per conv in all.  When the equalization does not stop
      after its two fused sweeps the correction reads the second conv once more (4N B = 2N B per conv on average, its range
      from the equalization's column extrema); 26N B with the fold, each sweep and the correction as passes of their own
      (the engine path, where the fold is not deferred).
    """

    def __init__(self, sess, n_blocks: int, channels: int = 512, k: int = 3, seed: int = 1234, quantize: bool = False):
        self.sess = sess
        self.n_blocks, self.C, self.k = n_blocks, channels, k
        self.n_layers = 2 * n_blocks
        C, kk = channels, k * k
        self.N = C * C * kk
        # arena layout: all weights | all biases | all BN vectors: the small per-channel state (what a multi-GPU step
        # exchanges) is ONE contiguous window behind the weights
        w_first = sess.alloc(0)
        bias_block = None
        self.layers = []
        for i in range(self.n_layers):
            self.layers.append(sess.alloc_layer(C, C, kk, bias_off=-1))
        bias_block = sess.alloc(self.n_layers * C)
        for i, li in enumerate(self.layers):
            sess.layer(li)["bias_off"] = bias_block + i * C
        self.bias_begin = bias_block
        self.w_begin = sess.layer(self.layers[0])["w_off"]
        # per-layer BN vectors: gamma, beta, mean, var, fake_w, fake_b
        self.vec = [dict((n, sess.alloc(C)) for n in ("gamma", "beta", "mean", "var", "fake_w", "fake_b"))
                    for _ in range(self.n_layers)]
        self.vec_begin = self.vec[0]["gamma"]
        self.vec_end = self.vec[-1]["fake_b"] + C
        self.seed = seed
        folds = [dict(layer=li, bn_eps=1e-5, gamma_off=v["gamma"], beta_off=v["beta"], mean_off=v["mean"], var_off=v["var"],
                      fake_w_off=v["fake_w"], fake_b_off=v["fake_b"]) for li, v in zip(self.layers, self.vec)]
        rels = [(self.layers[2 * b], self.layers[2 * b + 1], self.vec[2 * b]["fake_w"], self.vec[2 * b]["fake_b"])
                for b in range(n_blocks)]
        # every block is an independent model: its own convergence group (the reference would be called per model)
        self.cle_plan = sess.plan_cle(rels, groups=list(range(n_blocks)))
        # the fold also writes the column extrema of every block's second conv: the equalization starts without a scan
        self.fold_plan = sess.plan_bn_fold(folds, cle_plan=self.cle_plan)
        items = [dict(layer=self.layers[2 * b + 1], signed=False, level=0, next_bn_b_off=self.vec[2 * b + 1]["fake_b"],
                      terms=[dict(bn_w_off=self.vec[2 * b]["fake_w"], bn_b_off=self.vec[2 * b]["fake_b"], n=C, relu=True, op="set")])
                 for b in range(n_blocks)]
        # ... and the correction of the second convs rides on the equalization's pass (Session.plan_bias_correct)
        self.bc_plan = sess.plan_bias_correct(items, cle_plan=self.cle_plan)
        self.quant_plan = None
        if quantize:
            tasks = []
            for li in self.layers:
                l = sess.layer(li)
                tasks.append((l["w_off"], self.N, 8, False))
                tasks.append((l["bias_off"], C, 8, False))
            self.quant_plan = sess.plan_quantize(tasks)
        sess.materialize()
        self.state_floats = self.vec_end - self.w_begin

    def generate(self, chunk_layers: int = 64):
        """Seeded random weights/BN statistics written straight into the arena (device RNG)."""
        sess, C, kk = self.sess, self.C, self.k * self.k
        g = torch.Generator(device=sess.device).manual_seed(self.seed)
        std = math.sqrt(2.0 / (kk * C))
        for i, (li, v) in enumerate(zip(self.layers, self.vec)):
            l = sess.layer(li)
            w = sess.view(l["w_off"], self.N).view(C, C * kk)
            w.normal_(0.0, std, generator=g)
            gain = 10 ** torch.empty(C, device=sess.device).uniform_(-1.0, 1.0, generator=g)
            w.mul_(gain.view(-1, 1))
            sess.view(l["bias_off"], C).zero_()
            sess.view(v["gamma"], C).uniform_(0.5, 1.5, generator=g)
            sess.view(v["beta"], C).normal_(0.0, 0.2, generator=g)
            sess.view(v["mean"], C).normal_(0.0, 0.1, generator=g)
            sess.view(v["var"], C).uniform_(0.5, 1.5, generator=g)

    def state(self) -> torch.Tensor:
        """The mutable region (weights, biases, BN vectors) as one flat view - what a step reads and writes."""
        return self.sess.view(self.w_begin, self.state_floats)

    def channel_state(self) -> torch.Tensor:
        """Everything a calibration step produces besides the weights: corrected biases and the BN vectors
        (fake_weight / fake_bias after the fold) of every layer, one contiguous window (SURVEY 8(e) "Collective")."""
        return self.sess.view(self.bias_begin, self.vec_end - self.bias_begin)

    def scale_state(self) -> torch.Tensor:
        """The accumulated scale vectors Relation.S of every block (relation.py:20-24), one contiguous window."""
        lo = min(self.cle_plan["s_offs"])
        return self.sess.view(lo, max(self.cle_plan["s_offs"]) + self.C - lo)

    def block_arrays(self, state: torch.Tensor, b: int):
        """Block `b` of a flat state image (state() or a saved copy of it) as host numpy arrays: a list of two dicts
        (conv1, conv2) with w [C,C,k,k], bias, gamma, beta, mean, var, fake_w, fake_b.  Checker-side helper: the parity
        tests and bench.py's parity_check feed these to the oracle."""
        C, k = self.C, self.k
        out = []
        for li, v in zip(self.layers[2 * b: 2 * b + 2], self.vec[2 * b: 2 * b + 2]):
            l = self.sess.layer(li)
            take = lambda off, n: state[off - self.w_begin: off - self.w_begin + n].detach().cpu().numpy().copy()
            d = dict((n, take(v[n], C)) for n in ("gamma", "beta", "mean", "var", "fake_w", "fake_b"))
            d["w"] = take(l["w_off"], self.N).reshape(C, C, k, k)
            d["bias"] = take(l["bias_off"], C)
            out.append(d)
        return out

    def run(self, converge_thres=2e-7):
        """One calibration step over the whole stack; returns the CleResult."""
        s = self.sess
        s.run_bn_fold(self.fold_plan)
        res = s.run_cle_plan(self.cle_plan, converge_thres=converge_thres, cols_ready=self.fold_plan["scanned"])
        # the corrected layers are the `second` convs: their range comes from the column extrema the equalization kept
        s.run_bias_correct_plan(self.bc_plan, 8, col_hints=s.cle_col_hints(self.cle_plan, res))
        if self.quant_plan is not None:
            s.run_quantize(self.quant_plan)
        return res

    @property
    def launches_per_step(self) -> int:
        """Kernels of this library per step: fold prologue (column-range reset, the deferred fold's vectors) + fold pass
        (the read-only scan when deferred), equalization engine, correction engine (its retirement when the equalization
        prepared it) [+ range init, min/max, quantize], plus
        the small copy kernel (k_copy_words) that moves each call's descriptor tables (fold, equalization, correction
        [, quantize]) and the equalization's two result blocks through mapped pinned memory."""
        return 4 + 5 + (4 if self.quant_plan is not None else 0)


class HostStackCalibrator:
    """Calibrate a stack that lives in HOST memory, streaming it through the GPU in chunks.

    The host image is the concatenation of per-chunk state images (what ``DeviceStack.state()`` looks like).  Three
    streams form a pipeline over the chunks: H2D of chunk i+1, the kernels on chunk i, D2H of chunk i-1, each chunk in its
    own arena slot.  THREE slots are needed for the two copy directions to overlap (with two, the load of chunk i+1 has to
    wait for the store of chunk i-1 to vacate its slot); PCIe is full duplex, so a step is then bound by
    max(H2D, D2H, compute) per chunk instead of their sum.
    """

    def __init__(self, device, chunk_blocks: int = 32, channels: int = 512, k: int = 3, quantize: bool = False,
                 n_slots: int = 4):
        from .engine import Session
        self.device = device
        self.slots = []
        self.n_slots = n_slots
        for _ in range(n_slots):
            sess = Session(device)
            st = DeviceStack(sess, chunk_blocks, channels, k, quantize=quantize)
            self.slots.append(st)
        self.chunk_floats = self.slots[0].state_floats
        self.chunk_layers = 2 * chunk_blocks
        self.s_in = torch.cuda.Stream(device)
        self.s_run = torch.cuda.Stream(device)
        self.s_out = torch.cuda.Stream(device)

    def run(self, host_in: torch.Tensor, host_out: torch.Tensor, copy_only: bool = False):
        """host_in/host_out: pinned fp32 tensors of n_chunks * chunk_floats elements.  ``copy_only`` moves the same chunks
        through the same three streams without launching the kernels (the transfer ceiling of the box, for bench.py)."""
        n = host_in.numel() // self.chunk_floats
        F, S = self.chunk_floats, self.n_slots
        loaded = [torch.cuda.Event() for _ in range(n)]
        computed = [torch.cuda.Event() for _ in range(n)]
        stored = [torch.cuda.Event() for _ in range(n)]
        cur = torch.cuda.current_stream(self.device)
        self.s_in.wait_stream(cur); self.s_run.wait_stream(cur); self.s_out.wait_stream(cur)

        def load(i):
            with torch.cuda.stream(self.s_in):
                if i >= S:
                    self.s_in.wait_event(stored[i - S])          # the slot's previous tenant has left
                self.slots[i % S].state().copy_(host_in[i * F:(i + 1) * F], non_blocking=True)
                loaded[i].record(self.s_in)

        load(0)
        for i in range(n):
            if i + 1 < n:
                load(i + 1)
            with torch.cuda.stream(self.s_run):
                self.s_run.wait_event(loaded[i])
                if not copy_only:
                    self.slots[i % S].run()                       # returns when the equalization result is back
                computed[i].record(self.s_run)
            with torch.cuda.stream(self.s_out):
                self.s_out.wait_event(computed[i])
                host_out[i * F:(i + 1) * F].copy_(self.slots[i % S].state(), non_blocking=True)
                stored[i].record(self.s_out)
        cur.wait_stream(self.s_out)
