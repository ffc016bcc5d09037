"""Throughput of int8 execution (dfq_b200.int8) on the H100: prints one JSON line.

    python tools/bench_int8.py [--batch 256] [--reps 10]

images/s of torchvision MobileNetV2 and ResNet-18 (seeded weights, 224x224) run three ways - int8 execution, the fake-quant path
of the reference's QuantN* layers, plain fp32 with TF32 off - and the achieved int8 TOPS of dfq_i8_conv on ResNet-18's largest
GEMM layers against the data-sheet dense peak, and the relative logit error (2-norm over 64 random images) of int8 and of
fake-quant against fp32.  `chained`: per-layer int8 against int8.chain_int8 (activations kept in int8 between fused
convolutions) on the same nets with BN folded - images/s, fused edges, fp32 bytes avoided, bit-identity of the logits.
`residual`: per-layer against chain_int8 and chain_int8(residual=True) (residual adds and tensors with several consumers
fused too), the same way, with the fused adds.  `pool_cat`: per-layer against chain_int8(residual=True) and
chain_int8(residual=True, pool_cat=True) (max pools and channel concatenations carried in int8 too) on ResNet-18, SqueezeNet
1.1 and GoogLeNet.  `upsample`: per-layer against chain_int8(residual=True, pool_cat=True) and chain_int8(..., upsample=True)
(bilinear upsamples feeding concatenations carried in int8 too) on two segmentation networks at 513x513: the DeepLab-v3+-shaped
network of tests/deeplab_v3plus_like.py and torchvision's DeepLab-v3 ResNet-50.  `layout`: per-layer against
chain_int8(..., upsample=True) and chain_int8(..., layout=True) (zero pads folded into convolutions, detection heads written
into their concatenation) on the networks of tests/deeplab_mobilenet_padded.py (8 x 513x513) and tests/ssd_lite_like.py
(256 x 300x300).  `affine` (only when asked for: --sections affine): the reference's own asymmetric min / max quantization
executed in integers (int8.convert_affine) against the fake-quantized model and the ncnn per-layer int8 model on
MobileNetV2 and ResNet-18, with the logit errors against the fake-quantized model.  `affine_chained` (only when asked
for): the fake-quantized model, convert_affine per layer, int8.chain_affine and chain_affine(residual=True) on the same
networks, the three affine arms' logits asserted bit-identical.  `affine_observed` (only when asked for): the same
networks in the reference's evaluation state (tests/affine_observed_state.py: replace_op() active, the functional-op
observers on every residual add and, for MobileNetV2 with the reference's head, on the mean's input), timing the
fake-quantized model, the per-layer convert_affine model and chain_affine(residual=True), which runs the observers in its
epilogues; the two affine arms' logits asserted bit-identical.  `affine_pool_heads` (only when asked for):
ResNet-18 and GoogLeNet in that state, per-layer against chain_affine(residual=True[, concat=True]) and the same with
pools=True (max pools carried as affine codes), and SSD-Lite at 300x300 against chain_affine(residual=True, concat=True,
fold_pads=True) and the same with heads=True (detection heads written in place), outputs asserted bit-identical, with
the fp32 bytes the flags avoid.  `affine_distilled` (only when asked for): MobileNetV2 and ResNet-18 in the reference's
--distill_range state (tests/affine_distilled_state.py: QConv2d / QLinear, which re-quantize every weight and bias on each
forward), timing the fake-quantized model, the per-layer convert_affine model and chain_affine(residual=True), the two
affine arms' logits asserted bit-identical.  The card's name and power limit are read in the same run and reported beside the numbers.  Needs a CUDA
device; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def int8_inference(dev, reps=10, batch=256):
    """images/s of int8 execution (dfq_b200.int8) vs the fake-quant path (QuantN* layers) vs fp32 with TF32 off, for
    torchvision MobileNetV2 and ResNet-18 (seeded weights, batch 256, 224x224), their relative logit errors against fp32, and
    the achieved int8 TOPS of dfq_i8_conv on ResNet-18's largest GEMM layers against the data-sheet dense peak."""
    import copy
    import ctypes as C
    import torch
    import torch.nn as nn
    import torchvision
    from dfq_b200 import _lib, int8
    from dfq_b200.utils import quantize as Q

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def fake_quant(model, amax):
        for name, m in list(model.named_modules()):
            if type(m) in (nn.Conv2d, nn.Linear):
                q = (Q.QuantNConv2d(m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding, m.dilation, m.groups,
                                    m.bias is not None) if isinstance(m, nn.Conv2d) else
                     Q.QuantNLinear(m.in_features, m.out_features, m.bias is not None)).to(dev).eval()
                q.load_state_dict(m.state_dict(), strict=False)
                q.quant.running_min.fill_(-amax[name]); q.quant.running_max.fill_(amax[name])
                parent, _, attr = name.rpartition(".")
                setattr(model.get_submodule(parent) if parent else model, attr, q)
        return model

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps}
    try:
        x = torch.randn(batch, 3, 224, 224, device=dev)
        for net in ("mobilenet_v2", "resnet18"):
            torch.manual_seed(0)
            fp32 = getattr(torchvision.models, net)(num_classes=1000).to(dev).eval()
            graph, amax, hooks = {}, {}, []
            for name, m in fp32.named_modules():
                if type(m) in (nn.Conv2d, nn.Linear):
                    graph[id(m)] = m
                    hooks.append(m.register_forward_pre_hook(
                        lambda m, i, name=name: amax.__setitem__(name, max(amax.get(name, 0.0), float(i[0].abs().max())))))
            with torch.no_grad():
                fp32(x[:32])
            for h in hooks:
                h.remove()
            fq = fake_quant(copy.deepcopy(fp32), amax)
            i8 = copy.deepcopy(fp32)
            graph = {id(m): m for n, m in i8.named_modules() if type(m) in (nn.Conv2d, nn.Linear)}
            int8.convert_to_int8(i8, graph, [nn.Conv2d, nn.Linear], act_scales=[128. / amax[n] for n, m in fp32.named_modules()
                                                                                 if type(m) in (nn.Conv2d, nn.Linear)])
            with torch.no_grad():
                ms = {k: timed(lambda mod=mod: mod(x)) for k, mod in (("int8", i8), ("fake_quant", fq), ("fp32_no_tf32", fp32))}
                ref = fp32(x[:64])
                err = {k: float((mod(x[:64]) - ref).norm() / ref.norm()) for k, mod in (("int8", i8), ("fake_quant", fq))}
            out[net] = {k: batch / (v * 1e-3) for k, v in ms.items()}
            out[net]["ms_per_batch"] = ms
            out[net]["rel_logit_error_vs_fp32_64_random_images"] = err
            if net == "resnet18":
                lib, layers = _lib.load(), []
                shapes = {}
                hooks = [m.register_forward_pre_hook(lambda m, i: shapes.__setitem__(id(m), tuple(i[0].shape)))
                         for m in i8.modules() if isinstance(m, int8.Int8Conv2d)]
                with torch.no_grad():
                    i8(x)
                for h in hooks:
                    h.remove()
                for name, m in i8.named_modules():
                    if isinstance(m, int8.Int8Conv2d):
                        N, Cn, H, W = shapes[id(m)]
                        g = m._geometry(N, H, W)
                        M = N * int(g[0]["OH"]) * int(g[0]["OW"])
                        K = m.kernel_size[0] * m.kernel_size[1] * m.cpad
                        layers.append((2 * M * m.out_channels * K, name, m, g, (N, Cn, H, W)))
                tops = []
                for ops, name, m, g, shp in sorted(layers, key=lambda t: -t[0])[:4]:
                    xq = torch.zeros(shp[0] * shp[2] * shp[3] * m.cpad, dtype=torch.int8, device=dev)
                    y = torch.empty(shp[0], m.out_channels, int(g[0]["OH"]), int(g[0]["OW"]), device=dev)
                    st = _lib.stream_ptr()
                    call = lambda: lib.dfq_i8_conv(C.c_void_p(xq.data_ptr()), C.c_void_p(m.weight_codes.data_ptr()),
                                                   C.c_void_p(m.dq.data_ptr()), C.c_void_p(m.bias.data_ptr()),
                                                   C.c_void_p(y.data_ptr()), None, _lib.table_ptr(g), st)
                    t = timed(call)
                    tops.append({"layer": name, "input": list(shp), "out_channels": m.out_channels, "gemm_ops": ops,
                                 "ms": t, "TOPS": ops / (t * 1e-3) / 1e12})
                out["resnet18_largest_gemm_layers"] = {
                    "kernel": "k_i8_conv_mma (dfq_i8_conv, mma.sync m16n8k32 s8; epilogue and fp32 NCHW store included)",
                    "layers": tops, "datasheet_peak_int8_dense_TOPS": 1979.0,
                    "peak_note": "NVIDIA H100 SXM data-sheet figure (700 W), not a measured peak"}
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def chained_inference(dev, reps=10, batch=256, rounds=5):
    """Per-layer int8 execution against int8.chain_int8 (activations kept in int8 between fused convolutions) on torchvision
    MobileNetV2 (ReLU6 kept) and ResNet-18, BN folded by trace_graph + merge_batchnorm, activation scales 128 / max|input|
    from forward hooks: images/s and ms per batch of both arms (timed alternately, `rounds` rounds of `reps` passes, median),
    the fused edges, the fp32 traffic they avoid per batch (computed from shapes) and whether the logits are bit-identical."""
    import statistics
    from collections import OrderedDict
    import torch
    import torch.nn as nn
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds,
           "fp32_bytes_avoided_note": "per fused edge and element of the carried tensor: the producer's fp32 store and the "
                                      "quantizer's fp32 read (8 B) plus a read and a write (8 B) per deleted pass-through op; "
                                      "the int8 codes (1 B) are written either way"}
    x = torch.randn(batch, 3, 224, 224, device=dev)
    for net in ("mobilenet_v2", "resnet18"):
        torch.manual_seed(0)
        model = getattr(torchvision.models, net)(num_classes=1000).to(dev).eval()
        graph, bottoms = trace_graph(model)
        merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
        layers = OrderedDict((n, m) for n, m in model.named_modules() if type(m) in (nn.Conv2d, nn.Linear))
        amax = {}
        hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, max(amax.get(n, 0.0), float(i[0].abs().max()))))
                 for n, m in layers.items()]
        with torch.no_grad():
            model(x[:32])
        for h in hooks:
            h.remove()
        int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                             act_scales=[128. / amax[n] for n in layers])
        gm = int8.chain_int8(model)
        edges = gm.requantized_edges
        traced = int8._Int8Tracer().trace(model)
        node_of = {n.target: n for n in traced.nodes if n.op == "call_module"}
        numel, mods = {}, dict(model.named_modules())
        hooks = [mods[q].register_forward_pre_hook(lambda m, i, q=q: numel.__setitem__(q, i[0].numel())) for _, q, _ in edges]
        with torch.no_grad():
            ref = model(x)
            for h in hooks:
                h.remove()
            got = gm(x)
            torch.cuda.synchronize(dev)
            avoided = 0
            for p, q, _ in edges:
                k, node = 0, node_of[q].args[0]
                while not (node.op == "call_module" and node.target == p):
                    k, node = k + 1, node.args[0]
                avoided += numel[q] * (8 + 8 * k)
            for _ in range(2):
                model(x), gm(x)
            torch.cuda.synchronize(dev)
            ms = {"per_layer": [], "chained": []}
            for _ in range(rounds):
                ms["per_layer"].append(timed(lambda: model(x)))
                ms["chained"].append(timed(lambda: gm(x)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                    "ms_per_batch_rounds": ms, "fused_edges": len(edges), "fp32_bytes_avoided_per_batch": avoided,
                    "logits_bit_identical": bool(torch.equal(ref.view(torch.int32), got.view(torch.int32)))}
    return out


def residual_inference(dev, reps=10, batch=256, rounds=5):
    """Per-layer int8 execution against int8.chain_int8 and int8.chain_int8(residual=True) on the nets of chained_inference
    (timed alternately, `rounds` rounds of `reps` passes, median): images/s, ms per batch, edges and fused adds, the fp32
    traffic the residual arm avoids per batch against the per-layer path (computed from shapes) and bit-identity of the
    logits."""
    import statistics
    from collections import OrderedDict
    import torch
    import torch.nn as nn
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds,
           "fp32_bytes_avoided_note": "fp32 bytes of the per-layer path that the residual arm does not move, per batch: per "
                                      "element of every carried tensor, the quantizer's fp32 read (4 B) per carried consumer, "
                                      "plus the producer's fp32 store (4 B) when no fp32 consumer is left; a read and a write "
                                      "(8 B) per deleted pass-through and per deleted identity on a residual; per fused add, "
                                      "its two reads and its write (12 B)"}
    x = torch.randn(batch, 3, 224, 224, device=dev)
    for net in ("mobilenet_v2", "resnet18"):
        torch.manual_seed(0)
        model = getattr(torchvision.models, net)(num_classes=1000).to(dev).eval()
        graph, bottoms = trace_graph(model)
        merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
        layers = OrderedDict((n, m) for n, m in model.named_modules() if type(m) in (nn.Conv2d, nn.Linear))
        amax = {}
        hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, max(amax.get(n, 0.0), float(i[0].abs().max()))))
                 for n, m in layers.items()]
        with torch.no_grad():
            model(x[:32])
        for h in hooks:
            h.remove()
        int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                             act_scales=[128. / amax[n] for n in layers])
        chained = int8.chain_int8(model)
        gm = int8.chain_int8(model, residual=True)
        # bytes from shapes: every node of the per-layer graph the residual arm deleted or made int8
        traced = int8._Int8Tracer().trace(model)
        kept = {n.name for n in gm.graph.nodes}
        numel, mods = {}, dict(model.named_modules())
        hooks = [m.register_forward_hook(lambda m, i, o, n=n: numel.__setitem__(n, o.numel())) for n, m in mods.items()
                 if isinstance(m, int8.Int8Conv2d)]
        with torch.no_grad():
            ref = model(x)
            for h in hooks:
                h.remove()
            got = {"chained": chained(x), "residual": gm(x)}
            torch.cuda.synchronize(dev)
            avoided = 0
            for p, q, _ in gm.requantized_edges:
                avoided += 4 * numel[p]
            for p, epi in ((n, getattr(m, "epilogue", None)) for n, m in gm.named_modules()):
                if isinstance(mods.get(p), int8.Int8Conv2d) and (epi is None or not epi.fp32) and \
                        p in {e[0] for e in gm.requantized_edges}:
                    avoided += 4 * numel[p]
            node_out = {n.target: n for n in traced.nodes if n.op == "call_module"}
            for n in traced.nodes:
                if n.name in kept or n.op not in ("call_module", "call_function", "call_method"):
                    continue
                src = n.args[0] if n.args and isinstance(n.args[0], torch.fx.Node) else None
                while src is not None and not (src.op == "call_module" and src.target in node_out and
                                               isinstance(mods.get(src.target), int8.Int8Conv2d)):
                    src = src.args[0] if src.args and isinstance(src.args[0], torch.fx.Node) else None
                if src is not None:
                    avoided += numel[src.target] * (12 if int8._is_add(n) else 8)
            for _ in range(2):
                model(x), chained(x), gm(x)
            torch.cuda.synchronize(dev)
            ms = {"per_layer": [], "chained": [], "residual": []}
            for _ in range(rounds):
                ms["per_layer"].append(timed(lambda: model(x)))
                ms["chained"].append(timed(lambda: chained(x)))
                ms["residual"].append(timed(lambda: gm(x)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                    "ms_per_batch_rounds": ms, "edges": {"chained": len(chained.requantized_edges),
                                                         "residual": len(gm.requantized_edges)},
                    "fused_adds": len(gm.fused_adds), "fp32_bytes_avoided_per_batch": avoided,
                    "logits_bit_identical": {k: bool(torch.equal(ref.view(torch.int32), v.view(torch.int32)))
                                             for k, v in got.items()}}
    return out


def pool_cat_inference(dev, reps=10, batch=256, rounds=5):
    """Per-layer int8 execution against chain_int8(residual=True) and chain_int8(residual=True, pool_cat=True) on ResNet-18,
    SqueezeNet 1.1 and GoogLeNet (BN folded, scales 128 / max|input|), timed alternately (`rounds` rounds of `reps` passes,
    median): images/s, ms per batch, fused cats and pools, the fp32 bytes the pool_cat arm avoids against the residual arm
    (from shapes) and bit-identity of the logits."""
    import statistics
    from collections import OrderedDict
    import torch
    import torch.nn as nn
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds,
           "fp32_bytes_avoided_note": "fp32 bytes the residual arm moves through torch.cat, max_pool2d and the pass-throughs "
                                      "and quantizers around them that the pool_cat arm does not, per batch, from the "
                                      "traced tensors' sizes: per deleted node a read and a write of its output (cat: of "
                                      "its output twice), per fused pool its fp32 read and write unless it runs in fp32 mode, "
                                      "per carried consumer of a pool or cat the quantizer's read"}
    x = torch.randn(batch, 3, 224, 224, device=dev)
    for net in ("resnet18", "squeezenet1_1", "googlenet"):
        torch.manual_seed(0)
        kw = dict(aux_logits=False, init_weights=True) if net == "googlenet" else {}
        model = getattr(torchvision.models, net)(num_classes=1000, **kw).to(dev).eval()
        graph, bottoms = trace_graph(model)
        merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
        layers = OrderedDict((n, m) for n, m in model.named_modules() if type(m) in (nn.Conv2d, nn.Linear))
        amax = {}
        hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, max(amax.get(n, 0.0), float(i[0].abs().max()))))
                 for n, m in layers.items()]
        with torch.no_grad():
            model(x[:32])
        for h in hooks:
            h.remove()
        int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                             act_scales=[128. / amax[n] for n in layers])
        res = int8.chain_int8(model, residual=True)
        gm = int8.chain_int8(model, residual=True, pool_cat=True)
        # sizes of every traced node's output, from one fp32 run of the traced per-layer model
        traced = torch.fx.GraphModule(model, int8._Int8Tracer().trace(model))
        size = {}
        interp = torch.fx.Interpreter(traced)
        run_node = interp.run_node

        def record(n):
            v = run_node(n)
            if isinstance(v, torch.Tensor):
                size[n.name] = v.numel() * 4
            return v
        interp.run_node = record
        with torch.no_grad():
            interp.run(x)
            kept_res = {n.name for n in res.graph.nodes}
            kept = {n.name for n in gm.graph.nodes}
            avoided = sum(2 * size.get(n, 0) for n in kept_res - kept)
            avoided += sum(2 * size.get(c[0], 0) for c in gm.fused_cats)
            avoided += sum(size.get(p[0], 0) // 4 * 4 for p in gm.fused_pools if p[1] == "codes")
            avoided += sum(size.get(p, 0) for p, q, _ in gm.requantized_edges
                           if q not in {e[1] for e in res.requantized_edges})
            ref = model(x)
            got = {"residual": res(x), "pool_cat": gm(x)}
            for _ in range(2):
                model(x), res(x), gm(x)
            torch.cuda.synchronize(dev)
            ms = {"per_layer": [], "residual": [], "pool_cat": []}
            for _ in range(rounds):
                ms["per_layer"].append(timed(lambda: model(x)))
                ms["residual"].append(timed(lambda: res(x)))
                ms["pool_cat"].append(timed(lambda: gm(x)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                    "ms_per_batch_rounds": ms, "fused_cats": len(gm.fused_cats),
                    "fused_pools": [p[:2] for p in gm.fused_pools],
                    "carried_conv_inputs": {"residual": len({e[1] for e in res.requantized_edges}),
                                            "pool_cat": len({e[1] for e in gm.requantized_edges})},
                    "fp32_bytes_avoided_per_batch_vs_residual": avoided,
                    "logits_bit_identical": {k: bool(torch.equal(ref.view(torch.int32), v.view(torch.int32)))
                                             for k, v in got.items()}}
    return out


def upsample_inference(dev, reps=10, batch=8, rounds=5, size=513):
    """Per-layer int8 execution against chain_int8(residual=True, pool_cat=True) and chain_int8(..., upsample=True) on the
    DeepLab-v3+-shaped network of tests/deeplab_v3plus_like.py and torchvision's deeplabv3_resnet50 (seeded weights, BN
    folded, scales 128 / max|input|), `batch` images of size x size, timed alternately (`rounds` rounds of `reps` passes,
    median): images/s, ms per batch, fused cats and upsamples, carried convolution inputs, the fp32 bytes the upsample arm
    avoids against the pool_cat arm (from the traced tensors' sizes) and bit-identity of the output."""
    import statistics
    from collections import OrderedDict
    import torch
    import torch.nn as nn
    import torchvision
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from deeplab_v3plus_like import DeepLabV3PlusLike

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def out_of(t):
        return t["out"] if isinstance(t, dict) else t

    out = {"batch": batch, "image": "3x%dx%d" % (size, size), "unit": "images/s", "reps": reps, "rounds": rounds,
           "fp32_bytes_avoided_note": "fp32 bytes the pool_cat arm moves that the upsample arm does not, per batch, from the "
                                      "traced tensors' sizes: per deleted node a read and a write of its output (cat: of its "
                                      "output twice), per fused upsample its fp32 output's write, per carried consumer of a "
                                      "fused cat or upsample the quantizer's read"}
    x = torch.randn(batch, 3, size, size, device=dev)
    for net in ("deeplab_v3plus_like", "deeplabv3_resnet50"):
        torch.manual_seed(0)
        model = (DeepLabV3PlusLike(num_classes=21) if net == "deeplab_v3plus_like" else
                 torchvision.models.segmentation.deeplabv3_resnet50(weights=None, weights_backbone=None, aux_loss=False))
        model = model.to(dev).eval()
        graph, bottoms = trace_graph(model)
        merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
        layers = OrderedDict((n, m) for n, m in model.named_modules() if type(m) in (nn.Conv2d, nn.Linear))
        amax = {}
        hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, max(amax.get(n, 0.0), float(i[0].abs().max()))))
                 for n, m in layers.items()]
        with torch.no_grad():
            model(x[:2])
        for h in hooks:
            h.remove()
        int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                             act_scales=[128. / amax[n] for n in layers])
        base = int8.chain_int8(model, residual=True, pool_cat=True)
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
        traced = torch.fx.GraphModule(model, int8._Int8Tracer().trace(model))
        nbytes = {}
        interp = torch.fx.Interpreter(traced)
        run_node = interp.run_node

        def record(n):
            v = run_node(n)
            if isinstance(v, torch.Tensor):
                nbytes[n.name] = v.numel() * 4
            return v
        interp.run_node = record
        with torch.no_grad():
            interp.run(x)
            kept_base, kept = {n.name for n in base.graph.nodes}, {n.name for n in gm.graph.nodes}
            avoided = sum(2 * nbytes.get(n, 0) for n in kept_base - kept)
            avoided += sum(2 * nbytes.get(c[0], 0) for c in gm.fused_cats)
            avoided += sum(nbytes.get(u[0], 0) for u in gm.fused_upsamples)
            avoided += sum(nbytes.get(p, 0) for p, q, _ in gm.requantized_edges
                           if q not in {e[1] for e in base.requantized_edges})
            del interp, nbytes
            ref = out_of(model(x))
            got = {"pool_cat": out_of(base(x)), "upsample": out_of(gm(x))}
            for _ in range(2):
                model(x), base(x), gm(x)
            torch.cuda.synchronize(dev)
            ms = {"per_layer": [], "pool_cat": [], "upsample": []}
            for _ in range(rounds):
                ms["per_layer"].append(timed(lambda: model(x)))
                ms["pool_cat"].append(timed(lambda: base(x)))
                ms["upsample"].append(timed(lambda: gm(x)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                    "ms_per_batch_rounds": ms, "fused_cats": len(gm.fused_cats),
                    "fused_upsamples": [u[:3] for u in gm.fused_upsamples],
                    "carried_conv_inputs": {"pool_cat": len({e[1] for e in base.requantized_edges}),
                                            "upsample": len({e[1] for e in gm.requantized_edges}),
                                            "convolutions": sum(isinstance(m, int8.Int8Conv2d) for m in model.modules())},
                    "fp32_bytes_avoided_per_batch_vs_pool_cat": avoided,
                    "output_bit_identical": {k: bool(torch.equal(ref.view(torch.int32), v.view(torch.int32)))
                                             for k, v in got.items()}}
        del model, base, gm, ref, got
        torch.cuda.empty_cache()
    return out


def layout_inference(dev, reps=10, rounds=5, seg_batch=8, ssd_batch=256):
    """Per-layer int8 execution against chain_int8(residual=True, pool_cat=True, upsample=True) and chain_int8(...,
    layout=True) on the DeepLab-v3+ (MobileNetV2, fixed padding) of tests/deeplab_mobilenet_padded.py at seg_batch x
    513x513 and the MobileNetV2-SSD-Lite of tests/ssd_lite_like.py (is_test) at ssd_batch x 300x300 (seeded weights, BN
    folded, scales 128 / max|input|), timed alternately (`rounds` rounds of `reps` passes, median): images/s, ms per batch,
    folded pads and fused heads, carried convolution inputs, the fp32 bytes and launches the layout arm avoids against the
    upsample arm (from the traced tensors' sizes) and bit-identity of the outputs."""
    import statistics
    from collections import OrderedDict
    import torch
    import torch.nn as nn
    from dfq_b200 import int8
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils.layer_transform import merge_batchnorm
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from deeplab_mobilenet_padded import DeepLabMobileNetPadded
    from ssd_lite_like import SSDLiteLike

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def same(a, b):
        a, b = (t if isinstance(t, tuple) else (t,) for t in (a, b))
        return all(x.shape == y.shape and bool(torch.equal(x.view(torch.int32), y.view(torch.int32))) for x, y in zip(a, b))

    out = {"unit": "images/s", "reps": reps, "rounds": rounds,
           "avoided_note": "fp32 bytes and launches the upsample arm spends that the layout arm does not, per batch, from the "
                           "traced tensors' sizes: per folded pad the pad's read of its input, its write and the quantizer's "
                           "read of the padded tensor (2 launches); per fused head the contiguous copy's read and write and "
                           "the cat's read and write of its output (1 launch, plus 1 per cat)"}
    for net, batch, size in (("deeplab_mobilenet_padded", seg_batch, 513), ("ssd_lite", ssd_batch, 300)):
        torch.manual_seed(0)
        model = (DeepLabMobileNetPadded(21) if net == "deeplab_mobilenet_padded" else SSDLiteLike(21, is_test=True))
        model = model.to(dev).eval()
        x = torch.randn(batch, 3, size, size, device=dev)
        graph, bottoms = trace_graph(model)
        merge_batchnorm(model, graph, bottoms, [nn.Conv2d])
        layers = OrderedDict((n, m) for n, m in model.named_modules() if type(m) in (nn.Conv2d, nn.Linear))
        amax = {}
        hooks = [m.register_forward_pre_hook(lambda m, i, n=n: amax.__setitem__(n, max(amax.get(n, 0.0), float(i[0].abs().max()))))
                 for n, m in layers.items()]
        with torch.no_grad():
            model(x[:2])
        for h in hooks:
            h.remove()
        int8.convert_to_int8(model, OrderedDict((id(m), m) for m in layers.values()), [nn.Conv2d, nn.Linear],
                             act_scales=[128. / amax[n] for n in layers])
        base = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
        gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True)
        traced = torch.fx.GraphModule(model, int8._Int8Tracer().trace(model))
        numel = {}
        interp = torch.fx.Interpreter(traced)
        run_node = interp.run_node

        def record(n):
            v = run_node(n)
            if isinstance(v, torch.Tensor):
                numel[n.name] = v.numel()
            return v
        interp.run_node = record
        with torch.no_grad():
            interp.run(x[:1])                                   # sizes of one image, scaled to the batch below
            nodes = {n.name: n for n in traced.graph.nodes}
            avoided = sum(4 * (numel[nodes[p].args[0].name] + 2 * numel[p]) for p, _, _ in gm.folded_pads)
            launches = 2 * len(gm.folded_pads)
            heads = {q: n.name for n in traced.graph.nodes if n.op == "call_module" for q in [n.target]}
            for _, prods, _ in gm.fused_heads:
                avoided += sum(16 * numel[heads[q]] for q in prods)
                launches += len(prods) + 1
            del interp, numel
            ref = model(x)
            got = {"upsample": base(x), "layout": gm(x)}
            for _ in range(2):
                model(x), base(x), gm(x)
            torch.cuda.synchronize(dev)
            ms = {"per_layer": [], "upsample": [], "layout": []}
            for _ in range(rounds):
                ms["per_layer"].append(timed(lambda: model(x)))
                ms["upsample"].append(timed(lambda: base(x)))
                ms["layout"].append(timed(lambda: gm(x)))
        med = {k: statistics.median(v) for k, v in ms.items()}
        out[net] = {"batch": batch, "image": "3x%dx%d" % (size, size),
                    "images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                    "ms_per_batch_rounds": ms, "folded_pads": len(gm.folded_pads),
                    "fused_heads": [(c, len(p), k) for c, p, k in gm.fused_heads],
                    "carried_conv_inputs": {"upsample": len({e[1] for e in base.requantized_edges}),
                                            "layout": len({e[1] for e in gm.requantized_edges}),
                                            "convolutions": sum(isinstance(m, int8.Int8Conv2d) for m in model.modules())},
                    "fp32_bytes_avoided_per_batch_vs_upsample": avoided * batch,
                    "launches_avoided_per_forward_vs_upsample": launches,
                    "output_bit_identical": {k: same(v, ref) for k, v in got.items()}}
        del model, base, gm, ref, got, x
        torch.cuda.empty_cache()
    return out


def affine_inference(dev, reps=10, batch=256, rounds=5):
    """The reference's own quantization executed in integers (int8.convert_affine) on torchvision MobileNetV2 and ResNet-18 in
    the reference's inference state (tests/affine_calibrated.py: BN fold, equalization, bias correction, quantize_targ_layer's
    8-bit weights, observer ranges over synthetic images), timed alternately with the fake-quantized model it replaces
    (QuantN* layers: only the inputs of the target layers are quantized, no functional-op observers) and with the ncnn
    per-layer int8 model (convert_to_int8 on the same equalized fp32 weights, activation scales from the same observers),
    `rounds` rounds of `reps` passes, median; and the relative logit error (2-norm over the batch) of each against the
    fake-quantized model."""
    import copy
    import statistics
    from collections import OrderedDict
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_calibrated
    from dfq_b200 import int8
    from dfq_b200.utils import quantize as Q

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds}
    try:
        x = torch.randn(batch, 3, 224, 224, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).clamp_(-2.5, 2.5)
        for net in ("mobilenet_v2", "resnet18"):
            fq, _, qtarg, pre = affine_calibrated.calibrated(net, keep_unquantized=True)
            aff = copy.deepcopy(fq)
            int8.convert_affine(aff, OrderedDict((id(m), m) for m in aff.modules() if type(m) in qtarg), qtarg)
            int8.convert_to_int8(pre, OrderedDict((id(m), m) for m in pre.modules() if type(m) in qtarg), qtarg)
            arms = (("fake_quant", fq), ("affine_int8", aff), ("ncnn_int8_per_layer", pre))
            with torch.no_grad():
                ref = fq(x)
                err = {k: float((m(x) - ref).norm() / ref.norm()) for k, m in arms[1:]}
                for _ in range(2):
                    for _, m in arms:
                        m(x)
                torch.cuda.synchronize(dev)
                ms = {k: [] for k, _ in arms}
                for _ in range(rounds):
                    for k, m in arms:
                        ms[k].append(timed(lambda m=m: m(x)))
            med = {k: statistics.median(v) for k, v in ms.items()}
            out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                        "ms_per_batch_rounds": ms, "rel_logit_error_vs_fake_quant": err,
                        "layers": sum(1 for m in aff.modules() if isinstance(m, int8._AffineInt8Layer))}
            del fq, aff, pre
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def affine_chained_inference(dev, reps=10, batch=256, rounds=5):
    """The affine int8 path with activations carried as the consumers' shifted codes (int8.chain_affine) on the networks of
    affine_inference, timed alternately with the fake-quantized model and the per-layer convert_affine model, `rounds`
    rounds of `reps` passes, median: images/s, ms per batch, edges and fused adds, the fp32 traffic the residual arm avoids
    per batch against the per-layer path (computed from shapes), and bit-identity of the three affine arms' logits
    (asserted)."""
    import copy
    import statistics
    from collections import OrderedDict
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_calibrated
    from dfq_b200 import int8

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds,
           "fp32_bytes_avoided_note": "fp32 bytes of the per-layer path that the residual arm does not move, per batch: per "
                                      "element of every carried tensor, the quantizer's fp32 read (4 B) per carried consumer, "
                                      "plus the producer's fp32 store (4 B) when no fp32 consumer is left; a read and a write "
                                      "(8 B) per deleted pass-through; per fused add, its two reads and its write (12 B)"}
    try:
        x = torch.randn(batch, 3, 224, 224, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).clamp_(-2.5, 2.5)
        for net in ("mobilenet_v2", "resnet18"):
            fq, _, qtarg = affine_calibrated.calibrated(net)
            aff = copy.deepcopy(fq)
            int8.convert_affine(aff, OrderedDict((id(m), m) for m in aff.modules() if type(m) in qtarg), qtarg)
            chained = int8.chain_affine(aff)
            gm = int8.chain_affine(aff, residual=True)
            arms = (("fake_quant", fq), ("affine_per_layer", aff), ("affine_chained", chained), ("affine_residual", gm))
            numel, mods = {}, dict(aff.named_modules())
            hooks = [m.register_forward_hook(lambda m, i, o, n=n: numel.__setitem__(n, o.numel())) for n, m in mods.items()
                     if isinstance(m, int8.AffineInt8Conv2d)]
            with torch.no_grad():
                ref = aff(x)
                for h in hooks:
                    h.remove()
                logits = {k: m(x) for k, m in arms[2:]}
                same = {k: bool(torch.equal(ref.view(torch.int32), v.view(torch.int32))) for k, v in logits.items()}
                assert all(same.values()), same
                traced, kept = int8._Int8Tracer().trace(aff), {n.name for n in gm.graph.nodes}
                avoided = sum(4 * numel[p] for p, _, _ in gm.requantized_edges)
                avoided += sum(4 * numel[n] for n, m in gm.named_modules() if isinstance(m, int8.AffineInt8Conv2d) and
                               m.epilogue is not None and m.epilogue.out_scale is not None and not m.epilogue.fp32)
                for n in traced.nodes:
                    if n.name in kept or n.op not in ("call_module", "call_function", "call_method"):
                        continue
                    src = n.args[0] if n.args and isinstance(n.args[0], torch.fx.Node) else None
                    while src is not None and not (src.op == "call_module" and src.target in numel):
                        src = src.args[0] if src.args and isinstance(src.args[0], torch.fx.Node) else None
                    if src is not None:
                        avoided += numel[src.target] * (12 if int8._is_add(n) else 8)
                for _ in range(2):
                    for _, m in arms:
                        m(x)
                torch.cuda.synchronize(dev)
                ms = {k: [] for k, _ in arms}
                for _ in range(rounds):
                    for k, m in arms:
                        ms[k].append(timed(lambda m=m: m(x)))
            med = {k: statistics.median(v) for k, v in ms.items()}
            out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                        "ms_per_batch_rounds": ms, "edges": {"chained": len(chained.requantized_edges),
                                                             "residual": len(gm.requantized_edges)},
                        "fused_adds": len(gm.fused_adds), "fp32_bytes_avoided_per_batch": avoided,
                        "logits_bit_identical_to_per_layer": same}
            del fq, aff, chained, gm, logits
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def affine_observed_inference(dev, reps=10, batch=256, rounds=5):
    """MobileNetV2 (the reference's mean head) and ResNet-18 in the reference's evaluation state: the fake-quantized model,
    convert_affine per layer and chain_affine(residual=True), all with replace_op() active, timed alternately, `rounds`
    rounds of `reps` passes, median; the fused adds and observers, and bit-identity of the two affine arms' logits
    (asserted)."""
    import copy
    import statistics
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_observed_state
    from dfq_b200 import int8

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds}
    try:
        x = torch.randn(batch, 3, 224, 224, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).clamp_(-2.5, 2.5)
        for net in ("mobilenet_v2", "resnet18"):
            with affine_observed_state.evaluation_state(net) as (model, qgraph, qtarg):
                fq = copy.deepcopy(model)
                int8.convert_affine(model, qgraph, qtarg)
                gm = int8.chain_affine(model, residual=True)
                arms = (("fake_quant", fq), ("affine_per_layer", model), ("affine_observed", gm))
                with torch.no_grad():
                    same = bool(torch.equal(model(x).view(torch.int32), gm(x).view(torch.int32)))
                    assert same, net
                    for _ in range(2):
                        for _, m in arms:
                            m(x)
                    torch.cuda.synchronize(dev)
                    ms = {k: [] for k, _ in arms}
                    for _ in range(rounds):
                        for k, m in arms:
                            ms[k].append(timed(lambda m=m: m(x)))
                med = {k: statistics.median(v) for k, v in ms.items()}
                kinds = [w for _, w, _ in gm.fused_observers]
                out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                            "ms_per_batch_rounds": ms, "observers": model.custom_tensor_op.len,
                            "fused_observers": {k: kinds.count(k) for k in ("operand", "residual", "output")},
                            "fused_adds": len(gm.fused_adds), "edges": len(gm.requantized_edges),
                            "logits_bit_identical_to_per_layer": same}
                del fq, gm
            del model
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def affine_distilled_inference(dev, reps=10, batch=256, rounds=5):
    """MobileNetV2 (the reference's mean head) and ResNet-18 in the reference's --distill_range state
    (tests/affine_distilled_state.py: QConv2d / QLinear, which quantize their weights and bias on every forward, ranges from
    update_quant_range, replace_op() active): the fake-quantized model, convert_affine per layer and
    chain_affine(residual=True), timed alternately, `rounds` rounds of `reps` passes, median; bit-identity of the two
    affine arms' logits (asserted)."""
    import copy
    import statistics
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_distilled_state
    from dfq_b200 import int8

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x224x224", "unit": "images/s", "reps": reps, "rounds": rounds}
    try:
        for net in ("mobilenet_v2", "resnet18"):
            x = affine_distilled_state.inputs(net, batch, 224, torch.Generator(device=dev).manual_seed(3))
            with affine_distilled_state.distilled_state(net) as (model, qgraph, qtarg):
                fq = copy.deepcopy(model)
                int8.convert_affine(model, qgraph, qtarg)
                gm = int8.chain_affine(model, residual=True)
                arms = (("fake_quant", fq), ("affine_per_layer", model), ("affine_chained", gm))
                with torch.no_grad():
                    same = bool(torch.equal(model(x).view(torch.int32), gm(x).view(torch.int32)))
                    assert same, net
                    for _ in range(2):
                        for _, m in arms:
                            m(x)
                    torch.cuda.synchronize(dev)
                    ms = {k: [] for k, _ in arms}
                    for _ in range(rounds):
                        for k, m in arms:
                            ms[k].append(timed(lambda m=m: m(x)))
                med = {k: statistics.median(v) for k, v in ms.items()}
                out[net] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                            "ms_per_batch_rounds": ms, "observers": model.custom_tensor_op.len,
                            "fused_observers": len(gm.fused_observers), "fused_adds": len(gm.fused_adds),
                            "logits_bit_identical_to_per_layer": same}
                del fq, gm
            del model
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def affine_layout_inference(dev, reps=10, batch=8, rounds=5, size=513):
    """DeepLab-v3+ (tests/deeplab_mobilenet_padded.py) in the reference's evaluation state at batch x 3 x size x size:
    convert_affine per layer, chain_affine(residual=True) and chain_affine(residual=True, concat=True, fold_pads=True),
    timed alternately, `rounds` rounds of `reps` passes, median; the three outputs asserted bit-identical.  What the new
    flags avoid is counted from the shapes of chain_affine(residual=True)'s graph (torch.fx ShapeProp): per folded pad,
    fused concatenation or fused upsample, its fp32 input read, its fp32 output written and read again by the consumer's
    quantizer, one launch for the node and one for that quantizer; per fused operand observer, its fp32 tensor read and
    written and one launch."""
    import statistics
    import torch
    from torch.fx.passes.shape_prop import ShapeProp
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_observed_state
    from dfq_b200 import int8

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def nbytes(n):
        m = n.meta.get("tensor_meta") if isinstance(n, torch.fx.Node) else None
        return 4 * int(torch.Size(m.shape).numel()) if m is not None and hasattr(m, "shape") else 0

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"batch": batch, "image": "3x%dx%d" % (size, size), "unit": "images/s", "reps": reps, "rounds": rounds}
    try:
        x = torch.randn(batch, 3, size, size, device=dev, generator=torch.Generator(device=dev).manual_seed(3)).clamp_(-2.5,
                                                                                                                   2.5)
        with affine_observed_state.evaluation_state("deeplab", size=129) as (model, qgraph, qtarg):
            int8.convert_affine(model, qgraph, qtarg)
            base = int8.chain_affine(model, residual=True)
            gm = int8.chain_affine(model, residual=True, concat=True, fold_pads=True)
            arms = (("affine_per_layer", model), ("chain_affine_residual", base), ("chain_affine_concat_fold_pads", gm))
            with torch.no_grad():
                ys = [m(x) for _, m in arms]
                same = all(torch.equal(ys[0].view(torch.int32), y.view(torch.int32)) for y in ys[1:])
                assert same, "the three arms differ"
                del ys
                ShapeProp(base).propagate(x)
                for _ in range(2):
                    for _, m in arms:
                        m(x)
                torch.cuda.synchronize(dev)
                ms = {k: [] for k, _ in arms}
                for _ in range(rounds):
                    for k, m in arms:
                        ms[k].append(timed(lambda m=m: m(x)))
            fused = {t[0] for t in gm.folded_pads} | {t[0] for t in gm.fused_cats} | {t[0] for t in gm.fused_upsamples}
            avoided, launches = 0, 0
            for n in base.graph.nodes:
                if n.name in fused:
                    ins = n.args[0] if n.args and isinstance(n.args[0], (list, tuple)) else n.args[:1]
                    avoided += sum(nbytes(a) for a in ins) + 2 * nbytes(n)
                    launches += 2
            cat_obs = [o for o, w, _ in gm.fused_observers if w == "cat"]
            for n in base.graph.nodes:
                if n.op == "call_module" and n.target in cat_obs:
                    avoided += 2 * nbytes(n)
                    launches += 1
            med = {k: statistics.median(v) for k, v in ms.items()}
            out["deeplab"] = {"images_per_s": {k: batch / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                              "ms_per_batch_rounds": ms, "folded_pads": len(gm.folded_pads),
                              "fused_cats": len(gm.fused_cats), "fused_upsamples": len(gm.fused_upsamples),
                              "fused_observers": len(gm.fused_observers), "edges": len(gm.requantized_edges),
                              "edges_residual_only": len(base.requantized_edges),
                              "fp32_bytes_avoided_per_batch": avoided, "launches_avoided_per_batch": launches,
                              "outputs_bit_identical": same}
            del base, gm
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def affine_pool_heads_inference(dev, reps=10, batch=256, rounds=5, ssd_batch=256):
    """Networks in the reference's evaluation state, replace_op() active, each timed alternately in three arms (per-layer
    convert_affine, chain_affine without the new flag, the same call with it), `rounds` rounds of `reps` passes, median,
    the arms' outputs asserted bit-identical: ResNet-18 (residual=True, then pools=True) and GoogLeNet (residual=True,
    concat=True, then pools=True) at batch x 3 x 224 x 224, SSD-Lite (tests/ssd_lite_like.py, is_test; residual=True,
    concat=True, fold_pads=True, then heads=True) at ssd_batch x 3 x 300 x 300.  The fp32 bytes the flag avoids are counted
    from the shapes of the arm without it (torch.fx ShapeProp): per fused pool its fp32 output written and read by its
    consumers' quantizer, and in codes mode its fp32 input written and read; per fused head its NCHW output written and
    read by the permute copy, that copy written and read by the cat (and by the operand's observer, written and read
    again, when it has one); per fused tail observer the concatenation read and written."""
    import statistics
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affine_observed_state
    from dfq_b200 import int8

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def same(a, b):
        if isinstance(a, (tuple, list)):
            return all(same(u, v) for u, v in zip(a, b))
        return bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))

    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    out = {"unit": "images/s", "reps": reps, "rounds": rounds}
    nets = (("resnet18", 224, batch, {}, "pools"), ("googlenet", 224, batch, {"concat": True}, "pools"),
            ("ssd", 300, ssd_batch, {"concat": True, "fold_pads": True}, "heads"))
    try:
        for net, size, n, kw, flag in nets:
            x = torch.randn(n, 3, size, size, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
            x.clamp_(-2.5, 2.5)
            with affine_observed_state.evaluation_state(net, size=size) as (model, qgraph, qtarg):
                int8.convert_affine(model, qgraph, qtarg)
                base = int8.chain_affine(model, residual=True, **kw)
                gm = int8.chain_affine(model, residual=True, **kw, **{flag: True})
                arms = (("affine_per_layer", model), ("affine_chained", base), ("affine_chained_" + flag, gm))
                with torch.no_grad():
                    ref = model(x)
                    ok = all(same(ref, m(x)) for _, m in arms[1:])
                    assert ok, net
                    for _, m in arms:
                        m(x)
                    torch.cuda.synchronize(dev)
                    ms = {k: [] for k, _ in arms}
                    for _ in range(rounds):
                        for k, m in arms:
                            ms[k].append(timed(lambda m=m: m(x)))
                    size_of = _fp32_bytes(base, x)
                med = {k: statistics.median(v) for k, v in ms.items()}
                avoided = 0
                for name, mode, _ in getattr(gm, "fused_pools", []):
                    i_bytes, o_bytes = size_of[name]
                    avoided += 2 * o_bytes + (2 * i_bytes if mode == "codes" else 0)
                heads = getattr(gm, "fused_heads", [])
                observed = {(what, p) for _, what, p in gm.fused_observers}
                for _, producers, _ in heads:
                    for p in producers:
                        e = size_of[p][1]
                        avoided += 4 * e + (2 * e if ("head", p) in observed else 0) + \
                            (2 * e if ("tail", p) in observed else 0)
                rec = {"batch": n, "image": "3x%dx%d" % (size, size),
                       "images_per_s": {k: n / (v * 1e-3) for k, v in med.items()}, "ms_per_batch": med,
                       "ms_per_batch_rounds": ms, "fused_observers": len(gm.fused_observers),
                       "observers": model.custom_tensor_op.len,
                       "edges": [len(base.requantized_edges), len(gm.requantized_edges)],
                       "fp32_bytes_avoided_per_batch": avoided, "outputs_bit_identical": ok}
                if flag == "pools":
                    rec["fused_pools"] = [p[:2] for p in gm.fused_pools]
                    rec["fused_cats"] = len(getattr(gm, "fused_cats", []))
                else:
                    rec["fused_heads"] = [(c, len(ps), k) for c, ps, k in heads]
                    rec["fused_observers_by_kind"] = {w: sum(1 for _, v, _ in gm.fused_observers if v == w)
                                                      for w in ("residual", "operand", "output", "cat", "head", "tail")}
                out[net] = rec
                del base, gm
            del model, x
            torch.cuda.empty_cache()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return out


def _fp32_bytes(gm, x):
    """{node name and call_module target: (bytes of its first tensor argument, of its output)} of gm's nodes with a
    single tensor output, from torch.fx ShapeProp on x."""
    from torch.fx.passes.shape_prop import ShapeProp
    ShapeProp(gm).propagate(x)
    out = {}
    for n in gm.graph.nodes:
        meta = n.meta.get("tensor_meta")
        if not hasattr(meta, "shape"):
            continue
        a = n.args[0] if n.args and hasattr(n.args[0], "meta") else None
        am = a.meta.get("tensor_meta") if a is not None else None
        nbytes = (am.shape.numel() * am.dtype.itemsize if hasattr(am, "shape") else 0, meta.shape.numel() * meta.dtype.itemsize)
        out[n.name] = nbytes
        if n.op == "call_module":
            out[n.target] = nbytes
    return out


def card():
    """Name and power limit of the GPU (read only)."""
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0:
            out["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        pass
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--reps", type=int, default=10, help="timed forward passes per arm (after 2 warm-up passes)")
    p.add_argument("--seg-batch", type=int, default=8, help="batch of the 513x513 segmentation networks (upsample, layout)")
    p.add_argument("--ssd-batch", type=int, default=256, help="batch of the 300x300 SSD-Lite (layout)")
    p.add_argument("--sections", default="int8,chained,residual,pool_cat,upsample,layout",
                   help="comma-separated sections to run (default: all but affine, affine_chained, affine_observed, "
                        "affine_layout, affine_pool_heads and affine_distilled)")
    args = p.parse_args()
    want = set(args.sections.split(","))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_int8.py needs a CUDA device (H100)")
    dev = torch.device("cuda", 0)
    res = int8_inference(dev, reps=args.reps, batch=args.batch) if "int8" in want else {}
    if "chained" in want:
        res["chained"] = chained_inference(dev, reps=args.reps, batch=args.batch)
    if "residual" in want:
        res["residual"] = residual_inference(dev, reps=args.reps, batch=args.batch)
    if "pool_cat" in want:
        res["pool_cat"] = pool_cat_inference(dev, reps=args.reps, batch=args.batch)
    if "upsample" in want:
        res["upsample"] = upsample_inference(dev, reps=args.reps, batch=args.seg_batch)
    if "layout" in want:
        res["layout"] = layout_inference(dev, reps=args.reps, seg_batch=args.seg_batch, ssd_batch=args.ssd_batch)
    if "affine" in want:
        res["affine"] = affine_inference(dev, reps=args.reps, batch=args.batch)
    if "affine_chained" in want:
        res["affine_chained"] = affine_chained_inference(dev, reps=args.reps, batch=args.batch)
    if "affine_observed" in want:
        res["affine_observed"] = affine_observed_inference(dev, reps=args.reps, batch=args.batch)
    if "affine_layout" in want:
        res["affine_layout"] = affine_layout_inference(dev, reps=args.reps, batch=args.seg_batch)
    if "affine_pool_heads" in want:
        res["affine_pool_heads"] = affine_pool_heads_inference(dev, reps=args.reps, batch=args.batch,
                                                               ssd_batch=args.ssd_batch)
    if "affine_distilled" in want:
        res["affine_distilled"] = affine_distilled_inference(dev, reps=args.reps, batch=args.batch)
    res["gpu"] = card()
    print(json.dumps({"int8": res}))


if __name__ == "__main__":
    main()
