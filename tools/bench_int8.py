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
1.1 and GoogLeNet.  The card's name and power limit are read in the same run and reported beside the numbers.  Needs a CUDA device; writes nothing.
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
    args = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_int8.py needs a CUDA device (H100)")
    dev = torch.device("cuda", 0)
    res = int8_inference(dev, reps=args.reps, batch=args.batch)
    res["chained"] = chained_inference(dev, reps=args.reps, batch=args.batch)
    res["residual"] = residual_inference(dev, reps=args.reps, batch=args.batch)
    res["pool_cat"] = pool_cat_inference(dev, reps=args.reps, batch=args.batch)
    res["gpu"] = card()
    print(json.dumps({"int8": res}))


if __name__ == "__main__":
    main()
