"""Data-free calibration passes: drop-in for the reference's ``dfq.py``.

Same public names, signatures, prints and in-place semantics as jakc4103/DFQ ``dfq.py``:

    _quantize_error            dfq.py:8-25
    _layer_equalization        dfq.py:28-75
    cross_layer_equalization   dfq.py:78-117
    bias_absorption            dfq.py:121-164
    clip_weight                dfq.py:167-170
    bias_correction            dfq.py:173-293

Host code walks the graph and builds descriptor tables; every tensor operation runs in
libdfq_sm90.so (include/dfq_b200.h).  Parameters may live on the CPU (as in main_cls.py, where
calibration happens before ``model.cuda()``) or on the GPU: they are staged into a device arena, the
kernels run there, and the results are written back into the SAME parameter storages.
"""
import torch
import torch.nn as nn

from . import _lib
from .engine import Session
from .graphwalk import bias_correction_recipe, relu_between
from .utils import visualize_per_layer   # noqa: F401  (dfq.py:5 imports it; kept for API parity)
from .utils import quantize as _Q
from .utils.quantize import UniformQuantize, tensor_minmax, _ptr  # noqa: F401


def _zero_bias(layer):
    """dfq.py:91-92 / :160-161 / :290-291: a missing bias becomes a zero Parameter(requires_grad=False)."""
    layer.bias = nn.Parameter(data=torch.zeros((layer.weight.size(0)), dtype=torch.float32, device=layer.weight.device),
                              requires_grad=False)
    return layer.bias


def _quantize_error(param, num_bits=8, reduction='sum', signed=False):
    """!
    reduction should be one of 'sum', 'mean', 'none', 'channel', default to 'sum'
    """
    lib = _lib.load()
    _lib.require_cuda()
    src = param.detach()
    dev, _ = _Q._dev_f32(src)
    with torch.no_grad():
        mm = tensor_minmax(dev)
        eps = torch.empty_like(dev)
        # CPU tensors: true division; CUDA tensors: the reference would run div_(float) as a reciprocal multiply
        if src.is_cuda:
            eps = _Q.fake_quant_device_range(dev, num_bits, mm[0:1], mm[1:2], signed, prologue=0, div_mode=1) - dev
        else:
            _lib.check(lib.dfq_quant_error(_ptr(dev), _ptr(eps), dev.numel(), _ptr(mm), int(num_bits), 1 if signed else 0,
                                           _lib.stream_ptr()), "dfq_quant_error")
        if reduction == 'sum':
            eps = torch.sum(torch.abs(eps))
        elif reduction == 'mean':
            eps = torch.mean(eps)
        elif reduction == 'channel':
            eps = torch.sum(torch.abs(torch.sum(eps.view(eps.size(0), -1), -1)))
        elif reduction == 'spatial':
            eps = torch.sum(torch.abs(torch.sum(eps.view(eps.size(0), eps.size(1), -1), -1)))
        return eps if src.is_cuda else eps.cpu()   # a no-op copy when the tensors are already on the host


def _layer_equalization(weight_first, weight_second, bias_first, bn_weight=None, bn_bias=None, s_range=(1e-8, 1e8), signed=False, eps=0):
    """One equalization pass over a pair of layers, in place; returns (W1, W2, b1, S) like dfq.py:28-75."""
    with torch.no_grad():
        sess = Session()
        l1 = sess.add_layer(weight_first, bias_first)
        l2 = sess.add_layer(weight_second, None)
        obw = sess.bind(bn_weight) if bn_weight is not None else -1
        obb = sess.bind(bn_bias) if bn_bias is not None else -1
        sess.upload()
        _, s_offs = sess.run_cle([(l1, l2, obw, obb)], s_range=s_range, signed=signed, eps=eps, max_sweeps=1)
        S = sess.view(s_offs[0], weight_first.shape[0]).clone()
        sess.download()
    return weight_first, weight_second, bias_first, (S if weight_first.is_cuda else S.cpu())


def cross_layer_equalization(graph, relations, targ_type, s_range=[1e-8, 1e8], range_thres=0, converge_thres=2e-7, converge_count=20, signed=False, eps=0, visualize_state=False):
    print("Start cross layer equalization")
    with torch.no_grad():
        if not relations:
            return
        if not (10 > converge_thres and 0 < converge_count):      # dfq.py:81-83: the loop body never runs
            return
        sess = Session()
        index = {}

        def layer_of(key, need_bias):
            if key not in index:
                mod = graph[key]
                if need_bias and mod.bias is None:                  # only `first` layers get one (dfq.py:91-92)
                    _zero_bias(mod)
                index[key] = sess.add_layer(mod.weight, mod.bias)
            elif need_bias and graph[key].bias is None:
                sess.attach_bias(index[key], _zero_bias(graph[key]))
            return index[key]

        table = []
        bn_bound = {}
        for rr in relations:
            first, second, bn_idx = rr.get_idxs()
            if visualize_state:
                visualize_per_layer(graph[first].weight.detach(), 'Before equalization')
            l1 = layer_of(first, True)
            l2 = layer_of(second, False)
            if bn_idx not in bn_bound:
                bn = graph[bn_idx]
                bn_bound[bn_idx] = (sess.bind(bn.fake_weight), sess.bind(bn.fake_bias))
            table.append((l1, l2) + bn_bound[bn_idx])
        sess.upload()
        if _forward_chain_order(table):
            res, s_offs = sess.run_cle(table, s_range=s_range, converge_thres=converge_thres, converge_count=converge_count,
                                       signed=signed, eps=eps)
            scale_vecs = [sess.view(off, sess.layer(t[0])["rows"]).clone() for off, t in zip(s_offs, table)]
        else:
            res, scale_vecs = _equalize_any_order(sess, table, s_range, converge_thres, converge_count, signed, eps)
        sess.download()
        for rr, S in zip(relations, scale_vecs):
            first = rr.get_idxs()[0]
            # the reference builds S on the CPU (dfq.py:37) and re-assigns the parameters (dfq.py:95)
            rr.set_scale_vec(S if graph[first].weight.is_cuda else S.cpu())
            if visualize_state:
                visualize_per_layer(graph[first].weight.detach(), 'After equalization')
        cross_layer_equalization.last_result = res


def _forward_chain_order(table):
    """True when the fused persistent kernel applies: every layer is `first` of at most one relation and `second` of at
    most one, and a layer's incoming relation precedes its outgoing one (what create_relation emits)."""
    as_first, as_second = {}, {}
    for i, (a, b, _, _) in enumerate(table):
        if a in as_first or b in as_second:
            return False
        as_first[a] = i
        as_second[b] = i
    return all(as_second[l] < as_first[l] for l in as_first if l in as_second)


def _equalize_any_order(sess, table, s_range, converge_thres, converge_count, signed, eps):
    """Relation lists in an arbitrary order (hand-written lists; never produced by create_relation): the Gauss-Seidel
    order of dfq.py:85-103 is kept by running ONE relation per launch (dfq_cle_run with max_sweeps=1), and the exit rule of
    dfq.py:105-115 on the host from dfq_mean_abs_diff over device snapshots.  Slow path: one launch per relation."""
    import ctypes as C
    from .engine import CleResult
    lib = _lib.load()
    plans = [sess.plan_cle([t]) for t in table]
    sess._ensure_room()
    layers = sorted({t[0] for t in table} | {t[1] for t in table})
    S = [None] * len(table)
    out = torch.zeros(1, dtype=torch.float64, device=sess.device)
    diff, count, n, diffs = 10, 0, 0, []
    while diff > converge_thres and count < converge_count:
        prev = {l: sess.view(sess.layer(l)["w_off"], sess.layer(l)["rows"] * sess.layer(l)["cols"] * sess.layer(l)["kk"]).clone()
                for l in layers}
        for i, plan in enumerate(plans):
            sess.run_cle_plan(plan, s_range, converge_thres, converge_count, signed, eps, max_sweeps=1)
            s = sess.view(plan["s_offs"][0], sess.layer(table[i][0])["rows"]).clone()
            S[i] = s if S[i] is None else S[i] * s                       # relation.py:20-24
        diff_tmp = 0.0
        for l in layers:
            cur = sess.view(sess.layer(l)["w_off"], prev[l].numel())
            _lib.check(lib.dfq_mean_abs_diff(_ptr(cur), _ptr(prev[l]), prev[l].numel(), C.c_void_p(out.data_ptr()),
                                             _lib.stream_ptr()), "dfq_mean_abs_diff")
            diff_tmp += float(out.item())
        diffs.append(diff_tmp)
        n += 1
        if abs(diff - diff_tmp) > 1e-9:
            count, diff = 0, diff_tmp
        else:
            count += 1
    return CleResult(n, True, float(diff), diffs), S


def bias_absorption(graph, relations, bottoms, N=3):
    print("Absorbing bias")
    with torch.no_grad():
        todo = []
        for rr in relations:
            first, second, bn_idx = rr.get_idxs()
            if not relu_between(graph, bottoms, second, first):
                continue
            bn = graph[bn_idx]
            # c = clamp(beta - N*gamma, 0)   (dfq.py:143-144), a [C] vector
            c = (bn.fake_bias.detach().clone() - N * bn.fake_weight.detach().clone())
            c.clamp_(0)
            for key in (first, second):
                if graph[key].bias is None:
                    _zero_bias(graph[key])
            todo.append((first, second, bn, c))
        if not todo:
            return
        # wc = (sum_k W2) @ c per group (dfq.py:139-153): one pass over every W2, all relations in ONE launch.  The
        # relations are independent (c reads the FIRST layer's BN, which no relation writes before its own turn) except
        # for the order of the two updates that land in a middle layer's bias: `+= wc` as second of relation k, then
        # `-= c` as first of relation k+1 (dfq.py:162-164).  Device first (all the `+= wc`), host afterwards (all the
        # `-= c`) keeps that order whenever a layer's incoming relation precedes its outgoing one (create_relation's
        # order); any other list falls back to one launch per relation.
        seconds = [t[1] for t in todo]
        batched = len(set(seconds)) == len(seconds) and all(
            t[0] not in seconds or seconds.index(t[0]) < i for i, t in enumerate(todo))
        for group in ([todo] if batched else [[t] for t in todo]):
            sess = Session()
            items = []
            for first, second, bn, c in group:
                l2 = sess.add_layer(graph[second].weight, graph[second].bias, weight_writeback=False)
                oc = sess.bind(c, writeback=False)
                items.append(dict(layer=l2, signed=False, level=0, next_bn_b_off=-1, raw_sum=True, add=True,
                                  terms=[dict(bn_w_off=oc, bn_b_off=oc, n=c.numel(), relu=False, op="set")]))
            sess.upload()
            sess.run_bias_correct(items)
            sess.download()
            for first, second, bn, c in group:
                graph[first].bias.data.add_(-c.to(graph[first].bias.device))
                bn.fake_bias.data.add_(-c)


def clip_weight(graph, range_clip=[-15, 15], targ_type=[nn.Conv2d, nn.Linear]):
    lib = _lib.load()
    _lib.require_cuda()
    for idx in graph:
        if type(graph[idx]) in targ_type:
            w = graph[idx].weight.data
            dev, _ = _Q._dev_f32(w)
            if dev.data_ptr() == w.data_ptr():
                dev = dev.clone()
            _lib.check(lib.dfq_clamp(_ptr(dev), dev.numel(), float(range_clip[0]), float(range_clip[1]), _lib.stream_ptr()),
                       "dfq_clamp")
            w.copy_(dev.view(w.shape))


def bias_correction(graph, bottoms, targ_type, bits_weight=8, bn_type=torch.nn.BatchNorm2d, signed=False):
    """
    Perform bias correction.
    Expectation of input activations will be summed for elementwise addition, concate for torch.cat
    """
    print("Start bias correction")
    with torch.no_grad():
        recipe = bias_correction_recipe(graph, bottoms, targ_type, bn_type)
        if not recipe:
            return
        sess = Session()
        bn_bound = {}

        def bn_offsets(key):
            if key not in bn_bound:
                bn = graph[key]
                bn_bound[key] = (sess.bind(bn.fake_weight), sess.bind(bn.fake_bias))
            return bn_bound[key]

        items = []
        for step in recipe:
            mod = graph[step["layer"]]
            if mod.bias is None:
                _zero_bias(mod)                                       # dfq.py:290-291
            li = sess.add_layer(mod.weight, mod.bias, weight_writeback=False)
            terms = []
            for t in step["terms"]:
                ow, ob = bn_offsets(t["bn"])
                terms.append(dict(bn_w_off=ow, bn_b_off=ob, n=graph[t["bn"]].fake_bias.numel(), relu=t["relu"], op=t["op"]))
            nxt = bn_offsets(step["next_bn"])[1] if step["next_bn"] is not None else -1
            if step["next_bn"] is not None:
                assert graph[step["next_bn"]].fake_bias.numel() == mod.weight.size(0), \
                    "bias correction: the batch norm that follows has a different channel count"
            items.append(dict(layer=li, signed=signed, level=step["level"], next_bn_b_off=nxt, terms=terms))
        sess.upload()
        # quirk Q2 (dfq.py:218): the quantization error is always taken at 8 bits, whatever bits_weight says
        sess.run_bias_correct(items, num_bits=8)
        sess.download()
