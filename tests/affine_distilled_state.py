"""Models in the reference's --distill_range and --trainable evaluation states (main_cls.py / main_seg.py / main_ssd.py),
for the per-forward affine tests and tools/bench_int8.py (needs a CUDA device; torchvision for the classifiers and
SSD-Lite).  The networks and the functional-op records are tests/affine_observed_state.py's.

The state: BN fold, equalization (create_relation(..., delete_single=False)) and bias correction, then the layers swapped
for the ones that quantize their own weights and bias on every forward - QConv2d / QLinear (distill_range; the
segmentation main swaps the convolutions only) or QuantConv2d / QuantLinear (trainable) - with set_layer_bits, a
CustomTensorOP of one QuantMeasure per functional-op operand installed as `custom_tensor_op`, and the ranges of every
observer driven by update_quant_range (replace_op() active) over seeded synthetic batches in the preprocessing range,
which then pins the data-input observer ([-2.11790393, 2.64], detection [-1, 1]); finally update_stat off, as the mains
do.  Distilled images are not needed: the range mechanics are the same for any batches."""
from collections import OrderedDict
from contextlib import contextmanager

import torch
import torch.nn as nn

from affine_observed_state import build, record_ops

KINDS = ("distill_range", "trainable")


def data_range(net):
    """(lo, hi) of the network's preprocessed input: what update_quant_range pins the data-input observer to."""
    return (-1.0, 1.0) if net == "ssd" else (-2.11790393, 2.64)


def inputs(net, n, size, generator):
    """n seeded images uniform in the network's preprocessing range."""
    lo, hi = data_range(net)
    return torch.rand(n, 3, size, size, device="cuda", generator=generator) * (hi - lo) + lo


def layer_types(net, kind):
    """(nn type -> per-forward type) of the main's swap for this network and state."""
    from dfq_b200.utils import quantize as Q
    conv, lin = (Q.QConv2d, Q.QLinear) if kind == "distill_range" else (Q.QuantConv2d, Q.QuantLinear)
    return {nn.Conv2d: conv} if net == "deeplab" else {nn.Conv2d: conv, nn.Linear: lin}


@contextmanager
def distilled_state(net, kind="distill_range", batches=3, size=224, batch=8, bits_weight=8, bits_bias=16):
    """Yields (model, qgraph, qtarg) in the state with replace_op() active; restores the ops afterwards."""
    from dfq_b200 import dfq
    from dfq_b200.improve_dfq import set_update_stat, update_quant_range
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
    if kind not in KINDS:
        raise ValueError("kind must be one of %s" % (KINDS,))
    torch.manual_seed(0)
    model = build(net).eval()
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    targ = [nn.Conv2d, nn.Linear]
    graph, bottoms = trace_graph(model)
    LT.merge_batchnorm(model, graph, bottoms, targ)
    dfq.cross_layer_equalization(graph, create_relation(graph, bottoms, targ, delete_single=False), targ, converge_thres=2e-7)
    dfq.bias_correction(graph, bottoms, targ, bits_weight=bits_weight)
    types = layer_types(net, kind)
    swapped = {}

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d and nn.Conv2d in types:
                q = types[nn.Conv2d](ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation,
                                     ch.groups, ch.bias is not None)
            elif type(ch) is nn.Linear and nn.Linear in types:
                q = types[nn.Linear](ch.in_features, ch.out_features, ch.bias is not None)
            else:
                swap(ch)
                continue
            q.load_state_dict(ch.state_dict(), strict=False)
            swapped[id(ch)] = q
            setattr(parent, name, q)
    swap(model)
    qtarg = list(types.values())
    qgraph = OrderedDict((id(m), m) for m in model.modules() if type(m) in qtarg)
    Q.set_layer_bits(qgraph, bits_weight, 8, bits_bias, qtarg)
    model = model.cuda().eval()
    set_update_stat(model, [Q.QuantMeasure], False)         # the records' forward must not move any range
    g = torch.Generator(device="cuda").manual_seed(1)
    recs = record_ops(model, inputs(net, 2, size, g))
    observers = [Q.QuantMeasure(num_bits=8, momentum=0.1) for _, name in recs for _ in range(int(name.split("_")[-1]))]
    ct = LT.CustomTensorOP(observers, recs).cuda().eval()
    model.add_module("custom_tensor_op", ct)
    prev = LT.module_tensor_op
    LT.module_tensor_op = ct
    try:
        # the traced graph with the swapped layers in place: update_quant_range pins the layer fed by "Data"
        rgraph = OrderedDict((k, swapped.get(id(v), v)) for k, v in graph.items())
        set_update_stat(model, [Q.QuantMeasure], True)
        update_quant_range(model, [inputs(net, batch, size, g) for _ in range(batches)], rgraph, bottoms,
                           is_detection=net == "ssd")
        set_update_stat(model, [Q.QuantMeasure], False)
        LT.replace_op()
        try:
            yield model, qgraph, qtarg
        finally:
            LT.restore_op()
    finally:
        LT.module_tensor_op = prev
