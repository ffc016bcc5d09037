"""A calibrated torchvision network in the reference's inference state, for the affine int8 tests and tools/bench_int8.py
(needs a CUDA device and torchvision)."""
import copy
from collections import OrderedDict

import torch
import torch.nn as nn


def calibrated(net, batches=4, keep_unquantized=False, bits_weight=8, bits_bias=16, quantize_on_cpu=False):
    """torchvision `net` (seeded, ReLU6 -> ReLU for MobileNetV2 as main_cls.py --relu does) through BN fold, equalization and
    bias correction on its Conv2d / Linear layers, then QuantNConv2d / QuantNLinear layers with quantize_targ_layer's
    `bits_weight`-bit weights (`bits_bias`-bit biases) and observer ranges driven over `batches` batches of 16 synthetic
    images (update_quant_range's way).  quantize_on_cpu: quantize_targ_layer runs before the model moves to the GPU, as in
    the reference's main_cls.py / main_seg.py / main_ssd.py, so the parameters are fake-quantized with true division (the
    CPU recipe) instead of the reciprocal multiply of CUDA tensors.  Returns (model, graph of its target layers, target
    types) and, with keep_unquantized, a copy of the model from before quantize_targ_layer whose observers hold the same
    ranges (the input of int8.convert_to_int8)."""
    import torchvision
    from dfq_b200 import dfq
    from dfq_b200.improve_dfq import set_update_stat
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
    torch.manual_seed(0)
    model = getattr(torchvision.models, net)(num_classes=1000).eval()
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)

    def relu(parent):
        for name, ch in list(parent.named_children()):
            if isinstance(ch, nn.ReLU6):
                setattr(parent, name, nn.ReLU(inplace=True))
            else:
                relu(ch)
    relu(model)
    targ = [nn.Conv2d, nn.Linear]
    graph, bottoms = trace_graph(model)
    LT.merge_batchnorm(model, graph, bottoms, targ)
    dfq.cross_layer_equalization(graph, create_relation(graph, bottoms, targ, delete_single=False), targ, converge_thres=2e-7)
    dfq.bias_correction(graph, bottoms, targ)

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d:
                q = Q.QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation, ch.groups,
                                   ch.bias is not None)
            elif type(ch) is nn.Linear:
                q = Q.QuantNLinear(ch.in_features, ch.out_features, ch.bias is not None)
            else:
                swap(ch)
                continue
            q.load_state_dict(ch.state_dict(), strict=False)
            setattr(parent, name, q)
    swap(model)
    model = model.eval() if quantize_on_cpu else model.cuda().eval()
    qtarg = [Q.QuantNConv2d, Q.QuantNLinear]
    qgraph = OrderedDict((id(m), m) for m in model.modules() if type(m) in qtarg)
    pre = copy.deepcopy(model) if keep_unquantized else None
    LT.quantize_targ_layer(qgraph, bits_weight, bits_bias, qtarg)
    if quantize_on_cpu:
        model.cuda()
        pre = None if pre is None else pre.cuda()
    set_update_stat(model, [Q.QuantMeasure], True)
    g = torch.Generator(device="cuda").manual_seed(1)
    with torch.no_grad():
        for _ in range(batches):
            model(torch.randn(16, 3, 224, 224, device="cuda", generator=g).clamp_(-2.5, 2.5))
    set_update_stat(model, [Q.QuantMeasure], False)
    if pre is None:
        return model, qgraph, qtarg
    for a, b in zip(model.modules(), pre.modules()):
        if isinstance(a, Q.QuantMeasure):
            b.running_min.copy_(a.running_min); b.running_max.copy_(a.running_max)
    return model, qgraph, qtarg, pre
