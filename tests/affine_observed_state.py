"""Models in the reference's evaluation state (main_cls.py / main_seg.py / main_ssd.py --quantize), for the affine observer
tests and tools/bench_int8.py (needs a CUDA device; torchvision for the classifiers and SSD-Lite).

The state: BN fold, equalization and bias correction, QuantNConv2d / QuantNLinear layers with quantize_targ_layer's 8-bit
weights, a CustomTensorOP of one QuantMeasure per functional-op operand installed as `custom_tensor_op` (switch_layers'
way), every observer's range driven with update_stat over seeded synthetic batches while replace_op() is active
(update_quant_range's way), then update_stat off.  The functional-op records are taken from an eager run of the model's
own forwards: each Tensor.__add__ / __iadd__, torch.cat, torch.mean, F.interpolate and F.softmax called directly from a
function named `forward`, named <op>_<line>_<n> (add_<line>_2, torch_cat_<line>_<n>, ...).  This is the rule the patched
ops match records with (utils/layer_transform.py _called_from_forward_as), not the reference's tracer or trace_graph's
keys: the records' provenance is this package's reading of the reference's naming.  The keys (first elements) are not
read by the patched ops."""
import sys
from collections import OrderedDict
from contextlib import contextmanager

import torch
import torch.nn as nn
import torch.nn.functional as F


def mobilenet_v2_ref_head():
    """torchvision MobileNetV2 with the reference's head: torch.mean(x.view(N, C, -1), -1) instead of adaptive pooling."""
    import torchvision

    class MobileNetV2RefHead(torchvision.models.MobileNetV2):
        def forward(self, x):
            x = self.features(x)
            x = torch.mean(x.view(x.size(0), x.size(1), -1), -1)
            return self.classifier(x)
    return MobileNetV2RefHead(num_classes=1000)


def build(net):
    if net == "mobilenet_v2":
        return mobilenet_v2_ref_head()
    if net == "deeplab":
        from deeplab_mobilenet_padded import DeepLabMobileNetPadded
        return DeepLabMobileNetPadded()
    if net == "ssd":
        from ssd_lite_like import SSDLiteLike
        return SSDLiteLike(21, is_test=True)
    import torchvision
    return getattr(torchvision.models, net)(num_classes=1000)


def record_ops(model, x):
    """[(key, op name)] of the functional ops an eager forward of `model` on x calls directly from a `forward`, in order."""
    recs = []
    raw = {"__add__": torch.Tensor.__add__, "__iadd__": torch.Tensor.__iadd__, "cat": torch.cat, "mean": torch.mean,
           "interpolate": F.interpolate, "softmax": F.softmax}

    def note(stem, n):
        f = sys._getframe(2)
        if f.f_code.co_name == "forward":
            recs.append(("%s_%d" % (stem, len(recs) + 1), "%s_%d_%d" % (stem, f.f_lineno, n)))

    def add(a, b):
        note("add", 2)
        return raw["__add__"](a, b)

    def iadd(a, b):
        note("iadd", 2)
        return raw["__iadd__"](a, b)

    def cat(ts, dim=0):
        note("torch_cat", len(ts))
        return raw["cat"](ts, dim)

    def mean(t, *a, **k):
        note("torch_mean", 1)
        return raw["mean"](t, *a, **k)

    def interpolate(t, *a, **k):
        note("F_interpolate", 1)
        return raw["interpolate"](t, *a, **k)

    def softmax(t, *a, **k):
        note("F_softmax", 1)
        return raw["softmax"](t, *a, **k)
    torch.Tensor.__add__, torch.Tensor.__iadd__, torch.cat, torch.mean = add, iadd, cat, mean
    F.interpolate, F.softmax = interpolate, softmax
    try:
        with torch.no_grad():
            model(x)
    finally:
        torch.Tensor.__add__, torch.Tensor.__iadd__, torch.cat, torch.mean = (raw[k] for k in ("__add__", "__iadd__", "cat",
                                                                                                  "mean"))
        F.interpolate, F.softmax = raw["interpolate"], raw["softmax"]
    return recs


@contextmanager
def evaluation_state(net, batches=3, size=224, batch=8):
    """Yields (model, qgraph, qtarg) in the evaluation state with replace_op() active; restores the ops afterwards."""
    from dfq_b200 import dfq
    from dfq_b200.improve_dfq import set_update_stat
    from dfq_b200.trace import trace_graph
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
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
    dfq.bias_correction(graph, bottoms, targ)

    def swap(parent):
        for name, ch in list(parent.named_children()):
            if type(ch) is nn.Conv2d:
                q = Q.QuantNConv2d(ch.in_channels, ch.out_channels, ch.kernel_size, ch.stride, ch.padding, ch.dilation,
                                   ch.groups, ch.bias is not None)
            elif type(ch) is nn.Linear:
                q = Q.QuantNLinear(ch.in_features, ch.out_features, ch.bias is not None)
            else:
                swap(ch)
                continue
            q.load_state_dict(ch.state_dict(), strict=False)
            setattr(parent, name, q)
    swap(model)
    model = model.cuda().eval()
    qtarg = [Q.QuantNConv2d, Q.QuantNLinear]
    qgraph = OrderedDict((id(m), m) for m in model.modules() if type(m) in qtarg)
    LT.quantize_targ_layer(qgraph, 8, 16, qtarg)
    g = torch.Generator(device="cuda").manual_seed(1)
    recs = record_ops(model, torch.randn(2, 3, size, size, device="cuda", generator=g))
    observers = [Q.QuantMeasure(num_bits=8, momentum=0.1) for _, name in recs for _ in range(int(name.split("_")[-1]))]
    ct = LT.CustomTensorOP(observers, recs).cuda().eval()
    model.add_module("custom_tensor_op", ct)
    prev = LT.module_tensor_op
    LT.module_tensor_op = ct
    LT.replace_op()
    try:
        set_update_stat(model, [Q.QuantMeasure], True)
        with torch.no_grad():
            for _ in range(batches):
                model(torch.randn(batch, 3, size, size, device="cuda", generator=g).clamp_(-2.5, 2.5))
        set_update_stat(model, [Q.QuantMeasure], False)
        yield model, qgraph, qtarg
    finally:
        LT.restore_op()
        LT.module_tensor_op = prev
