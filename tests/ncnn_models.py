"""Seeded models for ncnn.write round trips  --  TEST INFRASTRUCTURE.

resnet18_int8(): torchvision ResNet-18 (weights=None, seed 0) with each BatchNorm folded into its convolution, converted by
int8.convert_to_int8 with seeded activation scales: Convolution, max pool, residual adds, global average Pooling, Flatten
and InnerProduct in one model.
mobilenetv2_int8(): the reference's MobileNetV2 with `--relu` (its mean-over-a-view head and a Softmax) on the calibrated
layers of the bundled checkpoint: what convert_ncnn.py exported as modeling/ncnn/model_quant_relu_equal.
"""
import numpy as np
import torch
import torch.nn as nn


def resnet18_folded(seed=0):
    import torchvision
    from torch.nn.utils.fusion import fuse_conv_bn_eval
    torch.manual_seed(seed)
    m = torchvision.models.resnet18(weights=None).eval()
    g = torch.Generator().manual_seed(seed)
    pairs = [("conv1", "bn1")] + [("%s.%d.conv%d" % (l, b, i), "%s.%d.bn%d" % (l, b, i)) for l in
                                  ("layer1", "layer2", "layer3", "layer4") for b in (0, 1) for i in (1, 2)] + \
        [("%s.0.downsample.0" % l, "%s.0.downsample.1" % l) for l in ("layer2", "layer3", "layer4")]
    for cname, bname in pairs:
        bn = m.get_submodule(bname)
        bn.running_mean.copy_(torch.randn(bn.num_features, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
        bn.weight.data.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
        bn.bias.data.copy_(torch.randn(bn.num_features, generator=g) * 0.1)
        conv = fuse_conv_bn_eval(m.get_submodule(cname), bn)
        parent, _, leaf = cname.rpartition(".")
        setattr(m.get_submodule(parent) if parent else m, leaf, conv)
        parent, _, leaf = bname.rpartition(".")
        setattr(m.get_submodule(parent) if parent else m, leaf, nn.Identity())
    return m


def resnet18_int8(seed=0):
    """(converted model, graph, targ_type): the graph is {name: layer} of the target layers in forward order."""
    from dfq_b200 import int8 as I
    m = resnet18_folded(seed)
    graph = {n: l for n, l in m.named_modules() if isinstance(l, (nn.Conv2d, nn.Linear))}
    rng = np.random.default_rng(seed)
    scales = [float(np.float32(s)) for s in rng.uniform(4.0, 64.0, len(graph))]
    I.convert_to_int8(m, graph, (nn.Conv2d, nn.Linear), act_scales=scales)
    return m, graph, (nn.Conv2d, nn.Linear)


class RefTailMobileNetV2(nn.Module):
    """torchvision MobileNetV2's features with the reference's head: the mean of x.view(N, C, -1) over the last dim
    (modeling/classification/MobileNetV2.py), the classifier, and the Softmax convert_ncnn.py's model ends with."""

    def __init__(self, features, classifier):
        super().__init__()
        self.features, self.classifier, self.softmax = features, classifier, nn.Softmax(dim=1)

    def forward(self, x):
        x = self.features(x)
        x = torch.mean(x.view(x.size(0), x.size(1), -1), -1)
        return self.softmax(self.classifier(x))


def mobilenetv2_int8(graph, targ, act_scales):
    """(converted model, its {name: layer} graph, targ): the calibrated target layers of `graph` (the bundled checkpoint
    after BN fold and equalization, tests/ncnn_int8_case.calibrated_graph) in the reference's MobileNetV2 with `--relu`
    (ReLU6 -> ReLU, BatchNorm folded away), converted by int8.convert_to_int8 at `act_scales`."""
    import copy
    import torchvision
    from dfq_b200 import int8 as I
    tv = torchvision.models.mobilenet_v2(weights=None).eval()
    model = RefTailMobileNetV2(tv.features, tv.classifier[1])
    for name, m in list(model.named_modules()):
        if isinstance(m, (nn.BatchNorm2d, nn.ReLU6)):
            parent, _, leaf = name.rpartition(".")
            setattr(model.get_submodule(parent), leaf, nn.Identity() if isinstance(m, nn.BatchNorm2d) else nn.ReLU())
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    mine = [(n, m) for n, m in model.named_modules() if isinstance(m, (nn.Conv2d, nn.Linear))]
    assert len(mine) == len(layers) == 53
    for (name, m), src in zip(mine, layers):
        assert m.weight.shape == src.weight.shape, name
        m.weight = nn.Parameter(copy.deepcopy(src.weight.detach()).float().cpu())
        m.bias = nn.Parameter(copy.deepcopy(src.bias.detach()).float().cpu())
    mgraph = dict(mine)
    I.convert_to_int8(model, mgraph, (nn.Conv2d, nn.Linear), act_scales=list(act_scales))
    return model, mgraph, (nn.Conv2d, nn.Linear)
