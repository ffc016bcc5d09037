"""MobileNetV2-SSD-Lite as the reference's main_ssd.py builds it, written from the architecture (torchvision's
mobilenet_v2().features and InvertedResidual) for the int8 layout tests and tools/bench_int8.py.

The base net is torchvision's MobileNetV2 features.  Detection heads read two taps of it: the 576-channel expansion inside
block 14 (its 1x1 convolution, BN and ReLU6, before the stride-2 depthwise convolution), and the 1280-channel output; then
four extra inverted residual blocks (stride 2, expansion 0.2, 0.25, 0.5, 0.25) each feed one more pair.  Every source has a
classification head (6 anchors x num_classes) and a regression head (6 x 4): separable 3x3 heads (depthwise 3x3 with bias,
BN, ReLU6, 1x1 with bias) on the first five sources, plain 1x1 convolutions on the last.  Each head's output is laid out as
`permute(0, 2, 3, 1).contiguous().view(x.size(0), -1, k)` and the six of each kind are concatenated along dim 1; with
is_test the confidences go through a softmax over the classes.  Conv2d and BatchNorm2d arguments in execution order equal
tests/golden/topology_ssd.json (tests/test_int8_layout_host.py checks them).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


def separable(cin, cout):
    return nn.Sequential(nn.Conv2d(cin, cin, 3, padding=1, groups=cin), nn.BatchNorm2d(cin), nn.ReLU6(),
                         nn.Conv2d(cin, cout, 1))


class SSDLiteLike(nn.Module):
    def __init__(self, num_classes=21, is_test=False):
        super().__init__()
        import torchvision
        from torchvision.models.mobilenetv2 import InvertedResidual
        self.num_classes, self.is_test = num_classes, is_test
        self.base_net = torchvision.models.mobilenet_v2(weights=None).features
        self.extras = nn.ModuleList([InvertedResidual(1280, 512, 2, 0.2), InvertedResidual(512, 256, 2, 0.25),
                                     InvertedResidual(256, 256, 2, 0.5), InvertedResidual(256, 64, 2, 0.25)])
        sources = [576, 1280, 512, 256, 256]
        self.classification_headers = nn.ModuleList([separable(c, 6 * num_classes) for c in sources] +
                                                    [nn.Conv2d(64, 6 * num_classes, 1)])
        self.regression_headers = nn.ModuleList([separable(c, 6 * 4) for c in sources] + [nn.Conv2d(64, 6 * 4, 1)])

    def _header(self, i, x, confidences, locations):
        c = self.classification_headers[i](x).permute(0, 2, 3, 1).contiguous()
        confidences.append(c.view(c.size(0), -1, self.num_classes))
        loc = self.regression_headers[i](x).permute(0, 2, 3, 1).contiguous()
        locations.append(loc.view(loc.size(0), -1, 4))

    def forward(self, x):
        confidences, locations = [], []
        for layer in self.base_net[:14]:
            x = layer(x)
        expand, *rest = self.base_net[14].conv          # block 14 has stride 2: no residual connection
        x = y = expand(x)                               # the 576-channel tap
        for layer in rest:
            x = layer(x)
        self._header(0, y, confidences, locations)
        for layer in self.base_net[15:]:
            x = layer(x)
        self._header(1, x, confidences, locations)
        for i, layer in enumerate(self.extras):
            x = layer(x)
            self._header(i + 2, x, confidences, locations)
        confidences, locations = torch.cat(confidences, 1), torch.cat(locations, 1)
        if self.is_test:
            confidences = F.softmax(confidences, dim=2)
        return confidences, locations
