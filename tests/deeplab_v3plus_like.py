"""A DeepLab-v3+-shaped segmentation network built from nn layers, for the int8 upsample tests and tools/bench_int8.py.

The shape of the network the reference's main_seg.py calibrates, scaled down: a MobileNetV2-like backbone at output stride 16
(inverted residual blocks, the last two with dilated depthwise convolutions) with a low-level feature tap at 1/4 scale; the
ASPP (a 1x1 branch, three dilated 3x3 branches, an image-pooling branch upsampled with align_corners=True, a 5-operand
channel concatenation and a 1x1 projection); and the decoder (a 48-channel 1x1 on the low-level features, a bilinear
upsample of the ASPP output to 1/4 scale, a concatenation, two 3x3 convolutions, a 1x1 classifier) and the final upsample of
the logits to the input size.  The upsample sizes are traced shape queries on a concatenation operand, as in the reference
(`size=x4.size()[2:]` in the ASPP, `size=low_level_feat.size()[2:]` in the decoder), so that the operand has a second user
that only reads its shape.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


def _cbr(cin, cout, k=1, stride=1, dilation=1, groups=1, act=nn.ReLU):
    pad = dilation * (k - 1) // 2
    layers = [nn.Conv2d(cin, cout, k, stride, pad, dilation=dilation, groups=groups, bias=False), nn.BatchNorm2d(cout)]
    return layers + ([act()] if act is not None else [])


class InvertedResidual(nn.Module):
    def __init__(self, cin, cout, stride, expand, dilation=1):
        super().__init__()
        hidden = cin * expand
        layers = _cbr(cin, hidden, act=nn.ReLU6) if expand != 1 else []
        layers += _cbr(hidden, hidden, 3, stride, dilation, groups=hidden, act=nn.ReLU6) + _cbr(hidden, cout, act=None)
        self.conv = nn.Sequential(*layers)
        self.use_res = stride == 1 and cin == cout

    def forward(self, x):
        return x + self.conv(x) if self.use_res else self.conv(x)


class ASPP(nn.Module):
    def __init__(self, cin, cout=64, rates=(6, 12, 18)):
        super().__init__()
        self.b0 = nn.Sequential(*_cbr(cin, cout))
        self.b1, self.b2, self.b3 = (nn.Sequential(*_cbr(cin, cout, 3, dilation=r)) for r in rates)
        self.pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), *_cbr(cin, cout))
        self.project = nn.Sequential(*_cbr(5 * cout, cout), nn.Dropout(0.5))

    def forward(self, x):
        x0, x1, x2, x3 = self.b0(x), self.b1(x), self.b2(x), self.b3(x)
        p = F.interpolate(self.pool(x), size=x3.size()[2:], mode="bilinear", align_corners=True)
        return self.project(torch.cat([x0, x1, x2, x3, p], dim=1))


class DeepLabV3PlusLike(nn.Module):
    def __init__(self, num_classes=21, aspp_channels=64):
        super().__init__()
        self.stem = nn.Sequential(*_cbr(3, 16, 3, 2, act=nn.ReLU6))
        self.low = nn.Sequential(InvertedResidual(16, 16, 1, 1), InvertedResidual(16, 24, 2, 6),
                                 InvertedResidual(24, 24, 1, 6))                                   # 1/4
        self.high = nn.Sequential(InvertedResidual(24, 32, 2, 6), InvertedResidual(32, 32, 1, 6),
                                  InvertedResidual(32, 64, 2, 6), InvertedResidual(64, 64, 1, 6, dilation=2),
                                  InvertedResidual(64, 96, 1, 6, dilation=2))                      # 1/16
        self.aspp = ASPP(96, aspp_channels)
        self.reduce = nn.Sequential(*_cbr(24, 48))
        self.last_conv = nn.Sequential(*_cbr(aspp_channels + 48, 64, 3), nn.Dropout(0.5), *_cbr(64, 64, 3),
                                       nn.Dropout(0.1), nn.Conv2d(64, num_classes, 1))

    def forward(self, x):
        low = self.low(self.stem(x))
        a = self.aspp(self.high(low))
        r = self.reduce(low)
        a = F.interpolate(a, size=r.size()[2:], mode="bilinear", align_corners=True)
        y = self.last_conv(torch.cat([a, r], dim=1))
        return F.interpolate(y, size=x.shape[-2:], mode="bilinear", align_corners=True)
