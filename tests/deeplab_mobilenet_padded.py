"""DeepLab-v3+ with a MobileNetV2 backbone at output stride 16, as the reference's main_seg.py builds it, written from the
architecture for the int8 layout tests and tools/bench_int8.py.

What sets it apart from tests/deeplab_v3plus_like.py is how the backbone pads: every inverted residual block first pads its
input with zeros by F.pad ("fixed padding": (k_eff - 1) // 2 on each side, k_eff = 3 + 2 (dilation - 1)) and then runs its
convolutions with padding 0, so each of the 17 blocks has an F.pad node in front of its first convolution (a 1x1 expansion,
or the depthwise 3x3 of the first block).  At output stride 16 the 160- and 320-channel stages keep stride 1; the 320-channel
block's depthwise convolution has dilation 2.  The low-level features (24 channels, 1/4 scale) are the output of the fourth
feature module.  The ASPP has a 1x1 branch, three dilated 3x3 branches (6, 12, 18), an image-pooling branch upsampled with
align_corners=True to a traced size, a 5 x 256-channel concatenation, a 1x1 projection and dropout; the decoder reduces the
low-level features to 48 channels, upsamples the ASPP output to their size, concatenates, and runs two 3x3 convolutions and
the classifier; the logits are upsampled to the input size.  Conv2d and BatchNorm2d arguments in execution order equal
tests/golden/topology_deeplab.json (tests/test_int8_layout_host.py checks them).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


def _conv_bn(cin, cout, k, stride=1, padding=0, dilation=1, groups=1, act=nn.ReLU6):
    layers = [nn.Conv2d(cin, cout, k, stride, padding, dilation, groups, bias=False), nn.BatchNorm2d(cout)]
    return layers + ([act()] if act is not None else [])


class PaddedInvertedResidual(nn.Module):
    """An inverted residual block whose convolutions have padding 0: the block zero-pads its input first."""

    def __init__(self, cin, cout, stride, dilation, expand):
        super().__init__()
        hidden = round(cin * expand)
        layers = _conv_bn(cin, hidden, 1) if expand != 1 else []
        layers += _conv_bn(hidden, hidden, 3, stride, 0, dilation, groups=hidden) + _conv_bn(hidden, cout, 1, act=None)
        self.conv = nn.Sequential(*layers)
        self.pad = dilation                      # (3 + 2 (dilation - 1) - 1) // 2 on each side
        self.use_res = stride == 1 and cin == cout

    def forward(self, x):
        x_pad = F.pad(x, (self.pad, self.pad, self.pad, self.pad))
        return x + self.conv(x_pad) if self.use_res else self.conv(x_pad)


class MobileNetV2OS16(nn.Module):
    # (expansion, channels, blocks, stride) of MobileNetV2
    STAGES = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]

    def __init__(self, output_stride=16):
        super().__init__()
        features = [nn.Sequential(*_conv_bn(3, 32, 3, 2, 1))]
        cin, cur, rate = 32, 2, 1
        for t, c, n, s in self.STAGES:
            if cur == output_stride:             # past the output stride: stride 1, dilate the later stages instead
                stride, dilation, rate = 1, rate, rate * s
            else:
                stride, dilation, cur = s, 1, cur * s
            for i in range(n):
                features.append(PaddedInvertedResidual(cin, c, stride if i == 0 else 1, dilation, t))
                cin = c
        self.features = nn.Sequential(*features)

    def forward(self, x):
        for i, f in enumerate(self.features):
            x = f(x)
            if i == 3:
                low = x
        return x, low


class ASPP(nn.Module):
    def __init__(self, cin=320, cout=256, rates=(6, 12, 18)):
        super().__init__()
        self.aspp1 = nn.Sequential(*_conv_bn(cin, cout, 1, act=nn.ReLU))
        self.aspp2, self.aspp3, self.aspp4 = (nn.Sequential(*_conv_bn(cin, cout, 3, 1, r, r, act=nn.ReLU)) for r in rates)
        self.image_pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), *_conv_bn(cin, cout, 1, act=nn.ReLU))
        self.project = nn.Sequential(*_conv_bn(5 * cout, cout, 1, act=nn.ReLU), nn.Dropout(0.5))

    def forward(self, x):
        x1, x2, x3, x4 = self.aspp1(x), self.aspp2(x), self.aspp3(x), self.aspp4(x)
        x5 = F.interpolate(self.image_pool(x), size=x4.size()[2:], mode="bilinear", align_corners=True)
        return self.project(torch.cat((x1, x2, x3, x4, x5), dim=1))


class Decoder(nn.Module):
    def __init__(self, num_classes, low_channels=24):
        super().__init__()
        self.reduce = nn.Sequential(*_conv_bn(low_channels, 48, 1, act=nn.ReLU))
        self.last_conv = nn.Sequential(*_conv_bn(256 + 48, 256, 3, 1, 1, act=nn.ReLU), nn.Dropout(0.5),
                                       *_conv_bn(256, 256, 3, 1, 1, act=nn.ReLU), nn.Dropout(0.1),
                                       nn.Conv2d(256, num_classes, 1))

    def forward(self, x, low):
        low = self.reduce(low)
        x = F.interpolate(x, size=low.size()[2:], mode="bilinear", align_corners=True)
        return self.last_conv(torch.cat((x, low), dim=1))


class DeepLabMobileNetPadded(nn.Module):
    def __init__(self, num_classes=21):
        super().__init__()
        self.backbone = MobileNetV2OS16()
        self.aspp = ASPP()
        self.decoder = Decoder(num_classes)

    def forward(self, x):
        high, low = self.backbone(x)
        y = self.decoder(self.aspp(high), low)
        return F.interpolate(y, size=x.size()[2:], mode="bilinear", align_corners=True)
