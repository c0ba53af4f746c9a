"""ResNet-50 / ResNet-152 (He et al.) for the benchmark configurations.  Own definition (not
torchvision's module) so that the stride-1 1x1 / 3x3 convolutions, BatchNorm(+add+ReLU), the stem pool and the classifier
run on this package's kernels; parameter order / shapes match torchvision's - bucket layouts of stock DDP
therefore hold.  The 7x7 stem runs on the wgmma tap-GEMM (``ops.StemConv7x7``); the six stride-2 convolutions stay on the library."""
from __future__ import annotations

import os
from typing import List

import torch
import torch.nn as nn

from ..ops import Conv3x3, FusedBatchNormAct2d, Linear, MaxPool3x3s2, PointwiseConv2d, StemConv7x7
from ..ops.bottleneck import bottleneck_forward, bottleneck_native_ok


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: nn.Module | None = None):
        super().__init__()
        # Convolutions: wgmma implicit GEMMs whose epilogue hands the following BatchNorm its statistics; BatchNorm + ReLU
        # (and, for bn3, the shortcut add) are single fused kernels on channels_last CUDA tensors.
        self.conv1 = PointwiseConv2d(inplanes, planes)
        self.bn1 = FusedBatchNormAct2d(planes, relu=True)
        self.conv2 = Conv3x3(planes, planes, stride=stride)
        self.bn2 = FusedBatchNormAct2d(planes, relu=True)
        self.conv3 = PointwiseConv2d(planes, planes * self.expansion)
        self.bn3 = FusedBatchNormAct2d(planes * self.expansion, relu=True)
        self.downsample = downsample

    def forward(self, x):
        if os.environ.get("B200DDP_BLOCK_FUSE", "0") == "1" and bottleneck_native_ok(self, x):
            return bottleneck_forward(self, x)             # one autograd node, hand-written backward (ops/bottleneck.py)
        if self.downsample is None:
            identity = x
        else:
            y, part = self.downsample[0].forward_with_stats(x)
            identity = self.downsample[1](y, partials=part)
        y, part = self.conv1.forward_with_stats(x)
        out = self.bn1(y, partials=part)
        y, part = self.conv2.forward_with_stats(out)
        out = self.bn2(y, partials=part)
        y, part = self.conv3.forward_with_stats(out)
        return self.bn3(y, residual=identity, partials=part)


class ResNet(nn.Module):
    def __init__(self, layers: List[int], num_classes: int = 1000, zero_init_residual: bool = False):
        super().__init__()
        self.inplanes = 64
        self.conv1 = StemConv7x7(3, 64)
        self.bn1 = FusedBatchNormAct2d(64, relu=True)
        self.maxpool = MaxPool3x3s2()
        self.layer1 = self._make_layer(64, layers[0], 1)
        self.layer2 = self._make_layer(128, layers[1], 2)
        self.layer3 = self._make_layer(256, layers[2], 2)
        self.layer4 = self._make_layer(512, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = Linear(512 * Bottleneck.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.zeros_(m.bn3.weight)

    def _make_layer(self, planes: int, blocks: int, stride: int) -> nn.Sequential:
        downsample = None
        if stride != 1 or self.inplanes != planes * Bottleneck.expansion:
            downsample = nn.Sequential(PointwiseConv2d(self.inplanes, planes * Bottleneck.expansion, stride=stride),
                                       FusedBatchNormAct2d(planes * Bottleneck.expansion))
        mods = [Bottleneck(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * Bottleneck.expansion
        mods += [Bottleneck(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*mods)

    def forward(self, x):
        if self.training:
            y, part = self.conv1.forward_with_stats(x)       # BatchNorm statistics ride on the stem's epilogue
        else:
            y, part = self.conv1(x), None                    # inference normalises with the running statistics
        x = self.maxpool(self.bn1(y, partials=part))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        x = torch.flatten(self.avgpool(x), 1)
        return self.fc(x)


def resnet50(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet([3, 4, 6, 3], num_classes, **kw)


def resnet152(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet([3, 8, 36, 3], num_classes, **kw)
