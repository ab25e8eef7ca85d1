"""ResNet-18 / ResNet-50 (BASELINE.json configs[2], configs[4]) written against plain
torch.nn so there is no torchvision dependency. BatchNorm(+residual)+ReLU and the global average
pool run on the fused sm_90a kernels of ``ops/resnet_ops.py`` when activations are NHWC bf16. BatchNorm running statistics are part of the
federated state (Keras ``get_weights`` includes moving mean/variance, FLPyfhelin.py:151)."""
from __future__ import annotations

from typing import List, Optional, Tuple, Type

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.fp8 import Conv1x1
from ..ops.tc_conv import Conv3x3
from ..ops.resnet_ops import bn_act, global_avgpool


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin: int, planes: int, stride: int = 1):
        super().__init__()
        self.conv1 = Conv3x3(cin, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = Conv3x3(planes, planes, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self.down = None
        if stride != 1 or cin != planes:
            self.down = nn.Sequential(Conv1x1(cin, planes, stride), nn.BatchNorm2d(planes))

    def forward(self, x):
        idt = x if self.down is None else bn_act(self.down[1], self.down[0](x), relu=False)
        out = bn_act(self.bn1, self.conv1(x))
        return bn_act(self.bn2, self.conv2(out), res=idt)      # relu(bn(.) + identity) in one kernel


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin: int, planes: int, stride: int = 1):
        super().__init__()
        self.conv1 = Conv1x1(cin, planes)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = Conv3x3(planes, planes, stride)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = Conv1x1(planes, planes * 4)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.down = None
        if stride != 1 or cin != planes * 4:
            self.down = nn.Sequential(Conv1x1(cin, planes * 4, stride), nn.BatchNorm2d(planes * 4))

    def forward(self, x):
        idt = x if self.down is None else bn_act(self.down[1], self.down[0](x), relu=False)
        out = bn_act(self.bn1, self.conv1(x))
        out = bn_act(self.bn2, self.conv2(out))
        return bn_act(self.bn3, self.conv3(out), res=idt)


class ResNet(nn.Module):
    def __init__(self, block: Type[nn.Module], layers: Tuple[int, ...], num_classes: int = 1000,
                 in_channels: int = 3):
        super().__init__()
        self.in_channels = in_channels
        self.num_classes = num_classes
        self.conv1 = nn.Conv2d(in_channels, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        cin = 64
        stages = []
        for i, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
            blocks = []
            for j in range(n):
                blocks.append(block(cin, planes, stride=2 if (j == 0 and i > 0) else 1))
                cin = planes * block.expansion
            stages.append(nn.Sequential(*blocks))
        self.stages = nn.Sequential(*stages)
        self.fc = nn.Linear(cin, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x):
        x = F.max_pool2d(bn_act(self.bn1, self.conv1(x)), 3, 2, 1)
        x = self.stages(x)
        return self.fc(global_avgpool(x))

    def keras_layers(self) -> List[Tuple[str, Optional[nn.Module]]]:
        """One entry per weight-bearing module, in definition order."""
        out: List[Tuple[str, Optional[nn.Module]]] = []
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                out.append(("conv", m))
            elif isinstance(m, nn.BatchNorm2d):
                out.append(("bn", m))
            elif isinstance(m, nn.Linear):
                out.append(("dense", m))
        return out


def resnet18(num_classes: int = 1000, in_channels: int = 3) -> ResNet:
    return ResNet(BasicBlock, (2, 2, 2, 2), num_classes, in_channels)


def resnet50(num_classes: int = 1000, in_channels: int = 3) -> ResNet:
    return ResNet(Bottleneck, (3, 4, 6, 3), num_classes, in_channels)
