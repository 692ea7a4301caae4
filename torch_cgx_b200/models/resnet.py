"""ResNet family (He et al. 2015) for the DDP benchmarks and the CIFAR example.

The reference trains torchvision ResNet-18 on CIFAR in its example
(/root/reference/examples/cifar_train.py:120-141) and BASELINE.json names
ResNet-50 as the headline DDP model; both are defined here so the framework has
no torchvision dependency. Weights are random-init (no network access).

Each block ends in the native residual join (``residual.py``) and returns the pair ``(y, alias of
y)``; the next block feeds the first to conv1 and the second to its identity or downsample path.
A block also accepts a plain tensor. Parameters and their order are torchvision's.

``forward`` runs every BatchNorm through ``batch_norm_act`` (``batchnorm.py``), with the ReLU that
follows it fused; the modules themselves (``stem``, ``bn1``, ``relu``, ``downsample``) are unchanged
and still compute the unfused model when called directly.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Type, Union

import torch
import torch.nn as nn

from .batchnorm import batch_norm_act
from .residual import residual_relu


def _conv3x3(cin: int, cout: int, stride: int = 1) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, 3, stride, 1, bias=False)


def _split(x: Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]]) -> Tuple[torch.Tensor, torch.Tensor]:
    """A block's input: a tensor, or the pair (for conv1, for the identity / downsample path) that
    the previous block returned (see ``residual.py``)."""
    return (x, x) if isinstance(x, torch.Tensor) else x


def _downsample(down: nn.Sequential, x: torch.Tensor) -> torch.Tensor:
    """``down(x)`` for the (1x1 conv, BatchNorm) downsample path."""
    return batch_norm_act(down[1], down[0](x), relu=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None):
        super().__init__()
        self.conv1 = _conv3x3(cin, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv3x3(planes, planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        xa, xb = _split(x)
        idt = xb if self.downsample is None else _downsample(self.downsample, xb)
        out = batch_norm_act(self.bn1, self.conv1(xa), relu=True)
        out = batch_norm_act(self.bn2, self.conv2(out), relu=False)
        return residual_relu(out, idt)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv3x3(planes, planes, stride)  # stride on the 3x3 (ResNet v1.5)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        xa, xb = _split(x)
        idt = xb if self.downsample is None else _downsample(self.downsample, xb)
        out = batch_norm_act(self.bn1, self.conv1(xa), relu=True)
        out = batch_norm_act(self.bn2, self.conv2(out), relu=True)
        out = batch_norm_act(self.bn3, self.conv3(out), relu=False)
        return residual_relu(out, idt)


class ResNet(nn.Module):
    def __init__(self, block: Type[Union[BasicBlock, Bottleneck]], layers: List[int], num_classes: int = 1000,
                 cifar_stem: bool = False):
        super().__init__()
        self.inplanes = 64
        if cifar_stem:  # 32x32 inputs: 3x3 stem, no max-pool
            self.stem = nn.Sequential(_conv3x3(3, 64), nn.BatchNorm2d(64), nn.ReLU(inplace=True))
        else:
            self.stem = nn.Sequential(
                nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
                nn.MaxPool2d(3, 2, 1),
            )
        self.layer1 = self._make(block, 64, layers[0], 1)
        self.layer2 = self._make(block, 128, layers[1], 2)
        self.layer3 = self._make(block, 256, layers[2], 2)
        self.layer4 = self._make(block, 512, layers[3], 2)
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        for m in self.modules():  # zero-init the last BN of each residual branch
            if isinstance(m, Bottleneck):
                nn.init.zeros_(m.bn3.weight)
            elif isinstance(m, BasicBlock):
                nn.init.zeros_(m.bn2.weight)

    def _make(self, block, planes: int, n: int, stride: int) -> nn.Sequential:
        down = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            down = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, 1, stride, bias=False),
                nn.BatchNorm2d(planes * block.expansion),
            )
        blocks = [block(self.inplanes, planes, stride, down)]
        self.inplanes = planes * block.expansion
        blocks += [block(self.inplanes, planes) for _ in range(1, n)]
        return nn.Sequential(*blocks)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = batch_norm_act(self.stem[1], self.stem[0](x), relu=True)  # conv, BN + ReLU
        for m in self.stem[3:]:  # the max-pool of the ImageNet stem
            x = m(x)
        x, _ = self.layer4(self.layer3(self.layer2(self.layer1(x))))  # the alias has no consumer
        return self.fc(torch.flatten(self.pool(x), 1))


def resnet18(num_classes: int = 1000, cifar_stem: bool = False) -> ResNet:
    return ResNet(BasicBlock, [2, 2, 2, 2], num_classes, cifar_stem)


def resnet50(num_classes: int = 1000, cifar_stem: bool = False) -> ResNet:
    return ResNet(Bottleneck, [3, 4, 6, 3], num_classes, cifar_stem)
