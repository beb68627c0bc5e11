"""
ResNet family (v1.5 bottleneck: the stride sits on the 3x3 conv), written for
the H100 execution model: NHWC (channels_last) activations and weights, bf16
tensor-core math under autocast with fp32 master weights in the gossip arena,
BatchNorm statistics and affine parameters kept in fp32.

Every BatchNorm is a :class:`~..ops.fused_bn.FusedBatchNormAct2d`: BN, the
residual add and the ReLU of a block run as one fused sm_90a op (2 reads + 1
write forward) instead of three framework kernels; parameters, buffers and
``state_dict`` keys are those of ``nn.BatchNorm2d``.

The reference trains ``torchvision.models.resnet50()`` (``gossip_sgd.py:693-707``)
initialised as in "ImageNet in 1 hour": zero gamma in the last BN of every
residual block and N(0, 0.01) weights in the classifier -- see
:func:`init_imagenet_in_1hr`.  ``resnet50()`` here has the same 25,557,032
parameters in the same order (161 tensors), so arenas, checkpoints and gossip
message sizes match the reference's.

Stochastic depth (``drop_path_rate=p > 0``, see :mod:`..ops.stochastic_depth`): a training forward draws
the ``[L, N]`` branch scales of its ``L`` blocks in one launch and hands block ``l`` its row, which the
block's last BN applies inside the fused kernels, ``relu(s_n * bn(conv(x)) + identity)``.  Eval-mode
forwards and forwards inside ``precise_bn_stats`` draw nothing and scale nothing.
"""

from __future__ import annotations

from typing import List, Type

import torch
import torch.nn as nn

from ..ops.fused_bn import (FusedBatchNormAct2d as _BN, MaxPool2dNHWC, conv_bn_act, conv_bn_act_split,
                             precise_bn_active, stem_conv)
from ..ops.stochastic_depth import StochasticDepth


def _conv3x3(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, 3, stride, 1, bias=False)


def _conv1x1(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, 1, stride, 0, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin, width, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv3x3(cin, width, stride)
        self.bn1 = _BN(width)
        self.conv2 = _conv3x3(width, width)
        self.bn2 = _BN(width)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    @property
    def last_bn(self):
        return self.bn2

    def forward(self, x, branch_scale=None):
        """``branch_scale``: the per-sample stochastic-depth scale of the residual branch, fp32 ``[N]``"""
        identity = x if self.downsample is None else conv_bn_act(self.downsample[0], self.downsample[1], x)
        out = self.bn1(self.conv1(x), relu=True)
        if branch_scale is None:
            return self.bn2(self.conv2(out), residual=identity, relu=True)
        return self.bn2(self.conv2(out), residual=identity, relu=True, branch_scale=branch_scale)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin, width, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv1x1(cin, width)
        self.bn1 = _BN(width)
        self.conv2 = _conv3x3(width, width, stride)
        self.bn2 = _BN(width)
        self.conv3 = _conv1x1(width, width * self.expansion)
        self.bn3 = _BN(width * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    @property
    def last_bn(self):
        return self.bn3

    def forward(self, x, branch_scale=None):
        """``branch_scale``: the per-sample stochastic-depth scale of the residual branch, fp32 ``[N]``"""
        # x feeds conv1 and the skip branch: the split op folds the skip gradient into conv1's dgrad
        out, skip = conv_bn_act_split(self.conv1, self.bn1, x, relu=True)
        identity = skip if self.downsample is None else conv_bn_act(self.downsample[0], self.downsample[1], skip)
        out = self.bn2(self.conv2(out), relu=True)
        return conv_bn_act(self.conv3, self.bn3, out, residual=identity, relu=True, branch_scale=branch_scale)


class ResNet(nn.Module):

    def __init__(self, block: Type[nn.Module], layers: List[int], num_classes=1000,
                 in_channels=3, base_width=64, drop_path_rate=0.0):
        """``drop_path_rate``: stochastic depth with timm's linear rule over the residual blocks (0 = off;
        :attr:`stochastic_depth` is then None).  Seed it with ``model.stochastic_depth.reseed(seed, rank)``."""
        super().__init__()
        self.inplanes = base_width
        self.conv1 = nn.Conv2d(in_channels, base_width, 7, 2, 3, bias=False)
        self.bn1 = _BN(base_width)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = MaxPool2dNHWC(3, 2, 1)
        self.layer1 = self._make_layer(block, base_width, layers[0])
        self.layer2 = self._make_layer(block, base_width * 2, layers[1], 2)
        self.layer3 = self._make_layer(block, base_width * 4, layers[2], 2)
        self.layer4 = self._make_layer(block, base_width * 8, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(base_width * 8 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        if not 0.0 <= drop_path_rate < 1.0:
            raise ValueError('drop_path_rate must be in [0, 1), got %r' % (drop_path_rate,))
        # a plain attribute: no parameters or buffers, so state_dict keys and the arena are unchanged
        self.stochastic_depth = StochasticDepth(sum(layers), drop_path_rate) if drop_path_rate > 0 else None

    def _make_layer(self, block, width, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != width * block.expansion:
            downsample = nn.Sequential(_conv1x1(self.inplanes, width * block.expansion, stride),
                                       _BN(width * block.expansion))
        layers = [block(self.inplanes, width, stride, downsample)]
        self.inplanes = width * block.expansion
        layers += [block(self.inplanes, width) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(self.bn1(stem_conv(self.conv1, x), relu=True))
        sd = self.stochastic_depth
        if sd is None or not self.training or precise_bn_active():
            x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        else:
            scales = sd.draw(x.shape[0], x.device)            # [L, N]: one launch
            blocks = [b for layer in (self.layer1, self.layer2, self.layer3, self.layer4) for b in layer]
            for l, (blk, rate) in enumerate(zip(blocks, sd.rates)):
                x = blk(x, scales[l] if rate > 0 else None)
        x = torch.flatten(self.avgpool(x), 1)
        return self.fc(x)


def resnet18(**kw):
    return ResNet(BasicBlock, [2, 2, 2, 2], **kw)


def resnet34(**kw):
    return ResNet(BasicBlock, [3, 4, 6, 3], **kw)


def resnet50(**kw):
    return ResNet(Bottleneck, [3, 4, 6, 3], **kw)


def resnet101(**kw):
    return ResNet(Bottleneck, [3, 4, 23, 3], **kw)


def resnet152(**kw):
    return ResNet(Bottleneck, [3, 8, 36, 3], **kw)


def init_imagenet_in_1hr(model: ResNet) -> ResNet:
    """Reference initialisation (``gossip_sgd.py:693-707``): zero the gamma of
    the last BN in every residual block, classifier weights ~ N(0, 0.01)."""
    for m in model.modules():
        if isinstance(m, (Bottleneck, BasicBlock)):
            nn.init.zeros_(m.last_bn.weight)
    model.fc.weight.data.normal_(0, 0.01)
    return model


class TinyConvNet(nn.Module):
    """Few-kernel CNN for smoke tests (same layer types as ResNet)."""

    def __init__(self, num_classes=10, width=16):
        super().__init__()
        self.features = nn.Sequential(
            nn.Conv2d(3, width, 3, 2, 1, bias=False), _BN(width), nn.ReLU(inplace=True),
            nn.Conv2d(width, 2 * width, 3, 2, 1, bias=False), _BN(2 * width),
            nn.ReLU(inplace=True), nn.AdaptiveAvgPool2d((1, 1)))
        self.fc = nn.Linear(2 * width, num_classes)

    def forward(self, x):
        return self.fc(torch.flatten(self.features(x), 1))


MODEL_ZOO = {
    'resnet18': resnet18, 'resnet34': resnet34, 'resnet50': resnet50,
    'resnet101': resnet101, 'resnet152': resnet152, 'tiny': TinyConvNet,
}
