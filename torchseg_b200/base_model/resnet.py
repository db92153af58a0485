"""ResNet v1 / v1c backbone with the reference's constructor and attribute names
(TorchSeg furnace/base_model/resnet.py); forward runs the fused libtsb path."""
import torch
import torch.nn as nn

from .. import ops
from ..seg_opr.seg_oprs import conv_bn_act, _as_act, _release_packed_image
from ..utils.pyt_utils import load_model

__all__ = ['ResNet', 'resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152']


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class BasicBlock(nn.Module):
    """resnet.py:17-53"""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, norm_layer=None, bn_eps=1e-5, bn_momentum=0.1, downsample=None,
                 inplace=True):
        super(BasicBlock, self).__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = norm_layer(planes, eps=bn_eps, momentum=bn_momentum)
        self.relu = nn.ReLU(inplace=inplace)
        self.relu_inplace = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = norm_layer(planes, eps=bn_eps, momentum=bn_momentum)
        self.downsample = downsample
        self.stride = stride
        self.inplace = inplace

    def forward(self, x):
        x = _as_act(x)
        # x is consumed twice inside the block (conv1 + shortcut): their input gradients share one buffer
        share = ops.GradShare(2) if (x.requires_grad and torch.is_grad_enabled()) else None
        out = conv_bn_act(x, self.conv1, self.bn1, True, in_share=share)
        if self.downsample is not None:
            residual = conv_bn_act(x, self.downsample[0], self.downsample[1], False, in_share=share)
            return conv_bn_act(out, self.conv2, self.bn2, True, residual=residual)
        # conv2 → bn2 → (+residual) → relu in one fused group (resnet.py:42-51)
        return conv_bn_act(out, self.conv2, self.bn2, True, residual=x, res_share=share)


class Bottleneck(nn.Module):
    """resnet.py:56-101"""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, norm_layer=None, bn_eps=1e-5, bn_momentum=0.1, downsample=None,
                 inplace=True):
        super(Bottleneck, self).__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = norm_layer(planes, eps=bn_eps, momentum=bn_momentum)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = norm_layer(planes, eps=bn_eps, momentum=bn_momentum)
        self.conv3 = nn.Conv2d(planes, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = norm_layer(planes * self.expansion, eps=bn_eps, momentum=bn_momentum)
        self.relu = nn.ReLU(inplace=inplace)
        self.relu_inplace = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride
        self.inplace = inplace

    def forward(self, x):
        x = _as_act(x)
        share = ops.GradShare(2) if (x.requires_grad and torch.is_grad_enabled()) else None   # see BasicBlock.forward
        out = conv_bn_act(x, self.conv1, self.bn1, True, in_share=share)
        out = conv_bn_act(out, self.conv2, self.bn2, True)
        if self.downsample is not None:
            residual = conv_bn_act(x, self.downsample[0], self.downsample[1], False, in_share=share)
            return conv_bn_act(out, self.conv3, self.bn3, True, residual=residual)
        return conv_bn_act(out, self.conv3, self.bn3, True, residual=x, res_share=share)


class ResNet(nn.Module):
    """resnet.py:104-184"""

    def __init__(self, block, layers, norm_layer=nn.BatchNorm2d, bn_eps=1e-5, bn_momentum=0.1, deep_stem=False,
                 stem_width=32, inplace=True):
        self.inplanes = stem_width * 2 if deep_stem else 64
        super(ResNet, self).__init__()
        self.deep_stem = deep_stem
        if deep_stem:
            self.conv1 = nn.Sequential(
                nn.Conv2d(3, stem_width, kernel_size=3, stride=2, padding=1, bias=False),
                norm_layer(stem_width, eps=bn_eps, momentum=bn_momentum),
                nn.ReLU(inplace=inplace),
                nn.Conv2d(stem_width, stem_width, kernel_size=3, stride=1, padding=1, bias=False),
                norm_layer(stem_width, eps=bn_eps, momentum=bn_momentum),
                nn.ReLU(inplace=inplace),
                nn.Conv2d(stem_width, stem_width * 2, kernel_size=3, stride=1, padding=1, bias=False),
            )
        else:
            self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = norm_layer(stem_width * 2 if deep_stem else 64, eps=bn_eps, momentum=bn_momentum)
        self.relu = nn.ReLU(inplace=inplace)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, norm_layer, 64, layers[0], inplace, bn_eps=bn_eps,
                                       bn_momentum=bn_momentum)
        self.layer2 = self._make_layer(block, norm_layer, 128, layers[1], inplace, stride=2, bn_eps=bn_eps,
                                       bn_momentum=bn_momentum)
        self.layer3 = self._make_layer(block, norm_layer, 256, layers[2], inplace, stride=2, bn_eps=bn_eps,
                                       bn_momentum=bn_momentum)
        self.layer4 = self._make_layer(block, norm_layer, 512, layers[3], inplace, stride=2, bn_eps=bn_eps,
                                       bn_momentum=bn_momentum)

    def _make_layer(self, block, norm_layer, planes, blocks, inplace=True, stride=1, bn_eps=1e-5, bn_momentum=0.1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                norm_layer(planes * block.expansion, eps=bn_eps, momentum=bn_momentum),
            )
        layers = [block(self.inplanes, planes, stride, norm_layer, bn_eps, bn_momentum, downsample, inplace)]
        self.inplanes = planes * block.expansion
        for i in range(1, blocks):
            layers.append(block(self.inplanes, planes, norm_layer=norm_layer, bn_eps=bn_eps, bn_momentum=bn_momentum,
                                inplace=inplace))
        return nn.Sequential(*layers)

    def forward(self, x):
        if self.deep_stem:
            # v1c stem (resnet.py:110-124): 3x3/2 (C_in = 3, space-to-depth stem kernel) → 3x3 → 3x3, then bn1 + relu
            c = self.conv1
            if c[3].in_channels % 64 != 0:
                raise NotImplementedError("deep stem needs stem_width % 64 == 0 (BASELINE configs use stem_width=64)")
            x = conv_bn_act(x, c[0], c[1], True)
            x = conv_bn_act(x, c[3], c[4], True)
            return self.forward_from_stem(conv_bn_act(x, c[6], self.bn1, True))
        return self.forward_from_stem(conv_bn_act(x, self.conv1, self.bn1, True))

    def forward_from_stem(self, x):
        """stages after conv1 → bn1 → relu (the stem may be computed elsewhere, fused with a sibling stem)"""
        _release_packed_image()   # every stem of this forward has consumed the space-to-depth image by now
        x = ops.MaxPool3x3S2Fn.apply(x)
        blocks = []
        x = self.layer1(x)
        blocks.append(x)
        x = self.layer2(x)
        blocks.append(x)
        x = self.layer3(x)
        blocks.append(x)
        x = self.layer4(x)
        blocks.append(x)
        return blocks


def _make(block, layers, pretrained_model, **kwargs):
    model = ResNet(block, layers, **kwargs)
    if pretrained_model is not None:
        model = load_model(model, pretrained_model)
    return model


def resnet18(pretrained_model=None, **kwargs):
    return _make(BasicBlock, [2, 2, 2, 2], pretrained_model, **kwargs)


def resnet34(pretrained_model=None, **kwargs):
    return _make(BasicBlock, [3, 4, 6, 3], pretrained_model, **kwargs)


def resnet50(pretrained_model=None, **kwargs):
    return _make(Bottleneck, [3, 4, 6, 3], pretrained_model, **kwargs)


def resnet101(pretrained_model=None, **kwargs):
    return _make(Bottleneck, [3, 4, 23, 3], pretrained_model, **kwargs)


def resnet152(pretrained_model=None, **kwargs):
    return _make(Bottleneck, [3, 8, 36, 3], pretrained_model, **kwargs)
