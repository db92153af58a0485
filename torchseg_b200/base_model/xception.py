"""Xception-39 backbone with the reference's constructor and attribute names (TorchSeg
furnace/base_model/xception.py); forward runs the fused libtsb path: depthwise 3x3 convs on tsb_dwconv_*, pointwise
convs with their BatchNorm (+ block residual + ReLU) on the conv / BN kernels."""
import torch
import torch.nn as nn

from .. import ops
from ..seg_opr.seg_oprs import ConvBnRelu, conv_bn_act, _as_act, _ceil_to, _release_packed_image
from ..utils.pyt_utils import load_model

__all__ = ['Xception', 'xception39']


class SeparableConvBnRelu(nn.Module):
    """xception.py:10-26: depthwise conv → pointwise ConvBnRelu (no BN after the depthwise conv)"""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=0, dilation=1, has_relu=True,
                 norm_layer=nn.BatchNorm2d):
        super(SeparableConvBnRelu, self).__init__()
        self.conv1 = nn.Conv2d(in_channels, in_channels, kernel_size, stride, padding, dilation, groups=in_channels,
                               bias=False)
        self.point_wise_cbr = ConvBnRelu(in_channels, out_channels, 1, 1, 0, has_bn=True, norm_layer=norm_layer,
                                         has_relu=has_relu, has_bias=False)

    def depthwise(self, x, share=None):
        """the depthwise conv; its output keeps the 64-padded channel layout the pointwise conv reads"""
        c = self.conv1
        if c.kernel_size != (3, 3) or c.padding != (1, 1) or c.dilation != (1, 1) or c.stride[0] != c.stride[1]:
            raise NotImplementedError("depthwise conv: only 3x3, padding 1, dilation 1 runs on libtsb")
        return ops.DWConvFn.apply(_as_act(x), c.weight, c.stride[0], _ceil_to(c.in_channels, 64), share)

    def forward(self, x, share=None):
        pw = self.point_wise_cbr
        return conv_bn_act(self.depthwise(x, share), pw.conv, pw.bn, pw.has_relu)


class Block(nn.Module):
    """xception.py:29-67"""
    expansion = 4

    def __init__(self, in_channels, mid_out_channels, has_proj, stride, dilation=1, norm_layer=nn.BatchNorm2d):
        super(Block, self).__init__()
        self.has_proj = has_proj
        if has_proj:
            self.proj = SeparableConvBnRelu(in_channels, mid_out_channels * self.expansion, 3, stride, 1,
                                            has_relu=False, norm_layer=norm_layer)
        self.residual_branch = nn.Sequential(
            SeparableConvBnRelu(in_channels, mid_out_channels, 3, stride, dilation, dilation, has_relu=True,
                                norm_layer=norm_layer),
            SeparableConvBnRelu(mid_out_channels, mid_out_channels, 3, 1, 1, has_relu=True, norm_layer=norm_layer),
            SeparableConvBnRelu(mid_out_channels, mid_out_channels * self.expansion, 3, 1, 1, has_relu=False,
                                norm_layer=norm_layer))
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        x = _as_act(x)
        # x feeds two consumers inside the block (the projection's or the shortcut's, and the residual branch's first
        # depthwise conv): their input gradients share one buffer, as in BasicBlock.forward
        share = ops.GradShare(2) if (x.requires_grad and torch.is_grad_enabled()) else None
        r0, r1, r2 = self.residual_branch
        if self.has_proj:
            shortcut = self.proj(x, share=share)
            res_share = None
        else:
            shortcut, res_share = x, share
        t = r2.depthwise(r1(r0(x, share=share)))
        # relu(shortcut + residual) is the BN-apply epilogue of the last pointwise conv
        pw = r2.point_wise_cbr
        return conv_bn_act(t, pw.conv, pw.bn, True, residual=shortcut, res_share=res_share)


class Xception(nn.Module):
    """xception.py:70-115"""

    def __init__(self, block, layers, channels, norm_layer=nn.BatchNorm2d):
        super(Xception, self).__init__()
        self.in_channels = 8
        self.conv1 = ConvBnRelu(3, self.in_channels, 3, 2, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                                has_bias=False)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, norm_layer, layers[0], channels[0], stride=2)
        self.layer2 = self._make_layer(block, norm_layer, layers[1], channels[1], stride=2)
        self.layer3 = self._make_layer(block, norm_layer, layers[2], channels[2], stride=2)

    def _make_layer(self, block, norm_layer, blocks, mid_out_channels, stride=1):
        layers = []
        has_proj = True if stride > 1 else False
        layers.append(block(self.in_channels, mid_out_channels, has_proj, stride=stride, norm_layer=norm_layer))
        self.in_channels = mid_out_channels * block.expansion
        for i in range(1, blocks):
            layers.append(block(self.in_channels, mid_out_channels, has_proj=False, stride=1, norm_layer=norm_layer))
        return nn.Sequential(*layers)

    def forward(self, x):
        # the 3x3/2 C_in = 3 stem runs on the space-to-depth image, which BiSeNet's spatial-path stem shares
        return self.forward_from_stem(self.conv1(x))

    def forward_from_stem(self, x):
        _release_packed_image()
        x = ops.MaxPool3x3S2Fn.apply(x)
        blocks = []
        x = self.layer1(x)
        blocks.append(x)
        x = self.layer2(x)
        blocks.append(x)
        x = self.layer3(x)
        blocks.append(x)
        return blocks


def xception39(pretrained_model=None, **kwargs):
    model = Xception(Block, [4, 8, 4], [16, 32, 64], **kwargs)
    if pretrained_model is not None:
        model = load_model(model, pretrained_model)
    return model
