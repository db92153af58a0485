"""DANet (ResNet-101 v1c, dilated-8) with its dual attention head (Fu et al., "Dual Attention Network for Scene
Segmentation", CVPR 2019) on the libtsb path, in the style of the reference's network lines:

  * backbone: `resnet101` with the deep stem, layer3 / layer4 dilated by 2 / 4 through PSPNet's `_nostride_dilate`
    (output stride 8);
  * head (DANetHead): conv5a and conv5c, 3x3 ConvBnRelu 2048 → 512; sa, the position attention (PAM_Module, attention
    over every pixel of the 1/8-resolution map at (d_k, d_v) = (64, 512) on tsb_attention_{fwd,bwd}) on conv5a, then
    conv51; sc, the channel attention (CAM_Module) on conv5c, then conv52 (3x3 ConvBnRelu 512 → 512 both); conv6, conv7
    and conv8, each Dropout2d(0.1) and a 1x1 classifier with bias (fp32 logits), on conv51, on conv52 and on their sum.

Training returns crit(sasc) + crit(sa) + crit(sc) with equal weights, as in DANet's multi-loss, each through the
criterion's fused up-sampling pair (`forward_lowres`, ProbOhemCrossEntropy2d) when it has one and through the fused
up-sampling cross-entropy (`head_loss`) otherwise, so the full-resolution logits are never written. Eval (label None)
returns the log_softmax of the sasc logits up-sampled to the input size, and runs neither conv6 nor conv7."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import CAM_Module, ConvBnRelu, PAM_Module, conv_plain
from .pspnet import PSPNet, _config, _dropout2d, _ignore_index_of, head_loss


def _cbr3x3(cin, cout, norm_layer):
    return ConvBnRelu(cin, cout, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer)


def _classifier(cin, classes):
    return nn.Sequential(nn.Dropout2d(0.1, False), nn.Conv2d(cin, classes, kernel_size=1))


class DANetHead(nn.Module):
    """DANet's head (`DANetHead`), children in its order: conv5a, conv5c, sa, sc, conv51, conv52, conv6, conv7, conv8.
    forward(x) returns the low-resolution fp32 logits (sasc, sa, sc), or sasc alone with aux=False."""

    def __init__(self, in_channels, out_channels, norm_layer=nn.BatchNorm2d):
        super(DANetHead, self).__init__()
        inter = in_channels // 4
        self.conv5a = _cbr3x3(in_channels, inter, norm_layer)
        self.conv5c = _cbr3x3(in_channels, inter, norm_layer)
        self.sa = PAM_Module(inter)
        self.sc = CAM_Module(inter)
        self.conv51 = _cbr3x3(inter, inter, norm_layer)
        self.conv52 = _cbr3x3(inter, inter, norm_layer)
        self.conv6 = _classifier(inter, out_channels)
        self.conv7 = _classifier(inter, out_channels)
        self.conv8 = _classifier(inter, out_channels)
        self.out_channels = out_channels

    def _logits(self, seq, x):
        K = self.out_channels
        return conv_plain(_dropout2d(x, seq[0].p, self.training), seq[1], out_f32=True, ocs=(K + 31) // 32 * 32)

    def forward(self, x, aux=True):
        sa_conv = self.conv51(self.sa(self.conv5a(x)))
        sc_conv = self.conv52(self.sc(self.conv5c(x)))
        sasc = self._logits(self.conv8, ops.AddFn.apply(sa_conv, sc_conv))
        if not aux:
            return sasc
        return sasc, self._logits(self.conv6, sa_conv), self._logits(self.conv7, sc_conv)


class DANet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(DANet, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.head = DANetHead(2048, out_planes, norm_layer)
        self.business_layer = [self.head]
        self.criterion = criterion
        self.out_planes = out_planes

    _nostride_dilate = PSPNet._nostride_dilate

    def _crit(self, lo, label, H, W):
        crit = self.criterion
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        return head_loss(lo, label, H, W, self.out_planes, _ignore_index_of(crit))

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        H, W = int(data.shape[2]), int(data.shape[3])
        if label is None:
            lo = self.head(blocks[-1], aux=False)
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        sasc, sa, sc = self.head(blocks[-1])
        return self._crit(sasc, label, H, W) + self._crit(sa, label, H, W) + self._crit(sc, label, H, W)
