"""DeepLabV3+ (ResNet-101 v1c, output stride 16) on the libtsb path, in the style of the reference's network lines.

The reference lists DeepLab v3 / v3+ on its To Do list and ships the block it is built from,
`seg_opr.seg_oprs.SeparableConvBnRelu` (furnace/seg_opr/seg_oprs.py:76-94); this line composes the reference's
`resnet101` (deep stem), `ConvBnRelu` and `SeparableConvBnRelu`:

  * backbone: layer4 de-strided and dilated by 2 (`_nostride_dilate`, as PSPNet does with 2 / 4), so layer4 runs at 1/16;
  * aspp: a 1x1 ConvBnRelu and three atrous separable convs (dilation 6, 12, 18) on layer4, an image-pooling branch
    (global average pool → 1x1 ConvBnRelu → bilinear back), concatenated in that order, a 1x1 projection to 256 channels
    and Dropout2d(0.1);
  * decoder: layer1 reduced to 48 channels by a 1x1 ConvBnRelu, the ASPP output up-sampled (bilinear, align_corners) to
    layer1's size and concatenated in front of it (304 channels), two 3x3 SeparableConvBnRelu to 256 channels and a 1x1
    classifier with bias.

Training returns `criterion(logits up-sampled to the label size)`; with ProbOhemCrossEntropy2d the up-sampling is fused
into the OHEM kernel pair (`forward_lowres`) and the full-resolution logits are never written. Eval (label None) returns
the log_softmax of the logits up-sampled to the input size."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, SeparableConvBnRelu, conv_plain, upsample_bilinear, _as_act
from .pspnet import PSPNet, _config, _dropout2d


class DeepLabV3Plus(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(DeepLabV3Plus, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=2))
        self.aspp = ASPP(2048, 256, (6, 12, 18), norm_layer=norm_layer)
        self.decoder = Decoder(out_planes, 256, 256, 48, norm_layer=norm_layer)
        self.business_layer = [self.aspp, self.decoder]
        self.criterion = criterion
        self.out_planes = out_planes

    _nostride_dilate = PSPNet._nostride_dilate

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        lo = self.decoder(self.aspp(blocks[-1]), blocks[0])
        if label is None:
            H, W = int(data.shape[2]), int(data.shape[3])
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        crit = self.criterion
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        return crit(ops.UpsampleLogitsFn.apply(lo, label.shape[-2], label.shape[-1]), label)


class ASPP(nn.Module):
    """atrous spatial pyramid pooling: branches[0] a 1x1 ConvBnRelu, branches[1..] 3x3 atrous SeparableConvBnRelu at
    `rates`, pool the image-level branch; concatenated, projected by a 1x1 ConvBnRelu, then Dropout2d(0.1)"""

    def __init__(self, in_planes, planes, rates, norm_layer=nn.BatchNorm2d):
        super(ASPP, self).__init__()
        self.branches = nn.ModuleList(
            [ConvBnRelu(in_planes, planes, 1, 1, 0, norm_layer=norm_layer)] +
            [SeparableConvBnRelu(in_planes, planes, 3, 1, d, d, norm_layer=norm_layer) for d in rates])
        self.pool = nn.Sequential(nn.AdaptiveAvgPool2d(1), ConvBnRelu(in_planes, planes, 1, 1, 0, norm_layer=norm_layer))
        self.project = ConvBnRelu(planes * (len(rates) + 2), planes, 1, 1, 0, norm_layer=norm_layer)
        self.dropout = nn.Dropout2d(0.1)

    def forward(self, x):
        x = _as_act(x)
        H, W = x.shape[2:]
        outs = [b(x) for b in self.branches]
        outs.append(upsample_bilinear(self.pool[1](ops.AdaptiveAvgPoolFn.apply(x, 1)), (H, W)))
        fm = self.project(ops.ConcatFn.apply(*outs))
        return _dropout2d(fm, self.dropout.p, self.training)


class Decoder(nn.Module):
    """reduce the 1/4-resolution layer1 features to `low_planes`, concatenate them behind the up-sampled ASPP output,
    refine with two 3x3 SeparableConvBnRelu and classify (1x1 conv with bias, fp32 logits)"""

    def __init__(self, out_planes, in_planes=256, planes=256, low_planes=48, norm_layer=nn.BatchNorm2d):
        super(Decoder, self).__init__()
        self.reduce = ConvBnRelu(256, low_planes, 1, 1, 0, norm_layer=norm_layer)
        self.refine = nn.Sequential(
            SeparableConvBnRelu(in_planes + low_planes, planes, 3, 1, 1, 1, norm_layer=norm_layer),
            SeparableConvBnRelu(planes, planes, 3, 1, 1, 1, norm_layer=norm_layer))
        self.classifier = nn.Conv2d(planes, out_planes, 1, bias=True)

    def forward(self, x, low):
        # the 48-channel reduction comes back in a 64-channel buffer whose last 16 channels are exact zeros (ragged
        # ConvBnRelu); behind the 256 ASPP channels those zeros are the channels the 304-channel refine conv does not read
        low = self.reduce(low)
        x = upsample_bilinear(x, low.shape[2:])
        fm = ops.ConcatFn.apply(x, low)
        fm = self.refine(fm)
        K = self.out_planes
        return conv_plain(fm, self.classifier, out_f32=True, ocs=(K + 31) // 32 * 32)

    @property
    def out_planes(self):
        return self.classifier.out_channels
