"""OCNet (ResNet-101 v1c, dilated-8) with the Base-OC object-context head (Yuan & Wang, "OCNet: Object Context Network
for Scene Parsing") on the libtsb path, in the style of the reference's network lines (the reference lists OCNet on its
To Do list):

  * backbone: `resnet101` with the deep stem, layer3 / layer4 dilated by 2 / 4 through PSPNet's `_nostride_dilate`
    (output stride 8);
  * context: a 3x3 ConvBnRelu 2048 → 512, then BaseOCModule(512, 512, key 256, value 256, Dropout2d 0.05): dense
    self-attention over every pixel of the 1/8-resolution map, fused on tsb_attention_{fwd,bwd};
  * cls: a 1x1 classifier with bias (fp32 logits); aux_layer: OCNet's deep supervision on layer3, ConvBnRelu 1024 → 512,
    Dropout2d(0.1) and a 1x1 classifier.

Training returns crit(logits) + aux_loss_ratio · crit(aux), each through the criterion's fused up-sampling pair
(`forward_lowres`, ProbOhemCrossEntropy2d) when it has one and through the fused up-sampling cross-entropy (`head_loss`)
otherwise, so the full-resolution logits are never written. Eval (label None) returns the log_softmax of the logits
up-sampled to the input size."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import BaseOCModule, ConvBnRelu, conv_plain
from .pspnet import PSPNet, _config, _dropout2d, _ignore_index_of, head_loss


class OCNet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d, aux_loss_ratio=0.4):
        super(OCNet, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.context = nn.Sequential(
            ConvBnRelu(2048, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer),
            BaseOCModule(512, 512, 256, 256, dropout=0.05, sizes=(1,), norm_layer=norm_layer))
        self.cls = nn.Conv2d(512, out_planes, kernel_size=1)
        self.aux_layer = nn.Sequential(
            ConvBnRelu(1024, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(512, out_planes, kernel_size=1))
        self.business_layer = [self.context, self.cls, self.aux_layer]
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio

    _nostride_dilate = PSPNet._nostride_dilate

    def _logits(self, x):
        K = self.out_planes
        return conv_plain(self.context(x), self.cls, out_f32=True, ocs=(K + 31) // 32 * 32)

    def _aux_logits(self, x):
        fm = _dropout2d(self.aux_layer[0](x), self.aux_layer[1].p, self.training)
        K = self.out_planes
        return conv_plain(fm, self.aux_layer[2], out_f32=True, ocs=(K + 31) // 32 * 32)

    def _crit(self, lo, label, H, W):
        crit = self.criterion
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        return head_loss(lo, label, H, W, self.out_planes, _ignore_index_of(crit))

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        H, W = int(data.shape[2]), int(data.shape[3])
        lo = self._logits(blocks[-1])
        if label is None:
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        loss = self._crit(lo, label, H, W)
        return loss + self.aux_loss_ratio * self._crit(self._aux_logits(blocks[-2]), label, H, W)
