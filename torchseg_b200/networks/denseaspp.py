"""DenseASPP (ResNet-101 v1c, dilated-8) with its densely connected atrous head (Yang et al., "DenseASPP for Semantic
Segmentation in Street Scenes", CVPR 2018) on the libtsb path, in the style of the reference's network lines (the
reference lists DenseASPP on its To Do list):

  * backbone: `resnet101` with the deep stem, layer3 / layer4 dilated by 2 / 4 through PSPNet's `_nostride_dilate`
    (output stride 8);
  * aspp: DenseASPPModule(2048, 512, 128, rates 3, 6, 12, 18, 24, Dropout2d 0.1), 2688 output channels;
  * dropout: Dropout2d(0.1); cls: a 1x1 classifier with bias (fp32 logits). DenseASPP has no auxiliary head.

Training returns crit(logits) through the criterion's fused up-sampling pair (`forward_lowres`, ProbOhemCrossEntropy2d)
when it has one and through the fused up-sampling cross-entropy (`head_loss`) otherwise, so the full-resolution logits
are never written. Eval (label None) returns the log_softmax of the logits up-sampled to the input size."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import DenseASPPModule, conv_plain
from .pspnet import PSPNet, _config, _dropout2d, _ignore_index_of, head_loss


class DenseASPP(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(DenseASPP, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.aspp = DenseASPPModule(2048, 512, 128, (3, 6, 12, 18, 24), dropout=0.1, norm_layer=norm_layer)
        self.dropout = nn.Dropout2d(0.1)
        self.cls = nn.Conv2d(self.aspp.out_channels, out_planes, kernel_size=1)
        self.business_layer = [self.aspp, self.cls]
        self.criterion = criterion
        self.out_planes = out_planes

    _nostride_dilate = PSPNet._nostride_dilate

    def _logits(self, x):
        K = self.out_planes
        fm = _dropout2d(self.aspp(x), self.dropout.p, self.training)
        return conv_plain(fm, self.cls, out_f32=True, ocs=(K + 31) // 32 * 32)

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        H, W = int(data.shape[2]), int(data.shape[3])
        lo = self._logits(blocks[-1])
        if label is None:
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        crit = self.criterion
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        return head_loss(lo, label, H, W, self.out_planes, _ignore_index_of(crit))
