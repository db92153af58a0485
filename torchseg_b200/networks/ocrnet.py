"""OCRNet (ResNet-101 v1c, dilated-8) with the object-contextual head (Yuan, Chen & Wang, "Object-Contextual
Representations for Semantic Segmentation", ECCV 2020; the layout of the authors' ResNet-101 `SpatialOCRNet`) on the
libtsb path, in the style of the reference's network lines:

  * backbone: `resnet101` with the deep stem, layer3 / layer4 dilated by 2 / 4 through PSPNet's `_nostride_dilate`
    (output stride 8);
  * dsn_head on layer3: 3x3 ConvBnRelu 1024 → 512, Dropout2d(0.05) and a 1x1 classifier with bias: the fp32 aux logits,
    which are also the soft object regions;
  * conv_3x3 on layer4: 3x3 ConvBnRelu 2048 → 512;
  * spatial_context_head (SpatialGatherModule): the object-region proxy, a soft-max over the pixels of each image of
    the aux logits (tsb_spatial_softmax_*) and a per-image GEMM with the features, [B, 512, K, 1];
  * spatial_ocr_head (SpatialOCRModule(512, 256, 512, dropout 0.05)): every pixel attends over the K regions of its
    image (the cross form of the fused attention kernels), then 1x1 ConvBnRelu on [context, features];
  * head: a 1x1 classifier with bias (fp32 logits).

Training returns crit(logits) + aux_loss_ratio · crit(aux), each through the criterion's fused up-sampling pair
(`forward_lowres`, ProbOhemCrossEntropy2d) when it has one and through the fused up-sampling cross-entropy (`head_loss`)
otherwise; the aux logits get gradient from both their loss and the gather. Eval (label None) still runs dsn_head,
whose logits the gather needs, and returns the log_softmax of the logits up-sampled to the input size."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, SpatialGatherModule, SpatialOCRModule, conv_plain
from .pspnet import PSPNet, _config, _dropout2d, _ignore_index_of, head_loss


def _cbr3x3(cin, cout, norm_layer):
    return ConvBnRelu(cin, cout, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer)


class OCRNet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d, aux_loss_ratio=0.4):
        super(OCRNet, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.conv_3x3 = _cbr3x3(2048, 512, norm_layer)
        self.spatial_context_head = SpatialGatherModule(out_planes)
        self.spatial_ocr_head = SpatialOCRModule(512, 256, 512, dropout=0.05, norm_layer=norm_layer)
        self.head = nn.Conv2d(512, out_planes, kernel_size=1)
        self.dsn_head = nn.Sequential(
            _cbr3x3(1024, 512, norm_layer),
            nn.Dropout2d(0.05, inplace=False),
            nn.Conv2d(512, out_planes, kernel_size=1))
        self.business_layer = [self.conv_3x3, self.spatial_ocr_head, self.head, self.dsn_head]
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio

    _nostride_dilate = PSPNet._nostride_dilate

    def _classify(self, x, conv):
        K = self.out_planes
        return conv_plain(x, conv, out_f32=True, ocs=(K + 31) // 32 * 32)

    def _crit(self, lo, label, H, W):
        crit = self.criterion
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        return head_loss(lo, label, H, W, self.out_planes, _ignore_index_of(crit))

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        H, W = int(data.shape[2]), int(data.shape[3])
        fm = _dropout2d(self.dsn_head[0](blocks[-2]), self.dsn_head[1].p, self.training)
        dsn = self._classify(fm, self.dsn_head[2])
        f = self.conv_3x3(blocks[-1])
        ctx = self.spatial_context_head(f, dsn)
        lo = self._classify(self.spatial_ocr_head(f, ctx), self.head)
        if label is None:
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        return self._crit(lo, label, H, W) + self.aux_loss_ratio * self._crit(dsn, label, H, W)
