"""EncNet (ResNet-101 v1c, dilated-8) with the Context Encoding layer and the SE-loss (Zhang et al., CVPR 2018) on the
libtsb path, in the style of the reference's ADE network lines (the reference lists EncNet on its To Do list):

  * backbone: `resnet101` with the deep stem, layer3 / layer4 dilated by 2 / 4 through PSPNet's `_nostride_dilate`;
  * head.conv5: a 3x3 ConvBnRelu 2048 → 512 (f);
  * head.encmodule: a 1x1 ConvBnRelu, Encoding(D=512, K=32), a BatchNorm over the codewords (`norm_layer(32)` with
    BatchNorm1d(K) semantics on [B, K, D]: statistics over B and D), ReLU and the mean over the codewords (en [B, 512]);
    `fc` (Linear 512 → 512) + sigmoid gives the channel gate γ, the head's output is relu(f + f·γ); `selayer`
    (Linear 512 → classes) gives the SE logits;
  * head.conv6: Dropout2d(0.1) + a 1x1 classifier with bias; aux_layer: PSPNet's, on layer3.

Training returns CE(up(logits)) + aux_loss_ratio · CE(up(aux)) + se_loss_ratio · BCELoss(sigmoid(se), presence(label)),
each CE on the fused up-sampling kernels (`head_loss`) and the SE-loss with the presence vector built on the device. Eval
(label None) returns the log_softmax of the logits up-sampled to the input size."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, Encoding, SELayer, conv_plain, _as_act, _bn_momentum
from .pspnet import PSPNet, _config, _dropout2d, _ignore_index_of, head_loss


class EncNet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d, aux_loss_ratio=0.2,
                 se_loss_ratio=0.2):
        super(EncNet, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.head = EncHead(2048, out_planes, norm_layer=norm_layer)
        self.aux_layer = nn.Sequential(
            ConvBnRelu(1024, 1024, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(1024, out_planes, kernel_size=1))
        self.business_layer = [self.head, self.aux_layer]
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio
        self.se_loss_ratio = se_loss_ratio

    _nostride_dilate = PSPNet._nostride_dilate
    _aux_logits = PSPNet._aux_logits

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        H, W = int(data.shape[2]), int(data.shape[3])
        lo, se = self.head(blocks[-1], with_se=label is not None)
        if label is None:
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(lo, H, W), dim=1)
        ign = _ignore_index_of(self.criterion)
        loss = head_loss(lo, label, H, W, self.out_planes, ign)
        aux_loss = head_loss(self._aux_logits(blocks[-2]), label, H, W, self.out_planes, ign)
        se_loss = ops.SELossFn.apply(se, label, self.out_planes)
        return loss + self.aux_loss_ratio * aux_loss + self.se_loss_ratio * se_loss


class EncModule(nn.Module):
    """conv → Encoding → BN over the codewords → ReLU → mean over the codewords (en); forward(f) returns
    (relu(f + f·sigmoid(fc(en))), selayer(en)), the SE logits as fp32 [B, classes, 1, 1] (None unless with_se)"""

    def __init__(self, in_planes, out_planes, num_codes=32, norm_layer=nn.BatchNorm2d):
        super(EncModule, self).__init__()
        self.conv = ConvBnRelu(in_planes, in_planes, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                               norm_layer=norm_layer)
        self.encoding = Encoding(D=in_planes, K=num_codes)
        self.bn = norm_layer(num_codes)
        self.fc = nn.Linear(in_planes, in_planes)
        self.selayer = nn.Linear(in_planes, out_planes)

    def forward(self, f, with_se=True):
        f = _as_act(f)
        E = self.encoding(self.conv(f))                 # [B, K, D, 1]: rows b·D + d, channel k
        bn = self.bn
        e = ops.BNFn.apply(E, bn.weight, bn.bias, bn.running_mean, bn.running_var, float(bn.eps), _bn_momentum(bn),
                           bool(bn.training), True)
        en = ops.ChanMeanFn.apply(e)                     # [B, D, 1, 1]
        # relu(f + f·γ) is f·(1 + γ): f is a ReLU output and 1 + γ > 0, so the relu is the identity, and its backward
        # mask is conv5's own ReLU mask; the FFM kernel with base 1 computes exactly these values and gradients
        y = ops.ChanScaleFn.apply(f, SELayer._linear(en, self.fc), None, 1.0)
        if not with_se:
            return y, None
        K = self.selayer.out_features
        w = self.selayer.weight
        se = ops.ConvFn.apply(en, w.view(K, w.shape[1], 1, 1), self.selayer.bias, 1, 0, 1, True, (K + 31) // 32 * 32)
        return y, se


class EncHead(nn.Module):
    def __init__(self, in_planes, out_planes, norm_layer=nn.BatchNorm2d):
        super(EncHead, self).__init__()
        self.conv5 = ConvBnRelu(in_planes, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False,
                                norm_layer=norm_layer)
        self.encmodule = EncModule(512, out_planes, num_codes=32, norm_layer=norm_layer)
        self.conv6 = nn.Sequential(nn.Dropout2d(0.1, inplace=False), nn.Conv2d(512, out_planes, kernel_size=1))
        self.out_planes = out_planes

    def forward(self, x, with_se=True):
        y, se = self.encmodule(self.conv5(x), with_se)
        y = _dropout2d(y, self.conv6[0].p, self.training)
        K = self.out_planes
        return conv_plain(y, self.conv6[1], out_f32=True, ocs=(K + 31) // 32 * 32), se
