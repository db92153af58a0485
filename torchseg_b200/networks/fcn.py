"""FCN-32s with the reference's class / attribute names (TorchSeg model/fcn/voc.fcn32s.R101_v1c/network.py:13-68).
BASELINE configs[0] uses the ResNet-18 variant (SURVEY.md §8 a15): resnet18(deep_stem=False) with
_FCNHead(512, .) / _FCNHead(256, .). Training forward returns `loss + aux_ratio * aux_loss` (network.py:43-47)
through the fused bilinear-upsample + cross-entropy kernels (plain CE == OHEM with min_kept = 0)."""
import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet18, resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, conv_plain


class FCN(nn.Module):
    def __init__(self, out_planes, criterion=None, inplace=True, pretrained_model=None, norm_layer=nn.BatchNorm2d,
                 backbone="R18", aux_loss_ratio=0.5, ignore_label=255, bn_eps=1e-5, bn_momentum=0.1):
        super(FCN, self).__init__()
        if backbone == "R18":
            self.backbone = resnet18(pretrained_model, norm_layer=norm_layer, bn_eps=bn_eps, bn_momentum=bn_momentum,
                                     deep_stem=False, stem_width=64)
            chans = (512, 256)
        else:
            self.backbone = resnet101(pretrained_model, inplace=inplace, norm_layer=norm_layer, bn_eps=bn_eps,
                                      bn_momentum=bn_momentum, deep_stem=True, stem_width=64)
            chans = (2048, 1024)
        self.business_layer = []
        self.head = _FCNHead(chans[0], out_planes, inplace, norm_layer=norm_layer)
        self.aux_head = _FCNHead(chans[1], out_planes, inplace, norm_layer=norm_layer)
        self.business_layer.append(self.head)
        self.business_layer.append(self.aux_head)
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio
        # train.py:45-47 passes nn.CrossEntropyLoss(reduction='mean', ignore_index=255): its ignore_index wins
        self.ignore_label = int(getattr(criterion, "ignore_index", ignore_label))

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        lo = self.head.lowres_logits(blocks[-1])
        if label is None:
            return ops.UpsampleLogitsFn.apply(lo, lo.shape[2] * 32, lo.shape[3] * 32)
        lo_aux = self.aux_head.lowres_logits(blocks[-2])
        H, W = label.shape[-2:]
        K = self.out_planes
        loss = ops.OhemUpCEFn.apply(lo, label, H, W, K, self.ignore_label, 0.7, 0, None)
        aux = ops.OhemUpCEFn.apply(lo_aux, label, H, W, K, self.ignore_label, 0.7, 0, None)
        return loss + self.aux_loss_ratio * aux


class _FCNHead(nn.Module):
    """network.py:52-68 — children named cbr / dropout / conv1x1"""

    def __init__(self, in_planes, out_planes, inplace=True, norm_layer=nn.BatchNorm2d):
        super(_FCNHead, self).__init__()
        inter_planes = in_planes // 4
        self.cbr = ConvBnRelu(in_planes, inter_planes, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                              has_bias=False)
        self.dropout = nn.Dropout2d(0.1)
        self.conv1x1 = nn.Conv2d(inter_planes, out_planes, kernel_size=1, stride=1, padding=0)

    def lowres_logits(self, x):
        x = self.cbr(x)
        if self.training and self.dropout.p > 0:
            # channel mask drawn by PyTorch's RNG (parity needs identical masks, SURVEY §2.2b); applied as a scale
            N, C = x.shape[:2]
            mask = torch.bernoulli(torch.full((N, C, 1, 1), 1 - self.dropout.p, device=x.device)) / (1 - self.dropout.p)
            x = x * mask.to(x.dtype)
        K = self.conv1x1.out_channels
        return conv_plain(x, self.conv1x1, out_f32=True, ocs=(K + 31) // 32 * 32)
