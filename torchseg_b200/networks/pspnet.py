"""PSPNet (ResNet-101 v1c, dilated-8) with the reference's class / attribute / state_dict names
(TorchSeg model/pspnet/ade.pspnet.R101_v1c/network.py:14-109) on the libtsb path.

Training forward returns `loss + 0.4 * aux_loss` (network.py:53-57). The reference applies log_softmax and then
nn.CrossEntropyLoss (a second, idempotent log_softmax); here each head ends in ONE fused kernel pair (bilinear up-sampling to
the input size + cross-entropy with the criterion's ignore_index, `ops.CEUpFn`): the 150-class full-resolution logits are
never materialised. (`FUSED_CE = False` restores the materialised form: NCHW fp32 logits + the OHEM kernels with min_kept = 0.)"""
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet50, resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, conv_plain, upsample_bilinear, _as_act
from .bisenet import _UpsampleLogitsFn


class _Cfg(object):
    bn_eps = 1e-5
    bn_momentum = 0.1


try:
    from config import config as _config
except Exception:  # noqa: BLE001
    _config = _Cfg()


def _ignore_index_of(criterion, default=-1):
    return int(getattr(criterion, "ignore_index", getattr(criterion, "ignore_label", default)))


FUSED_CE = True   # training heads: fused bilinear up-sampling + cross-entropy (tsb_ce_up_*); False = materialised logits


def head_loss(lo, label, H, W, num_classes, ignore_index):
    """bilinear(align_corners) up-sampling of the low-resolution fp32 logits to H x W + CrossEntropyLoss(mean, ignore_index)
    (network.py:46-55). Fused: the [N, C, H, W] logits are never written (C <= 152); otherwise the up-sampled NCHW fp32
    logits go through the OHEM kernels with min_kept = 0, which is exactly CrossEntropyLoss."""
    if FUSED_CE and num_classes <= ops.FUSED_CE_MAX_CLASSES:
        return ops.CEUpFn.apply(lo, label, H, W, num_classes, ignore_index)
    return ops.OhemCEFn.apply(_UpsampleLogitsFn.apply(lo, H, W), label, ignore_index, 1.0, 0, None)


def _dropout2d(x, p, training):
    """nn.Dropout2d as a per-(sample, channel) scale drawn from PyTorch's RNG (parity needs identical masks)"""
    if not training or p <= 0:
        return x
    N, C = x.shape[:2]
    mask = torch.bernoulli(torch.full((N, C, 1, 1), 1 - p, device=x.device)) / (1 - p)
    return x * mask.to(x.dtype)


class PSPNet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d, backbone="R101",
                 aux_loss_ratio=0.4):
        super(PSPNet, self).__init__()
        make = resnet101 if backbone == "R101" else resnet50
        self.backbone = make(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                             bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.business_layer = []
        self.psp_layer = PyramidPooling('psp', out_planes, 2048, norm_layer=norm_layer)
        self.aux_layer = nn.Sequential(
            ConvBnRelu(1024, 1024, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(1024, out_planes, kernel_size=1))
        self.business_layer.append(self.psp_layer)
        self.business_layer.append(self.aux_layer)
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio

    def _aux_logits(self, x):
        fm = self.aux_layer[0](x)
        fm = _dropout2d(fm, self.aux_layer[1].p, self.training)
        K = self.out_planes
        return conv_plain(fm, self.aux_layer[2], out_f32=True, ocs=(K + 31) // 32 * 32)

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        # network.py:46-49 upsample by scale_factor=8, which only reproduces the input size when it is a multiple of 8
        # (480); `size=` semantics — identical numbers for those sizes — also admit the 713 / 473 crops of BASELINE.json
        H, W = int(data.shape[2]), int(data.shape[3])
        psp_lo = self.psp_layer(blocks[-1])
        if label is None:
            return torch.log_softmax(_UpsampleLogitsFn.apply(psp_lo, H, W), dim=1)   # network.py:46-51
        ign = _ignore_index_of(self.criterion)
        loss = head_loss(psp_lo, label, H, W, self.out_planes, ign)
        aux_loss = head_loss(self._aux_logits(blocks[-2]), label, H, W, self.out_planes, ign)
        return loss + self.aux_loss_ratio * aux_loss           # network.py:56

    def _nostride_dilate(self, m, dilate):
        """network.py:62-72"""
        if isinstance(m, nn.Conv2d):
            if m.stride == (2, 2):
                m.stride = (1, 1)
                if m.kernel_size == (3, 3):
                    m.dilation = (dilate // 2, dilate // 2)
                    m.padding = (dilate // 2, dilate // 2)
            else:
                if m.kernel_size == (3, 3):
                    m.dilation = (dilate, dilate)
                    m.padding = (dilate, dilate)


class PyramidPooling(nn.Module):
    """network.py:75-109 — same child names (the Sequential keys literally contain a slash, SURVEY App. D)"""

    def __init__(self, name, out_planes, fc_dim=4096, pool_scales=[1, 2, 3, 6], norm_layer=nn.BatchNorm2d):
        super(PyramidPooling, self).__init__()
        self.ppm = []
        for scale in pool_scales:
            self.ppm.append(nn.Sequential(OrderedDict([
                ('{}/pool_1'.format(name), nn.AdaptiveAvgPool2d(scale)),
                ('{}/cbr'.format(name), ConvBnRelu(fc_dim, 512, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                                                   norm_layer=norm_layer))])))
        self.ppm = nn.ModuleList(self.ppm)
        self.pool_scales = list(pool_scales)
        self.out_planes = out_planes
        self.conv6 = nn.Sequential(
            ConvBnRelu(fc_dim + len(pool_scales) * 512, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False,
                       norm_layer=norm_layer),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(512, out_planes, kernel_size=1))

    def forward(self, x):
        x = _as_act(x)
        H, W = x.shape[2:]
        outs = [x]
        for scale, pooling in zip(self.pool_scales, self.ppm):
            pooled = ops.AdaptiveAvgPoolFn.apply(x, scale)     # one pass per scale over x (bins of S x S)
            outs.append(upsample_bilinear(pooling[1](pooled), (H, W)))
        fm = ops.ConcatFn.apply(*outs)                          # strided copies into one NHWC buffer
        fm = self.conv6[0](fm)
        fm = _dropout2d(fm, self.conv6[1].p, self.training)
        K = self.out_planes
        return conv_plain(fm, self.conv6[2], out_f32=True, ocs=(K + 31) // 32 * 32)
