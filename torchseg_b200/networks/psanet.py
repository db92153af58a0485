"""PSANet (ResNet-101 v1c, dilated-8, point-wise spatial attention head) with the reference's class / attribute /
state_dict names (TorchSeg model/psanet/ade.psanet.R101_v1c/network.py:14-144 — the reference class is still
called `PSPNet` there; both names are exported) on the libtsb path.

The PSA head needs exactly h*w = 3600 positions at 1/8 resolution (480x480 or 473x473 inputs, network.py:88,101):
the 3600-channel attention maps are soft-maxed over their channel dimension and contracted with the 512-channel
reduced feature map by `torch.bmm`; here both contractions (and their two backward GEMMs) run on the wgmma 1x1
convolution kernels (ops.PSABmmFn). Loss: `criterion(log_softmax(x8 up-sampled logits)) + 0.4 * aux` (network.py:41-57),
evaluated like PSPNet through the OHEM kernels with min_kept = 0."""
from functools import partial

import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet50, resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, conv_plain, _as_act
from .pspnet import _ignore_index_of, _dropout2d, _config, head_loss, PSPNet as _PSPNetBase


class PSANet(nn.Module):
    def __init__(self, out_planes, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d, backbone="R101",
                 aux_loss_ratio=0.4):
        super(PSANet, self).__init__()
        make = resnet101 if backbone == "R101" else resnet50
        self.backbone = make(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                             bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.backbone.layer3.apply(partial(self._nostride_dilate, dilate=2))
        self.backbone.layer4.apply(partial(self._nostride_dilate, dilate=4))
        self.business_layer = []
        self.psa_layer = PointwiseSpatialAttention('psa', out_planes, 2048, norm_layer=norm_layer)
        self.aux_layer = nn.Sequential(
            ConvBnRelu(1024, 1024, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(1024, out_planes, kernel_size=1))
        self.business_layer.append(self.psa_layer)
        self.business_layer.append(self.aux_layer)
        self.criterion = criterion
        self.out_planes = out_planes
        self.aux_loss_ratio = aux_loss_ratio

    _nostride_dilate = _PSPNetBase._nostride_dilate
    _aux_logits = _PSPNetBase._aux_logits

    def forward(self, data, label=None):
        blocks = self.backbone(data)
        # network.py:46-49 upsample by scale_factor=8, which only reproduces the input size when it is a multiple of 8
        # (480); `size=` semantics — identical numbers for those sizes — also admit the 713 / 473 crops of BASELINE.json
        H, W = int(data.shape[2]), int(data.shape[3])
        psa_lo = self.psa_layer(blocks[-1])
        if label is None:
            return torch.log_softmax(ops.UpsampleLogitsFn.apply(psa_lo, H, W), dim=1)   # network.py:46-51
        ign = _ignore_index_of(self.criterion)
        loss = head_loss(psa_lo, label, H, W, self.out_planes, ign)
        aux_loss = head_loss(self._aux_logits(blocks[-2]), label, H, W, self.out_planes, ign)
        return loss + self.aux_loss_ratio * aux_loss                         # network.py:55


PSPNet = PSANet   # the name the reference's psanet network.py / train.py use


class PointwiseSpatialAttention(nn.Module):
    """network.py:75-144 — same child names. (`pool_scales` only sizes conv6's input: 2048 + 4*512 = 4096 channels,
    which is what cat([x, proj(psa)]) provides.)"""

    def __init__(self, name, out_planes, fc_dim=4096, pool_scales=[1, 2, 3, 6], norm_layer=nn.BatchNorm2d,
                 positions=3600):
        super(PointwiseSpatialAttention, self).__init__()
        self.inner_channel = 512
        cbr = partial(ConvBnRelu, has_bias=False, norm_layer=norm_layer)
        self.collect_reduction = cbr(fc_dim, 512, 1, 1, 0, has_bn=True, has_relu=True)
        self.collect_attention = nn.Sequential(
            cbr(512, 512, 1, 1, 0, has_bn=True, has_relu=True),
            cbr(512, positions, 1, 1, 0, has_bn=False, has_relu=False))
        self.distribute_reduction = cbr(fc_dim, 512, 1, 1, 0, has_bn=True, has_relu=True)
        self.distribute_attention = nn.Sequential(
            cbr(512, 512, 1, 1, 0, has_bn=True, has_relu=True),
            cbr(512, positions, 1, 1, 0, has_bn=False, has_relu=False))
        self.proj = cbr(1024, 2048, 1, 1, 0, has_bn=True, has_relu=True)
        self.conv6 = nn.Sequential(
            cbr(fc_dim + len(pool_scales) * 512, 512, 3, 1, 1, has_bn=True, has_relu=True),
            nn.Dropout2d(0.1, inplace=False),
            nn.Conv2d(512, out_planes, kernel_size=1))
        self.out_planes = out_planes

    def _branch(self, x, reduction, attention):
        reduce_x = reduction(x)
        # [b, h*w, h, w] attention logits kept in fp32 like the reference: the soft-max over 3600 random-init logits is
        # peaky enough that bf16 logit rounding would show up as a few % in the attention weights
        att = conv_plain(attention[0](reduce_x), attention[1].conv, out_f32=True)
        return ops.PSABmmFn.apply(reduce_x, att)                  # bmm(reduce_x, softmax(att, dim=1))

    def forward(self, x):
        x = _as_act(x)
        collect_fm = self._branch(x, self.collect_reduction, self.collect_attention)
        distribute_fm = self._branch(x, self.distribute_reduction, self.distribute_attention)
        psa_fm = self.proj(ops.ConcatFn.apply(collect_fm, distribute_fm))
        fm = ops.ConcatFn.apply(x, psa_fm)
        fm = self.conv6[0](fm)
        fm = _dropout2d(fm, self.conv6[1].p, self.training)
        K = self.out_planes
        return conv_plain(fm, self.conv6[2], out_f32=True, ocs=(K + 31) // 32 * 32)
