"""DFN (ResNet-101 v1c) with the reference's class / attribute / state_dict names
(TorchSeg model/dfn/cityscapes.dfn.R101_v1c/network.py:15-172) on the libtsb path.

Training forward returns `Σ₄ criterion(smooth head) + alpha · Σ₄ aux_criterion(border head)` (network.py:139-152).
Smooth network (network.py:94-119): global context → per stage RRB → CAB(with the up-sampled deeper stage) → RRB →
DFNHead. Border network (network.py:121-137): bottom-up RRBs accumulated at 1/4 resolution → DFNHead(·, 1, 4).

The 21 / 171 / 9-channel layers of the border network and of every DFNHead run zero-padded to multiples of 64
channels (seg_oprs._ragged); parameters keep the reference shapes. When the smooth criterion is a plain
nn.CrossEntropyLoss (train.py:48-49) or ProbOhemCrossEntropy2d (the commented alternative, train.py:50-51) the ×4…×32
bilinear up-sampling of the 19-class logits is fused into the loss kernels and the full-resolution logits are never
written."""
import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet101
from ..seg_opr.seg_oprs import ConvBnRelu, RefineResidual, ChannelAttention, conv_plain, upsample_bilinear, _as_act
from .bisenet import _UpsampleLogitsFn
from .pspnet import _ignore_index_of


class _Cfg(object):
    bn_eps = 1e-5
    bn_momentum = 0.1


try:
    from config import config as _config
except Exception:  # noqa: BLE001
    _config = _Cfg()


class DFN(nn.Module):
    def __init__(self, out_planes, criterion, aux_criterion, alpha, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(DFN, self).__init__()
        self.backbone = resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                  bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64)
        self.business_layer = []
        smooth_inner_channel = 512
        self.global_context = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            ConvBnRelu(2048, smooth_inner_channel, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                       norm_layer=norm_layer))
        self.business_layer.append(self.global_context)

        stage = [2048, 1024, 512, 256]
        smooth_pre_rrbs, cabs, smooth_aft_rrbs, smooth_heads = [], [], [], []
        for i, channel in enumerate(stage):
            smooth_pre_rrbs.append(RefineResidual(channel, smooth_inner_channel, 3, has_bias=False, has_relu=True,
                                                  norm_layer=norm_layer))
            cabs.append(ChannelAttention(smooth_inner_channel * 2, smooth_inner_channel, 1))
            smooth_aft_rrbs.append(RefineResidual(smooth_inner_channel, smooth_inner_channel, 3, has_bias=False,
                                                  has_relu=True, norm_layer=norm_layer))
            smooth_heads.append(DFNHead(smooth_inner_channel, out_planes, 2 ** (5 - i), norm_layer=norm_layer))

        stage.reverse()
        border_inner_channel = 21
        border_pre_rrbs, border_aft_rrbs, border_heads = [], [], []
        for i, channel in enumerate(stage):
            border_pre_rrbs.append(RefineResidual(channel, border_inner_channel, 3, has_bias=False, has_relu=True,
                                                  norm_layer=norm_layer))
            border_aft_rrbs.append(RefineResidual(border_inner_channel, border_inner_channel, 3, has_bias=False,
                                                  has_relu=True, norm_layer=norm_layer))
            border_heads.append(DFNHead(border_inner_channel, 1, 4, norm_layer=norm_layer))

        self.smooth_pre_rrbs = nn.ModuleList(smooth_pre_rrbs)
        self.cabs = nn.ModuleList(cabs)
        self.smooth_aft_rrbs = nn.ModuleList(smooth_aft_rrbs)
        self.smooth_heads = nn.ModuleList(smooth_heads)
        self.border_pre_rrbs = nn.ModuleList(border_pre_rrbs)
        self.border_aft_rrbs = nn.ModuleList(border_aft_rrbs)
        self.border_heads = nn.ModuleList(border_heads)
        for m in (self.smooth_pre_rrbs, self.cabs, self.smooth_aft_rrbs, self.smooth_heads, self.border_pre_rrbs,
                  self.border_aft_rrbs, self.border_heads):
            self.business_layer.append(m)

        self.criterion = criterion
        self.aux_criterion = aux_criterion
        self.alpha = alpha
        self.out_planes = out_planes

    # ------------------------------------------------------------------------------------------
    def _smooth_features(self, blocks):
        """network.py:94-119 → the four DFNHead inputs, deepest first"""
        deep = blocks[::-1]
        gc = ops.AdaptiveAvgPoolFn.apply(_as_act(deep[0]), 1)
        gc = self.global_context[1](gc)
        last_fm = upsample_bilinear(gc, deep[0].shape[2:])
        feats = []
        for i, (fm, pre_rrb, cab, aft_rrb) in enumerate(zip(deep, self.smooth_pre_rrbs, self.cabs,
                                                            self.smooth_aft_rrbs)):
            fm = pre_rrb(fm)
            fm = cab(fm, last_fm)
            fm = aft_rrb(fm)
            feats.append(fm)
            if i != 3:
                H, W = fm.shape[2:]
                last_fm = upsample_bilinear(fm, (H * 2, W * 2))
        return feats

    def _border_features(self, blocks):
        """network.py:121-137 → the four border DFNHead inputs (all at 1/4 resolution, 21 → 64-padded channels)"""
        last_fm = None
        feats = []
        for i, (fm, pre_rrb, aft_rrb) in enumerate(zip(blocks, self.border_pre_rrbs, self.border_aft_rrbs)):
            fm = pre_rrb(fm)
            if last_fm is not None:
                H, W = fm.shape[2:]
                fm = upsample_bilinear(fm, (H * 2 ** i, W * 2 ** i))
                last_fm = ops.AddFn.apply(last_fm, fm)
                last_fm = aft_rrb(last_fm)
            else:
                last_fm = fm
            feats.append(last_fm)
        return feats

    def _smooth_loss(self, lo, label):
        crit = self.criterion
        H, W = label.shape[-2:]
        if hasattr(crit, "forward_lowres"):
            return crit.forward_lowres(lo, label, self.out_planes)
        if isinstance(crit, nn.CrossEntropyLoss) and crit.reduction == 'mean' and crit.label_smoothing == 0.0 and \
                self.out_planes <= 32:
            # CrossEntropyLoss(mean, ignore_index) == OHEM with thresh 1 / min_kept 0 (every valid pixel kept)
            return ops.OhemUpCEFn.apply(lo, label, H, W, self.out_planes, int(crit.ignore_index), 1.0, 0, crit.weight)
        return None

    def forward(self, data, label=None, aux_label=None):
        blocks = self.backbone(data)
        smooth = self._smooth_features(blocks)
        if label is None or aux_label is None:
            return torch.log_softmax(self.smooth_heads[3](smooth[3]), dim=1)
        border = self._border_features(blocks)
        loss = None
        for fm, head in zip(smooth, self.smooth_heads):
            lo = head.lowres_logits(fm)
            if lo.shape[2] * head.scale != label.shape[-2] or lo.shape[3] * head.scale != label.shape[-1]:
                raise ValueError("DFN: label size must be scale x the head resolution")
            li = self._smooth_loss(lo, label)
            if li is None:
                li = self.criterion(_UpsampleLogitsFn.apply(lo, lo.shape[2] * head.scale, lo.shape[3] * head.scale), label)
            loss = li if loss is None else loss + li
        aux_loss = None
        for fm, head in zip(border, self.border_heads):
            li = self.aux_criterion(head(fm), aux_label)
            aux_loss = li if aux_loss is None else aux_loss + li
        return loss + self.alpha * aux_loss


class DFNHead(nn.Module):
    """network.py:157-172: RRB(in → 9·out) → 1x1(9·out → out, bias) → bilinear ×scale"""

    def __init__(self, in_planes, out_planes, scale, norm_layer=nn.BatchNorm2d):
        super(DFNHead, self).__init__()
        self.rrb = RefineResidual(in_planes, out_planes * 9, 3, has_bias=False, has_relu=False, norm_layer=norm_layer)
        self.conv = nn.Conv2d(out_planes * 9, out_planes, kernel_size=1, stride=1, padding=0)
        self.scale = scale

    def lowres_logits(self, x):
        """fp32 NHWC logits at head resolution"""
        x = self.rrb(x)
        K = self.conv.out_channels
        return conv_plain(x, self.conv, out_f32=True, ocs=(K + 31) // 32 * 32)

    def forward(self, x):
        lo = self.lowres_logits(x)
        if self.scale > 1:
            return _UpsampleLogitsFn.apply(lo, lo.shape[2] * self.scale, lo.shape[3] * self.scale)
        return lo
