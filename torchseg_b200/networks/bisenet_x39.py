"""BiSeNet with the Xception-39 context path, with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.X39/network.py:18-169) on the libtsb path.

Differences from the R18 network: xception39 context path (256 / 128 / 64-channel stages), 128-channel aux heads, and
the three losses go through `ohem_criterion` (X39 train.py:48-54 passes CrossEntropyLoss as `criterion` and
ProbOhemCrossEntropy2d as `ohem_criterion`). As in R18, each head ends in the fused bilinear-upsample + OHEM loss when
the criterion supports it (`forward_lowres`), so the full-resolution logits are never materialised.
"""
import torch
import torch.nn as nn

from .. import ops
from ..base_model import xception39
from ..seg_opr.seg_oprs import ConvBnRelu, AttentionRefinement, FeatureFusion, upsample_bilinear
from .bisenet import SpatialPath, BiSeNetHead


class BiSeNet(nn.Module):
    def __init__(self, out_planes, is_training, criterion, ohem_criterion, pretrained_model=None,
                 norm_layer=nn.BatchNorm2d):
        super(BiSeNet, self).__init__()
        self.context_path = xception39(pretrained_model, norm_layer=norm_layer)
        self.business_layer = []
        self.is_training = is_training
        self.out_planes = out_planes
        self.spatial_path = SpatialPath(3, 128, norm_layer)
        conv_channel = 128
        self.global_context = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            ConvBnRelu(256, conv_channel, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer))
        arms = [AttentionRefinement(256, conv_channel, norm_layer), AttentionRefinement(128, conv_channel, norm_layer)]
        refines = [ConvBnRelu(conv_channel, conv_channel, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                              has_bias=False),
                   ConvBnRelu(conv_channel, conv_channel, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                              has_bias=False)]
        heads = [BiSeNetHead(conv_channel, out_planes, 16, True, norm_layer, aux_mid=128),
                 BiSeNetHead(conv_channel, out_planes, 8, True, norm_layer, aux_mid=128),
                 BiSeNetHead(conv_channel * 2, out_planes, 8, False, norm_layer)]
        self.ffm = FeatureFusion(conv_channel * 2, conv_channel * 2, 1, norm_layer)
        self.arms = nn.ModuleList(arms)
        self.refines = nn.ModuleList(refines)
        self.heads = nn.ModuleList(heads)
        self.business_layer.append(self.spatial_path)
        self.business_layer.append(self.global_context)
        self.business_layer.append(self.arms)
        self.business_layer.append(self.refines)
        self.business_layer.append(self.heads)
        self.business_layer.append(self.ffm)
        if is_training:
            self.criterion = criterion
            self.ohem_criterion = ohem_criterion

    def features(self, data):
        """network.py:75-98 up to the three head inputs. The spatial path's 7x7/2 stem and the context path's 3x3/2
        stem read the same space-to-depth image (packed once, seg_oprs._packed_image)."""
        spatial_out = self.spatial_path(data)
        context_blocks = self.context_path(data)
        context_blocks.reverse()
        gc = ops.AdaptiveAvgPoolFn.apply(context_blocks[0], 1)
        gc = self.global_context[1](gc)
        gc = upsample_bilinear(gc, context_blocks[0].shape[2:])
        last_fm = gc
        pred_out = []
        for i, (fm, arm, refine) in enumerate(zip(context_blocks[:2], self.arms, self.refines)):
            fm = arm(fm, add=last_fm)  # ARM scale and `fm += last_fm` in one kernel
            last_fm = upsample_bilinear(fm, context_blocks[i + 1].shape[2:])
            last_fm = refine(last_fm)
            pred_out.append(last_fm)
        concate_fm = self.ffm(spatial_out, last_fm)
        pred_out.append(concate_fm)
        return pred_out

    def forward(self, data, label=None):
        pred_out = self.features(data)
        if self.is_training:
            crit = self.ohem_criterion
            fused = hasattr(crit, "forward_lowres")
            losses = []
            for i in (0, 1, 2):
                if fused:
                    lo = self.heads[i].lowres_logits(pred_out[i])
                    losses.append(crit.forward_lowres(lo, label, self.out_planes))
                else:
                    losses.append(crit(self.heads[i](pred_out[i]), label))
            aux_loss0, aux_loss1, main_loss = losses
            return main_loss + aux_loss0 + aux_loss1  # network.py:106-107
        return torch.log_softmax(self.heads[-1](pred_out[-1]), dim=1)
