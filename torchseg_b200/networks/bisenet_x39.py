"""BiSeNet with the Xception-39 context path, with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.X39/network.py:18-169) on the libtsb path.

Differences from the R18 network: xception39 context path (256 / 128 / 64-channel stages), 128-channel aux heads, and
the three losses go through `ohem_criterion` (X39 train.py:48-54 passes CrossEntropyLoss as `criterion` and
ProbOhemCrossEntropy2d as `ohem_criterion`). As in R18, each head ends in the fused bilinear-upsample + OHEM loss when
the criterion supports it (`forward_lowres`), so the full-resolution logits are never materialised.
"""
import torch.nn as nn

from ..base_model import xception39
from .bisenet import BiSeNetBody


class BiSeNet(BiSeNetBody):
    loss_attr = "ohem_criterion"

    def __init__(self, out_planes, is_training, criterion, ohem_criterion, pretrained_model=None,
                 norm_layer=nn.BatchNorm2d):
        super(BiSeNet, self).__init__()
        self._build(xception39(pretrained_model, norm_layer=norm_layer), (256, 128), out_planes, is_training,
                    norm_layer, aux_mid=128)
        if is_training:
            self.criterion = criterion
            self.ohem_criterion = ohem_criterion
