"""BiSeNet-X39 real-time line with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.X39.speed/network.py:18-171) on the libtsb path.

The X39 network with the .speed changes: labels at 1/8 resolution (gt_down_sampling = 8), so the heads up-sample
x2 / x1 / x1 instead of x16 / x8 / x8, and an eval-mode network holds only the main head (`heads = [None, None, head]`)
and returns log-probabilities at 1/8 of the input. Head widths stay those of X39 (aux 128, main 64).
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
                    norm_layer, scales=(2, 1, 1), aux_mid=128, eval_aux_heads=False)
        if is_training:
            self.criterion = criterion
            self.ohem_criterion = ohem_criterion
