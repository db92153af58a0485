"""BiSeNet-R18 real-time line with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.R18.speed/network.py:18-171) on the libtsb path.

Differences from the R18 network: 768x1536 crops trained against labels at 1/8 resolution (config.py
gt_down_sampling = 8), so the heads up-sample x2 / x1 / x1 instead of x16 / x8 / x8; 128-channel aux heads; the three
losses go through `ohem_criterion`; and an eval-mode network holds only the main head (`heads = [None, None, head]`)
and returns log-probabilities at 1/8 of the input.
"""
import torch.nn as nn

from ..base_model import resnet18
from .bisenet import BiSeNetBody, _config


class BiSeNet(BiSeNetBody):
    loss_attr = "ohem_criterion"

    def __init__(self, out_planes, is_training, criterion, ohem_criterion, pretrained_model=None,
                 norm_layer=nn.BatchNorm2d):
        super(BiSeNet, self).__init__()
        self._build(resnet18(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                             bn_momentum=_config.bn_momentum, deep_stem=False, stem_width=64),
                    (512, 256), out_planes, is_training, norm_layer, scales=(2, 1, 1), aux_mid=128,
                    eval_aux_heads=False)
        if is_training:
            self.criterion = criterion
            self.ohem_criterion = ohem_criterion
