"""BiSeNet with the ResNet-101 context path, with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.R101/network.py:18-168) on the libtsb path.

Differences from the R18 network: resnet101(deep_stem=True, stem_width=64), not dilated (output stride 32), so the
ARMs and the global-context conv read the 2048 / 1024-channel stages; the main head is 256 channels wide. The rest is
the R18 recipe: full-resolution labels, heads x16 / x8 / x8, the losses through `criterion`.
"""
import torch.nn as nn

from ..base_model import resnet101
from .bisenet import BiSeNetBody, _config


class BiSeNet(BiSeNetBody):
    def __init__(self, out_planes, is_training, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(BiSeNet, self).__init__()
        self._build(resnet101(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                              bn_momentum=_config.bn_momentum, deep_stem=True, stem_width=64),
                    (2048, 1024), out_planes, is_training, norm_layer, main_mid=256)
        if is_training:
            self.criterion = criterion
