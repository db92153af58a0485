"""init_weight / group_weight with the reference semantics (TorchSeg furnace/utils/init_func.py:11-57)."""
import torch.nn as nn

_CONV = (nn.Conv2d, nn.Conv3d, nn.ConvTranspose2d)
_NORM_EXTRA = (nn.GroupNorm, nn.InstanceNorm2d, nn.LayerNorm)


def _init_one(feature, conv_init, norm_layer, bn_eps, bn_momentum, **kwargs):
    for _, m in feature.named_modules():
        if isinstance(m, _CONV):
            conv_init(m.weight, **kwargs)
        elif isinstance(m, norm_layer):
            m.eps = bn_eps
            m.momentum = bn_momentum
            nn.init.constant_(m.weight, 1)
            nn.init.constant_(m.bias, 0)


def init_weight(module_list, conv_init, norm_layer, bn_eps, bn_momentum, **kwargs):
    """init_func.py:23-31"""
    if isinstance(module_list, list):
        for feature in module_list:
            _init_one(feature, conv_init, norm_layer, bn_eps, bn_momentum, **kwargs)
    else:
        _init_one(module_list, conv_init, norm_layer, bn_eps, bn_momentum, **kwargs)


def group_weight(weight_group, module, norm_layer, lr, no_decay_lr=None):
    """init_func.py:34-57: [decay: conv/linear weights] + [no decay: biases, norm γ/β]; asserts completeness."""
    from ..seg_opr.seg_oprs import CAM_Module, Encoding, PAM_Module
    decay, no_decay = [], []
    for m in module.modules():
        if isinstance(m, Encoding):   # EncNet: the codewords decay, the smoothing factors do not
            decay.append(m.codewords)
            no_decay.append(m.scale)
        elif isinstance(m, (PAM_Module, CAM_Module)):   # DANet: gamma does not decay (the convs are visited on their own)
            no_decay.append(m.gamma)
        elif isinstance(m, nn.Linear) or isinstance(m, _CONV):
            decay.append(m.weight)
            if m.bias is not None:
                no_decay.append(m.bias)
        elif isinstance(m, norm_layer) or isinstance(m, _NORM_EXTRA):
            if m.weight is not None:
                no_decay.append(m.weight)
            if m.bias is not None:
                no_decay.append(m.bias)
    assert len(list(module.parameters())) == len(decay) + len(no_decay)
    weight_group.append(dict(params=decay, lr=lr))
    lr = lr if no_decay_lr is None else no_decay_lr
    weight_group.append(dict(params=no_decay, weight_decay=.0, lr=lr))
    return weight_group
