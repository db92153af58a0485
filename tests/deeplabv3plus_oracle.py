"""ORACLE — test infrastructure only: DeepLabV3+ (ResNet-101 v1c, output stride 16).

Functional fp32 PyTorch restatement of torchseg_b200/networks/deeplabv3plus.py composed from the reference's blocks
(TorchSeg furnace/base_model/resnet.py `resnet101` with the deep stem, furnace/seg_opr/seg_oprs.py `ConvBnRelu` and
`SeparableConvBnRelu`, furnace/seg_opr/loss_opr.py `ProbOhemCrossEntropy2d`), driven by a state_dict with the network's
key names. It builds on the shared blocks of oracle/torch_ref.py and honours its bf16-storage emulation
(`set_bf16_emulation`, re-exported here). Pinned to the live reference composition by tests/test_cpu_deeplabv3plus.py
through tests/golden/live_reference_deeplabv3plus.npz (tools/make_live_golden_deeplabv3plus.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import _bn, bottleneck, conv_bn_relu, ohem_ce, q, qw, set_bf16_emulation

__all__ = ["set_bf16_emulation", "separable_conv_bn_relu", "resnet101_os16", "aspp", "decoder",
           "deeplabv3plus_logits", "deeplabv3plus_loss", "deeplabv3plus_eval"]

RATES = (6, 12, 18)


def separable_conv_bn_relu(x, sd, prefix, dilation, has_relu=True, eps=1e-5, momentum=0.1, training=True, stats=None):
    """SeparableConvBnRelu.forward — seg_oprs.py:76-94 with a 3x3 depthwise conv, stride 1, padding = dilation:
    depthwise conv → BN (no ReLU) → pointwise ConvBnRelu"""
    C = x.shape[1]
    x = q(F.conv2d(x, qw(sd[prefix + ".conv1.weight"]), None, 1, dilation, dilation, C))
    x = q(_bn(x, sd, prefix + ".bn", eps, momentum, training, stats))
    return conv_bn_relu(x, sd, prefix + ".point_wise_cbr", 1, 0, has_relu=has_relu, eps=eps, momentum=momentum,
                        training=training, stats=stats)


def resnet101_os16(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None, layers=(3, 4, 23, 3)):
    """ResNet.forward with the deep stem (resnet.py:110-124,168-184) after `_nostride_dilate(layer4, 2)`
    (pspnet network.py:62-72): layer4's stride-2 3x3 → stride 1 (dilation 1), its other 3x3 → dilation 2, its stride-2
    1x1 downsample → stride 1. Returns the four stage outputs."""
    c = prefix + ".conv1"
    x = q(F.conv2d(q(x), qw(sd[c + ".0.weight"]), None, 2, 1))
    x = q(F.relu(_bn(x, sd, c + ".1", eps, momentum, training, stats)))
    x = q(F.conv2d(x, qw(sd[c + ".3.weight"]), None, 1, 1))
    x = q(F.relu(_bn(x, sd, c + ".4", eps, momentum, training, stats)))
    x = q(F.conv2d(x, qw(sd[c + ".6.weight"]), None, 1, 1))
    x = q(F.relu(_bn(x, sd, prefix + ".bn1", eps, momentum, training, stats)))
    x = F.max_pool2d(x, 3, 2, 1)
    blocks = []
    for li, nblk in enumerate(layers, start=1):
        for bi in range(nblk):
            first = bi == 0
            if li == 1:
                stride, dil2, dstride = 1, 1, 1
            elif li < 4:
                stride, dil2, dstride = (2 if first else 1), 1, 2
            else:
                stride, dil2, dstride = 1, (1 if first else 2), 1
            x = bottleneck(x, sd, "%s.layer%d.%d" % (prefix, li, bi), stride, dil2, first, dstride, eps, momentum,
                           training, stats)
        blocks.append(x)
    return blocks


def aspp(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None, drop=None):
    """ASPP: [1x1 CBR, separable 3x3 at 6 / 12 / 18, image pool → 1x1 CBR → bilinear] → concat → 1x1 CBR → Dropout2d.
    drop: the Dropout2d as a function of the projected map (None: identity)"""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    outs = [conv_bn_relu(x, sd, prefix + ".branches.0", 1, 0, **kw)]
    for i, d in enumerate(RATES, start=1):
        outs.append(separable_conv_bn_relu(x, sd, "%s.branches.%d" % (prefix, i), d, **kw))
    p = q(F.adaptive_avg_pool2d(x, 1))
    p = conv_bn_relu(p, sd, prefix + ".pool.1", 1, 0, **kw)
    outs.append(q(F.interpolate(p, size=x.shape[2:], mode="bilinear", align_corners=True)))
    fm = conv_bn_relu(q(torch.cat(outs, dim=1)), sd, prefix + ".project", 1, 0, **kw)
    return drop(fm) if drop is not None else fm


def decoder(x, low, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """reduce(layer1) → 48 ch; bilinear(ASPP, layer1 size) ++ reduced (304 ch) → two separable 3x3 → 1x1 classifier"""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    low = conv_bn_relu(low, sd, prefix + ".reduce", 1, 0, **kw)
    x = q(F.interpolate(x, size=low.shape[2:], mode="bilinear", align_corners=True))
    fm = torch.cat([x, low], dim=1)
    fm = separable_conv_bn_relu(fm, sd, prefix + ".refine.0", 1, **kw)
    fm = separable_conv_bn_relu(fm, sd, prefix + ".refine.1", 1, **kw)
    return F.conv2d(fm, qw(sd[prefix + ".classifier.weight"]), sd[prefix + ".classifier.bias"])


def deeplabv3plus_logits(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None, drop=None):
    """the 1/4-resolution fp32 logits"""
    blocks = resnet101_os16(data, sd, "backbone", eps, momentum, training, stats)
    a = aspp(blocks[-1], sd, "aspp", eps, momentum, training, stats, drop)
    return decoder(a, blocks[0], sd, "decoder", eps, momentum, training, stats)


def deeplabv3plus_loss(data, label, sd, min_kept, ignore_label=255, thresh=0.7, eps=1e-5, momentum=0.1, stats=None,
                       drop=None):
    """training: ProbOhemCrossEntropy2d on the logits up-sampled (bilinear, align_corners) to the label size"""
    lo = deeplabv3plus_logits(data, sd, eps, momentum, True, stats, drop)
    up = F.interpolate(lo, size=label.shape[-2:], mode="bilinear", align_corners=True)
    return ohem_ce(up, label, ignore_label, thresh, min_kept), lo


def deeplabv3plus_eval(data, sd, eps=1e-5, stats=None):
    """eval: log_softmax of the logits up-sampled to the input size, BN on running statistics"""
    lo = deeplabv3plus_logits(data, sd, eps, 0.0, False, stats)
    return F.log_softmax(F.interpolate(lo, size=data.shape[2:], mode="bilinear", align_corners=True), dim=1)
