"""ORACLE — test infrastructure only: DenseASPP (ResNet-101 v1c, dilated-8) with its densely connected atrous head.

Functional fp32 PyTorch restatement of torchseg_b200/networks/denseaspp.py on the shared blocks of oracle/torch_ref.py
(`resnet_v1c_d8`, `conv_bn_relu`), driven by a state_dict with the network's key names. Each block is written in the
textbook pre-activation form: BN → ReLU on the concatenation (a materialised copy), the 1x1 ConvBnRelu, the dilated 3x3
conv with bias, then `cat((new, feature))`. Dropout2d is at p = 0. The bf16-storage emulation of oracle/torch_ref.py
(`set_bf16_emulation`, re-exported here) is honoured. Pinned to the network composed from the live reference modules
by tests/test_cpu_denseaspp.py through tests/golden/live_reference_denseaspp.npz (tools/make_live_golden_denseaspp.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import _bn, conv_bn_relu, q, qw, resnet_v1c_d8, set_bf16_emulation

__all__ = ["set_bf16_emulation", "denseaspp_case", "RATES", "dense_aspp", "denseaspp_logits", "denseaspp_loss",
           "denseaspp_eval"]

RATES = (3, 6, 12, 18, 24)


def denseaspp_case(N=2, HW=64, seed=29, classes=19):
    """Cityscapes-shaped input (19 classes, ignore 255)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, :4] = 255
    return x, y, seed


def dense_aspp(x, sd, prefix, rates=RATES, eps=1e-5, momentum=0.1, training=True, stats=None):
    """DenseASPPModule: block i = conv3x3_d(ConvBnRelu1x1(relu(pre_bn(feats)))) (no pre_bn in block 0), prepended to
    the running concatenation; returns [a_{n-1} | ... | a_0 | x]"""
    feats = x
    for i, d in enumerate(rates):
        p = "%s.blocks.%d" % (prefix, i)
        t = feats
        if i > 0:
            t = q(F.relu(_bn(feats, sd, p + ".pre_bn", eps, momentum, training, stats)))
        t = conv_bn_relu(t, sd, p + ".reduce", 1, 0, eps=eps, momentum=momentum, training=training, stats=stats)
        a = q(F.conv2d(t, qw(sd[p + ".conv.weight"]), sd[p + ".conv.bias"], 1, d, d))
        feats = torch.cat([a, feats], 1)
    return feats


def denseaspp_logits(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None, layers=(3, 4, 23, 3)):
    """low-resolution fp32 logits"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, training, stats)
    f = dense_aspp(blocks[-1], sd, "aspp", RATES, eps, momentum, training, stats)
    return F.conv2d(f, qw(sd["cls.weight"]), sd["cls.bias"])


def _up(x, data):
    return F.interpolate(x, size=data.shape[2:], mode="bilinear", align_corners=True)


def denseaspp_loss(data, label, sd, ignore_label=255, eps=1e-5, momentum=0.1, stats=None):
    """training: CE(up(logits)), Dropout2d at p = 0"""
    lo = denseaspp_logits(data, sd, eps, momentum, True, stats)
    return F.cross_entropy(_up(lo, data), label, ignore_index=ignore_label), lo


def denseaspp_eval(data, sd, eps=1e-5, stats=None):
    """eval: log_softmax of the logits up-sampled to the input size, BN on running statistics"""
    return F.log_softmax(_up(denseaspp_logits(data, sd, eps, 0.0, False, stats), data), dim=1)
