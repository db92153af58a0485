"""ORACLE — test infrastructure only: DANet (ResNet-101 v1c, dilated-8) with its dual attention head.

Functional fp32 PyTorch restatement of torchseg_b200/networks/danet.py on the shared blocks of oracle/torch_ref.py
(`resnet_v1c_d8`, `conv_bn_relu`), driven by a state_dict with the network's key names. The position attention is
written in DANet's materialised form (the [N, N] matrix is formed) and the channel attention with its [C, C] energy
and torch's `rowmax − E` soft-max; the bf16-storage emulation of oracle/torch_ref.py (`set_bf16_emulation`,
re-exported here) is honoured. Pinned to the network composed from the live reference modules by
tests/test_cpu_danet.py through tests/golden/live_reference_danet.npz (tools/make_live_golden_danet.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import conv_bn_relu, q, qw, resnet_v1c_d8, set_bf16_emulation

__all__ = ["set_bf16_emulation", "danet_case", "GAMMAS", "pam", "cam", "danet_head", "danet_loss", "danet_eval"]

# non-zero gammas for the parity cases: DANet zero-initialises both, and then nothing flows back into the attention
GAMMAS = {"head.sa.gamma": 0.5, "head.sc.gamma": 0.25}


def danet_case(N=2, HW=64, seed=29, classes=19):
    """Cityscapes-shaped input (19 classes, ignore 255)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, :4] = 255
    return x, y, seed


def _conv1x1(x, sd, prefix):
    return q(F.conv2d(x, qw(sd[prefix + ".weight"]), sd[prefix + ".bias"]))


def pam(x, sd, prefix):
    """PAM_Module: gamma · softmax(q kᵀ) v + x with the [N, N] attention materialised, no scale"""
    B, C, h, w = x.shape
    proj_query = _conv1x1(x, sd, prefix + ".query_conv").view(B, -1, h * w).permute(0, 2, 1)
    proj_key = _conv1x1(x, sd, prefix + ".key_conv").view(B, -1, h * w)
    attention = F.softmax(torch.bmm(proj_query, proj_key), dim=-1)
    proj_value = _conv1x1(x, sd, prefix + ".value_conv").view(B, -1, h * w)
    out = q(torch.bmm(proj_value, attention.permute(0, 2, 1)).view(B, C, h, w))
    return q(sd[prefix + ".gamma"] * out + x)


def cam(x, sd, prefix):
    """CAM_Module: gamma · softmax(rowmax(E) − E) X + x with E = X Xᵀ [C, C] materialised"""
    B, C, h, w = x.shape
    proj_query = x.view(B, C, -1)
    energy = torch.bmm(proj_query, x.view(B, C, -1).permute(0, 2, 1))
    energy_new = torch.max(energy, -1, keepdim=True)[0].expand_as(energy) - energy
    attention = q(F.softmax(energy_new, dim=-1))
    out = q(torch.bmm(attention, x.view(B, C, -1)).view(B, C, h, w))
    return q(sd[prefix + ".gamma"] * out + x)


def danet_head(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """DANetHead with Dropout2d at p = 0: the low-resolution fp32 logits (sasc, sa, sc)"""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    sa = conv_bn_relu(pam(conv_bn_relu(x, sd, prefix + ".conv5a", 1, 1, **kw), sd, prefix + ".sa"), sd,
                      prefix + ".conv51", 1, 1, **kw)
    sc = conv_bn_relu(cam(conv_bn_relu(x, sd, prefix + ".conv5c", 1, 1, **kw), sd, prefix + ".sc"), sd,
                      prefix + ".conv52", 1, 1, **kw)

    def cls(f, name):
        return F.conv2d(f, qw(sd[prefix + "." + name + ".1.weight"]), sd[prefix + "." + name + ".1.bias"])

    return cls(q(sa + sc), "conv8"), cls(sa, "conv6"), cls(sc, "conv7")


def _up(x, data):
    return F.interpolate(x, size=data.shape[2:], mode="bilinear", align_corners=True)


def danet_loss(data, label, sd, ignore_label=255, eps=1e-5, momentum=0.1, stats=None, layers=(3, 4, 23, 3)):
    """training: CE(up(sasc)) + CE(up(sa)) + CE(up(sc)), Dropout2d at p = 0"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, True, stats)
    heads = danet_head(blocks[-1], sd, "head", eps, momentum, True, stats)
    losses = [F.cross_entropy(_up(lo, data), label, ignore_index=ignore_label) for lo in heads]
    return losses[0] + losses[1] + losses[2], heads


def danet_eval(data, sd, eps=1e-5, stats=None, layers=(3, 4, 23, 3)):
    """eval: log_softmax of the sasc logits up-sampled to the input size, BN on running statistics"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, 0.0, False, stats)
    sasc, _, _ = danet_head(blocks[-1], sd, "head", eps, 0.0, False, stats)
    return F.log_softmax(_up(sasc, data), dim=1)
