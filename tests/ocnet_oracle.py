"""ORACLE — test infrastructure only: OCNet (ResNet-101 v1c, dilated-8) with the Base-OC object-context head.

Functional fp32 PyTorch restatement of torchseg_b200/networks/ocnet.py on the shared blocks of oracle/torch_ref.py
(`resnet_v1c_d8`, `conv_bn_relu`), driven by a state_dict with the network's key names. The self-attention is written
in the explicit materialised form softmax(scale · q kᵀ) v (the [N, N] matrix is formed), and the bf16-storage emulation
of oracle/torch_ref.py (`set_bf16_emulation`, re-exported here) is honoured. Pinned to the network composed from the
live reference modules by tests/test_cpu_ocnet.py through tests/golden/live_reference_ocnet.npz
(tools/make_live_golden_ocnet.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import conv_bn_relu, q, qw, resnet_v1c_d8, set_bf16_emulation

__all__ = ["set_bf16_emulation", "ocnet_case", "nonzero_w", "attention", "self_attention", "base_oc", "ocnet_logits",
           "ocnet_loss", "ocnet_eval"]

W_PREFIX = "context.1.stages.0.W"


def ocnet_case(N=2, HW=64, seed=23, classes=19):
    """Cityscapes-shaped input (19 classes, ignore 255)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, :4] = 255
    return x, y, seed


def nonzero_w(out_ch=512, in_ch=256, seed=5, std=0.05):
    """seeded non-zero (weight, bias) for the attention block's W: OCNet zero-initialises W, and then nothing flows back
    into f_key / f_value, so every parity case replaces it"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(out_ch, in_ch, 1, 1, generator=g) * std, torch.randn(out_ch, generator=g) * std


def attention(qq, kk, v, scale):
    """softmax(scale · q kᵀ) v over the h·w pixels of each image, the [N, N] matrix materialised"""
    B, C, h, w = qq.shape
    Q = qq.reshape(B, C, -1).permute(0, 2, 1)
    K = kk.reshape(B, C, -1)
    V = v.reshape(B, v.shape[1], -1).permute(0, 2, 1)
    sim = F.softmax(torch.matmul(Q, K) * scale, dim=-1)
    return q(torch.matmul(sim, V).permute(0, 2, 1).contiguous().view(B, v.shape[1], h, w))


def self_attention(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """SelfAttentionBlock: W(attention(f_key(x), f_key(x), f_value(x), key_channels^-0.5))"""
    k = conv_bn_relu(x, sd, prefix + ".f_key", 1, 0, eps=eps, momentum=momentum, training=training, stats=stats)
    v = q(F.conv2d(x, qw(sd[prefix + ".f_value.weight"]), sd[prefix + ".f_value.bias"]))
    ctx = attention(k, k, v, k.shape[1] ** -0.5)
    return q(F.conv2d(ctx, qw(sd[prefix + ".W.weight"]), sd[prefix + ".W.bias"]))


def base_oc(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """BaseOCModule with one stage and Dropout2d at p = 0: conv_bn_dropout(cat([stage(x), x]))"""
    ctx = self_attention(x, sd, prefix + ".stages.0", eps, momentum, training, stats)
    return conv_bn_relu(torch.cat([ctx, x], 1), sd, prefix + ".conv_bn_dropout.0", 1, 0, eps=eps, momentum=momentum,
                        training=training, stats=stats)


def ocnet_logits(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None, layers=(3, 4, 23, 3)):
    """(low-resolution fp32 logits, layer3 output)"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, training, stats)
    f = conv_bn_relu(blocks[-1], sd, "context.0", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    f = base_oc(f, sd, "context.1", eps, momentum, training, stats)
    return F.conv2d(f, qw(sd["cls.weight"]), sd["cls.bias"]), blocks[-2]


def _up(x, data):
    return F.interpolate(x, size=data.shape[2:], mode="bilinear", align_corners=True)


def ocnet_loss(data, label, sd, aux_ratio=0.4, ignore_label=255, eps=1e-5, momentum=0.1, stats=None):
    """training: CE(up(logits)) + aux_ratio · CE(up(aux)), Dropout2d at p = 0"""
    lo, l3 = ocnet_logits(data, sd, eps, momentum, True, stats)
    aux = conv_bn_relu(l3, sd, "aux_layer.0", 1, 1, eps=eps, momentum=momentum, training=True, stats=stats)
    aux = F.conv2d(aux, qw(sd["aux_layer.2.weight"]), sd["aux_layer.2.bias"])
    loss = F.cross_entropy(_up(lo, data), label, ignore_index=ignore_label)
    aux_loss = F.cross_entropy(_up(aux, data), label, ignore_index=ignore_label)
    return loss + aux_ratio * aux_loss, (lo, aux)


def ocnet_eval(data, sd, eps=1e-5, stats=None):
    """eval: log_softmax of the logits up-sampled to the input size, BN on running statistics"""
    lo, _ = ocnet_logits(data, sd, eps, 0.0, False, stats)
    return F.log_softmax(_up(lo, data), dim=1)
