"""ORACLE — test infrastructure only: EncNet (ResNet-101 v1c, dilated-8) with the Context Encoding layer and the SE-loss.

Functional fp32 PyTorch restatement of torchseg_b200/networks/encnet.py on the shared blocks of oracle/torch_ref.py
(`resnet_v1c_d8`, `conv_bn_relu`, `_bn`), driven by a state_dict with the network's key names. The Encoding layer is
written in the direct broadcast form (the [B, HW, K, D] residuals are formed), the class presence of the SE-loss comes
from `torch.histc`, and the bf16-storage emulation of oracle/torch_ref.py (`set_bf16_emulation`, re-exported here) is
honoured, E included. Pinned to the network composed from the live reference modules by tests/test_cpu_encnet.py through
tests/golden/live_reference_encnet.npz (tools/make_live_golden_encnet.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import _bn, conv_bn_relu, q, qw, resnet_v1c_d8, set_bf16_emulation

__all__ = ["set_bf16_emulation", "encnet_case", "encoding", "presence", "se_loss", "enc_module", "encnet_logits",
           "encnet_loss", "encnet_eval"]


def encnet_case(N=2, HW=64, seed=21, classes=150, present=40):
    """ADE-shaped input (150 classes, ignore -1) whose labels use only classes [0, present) and -1, so the SE target
    has absent classes"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(-1, present, (N, HW, HW), generator=g, dtype=torch.int64)
    return x, y, seed


def encoding(x, codewords, scale):
    """E_bk = Σ_i softmax_k(s_k ‖x_i − c_k‖²) (x_i − c_k) over the pixels of image b: [B, D, h, w] → [B, K, D]"""
    B, D = x.shape[:2]
    X = x.reshape(B, D, -1).transpose(1, 2)                    # [B, N, D]
    R = X.unsqueeze(2) - codewords[None, None]                 # [B, N, K, D]
    A = F.softmax(scale[None, None] * R.pow(2).sum(3), dim=2)  # [B, N, K]
    return q((A.unsqueeze(3) * R).sum(1))


def presence(label, C):
    """[B, C] fp32: 1 where class c occurs in label[b] (−1, 255 and values >= C count for nothing)"""
    return torch.stack([torch.histc(l.float(), bins=C, min=0, max=C - 1) > 0 for l in label]).float()


def se_loss(se, label, C):
    return F.binary_cross_entropy(torch.sigmoid(se), presence(label, C))


def enc_module(f, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """EncModule: (relu(f + f·sigmoid(fc(en))), selayer(en)) with en the mean over the codewords of relu(BN(E))"""
    x = conv_bn_relu(f, sd, prefix + ".conv", 1, 0, eps=eps, momentum=momentum, training=training, stats=stats)
    E = encoding(x, sd[prefix + ".encoding.codewords"], sd[prefix + ".encoding.scale"])
    e = q(F.relu(_bn(E, sd, prefix + ".bn", eps, momentum, training, stats)))
    en = q(e.mean(1))                                          # [B, D]
    gamma = torch.sigmoid(q(F.linear(en, qw(sd[prefix + ".fc.weight"]), sd[prefix + ".fc.bias"])))
    y = q(F.relu(f + f * gamma[:, :, None, None]))
    se = F.linear(en, qw(sd[prefix + ".selayer.weight"]), sd[prefix + ".selayer.bias"])
    return y, se


def encnet_logits(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None, layers=(3, 4, 23, 3)):
    """(low-resolution fp32 logits, SE logits, layer3 output)"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, training, stats)
    f = conv_bn_relu(blocks[-1], sd, "head.conv5", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    y, se = enc_module(f, sd, "head.encmodule", eps, momentum, training, stats)
    lo = F.conv2d(y, qw(sd["head.conv6.1.weight"]), sd["head.conv6.1.bias"])
    return lo, se, blocks[-2]


def _up(x, data):
    return F.interpolate(x, size=data.shape[2:], mode="bilinear", align_corners=True)


def encnet_loss(data, label, sd, aux_ratio=0.2, se_ratio=0.2, ignore_label=-1, eps=1e-5, momentum=0.1, stats=None):
    """training: CE(up(logits)) + aux_ratio · CE(up(aux)) + se_ratio · BCELoss(sigmoid(se), presence(label))"""
    C = sd["head.conv6.1.bias"].shape[0]
    lo, se, l3 = encnet_logits(data, sd, eps, momentum, True, stats)
    aux = conv_bn_relu(l3, sd, "aux_layer.0", 1, 1, eps=eps, momentum=momentum, training=True, stats=stats)
    aux = F.conv2d(aux, qw(sd["aux_layer.2.weight"]), sd["aux_layer.2.bias"])
    loss = F.cross_entropy(_up(lo, data), label, ignore_index=ignore_label)
    aux_loss = F.cross_entropy(_up(aux, data), label, ignore_index=ignore_label)
    return loss + aux_ratio * aux_loss + se_ratio * se_loss(se, label, C), (lo, se)


def encnet_eval(data, sd, eps=1e-5, stats=None):
    """eval: log_softmax of the logits up-sampled to the input size, BN on running statistics"""
    lo, _, _ = encnet_logits(data, sd, eps, 0.0, False, stats)
    return F.log_softmax(_up(lo, data), dim=1)
