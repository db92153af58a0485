"""ORACLE — test infrastructure only: BiSeNet-X39.

Functional fp32 PyTorch restatement of the reference's Xception-39 (TorchSeg furnace/base_model/xception.py) and of the
X39 BiSeNet wiring (model/bisenet/cityscapes.bisenet.X39/network.py), driven by a state_dict with the REFERENCE's key
names. It builds on the shared blocks of oracle/torch_ref.py and honours its bf16-storage emulation
(`set_bf16_emulation`, re-exported here). Pinned to the live reference X39 network by tests/test_cpu_x39.py through
tests/golden/live_reference_x39.npz (tools/make_live_golden_x39.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch.nn.functional as F

from oracle.torch_ref import (_bn, attention_refinement, bisenet_head_logits, conv_bn_relu, feature_fusion, ohem_ce, q,
                              qw, set_bf16_emulation)

__all__ = ["set_bf16_emulation", "separable_conv_bn_relu", "xception_block", "xception39", "bisenet_x39_forward",
           "bisenet_x39_loss", "bisenet_x39_eval"]


def _depthwise3x3(x, sd, prefix, stride):
    """the groups = C 3x3 conv (padding 1) of SeparableConvBnRelu — xception.py:14-16"""
    return q(F.conv2d(x, qw(sd[prefix + ".conv1.weight"]), None, stride, 1, 1, x.shape[1]))


def separable_conv_bn_relu(x, sd, prefix, stride, has_relu, eps=1e-5, momentum=0.1, training=True, stats=None):
    """SeparableConvBnRelu.forward — xception.py:23-26: depthwise 3x3 → pointwise ConvBnRelu (no BN after the dw)"""
    x = _depthwise3x3(x, sd, prefix, stride)
    return conv_bn_relu(x, sd, prefix + ".point_wise_cbr", 1, 0, has_relu=has_relu, eps=eps, momentum=momentum,
                        training=training, stats=stats)


def xception_block(x, sd, prefix, stride, has_proj, eps=1e-5, momentum=0.1, training=True, stats=None):
    """Block.forward — xception.py:58-67: relu(shortcut + residual_branch(x)), shortcut = proj(x) when projecting"""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    shortcut = x
    if has_proj:
        shortcut = separable_conv_bn_relu(x, sd, prefix + ".proj", stride, False, **kw)
    t = separable_conv_bn_relu(x, sd, prefix + ".residual_branch.0", stride, True, **kw)
    t = separable_conv_bn_relu(t, sd, prefix + ".residual_branch.1", 1, True, **kw)
    # the last separable conv without its ReLU; its BN output is added to the shortcut unrounded (one fused pass)
    p = prefix + ".residual_branch.2"
    t = _depthwise3x3(t, sd, p, 1)
    t = q(F.conv2d(t, qw(sd[p + ".point_wise_cbr.conv.weight"])))
    t = _bn(t, sd, p + ".point_wise_cbr.bn", eps, momentum, training, stats)
    return q(F.relu(shortcut + t))


def xception39(x, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """Xception.forward with Block, layers [4, 8, 4], mid channels [16, 32, 64] — xception.py:72-122"""
    x = conv_bn_relu(q(x), sd, prefix + ".conv1", 2, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    x = F.max_pool2d(x, 3, 2, 1)
    blocks = []
    for li, nblk in ((1, 4), (2, 8), (3, 4)):
        for bi in range(nblk):
            x = xception_block(x, sd, "%s.layer%d.%d" % (prefix, li, bi), 2 if bi == 0 else 1, bi == 0, eps, momentum,
                               training, stats)
        blocks.append(x)
    return blocks


def bisenet_x39_forward(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None):
    """BiSeNet.forward wiring — TorchSeg model/bisenet/cityscapes.bisenet.X39/network.py:74-101 (the R18 wiring on the
    256 / 128-channel Xception stages). Returns the three LOW-resolution logit tensors (aux0 @1/16, aux1 @1/8,
    main @1/8) and the head inputs."""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    sp = conv_bn_relu(q(data), sd, "spatial_path.conv_7x7", 2, 3, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_1", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_2", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_1x1", 1, 0, **kw)
    blocks = xception39(data, sd, "context_path", eps, momentum, training, stats)[::-1]
    gc = q(F.adaptive_avg_pool2d(blocks[0], 1))
    gc = conv_bn_relu(gc, sd, "global_context.1", 1, 0, **kw)
    last = q(F.interpolate(gc, size=blocks[0].shape[2:], mode="bilinear", align_corners=True))
    pred_out = []
    for i in range(2):
        fm = attention_refinement(blocks[i], sd, "arms.%d" % i, eps, momentum, training, stats)
        fm = q(fm + last)
        last = q(F.interpolate(fm, size=blocks[i + 1].shape[2:], mode="bilinear", align_corners=True))
        last = conv_bn_relu(last, sd, "refines.%d" % i, 1, 1, **kw)
        pred_out.append(last)
    pred_out.append(feature_fusion(sp, last, sd, "ffm", eps, momentum, training, stats))
    lo = [bisenet_head_logits(pred_out[i], sd, "heads.%d" % i, eps, momentum, training, stats) for i in range(3)]
    return lo, pred_out


def bisenet_x39_loss(data, label, sd, min_kept, ignore_label=255, thresh=0.7, eps=1e-5, momentum=0.1, stats=None):
    """training branch of the X39 BiSeNet.forward — network.py:100-107: three ProbOhemCrossEntropy2d losses
    (`ohem_criterion`) on the x16 / x8 / x8 upsampled heads, main + aux0 + aux1"""
    lo, _ = bisenet_x39_forward(data, sd, eps, momentum, True, stats)
    losses = []
    for l, s in zip(lo, (16, 8, 8)):
        up = F.interpolate(l, scale_factor=s, mode="bilinear", align_corners=True)
        losses.append(ohem_ce(up, label, ignore_label, thresh, min_kept))
    return losses[2] + losses[0] + losses[1], lo


def bisenet_x39_eval(data, sd, eps=1e-5, stats=None):
    """eval branch — network.py:109: log_softmax of the main head upsampled x8, BN on running statistics"""
    lo, _ = bisenet_x39_forward(data, sd, eps, 0.0, False, stats)
    return F.log_softmax(F.interpolate(lo[2], scale_factor=8, mode="bilinear", align_corners=True), dim=1)
