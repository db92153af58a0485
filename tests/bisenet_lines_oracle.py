"""ORACLE — test infrastructure only: the BiSeNet lines R18.speed, X39.speed and R101.

Functional fp32 PyTorch restatement of model/bisenet/cityscapes.bisenet.{R18.speed, X39.speed, R101}/network.py,
driven by a state_dict with the REFERENCE's key names. It builds on the shared blocks of oracle/torch_ref.py (the R18
and R101 context paths, heads, OHEM) and on tests/x39_oracle.py (the Xception-39 context path), and honours their
bf16-storage emulation (`set_bf16_emulation`, re-exported here). Pinned to the live reference networks by
tests/test_cpu_bisenet_lines.py through tests/golden/live_reference_bisenet_lines.npz
(tools/make_live_golden_bisenet_lines.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch.nn.functional as F

from oracle.torch_ref import (attention_refinement, bisenet_head_logits, conv_bn_relu, feature_fusion, ohem_ce, q,
                              resnet18, resnet_v1c_d8, set_bf16_emulation)
from x39_oracle import xception39

__all__ = ["set_bf16_emulation", "LINES", "bisenet_forward", "head_up", "bisenet_loss", "bisenet_eval"]


def _r101(x, sd, prefix, eps, momentum, training, stats=None):
    """resnet101(deep_stem=True, stem_width=64), not dilated — R101 network.py:23-26"""
    return resnet_v1c_d8(x, sd, prefix, (3, 4, 23, 3), eps, momentum, training, stats, dilated=False)


# line → (context path, up-scale factors of heads 0 / 1 / 2)
LINES = {
    "r18_speed": (resnet18, (2, 1, 1)),
    "x39_speed": (xception39, (2, 1, 1)),
    "r101": (_r101, (16, 8, 8)),
}


def bisenet_forward(line, data, sd, eps=1e-5, momentum=0.1, training=True, stats=None):
    """BiSeNet.forward wiring — network.py:75-103 of each line. Returns the LOW-resolution logits of the heads the
    network holds (all three in training; only the main head, as [None, None, main], in eval for the .speed lines,
    whose eval network builds no aux heads) and the three head inputs."""
    backbone, _ = LINES[line]
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    sp = conv_bn_relu(q(data), sd, "spatial_path.conv_7x7", 2, 3, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_1", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_2", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_1x1", 1, 0, **kw)
    blocks = backbone(data, sd, "context_path", eps, momentum, training, stats)[::-1]
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
    lo = [bisenet_head_logits(pred_out[i], sd, "heads.%d" % i, eps, momentum, training, stats)
          if "heads.%d.conv_1x1.weight" % i in sd else None for i in range(3)]
    return lo, pred_out


def head_up(lo, scale):
    """BiSeNetHead.forward tail — network.py:164-166: bilinear x scale (align_corners) only when scale > 1"""
    return F.interpolate(lo, scale_factor=scale, mode="bilinear", align_corners=True) if scale > 1 else lo


def bisenet_loss(line, data, label, sd, min_kept, ignore_label=255, thresh=0.7, eps=1e-5, momentum=0.1, stats=None):
    """training branch — network.py:103-111: three ProbOhemCrossEntropy2d losses on the up-scaled heads against
    `label` (1/8 resolution for the .speed lines), main + aux0 + aux1"""
    lo, _ = bisenet_forward(line, data, sd, eps, momentum, True, stats)
    losses = [ohem_ce(head_up(l, s), label, ignore_label, thresh, min_kept) for l, s in zip(lo, LINES[line][1])]
    return losses[2] + losses[0] + losses[1], lo


def bisenet_eval(line, data, sd, eps=1e-5, stats=None):
    """eval branch — network.py:113: log_softmax of the up-scaled main head, BN on running statistics"""
    lo, _ = bisenet_forward(line, data, sd, eps, 0.0, False, stats)
    return F.log_softmax(head_up(lo[2], LINES[line][1][2]), dim=1)
