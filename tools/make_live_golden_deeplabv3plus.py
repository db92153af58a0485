"""Write tests/golden/live_reference_deeplabv3plus.npz from DeepLabV3+ composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_deeplabv3plus.py

The reference has no DeepLab network, so this composes torchseg_b200/networks/deeplabv3plus.py's wiring from the live
reference's `resnet101`, `ConvBnRelu`, `SeparableConvBnRelu` and `ProbOhemCrossEntropy2d` (imported, nothing copied),
with the same child names and construction order, so the same seed gives the same initial weights. Stores what
tests/test_cpu_deeplabv3plus.py compares against, so that it runs without the reference: the seeded training loss
(Dropout2d at p = 0), every parameter gradient's norm and 64 seeded entries, and the state_dict keys and shapes.
"""
import json
import os
import sys
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from golden_cases import bisenet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_deeplabv3plus.npz")
CASE = dict(N=2, HW=64, seed=11)


def compose(num_classes, criterion):
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    # the reference PSPNet's de-striding helper (its `self` is unused)
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    class ASPP(nn.Module):
        def __init__(self):
            super().__init__()
            self.branches = nn.ModuleList(
                [so.ConvBnRelu(2048, 256, 1, 1, 0, norm_layer=BN)] +
                [so.SeparableConvBnRelu(2048, 256, 3, 1, d, d, norm_layer=BN) for d in (6, 12, 18)])
            self.pool = nn.Sequential(nn.AdaptiveAvgPool2d(1), so.ConvBnRelu(2048, 256, 1, 1, 0, norm_layer=BN))
            self.project = so.ConvBnRelu(1280, 256, 1, 1, 0, norm_layer=BN)
            self.dropout = nn.Dropout2d(0.1)

        def forward(self, x):
            outs = [b(x) for b in self.branches]
            outs.append(F.interpolate(self.pool(x), size=x.shape[2:], mode="bilinear", align_corners=True))
            return self.dropout(self.project(torch.cat(outs, dim=1)))

    class Decoder(nn.Module):
        def __init__(self):
            super().__init__()
            self.reduce = so.ConvBnRelu(256, 48, 1, 1, 0, norm_layer=BN)
            self.refine = nn.Sequential(so.SeparableConvBnRelu(304, 256, 3, 1, 1, 1, norm_layer=BN),
                                        so.SeparableConvBnRelu(256, 256, 3, 1, 1, 1, norm_layer=BN))
            self.classifier = nn.Conv2d(256, num_classes, 1, bias=True)

        def forward(self, x, low):
            low = self.reduce(low)
            x = F.interpolate(x, size=low.shape[2:], mode="bilinear", align_corners=True)
            return self.classifier(self.refine(torch.cat([x, low], dim=1)))

    class DeepLabV3Plus(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=2))
            self.aspp = ASPP()
            self.decoder = Decoder()
            self.criterion = criterion

        def forward(self, data, label):
            blocks = self.backbone(data)
            lo = self.decoder(self.aspp(blocks[-1]), blocks[0])
            return self.criterion(F.interpolate(lo, size=label.shape[-2:], mode="bilinear", align_corners=True), label)

    return DeepLabV3Plus()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    lo = rl.load_loss_opr()
    x, y, min_kept, seed = bisenet_case(**CASE)
    torch.manual_seed(seed)
    ohem = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    m = compose(19, ohem)
    m.aspp.dropout.p = 0.0
    m.train()
    loss = m(x, y)
    loss.backward()
    g = {"loss": np.float32(float(loss.detach()))}
    grads = {}
    for i, (n, p) in enumerate(m.named_parameters()):
        flat = p.grad.reshape(-1).double().numpy()
        idx = np.random.default_rng(i).choice(flat.size, min(flat.size, 64), replace=False)
        grads[n] = [float(np.linalg.norm(flat)), idx.tolist(), flat[idx].tolist()]
    g["grads"] = json.dumps(grads)
    g["keys"] = json.dumps([[k, list(v.shape)] for k, v in compose(19, None).state_dict().items()])
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
