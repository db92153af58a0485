"""Write tests/golden/live_reference_denseaspp.npz from DenseASPP composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_denseaspp.py

The reference has no DenseASPP, so this composes torchseg_b200/networks/denseaspp.py's wiring from the live reference's
`resnet101`, PSPNet's `_nostride_dilate`, `ConvBnRelu`, `nn.BatchNorm2d`, `nn.Conv2d` and
`nn.CrossEntropyLoss(ignore_index=255)` (imported, nothing copied). The pre-activation block is written here from its
definition (Yang et al., CVPR 2018: BN → ReLU → 1x1 conv → BN → ReLU → dilated 3x3 conv, output prepended to its input;
widths 512 / 128, rates 3, 6, 12, 18, 24, no leading BN in the first block). Child names and construction order are the
network's, so the same seed gives the same initial weights. Stores what tests/test_cpu_denseaspp.py compares against,
so that it runs without the reference: the seeded training loss (Dropout2d at p = 0), every parameter gradient's norm
and 64 seeded entries, and the state_dict keys and shapes.
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

from denseaspp_oracle import RATES, denseaspp_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_denseaspp.npz")
C = 19


def compose():
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    class DenseAsppBlock(nn.Module):
        def __init__(self, cin, d, bn_start):
            super().__init__()
            if bn_start:
                self.pre_bn = BN(cin)
            self.bn_start = bn_start
            self.reduce = so.ConvBnRelu(cin, 512, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)
            self.conv = nn.Conv2d(512, 128, 3, padding=d, dilation=d, bias=True)
            self.drop = nn.Dropout2d(0.0)

        def forward(self, x):
            if self.bn_start:
                x = F.relu(self.pre_bn(x))
            return self.drop(self.conv(self.reduce(x)))

    class DenseASPPModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.blocks = nn.ModuleList([DenseAsppBlock(2048 + 128 * i, d, i > 0) for i, d in enumerate(RATES)])

        def forward(self, x):
            for blk in self.blocks:
                x = torch.cat((blk(x), x), 1)
            return x

    class DenseASPP(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer3.apply(partial(nostride_dilate, dilate=2))
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=4))
            self.aspp = DenseASPPModule()
            self.dropout = nn.Dropout2d(0.0)
            self.cls = nn.Conv2d(2688, C, 1)
            self.criterion = nn.CrossEntropyLoss(ignore_index=255)

        def forward(self, data, label):
            blocks = self.backbone(data)
            lo = self.cls(self.dropout(self.aspp(blocks[-1])))
            up = F.interpolate(lo, size=data.shape[2:], mode="bilinear", align_corners=True)
            return self.criterion(up, label)

    return DenseASPP()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    x, y, seed = denseaspp_case()
    torch.manual_seed(seed)
    m = compose()
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
    g["keys"] = json.dumps([[k, list(v.shape)] for k, v in compose().state_dict().items()])
    np.savez_compressed(OUT, **g)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
