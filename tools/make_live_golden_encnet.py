"""Write tests/golden/live_reference_encnet.npz from EncNet composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_encnet.py

The reference has no EncNet, so this composes torchseg_b200/networks/encnet.py's wiring from the live reference's
`resnet101`, PSPNet's `_nostride_dilate`, `ConvBnRelu` and `nn.CrossEntropyLoss(ignore_index=-1)` (imported, nothing
copied). The Encoding layer, the BatchNorm over the codewords and the SE-loss are written here from their definitions
(Zhang et al., CVPR 2018), with `torch.histc` for the class presence and `nn.BCELoss`. Child names and construction order
are the network's, so the same seed gives the same initial weights. Stores what tests/test_cpu_encnet.py compares
against, so that it runs without the reference: the seeded training loss (Dropout2d at p = 0), every parameter gradient's
norm and 64 seeded entries, and the state_dict keys and shapes.
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

from encnet_oracle import encnet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_encnet.npz")
C = 150


def compose():
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    class Encoding(nn.Module):
        def __init__(self, D, K):
            super().__init__()
            self.D, self.K = D, K
            self.codewords = nn.Parameter(torch.empty(K, D, dtype=torch.float))
            self.scale = nn.Parameter(torch.empty(K, dtype=torch.float))
            std = 1.0 / (K * D) ** 0.5
            self.codewords.data.uniform_(-std, std)
            self.scale.data.uniform_(-1, 0)

        def forward(self, x):
            B, D = x.shape[:2]
            X = x.view(B, D, -1).transpose(1, 2)
            R = X.unsqueeze(2) - self.codewords[None, None]
            A = F.softmax(self.scale[None, None] * R.pow(2).sum(3), dim=2)
            return (A.unsqueeze(3) * R).sum(1)

    class EncModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = so.ConvBnRelu(512, 512, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)
            self.encoding = Encoding(512, 32)
            self.bn = nn.BatchNorm1d(32)   # the network's norm_layer(32): same parameters, statistics over B and D
            self.fc = nn.Linear(512, 512)
            self.selayer = nn.Linear(512, C)

        def forward(self, f):
            en = F.relu(self.bn(self.encoding(self.conv(f)))).mean(1)
            gamma = torch.sigmoid(self.fc(en))
            return F.relu(f + f * gamma[:, :, None, None]), self.selayer(en)

    class EncHead(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv5 = so.ConvBnRelu(2048, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)
            self.encmodule = EncModule()
            self.conv6 = nn.Sequential(nn.Dropout2d(0.1), nn.Conv2d(512, C, 1))

        def forward(self, x):
            y, se = self.encmodule(self.conv5(x))
            return self.conv6(y), se

    class EncNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer3.apply(partial(nostride_dilate, dilate=2))
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=4))
            self.head = EncHead()
            self.aux_layer = nn.Sequential(
                so.ConvBnRelu(1024, 1024, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN),
                nn.Dropout2d(0.1), nn.Conv2d(1024, C, 1))
            self.criterion = nn.CrossEntropyLoss(ignore_index=-1)

        def forward(self, data, label):
            blocks = self.backbone(data)
            lo, se = self.head(blocks[-1])
            aux = self.aux_layer(blocks[-2])
            up = partial(F.interpolate, size=data.shape[2:], mode="bilinear", align_corners=True)
            pres = torch.stack([torch.histc(l.float(), bins=C, min=0, max=C - 1) > 0 for l in label]).float()
            return (self.criterion(up(lo), label) + 0.2 * self.criterion(up(aux), label) +
                    0.2 * nn.BCELoss()(torch.sigmoid(se), pres))

    return EncNet()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    x, y, seed = encnet_case()
    torch.manual_seed(seed)
    m = compose()
    m.head.conv6[0].p = 0.0
    m.aux_layer[1].p = 0.0
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
