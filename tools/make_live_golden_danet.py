"""Write tests/golden/live_reference_danet.npz from DANet composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_danet.py

The reference has no DANet, so this composes torchseg_b200/networks/danet.py's wiring from the live reference's
`resnet101`, PSPNet's `_nostride_dilate`, `ConvBnRelu` and `nn.CrossEntropyLoss(ignore_index=255)` (imported, nothing
copied). The position and channel attention modules are written here from their definition (Fu et al., DANet's
`PAM_Module` and `CAM_Module`). Child names and construction order are the network's, so the same seed gives the same
initial weights; both gammas, zero at construction, are then set to `GAMMAS` so that the gradient reaches the
attention. Stores what tests/test_cpu_danet.py compares against, so that it runs without the reference: the seeded
training loss (Dropout2d at p = 0), every parameter gradient's norm and 64 seeded entries, and the state_dict keys and
shapes.
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

from danet_oracle import GAMMAS, danet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_danet.npz")
C = 19


def compose():
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    class PAM(nn.Module):
        def __init__(self, in_dim):
            super().__init__()
            self.query_conv = nn.Conv2d(in_dim, in_dim // 8, 1)
            self.key_conv = nn.Conv2d(in_dim, in_dim // 8, 1)
            self.value_conv = nn.Conv2d(in_dim, in_dim, 1)
            self.gamma = nn.Parameter(torch.zeros(1))

        def forward(self, x):
            b, c, h, w = x.shape
            proj_query = self.query_conv(x).view(b, -1, h * w).permute(0, 2, 1)
            proj_key = self.key_conv(x).view(b, -1, h * w)
            attention = F.softmax(torch.bmm(proj_query, proj_key), dim=-1)
            proj_value = self.value_conv(x).view(b, -1, h * w)
            out = torch.bmm(proj_value, attention.permute(0, 2, 1)).view(b, c, h, w)
            return self.gamma * out + x

    class CAM(nn.Module):
        def __init__(self):
            super().__init__()
            self.gamma = nn.Parameter(torch.zeros(1))

        def forward(self, x):
            b, c, h, w = x.shape
            proj_query = x.view(b, c, -1)
            energy = torch.bmm(proj_query, x.view(b, c, -1).permute(0, 2, 1))
            energy_new = torch.max(energy, -1, keepdim=True)[0].expand_as(energy) - energy
            attention = F.softmax(energy_new, dim=-1)
            out = torch.bmm(attention, x.view(b, c, -1)).view(b, c, h, w)
            return self.gamma * out + x

    def cbr(cin, cout):
        return so.ConvBnRelu(cin, cout, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)

    class Head(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv5a, self.conv5c = cbr(2048, 512), cbr(2048, 512)
            self.sa, self.sc = PAM(512), CAM()
            self.conv51, self.conv52 = cbr(512, 512), cbr(512, 512)
            self.conv6 = nn.Sequential(nn.Dropout2d(0.1, False), nn.Conv2d(512, C, 1))
            self.conv7 = nn.Sequential(nn.Dropout2d(0.1, False), nn.Conv2d(512, C, 1))
            self.conv8 = nn.Sequential(nn.Dropout2d(0.1, False), nn.Conv2d(512, C, 1))

        def forward(self, x):
            sa_conv = self.conv51(self.sa(self.conv5a(x)))
            sc_conv = self.conv52(self.sc(self.conv5c(x)))
            return self.conv8(sa_conv + sc_conv), self.conv6(sa_conv), self.conv7(sc_conv)

    class DANet(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer3.apply(partial(nostride_dilate, dilate=2))
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=4))
            self.head = Head()
            self.criterion = nn.CrossEntropyLoss(ignore_index=255)

        def forward(self, data, label):
            blocks = self.backbone(data)
            up = partial(F.interpolate, size=data.shape[2:], mode="bilinear", align_corners=True)
            sasc, sa, sc = self.head(blocks[-1])
            return self.criterion(up(sasc), label) + self.criterion(up(sa), label) + self.criterion(up(sc), label)

    return DANet()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    x, y, seed = danet_case()
    torch.manual_seed(seed)
    m = compose()
    for name in ("conv6", "conv7", "conv8"):
        getattr(m.head, name)[0].p = 0.0
    params = dict(m.named_parameters())
    with torch.no_grad():
        for k, v in GAMMAS.items():
            params[k].fill_(v)
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
