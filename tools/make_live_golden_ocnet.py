"""Write tests/golden/live_reference_ocnet.npz from OCNet composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_ocnet.py

The reference has no OCNet, so this composes torchseg_b200/networks/ocnet.py's wiring from the live reference's
`resnet101`, PSPNet's `_nostride_dilate`, `ConvBnRelu` and `nn.CrossEntropyLoss(ignore_index=255)` (imported, nothing
copied). The self-attention block is written here from its definition (OCNet's `_SelfAttentionBlock` at scale 1:
softmax(k kᵀ / √256) v with one f_key for queries and keys). Child names and construction order are the network's, so
the same seed gives the same initial weights; W, zero at construction, is then set to `nonzero_w()` so that the
gradient reaches f_key and f_value. Stores what tests/test_cpu_ocnet.py compares against, so that it runs without the
reference: the seeded training loss (Dropout2d at p = 0), every parameter gradient's norm and 64 seeded entries, and the
state_dict keys and shapes.
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

from ocnet_oracle import nonzero_w, ocnet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_ocnet.npz")
C = 19


def compose():
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    class SelfAttentionBlock(nn.Module):
        def __init__(self):
            super().__init__()
            self.f_key = so.ConvBnRelu(512, 256, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)
            self.f_value = nn.Conv2d(512, 256, 1)
            self.W = nn.Conv2d(256, 512, 1)
            nn.init.constant_(self.W.weight, 0)
            nn.init.constant_(self.W.bias, 0)

        def forward(self, x):
            b, _, h, w = x.shape
            key = self.f_key(x)
            query = key.view(b, 256, -1).permute(0, 2, 1)
            value = self.f_value(x).view(b, 256, -1).permute(0, 2, 1)
            sim = F.softmax(torch.matmul(query, key.view(b, 256, -1)) * 256 ** -0.5, dim=-1)
            context = torch.matmul(sim, value).permute(0, 2, 1).contiguous().view(b, 256, h, w)
            return self.W(context)

    class BaseOCModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.stages = nn.ModuleList([SelfAttentionBlock()])
            self.conv_bn_dropout = nn.Sequential(
                so.ConvBnRelu(1024, 512, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN),
                nn.Dropout2d(0.05))

        def forward(self, feats):
            return self.conv_bn_dropout(torch.cat([self.stages[0](feats), feats], 1))

    class OCNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer3.apply(partial(nostride_dilate, dilate=2))
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=4))
            self.context = nn.Sequential(
                so.ConvBnRelu(2048, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN),
                BaseOCModule())
            self.cls = nn.Conv2d(512, C, 1)
            self.aux_layer = nn.Sequential(
                so.ConvBnRelu(1024, 512, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN),
                nn.Dropout2d(0.1), nn.Conv2d(512, C, 1))
            self.criterion = nn.CrossEntropyLoss(ignore_index=255)

        def forward(self, data, label):
            blocks = self.backbone(data)
            lo = self.cls(self.context(blocks[-1]))
            aux = self.aux_layer(blocks[-2])
            up = partial(F.interpolate, size=data.shape[2:], mode="bilinear", align_corners=True)
            return self.criterion(up(lo), label) + 0.4 * self.criterion(up(aux), label)

    return OCNet()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    x, y, seed = ocnet_case()
    torch.manual_seed(seed)
    m = compose()
    m.context[1].conv_bn_dropout[1].p = 0.0
    m.aux_layer[1].p = 0.0
    W = m.context[1].stages[0].W
    w, b = nonzero_w()
    with torch.no_grad():
        W.weight.copy_(w)
        W.bias.copy_(b)
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
