"""Write tests/golden/live_reference_ocrnet.npz from OCRNet composed of the unmodified reference modules.

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_live_golden_ocrnet.py

The reference has no OCRNet, so this composes torchseg_b200/networks/ocrnet.py's wiring from the live reference's
`resnet101`, PSPNet's `_nostride_dilate`, `ConvBnRelu` and `nn.CrossEntropyLoss(ignore_index=255)` (imported, nothing
copied). The gather and the object attention are written here from their definitions (OCRNet's SpatialGather_Module
and ObjectAttentionBlock2D at scale 1: the soft-max over the pixels of each image of the aux logits, then
softmax_k(f_pixel(x) · f_object(proxy)ᵀ / √256) · f_down(proxy) and f_up). Child names and construction order are the
network's, so the same seed gives the same initial weights. Stores what tests/test_cpu_ocrnet.py compares against, so
that it runs without the reference: the seeded training loss (both Dropout2d at p = 0) on 2 x 3 x 72² (a 9 x 9 map),
every parameter gradient's norm and 64 seeded entries, and the state_dict keys and shapes.
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

from ocrnet_oracle import ocrnet_case  # noqa: E402
from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_ocrnet.npz")
C = 19


def compose():
    so, rn = rl.load_seg_oprs(), rl.load_resnet()
    nostride_dilate = partial(rl.load_network("pspnet/ade.pspnet.R101_v1c").PSPNet._nostride_dilate, None)
    BN = nn.BatchNorm2d

    def cbr1(cin, cout):
        return so.ConvBnRelu(cin, cout, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)

    def cbr3(cin, cout):
        return so.ConvBnRelu(cin, cout, 3, 1, 1, has_bn=True, has_relu=True, has_bias=False, norm_layer=BN)

    class SpatialGatherModule(nn.Module):
        def forward(self, feats, probs):
            b, k = probs.shape[:2]
            probs = F.softmax(probs.view(b, k, -1), dim=2)                 # [B, K, N]
            feats = feats.view(b, feats.shape[1], -1).permute(0, 2, 1)     # [B, N, C]
            return torch.matmul(probs, feats).permute(0, 2, 1).unsqueeze(3)

    class ObjectAttentionBlock(nn.Module):
        def __init__(self):
            super().__init__()
            self.f_pixel = nn.Sequential(cbr1(512, 256), cbr1(256, 256))
            self.f_object = nn.Sequential(cbr1(512, 256), cbr1(256, 256))
            self.f_down = cbr1(512, 256)
            self.f_up = cbr1(256, 512)

        def forward(self, x, proxy):
            b, _, h, w = x.shape
            query = self.f_pixel(x).view(b, 256, -1).permute(0, 2, 1)
            key = self.f_object(proxy).view(b, 256, -1)
            value = self.f_down(proxy).view(b, 256, -1).permute(0, 2, 1)
            sim = F.softmax(torch.matmul(query, key) * 256 ** -0.5, dim=-1)
            context = torch.matmul(sim, value).permute(0, 2, 1).contiguous().view(b, 256, h, w)
            return self.f_up(context)

    class SpatialOCRModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.object_context_block = ObjectAttentionBlock()
            self.conv_bn_dropout = nn.Sequential(cbr1(1024, 512), nn.Dropout2d(0.05))

        def forward(self, feats, proxy):
            return self.conv_bn_dropout(torch.cat([self.object_context_block(feats, proxy), feats], 1))

    class OCRNet(nn.Module):
        def __init__(self):
            super().__init__()
            self.backbone = rn.resnet101(None, norm_layer=BN, bn_eps=1e-5, bn_momentum=0.1, deep_stem=True,
                                         stem_width=64)
            self.backbone.layer3.apply(partial(nostride_dilate, dilate=2))
            self.backbone.layer4.apply(partial(nostride_dilate, dilate=4))
            self.conv_3x3 = cbr3(2048, 512)
            self.spatial_context_head = SpatialGatherModule()
            self.spatial_ocr_head = SpatialOCRModule()
            self.head = nn.Conv2d(512, C, 1)
            self.dsn_head = nn.Sequential(cbr3(1024, 512), nn.Dropout2d(0.05), nn.Conv2d(512, C, 1))
            self.criterion = nn.CrossEntropyLoss(ignore_index=255)

        def forward(self, data, label):
            blocks = self.backbone(data)
            dsn = self.dsn_head(blocks[-2])
            f = self.conv_3x3(blocks[-1])
            lo = self.head(self.spatial_ocr_head(f, self.spatial_context_head(f, dsn)))
            up = partial(F.interpolate, size=data.shape[2:], mode="bilinear", align_corners=True)
            return self.criterion(up(lo), label) + 0.4 * self.criterion(up(dsn), label)

    return OCRNet()


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    x, y, seed = ocrnet_case()
    torch.manual_seed(seed)
    m = compose()
    m.spatial_ocr_head.conv_bn_dropout[1].p = 0.0
    m.dsn_head[1].p = 0.0
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
