"""Seeded synthetic cases shared by tools/make_golden.py (live reference) and the parity tests."""
import torch
import torch.nn.functional as F

OHEM_REGIMES = ["A", "B", "C", "D", "E"]


def ohem_case(regime, N=2, C=19, H=48, W=64, seed=1234):
    """SURVEY.md §8d regimes: A all kept (thr 0.7), B k-th value threshold, C min_kept > valid, D min_kept = 0,
    E all ignored"""
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, C, (N, H, W), generator=g, dtype=torch.int64)
    labels[:, : H // 10 + 1, :] = 255
    logits = torch.randn(N, C, H, W, generator=g)
    min_kept = N * H * W // 16
    if regime == "B":
        onehot = F.one_hot(labels.clamp(max=C - 1), C).permute(0, 3, 1, 2).float()
        logits = 8 * onehot + logits
    elif regime == "C":
        min_kept = N * H * W
    elif regime == "D":
        min_kept = 0
    elif regime == "E":
        labels[:] = 255
    return logits, labels, min_kept


def bisenet_case(N=2, HW=128, seed=77):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, 19, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, : HW // 10, :] = 255
    return x, y, N * HW * HW // 16, seed


def fcn_case(N=2, HW=256, seed=304):
    """BASELINE configs[0]: 2 synthetic 256x256 19-class images"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, 19, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, : HW // 10, :] = 255
    return x, y, seed


def fcn_r101_case(N=2, HW=128, seed=304, classes=21):
    """the shipped FCN-32s (R101_v1c, VOC 21 classes, ignore 255) at a small size"""
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, : HW // 10, :] = 255
    return x, y, seed


def pspnet_case(N=2, HW=96, seed=4, classes=150):
    """BASELINE configs[2] shape family (PSPNet R101_v1c dilated-8, ADE 150 classes, ignore -1), small spatial size"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(-1, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    return x, y, seed


def dfn_case(N=2, HW=128, seed=12345):
    """BASELINE configs C4 shape family (DFN R101_v1c, Cityscapes 19 classes + {0,1,255} border labels), small size"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, 19, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, : HW // 10, :] = 255
    e = (torch.rand(N, HW, HW, generator=g) < 0.15).to(torch.int64)
    e[:, : HW // 10, :] = 255
    return x, y, e, seed


def psanet_case(N=1, HW=480, seed=304, classes=150):
    """SURVEY C5 (PSANet R101_v1c dilated-8, ADE 150 classes, ignore -1). The PSA head needs h*w = 3600 positions at
    1/8 resolution, so the spatial size cannot be reduced below the reference's 480x480 (psanet config.py)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(-1, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    return x, y, seed


def pipeline_case(H=100, W=160, crop=(96, 128), seed=1):
    """a decoded uint8 BGR frame + label map, the BiSeNet scale array and normalisation constants (config.py:61-62,86)"""
    import numpy as np
    rng = np.random.default_rng(seed)
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    gt = rng.integers(0, 20, (H, W), dtype=np.uint8)
    gt[rng.random((H, W)) < 0.05] = 255
    return (bgr, gt, crop, [0.75, 1, 1.25, 1.5, 1.75, 2.0], np.array([0.485, 0.456, 0.406]),
            np.array([0.229, 0.224, 0.225]))


def pipeline_case_dfn(H=100, W=160, crop=(96, 128), seed=2):
    """label map with regions (so that Canny finds borders) + the DFN scale array (dfn config.py:87)"""
    import numpy as np
    rng = np.random.default_rng(seed)
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    gt = np.zeros((H, W), np.uint8)
    for _ in range(30):
        y0, x0 = rng.integers(0, H), rng.integers(0, W)
        h, w = rng.integers(3, H // 2), rng.integers(3, W // 2)
        gt[y0:y0 + h, x0:x0 + w] = rng.integers(0, 19)
    gt[rng.random((H, W)) < 0.03] = 255
    return (bgr, gt, crop, [0.5, 0.75, 1, 1.5, 1.75, 2.0], np.array([0.485, 0.456, 0.406]),
            np.array([0.229, 0.224, 0.225]))


# ---- live-reference cases pinned by tests/golden/live_reference.npz (tools/make_live_golden.py) ----
OHEM_SAMPLE = 2000   # gradient entries stored per OHEM case


def metric_inputs():
    """seeded predictions for the metric functions, incl. ignore labels (255 → outside [0, n_cl), -1 for ADE) and
    classes that never occur"""
    import numpy as np
    rng = np.random.default_rng(5)
    n_cl = 19
    gt = rng.integers(0, 17, size=(3, 64, 80))          # classes 17, 18 never occur → NaN IoU, skipped by nanmean
    gt[:, :5] = 255
    pred = np.where(rng.random(gt.shape) < 0.7, np.clip(gt, 0, 16), rng.integers(0, 17, size=gt.shape))
    lab = rng.integers(-1, 150, size=(48, 64))
    pr = np.where(rng.random(lab.shape) < 0.6, np.clip(lab, 0, 149), rng.integers(0, 150, size=lab.shape))
    return n_cl, pred, gt, pr, lab


def eval_net():
    """small deterministic network for the Evaluator comparison"""
    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(0)
            self.c1 = torch.nn.Conv2d(3, 8, 3, padding=1)
            self.c2 = torch.nn.Conv2d(8, 5, 3, padding=2, dilation=2)

        def forward(self, x):
            return torch.log_softmax(self.c2(torch.relu(self.c1(x))) * 3.0, dim=1)
    return Net().double().float()


def eval_image():
    import numpy as np
    return np.random.default_rng(3).integers(0, 256, size=(150, 210, 3), dtype=np.uint8)


def _eval_kw():
    import numpy as np
    return dict(dataset=None, class_num=5, image_mean=np.array([0.485, 0.456, 0.406]),
                image_std=np.array([0.229, 0.224, 0.225]), network=None, multi_scales=[0.75, 1.0, 1.5], is_flip=True,
                devices=[0])


EVAL_KW = _eval_kw()
