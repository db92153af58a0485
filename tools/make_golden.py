"""Generate tests/golden/*.json from the LIVE reference (a TorchSeg checkout named by TSB_REFERENCE_DIR).

The reference ships no golden vectors (SURVEY.md §4); these fixtures pin the oracle to outputs of the reference
modules themselves on seeded synthetic inputs. Inputs are regenerated from seeds (torch CPU generator), only
outputs are stored. Run: python tools/make_golden.py
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from oracle import reference_live as rl  # noqa: E402
from golden_cases import ohem_case, bisenet_case, fcn_case, fcn_r101_case, pspnet_case, dfn_case, psanet_case, OHEM_REGIMES  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def main():
    assert rl.available(), "needs the reference checkout (TSB_REFERENCE_DIR)"
    torch.set_num_threads(8)
    lo = rl.load_loss_opr()
    gold = {"ohem": {}, "torch": torch.__version__}
    for regime in OHEM_REGIMES:
        logits, labels, min_kept = ohem_case(regime)
        crit = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
        x = logits.clone().requires_grad_(True)
        loss = crit(x, labels)
        entry = {"loss": float(loss) if loss == loss else "nan", "min_kept": min_kept}
        if loss == loss:
            loss.backward()
            kept = (x.grad.abs().sum(dim=1) > 0).reshape(-1)   # pixels that received gradient == kept set
            entry["kept_count"] = int(kept.sum())
            entry["kept_sha256"] = sha(kept.to(torch.uint8))
            entry["grad_abs_sum"] = float(x.grad.abs().sum())
        gold["ohem"][regime] = entry
    # weighted variant (use_weight=True, loss_opr.py:57-63)
    logits, labels, min_kept = ohem_case("B")
    crit = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=True)
    gold["ohem"]["B_weighted"] = {"loss": float(crit(logits, labels)), "min_kept": min_kept}
    # focal
    g = torch.Generator().manual_seed(10)
    pred = torch.randn(2, 1, 32, 40, generator=g)
    tgt = torch.randint(0, 2, (2, 32, 40), generator=g)
    tgt[:, :3] = 255
    gold["focal"] = {"loss": float(lo.SigmoidFocalLoss(255)(pred, tgt))}

    # BiSeNet-R18 tiny step through the reference network.py
    net = rl.load_network('bisenet/cityscapes.bisenet.R18')
    x, y, min_kept, seed = bisenet_case()
    torch.manual_seed(seed)
    crit = lo.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    m = net.BiSeNet(19, True, crit, None, nn.BatchNorm2d)
    m.train()
    loss = m(x, y)
    loss.backward()
    gn = {n: float(p.grad.norm()) for n, p in m.named_parameters()
          if n in ("context_path.conv1.weight", "spatial_path.conv_7x7.conv.weight", "heads.2.conv_1x1.weight", "ffm.conv_1x1.conv.weight")}
    gold["bisenet_r18"] = {"loss": float(loss), "grad_norms": gn, "n_params": sum(p.numel() for p in m.parameters()),
                           "n_state": len(m.state_dict())}

    # FCN-32s R18 (BASELINE configs[0]) assembled from the reference's own resnet18 + _FCNHead
    fcn = rl.load_network('fcn/voc.fcn32s.R101_v1c', num_classes=19, aux_loss_ratio=0.5)
    resnet = rl.load_resnet()
    x, y, seed = fcn_case()
    torch.manual_seed(seed)
    backbone = resnet.resnet18(None, norm_layer=nn.BatchNorm2d, bn_eps=1e-5, bn_momentum=0.1, deep_stem=False, stem_width=64)
    head = fcn._FCNHead(512, 19, True, nn.BatchNorm2d)
    aux_head = fcn._FCNHead(256, 19, True, nn.BatchNorm2d)
    for h in (head, aux_head):
        h.dropout.p = 0.0
    import torch.nn.functional as F
    blocks = backbone(x)
    pred = F.interpolate(head(blocks[-1]), scale_factor=32, mode='bilinear', align_corners=True)
    aux = F.interpolate(aux_head(blocks[-2]), scale_factor=16, mode='bilinear', align_corners=True)
    ce = nn.CrossEntropyLoss(ignore_index=255)
    gold["fcn_r18"] = {"loss": float(ce(pred, y) + 0.5 * ce(aux, y))}

    # the shipped FCN-32s R101_v1c (fcn network.py:13-47, train.py:45-47 criterion), Dropout2d disabled
    fcn21 = rl.load_network('fcn/voc.fcn32s.R101_v1c', num_classes=21, aux_loss_ratio=0.5)
    x, y, seed = fcn_r101_case()
    torch.manual_seed(seed)
    m = fcn21.FCN(21, nn.CrossEntropyLoss(reduction='mean', ignore_index=255), True, None, nn.BatchNorm2d)
    for mod in m.modules():
        if isinstance(mod, nn.Dropout2d):
            mod.p = 0.0
    m.train()
    loss = m(x, y)
    loss.backward()
    gold["fcn_r101"] = {"loss": float(loss), "n_params": sum(p.numel() for p in m.parameters()),
                        "n_state": len(m.state_dict()),
                        "grad_norms": {n: float(p.grad.norm()) for n, p in m.named_parameters()
                                       if n in ("backbone.conv1.0.weight", "backbone.layer4.2.conv3.weight",
                                                "head.cbr.conv.weight", "head.conv1x1.weight", "aux_head.conv1x1.bias")}}

    # PSPNet-R101_v1c dilated-8 (BASELINE configs[2] family), Dropout2d disabled
    psp = rl.load_network('pspnet/ade.pspnet.R101_v1c', num_classes=150)
    x, y, seed = pspnet_case()
    torch.manual_seed(seed)
    m = psp.PSPNet(150, nn.CrossEntropyLoss(reduction='mean', ignore_index=-1), None, nn.BatchNorm2d)
    for mod in m.modules():
        if isinstance(mod, nn.Dropout2d):
            mod.p = 0.0
    m.train()
    loss = m(x, y)
    loss.backward()
    gold["pspnet_r101"] = {"loss": float(loss), "n_params": sum(p.numel() for p in m.parameters()),
                           "n_state": len(m.state_dict()),
                           "grad_norms": {n: float(p.grad.norm()) for n, p in m.named_parameters()
                                          if n in ("backbone.conv1.0.weight", "backbone.layer3.5.conv2.weight",
                                                   "psp_layer.conv6.0.conv.weight", "aux_layer.2.weight")}}

    # DFN-R101_v1c (SURVEY C4): CrossEntropyLoss on the smooth heads + 0.1 * SigmoidFocalLoss on the border heads
    dfn = rl.load_network('dfn/cityscapes.dfn.R101_v1c', num_classes=19)
    x, y, e, seed = dfn_case()
    torch.manual_seed(seed)
    m = dfn.DFN(19, nn.CrossEntropyLoss(reduction='mean', ignore_index=255),
                lo.SigmoidFocalLoss(ignore_label=255, gamma=2.0, alpha=0.25), 0.1, None, nn.BatchNorm2d)
    m.train()
    loss = m(x, y, e)
    loss.backward()
    gold["dfn_r101"] = {"loss": float(loss), "n_params": sum(p.numel() for p in m.parameters()),
                        "n_state": len(m.state_dict()),
                        "grad_norms": {n: float(p.grad.norm()) for n, p in m.named_parameters()
                                       if n in ("backbone.conv1.0.weight", "backbone.layer4.2.conv3.weight",
                                                "smooth_pre_rrbs.0.cbr.conv.weight", "cabs.3.channel_attention.fc.0.weight",
                                                "border_aft_rrbs.3.conv_refine.weight", "smooth_heads.3.conv.weight",
                                                "border_heads.0.conv.bias")}}

    # PSANet-R101_v1c (SURVEY C5; the class is called PSPNet in psanet network.py), Dropout2d disabled
    psa = rl.load_network('psanet/ade.psanet.R101_v1c', num_classes=150)
    x, y, seed = psanet_case()
    torch.manual_seed(seed)
    m = psa.PSPNet(150, nn.CrossEntropyLoss(reduction='mean', ignore_index=-1), None, nn.BatchNorm2d)
    for mod in m.modules():
        if isinstance(mod, nn.Dropout2d):
            mod.p = 0.0
    m.train()
    loss = m(x, y)
    loss.backward()
    gold["psanet_r101"] = {"loss": float(loss), "n_params": sum(p.numel() for p in m.parameters()),
                           "n_state": len(m.state_dict()),
                           "grad_norms": {n: float(p.grad.norm()) for n, p in m.named_parameters()
                                          if n in ("backbone.layer4.2.conv3.weight",
                                                   "psa_layer.collect_attention.1.conv.weight",
                                                   "psa_layer.distribute_reduction.conv.weight",
                                                   "psa_layer.proj.conv.weight", "psa_layer.conv6.2.weight")}}

    # input pipeline: the LIVE TrainPre (bisenet dataloader.py:11-33) on a seeded synthetic frame, one entry per RNG seed
    import random
    import numpy as np
    from golden_cases import pipeline_case
    bgr, gt, crop, scales, mean, std = pipeline_case()
    dl = rl.load_train_pre('bisenet/cityscapes.bisenet.R18', train_scale_array=scales, image_height=crop[0],
                           image_width=crop[1], image_mean=mean, image_std=std)
    pre = dl.TrainPre(mean, std)
    pipe = {}
    for seed in range(16):
        random.seed(seed)
        p_img, p_gt, _ = pre(bgr[:, :, ::-1], gt)                      # BaseDataset.py:45 reverses the channels first
        a = torch.from_numpy(np.ascontiguousarray(p_img)).float()       # BaseDataset.py:50-51
        b = torch.from_numpy(np.ascontiguousarray(p_gt)).long()
        pipe[str(seed)] = {"data_sha256": sha(a), "label_sha256": sha(b), "shape": list(a.shape),
                           "data_sum": float(a.double().sum()), "label_sum": int(b.sum())}
    # speed config (cityscapes.bisenet.R18.speed/dataloader.py:11-36): the cropped label down-sampled x8 by INTER_NEAREST
    bgr, gt, crop, scales, mean, std = pipeline_case()
    dl = rl.load_train_pre('bisenet/cityscapes.bisenet.R18.speed', train_scale_array=scales, image_height=crop[0],
                           image_width=crop[1], image_mean=mean, image_std=std, gt_down_sampling=8)
    pre = dl.TrainPre(mean, std)
    pipe_speed = {}
    for seed in range(6):
        random.seed(seed)
        p_img, p_gt, _ = pre(bgr[:, :, ::-1], gt)
        b = torch.from_numpy(np.ascontiguousarray(p_gt)).long()
        pipe_speed[str(seed)] = {"label_sha256": sha(b), "label_shape": list(b.shape)}

    # DFN TrainPre (dfn dataloader.py:11-44): same pipeline + the Canny / dilate border label, its own scale array
    from golden_cases import pipeline_case_dfn
    bgr, gt, crop, scales, mean, std = pipeline_case_dfn()
    dl = rl.load_train_pre('dfn/cityscapes.dfn.R101_v1c', train_scale_array=scales, image_height=crop[0],
                           image_width=crop[1], image_mean=mean, image_std=std)
    pre = dl.TrainPre(mean, std)
    pipe_dfn = {}
    for seed in range(12):
        random.seed(seed)
        p_img, p_gt, extra = pre(bgr[:, :, ::-1], gt)
        a = torch.from_numpy(np.ascontiguousarray(p_img)).float()
        b = torch.from_numpy(np.ascontiguousarray(p_gt)).long()
        c = torch.from_numpy(np.ascontiguousarray(extra['aux_label'])).long()
        pipe_dfn[str(seed)] = {"data_sha256": sha(a), "label_sha256": sha(b), "aux_sha256": sha(c), "shape": list(a.shape),
                               "aux_ones": int((c == 1).sum()), "aux_pad": int((c == 255).sum())}
    with open(os.path.join(OUT, "data_pipeline.json"), "w") as f:
        json.dump({"cv2": __import__("cv2").__version__, "cases": pipe, "cases_dfn": pipe_dfn, "cases_speed": pipe_speed}, f, indent=1, sort_keys=True)

    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "reference_outputs.json"), "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
    print(json.dumps(gold, indent=1)[:1500])


if __name__ == "__main__":
    main()
