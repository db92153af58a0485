"""Segmentation metrics with the reference's function names and return conventions
(TorchSeg furnace/seg_opr/metric.py) — the host-side half of the Evaluator row (SURVEY.md §8f rank 2).

VOC / Cityscapes protocol: a confusion matrix over the labelled pixels (`hist_info`) reduced to per-class IoU, mean IoU
(with and without class 0) and pixel accuracy (`compute_score`). ADE protocol: per-image intersection / union areas with
the unlabeled class (-1) removed (`intersectionAndUnion`, `meanIoU`, `pixelAccuracy`, `mean_pixel_accuracy`,
`accuracy`). Pure numpy; the `*_torch` variant accumulates the confusion matrix on the device so that an evaluation loop
never copies full-resolution predictions to the host."""
import numpy as np


def hist_info(n_cl, pred, gt):
    """metric.py:9-18 → (confusion[n_cl, n_cl] with rows = ground truth, labelled pixel count, correct pixel count)"""
    if pred.shape != gt.shape:
        raise AssertionError("prediction and ground truth differ in shape")
    valid = np.logical_and(gt >= 0, gt < n_cl)
    g = gt[valid].astype(np.int64)
    p = pred[valid].astype(np.int64)
    conf = np.bincount(g * n_cl + p, minlength=n_cl * n_cl).reshape(n_cl, n_cl)
    return conf, int(valid.sum()), int((p == g).sum())


def compute_score(hist, correct, labeled):
    """metric.py:21-29 → (iu[n_cl], mean_IU, mean_IU_no_back, mean_pixel_acc); classes absent from both prediction and
    ground truth give NaN and are skipped by the means, like the reference"""
    hist = np.asarray(hist, dtype=np.float64)
    tp = np.diag(hist)
    with np.errstate(divide="ignore", invalid="ignore"):
        iu = tp / (hist.sum(axis=1) + hist.sum(axis=0) - tp)
        acc = np.float64(correct) / np.float64(labeled)
    return iu, np.nanmean(iu), np.nanmean(iu[1:]), acc


def hist_info_torch(n_cl, pred, gt):
    """device-side hist_info: pred / gt integer tensors of equal shape → (confusion int64 [n_cl, n_cl], labeled, correct)
    as 0-d tensors on the same device (no host sync)"""
    import torch
    valid = (gt >= 0) & (gt < n_cl)
    g = gt[valid].to(torch.int64)
    p = pred[valid].to(torch.int64)
    conf = torch.bincount(g * n_cl + p, minlength=n_cl * n_cl).reshape(n_cl, n_cl)
    return conf, valid.sum(), (p == g).sum()


def intersectionAndUnion(imPred, imLab, numClass):
    """metric.py:41-64: labels shifted by +1 so that the unlabeled class (-1) becomes 0 and drops out"""
    pred = np.asarray(imPred).astype(np.int64) + 1
    lab = np.asarray(imLab).astype(np.int64) + 1
    pred = pred * (lab > 0)
    inter = pred * (pred == lab)
    edges = dict(bins=numClass, range=(1, numClass))
    area_inter = np.histogram(inter, **edges)[0]
    area_pred = np.histogram(pred, **edges)[0]
    area_lab = np.histogram(lab, **edges)[0]
    return area_inter, area_pred + area_lab - area_inter


def meanIoU(area_intersection, area_union):
    """metric.py:33-38: areas are [numClass, numImages]"""
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = 1.0 * np.sum(area_intersection, axis=1) / np.sum(area_union, axis=1)
    return iou, np.nanmean(iou), np.nanmean(iou[1:])


def mean_pixel_accuracy(pixel_correct, pixel_labeled):
    """metric.py:67-71"""
    return 1.0 * np.sum(pixel_correct) / (np.spacing(1) + np.sum(pixel_labeled))


def pixelAccuracy(imPred, imLab):
    """metric.py:74-81"""
    labeled = imLab >= 0
    n_lab = np.sum(labeled)
    n_ok = np.sum((imPred == imLab) * labeled)
    with np.errstate(divide="ignore", invalid="ignore"):
        acc = 1.0 * n_ok / n_lab
    return acc, n_ok, n_lab


def accuracy(preds, label):
    """metric.py:84-89"""
    valid = label >= 0
    n_valid = valid.sum()
    return float((valid * (preds == label)).sum()) / (n_valid + 1e-10), n_valid
