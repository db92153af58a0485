"""Device-side training input pipeline (SURVEY §8 f4) behind the reference's TrainPre protocol.

`TrainPreGPU` restates TrainPre.__call__ (TorchSeg model/bisenet/cityscapes.bisenet.R18/dataloader.py:11-33): the
random draws (mirror, scale, crop position) are made on the host with Python's `random` module in the reference's order
(furnace/utils/img_utils.py:141, :119, :54-58 — same seed ⇒ same augmentation), everything that touches pixels —
cv2.flip, cv2.resize (INTER_LINEAR image / INTER_NEAREST label), normalize, crop + centred pad, HWC→CHW — runs as ONE
libtsb kernel (tsb_train_preprocess) over the whole batch of decoded uint8 frames, bit-exact with the cv2 path.

At ~900 img/s per GPU the reference's 24 cv2 worker processes are the bottleneck of the step; uploading the 6 MB uint8
frame instead of 20 MB of fp32 image + int64 label also cuts the H2D traffic 3.3x."""
import random

import numpy as np
import torch

from .. import ops


def normalize_lut(mean, std):
    """[3,256] float32 table of normalize() (img_utils.py:181-187) for every uint8 value: float32 division by 255,
    then float64 `- mean`, `/ std` (config.image_mean / image_std are float64 arrays), then the loader's `.float()`"""
    mean = np.asarray(mean, dtype=np.float64)
    std = np.asarray(std, dtype=np.float64)
    v = np.arange(256, dtype=np.float32) / 255.0
    lut = ((v[None, :].astype(np.float32) - mean[:, None]) / std[:, None])
    return np.ascontiguousarray(lut.astype(np.float32))


class TrainPreGPU(object):
    def __init__(self, img_mean, img_std, crop_size, scale_array, device, bgr_input=True, edge_labels=False,
                 gt_down_sampling=1):
        """edge_labels=True: DFN's TrainPre (model/dfn/cityscapes.dfn.R101_v1c/dataloader.py:11-44) — __call__ returns a
        third tensor 'aux_label' (Canny + 7x7 dilate border map ∈ {0, 1, 255}, tsb_edge_labels)"""
        self.edge_labels = bool(edge_labels)
        # speed config (cityscapes.bisenet.R18.speed/dataloader.py:28-30, config.py:66): the cropped label is resized to
        # (cw // ds, ch // ds) with INTER_NEAREST = index floor(d · ds) — every ds-th pixel, a strided view
        self.gt_down_sampling = int(gt_down_sampling)
        self._ws = None
        self.crop_h, self.crop_w = int(crop_size[0]), int(crop_size[1])
        self.scale_array = list(scale_array) if scale_array is not None else None
        self.device = torch.device(device)
        self.bgr_input = bool(bgr_input)
        self.lut = torch.from_numpy(normalize_lut(img_mean, img_std)).to(self.device)

    def draw(self, shape_hw, rng=random):
        """one sample's random parameters, consuming `random` exactly like random_mirror → random_scale →
        generate_random_crop_pos (two randint draws only when the scaled image exceeds the crop)"""
        H, W = int(shape_hw[0]), int(shape_hw[1])
        flip = rng.random() >= 0.5
        if self.scale_array is not None:
            scale = rng.choice(self.scale_array)
            sh, sw = int(H * scale), int(W * scale)
        else:
            sh, sw = H, W
        pos_h = rng.randint(0, sh - self.crop_h + 1) if sh > self.crop_h else 0
        pos_w = rng.randint(0, sw - self.crop_w + 1) if sw > self.crop_w else 0
        return dict(flip=bool(flip), sh=sh, sw=sw, pos_h=pos_h, pos_w=pos_w)

    def __call__(self, imgs, gts, params=None):
        """imgs: list of uint8 [H,W,3] tensors on the device (decoded frames; BGR when bgr_input), gts: uint8 [H,W].
        Returns (data float32 [B,3,crop_h,crop_w], label int64 [B,crop_h,crop_w]) — the 'data' / 'label' entries of the
        reference minibatch (BaseDataset.py:49-57)."""
        n = len(imgs)
        assert n == len(gts) and n > 0
        if params is None:
            params = [self.draw(im.shape[:2]) for im in imgs]
        rows = []
        keep = []
        for im, gt, p in zip(imgs, gts, params):
            if im.dtype != torch.uint8 or gt.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise TypeError("TrainPreGPU expects uint8 [H,W,3] frames and uint8 [H,W] labels")
            im, gt = im.contiguous(), gt.contiguous()
            keep += [im, gt]
            H, W = int(im.shape[0]), int(im.shape[1])
            if not (0 <= p["pos_h"] < p["sh"] and 0 <= p["pos_w"] < p["sw"]):      # img_utils.py:27-28
                raise AssertionError("crop origin outside the scaled image")
            rows.append([im.data_ptr(), gt.data_ptr(), H, W, int(p["flip"]), p["sh"], p["sw"], p["pos_h"], p["pos_w"], 0])
        desc = torch.tensor(rows, dtype=torch.int64).to(self.device, non_blocking=False)
        data = torch.empty((n, 3, self.crop_h, self.crop_w), dtype=torch.float32, device=self.device)
        label = torch.empty((n, self.crop_h, self.crop_w), dtype=torch.int64, device=self.device)
        ops.call("tsb_train_preprocess", ops.ptr(desc), n, self.crop_h, self.crop_w, int(self.bgr_input), ops.ptr(self.lut),
                 0.0, 255, ops.ptr(data), ops.ptr(label), ops.stream())
        ds = self.gt_down_sampling
        if ds > 1:
            label = label[:, ::ds, ::ds][:, :self.crop_h // ds, :self.crop_w // ds].contiguous()
        if not self.edge_labels:
            return data, label
        need = int(ops._lib.lib().tsb_edge_labels_workspace_bytes(n, self.crop_h, self.crop_w))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        aux = torch.empty((n, self.crop_h, self.crop_w), dtype=torch.int64, device=self.device)
        ops.call("tsb_edge_labels", ops.ptr(desc), n, self.crop_h, self.crop_w, 255, ops.ptr(self._ws), need, ops.ptr(aux),
                 ops.stream())
        return data, label, aux
