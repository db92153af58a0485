"""Host-side image helpers used by the evaluator (TorchSeg furnace/utils/img_utils.py:8-21,60-74,181-187):
shape canonicalisation, centred constant padding up to a crop size, 0-1 scaling + mean / std normalisation.
cv2 is only needed by pad_image_to_shape (and is imported lazily)."""
from collections.abc import Iterable

import numpy as np


def get_2dshape(shape, *, zero=True):
    """int or (h, w) → (h, w); img_utils.py:8-21"""
    if isinstance(shape, Iterable):
        h, w = (int(v) for v in shape)
    else:
        h = w = int(shape)
    if min(h, w) < (0 if zero else 1):
        raise AssertionError('invalid shape: {}'.format((h, w)))
    return h, w


def pad_image_to_shape(img, shape, border_mode, value):
    """pad (centred; the odd pixel goes to the bottom / right) up to `shape`; returns (image, margin[top, bottom, left,
    right]); img_utils.py:60-74"""
    import cv2
    th, tw = get_2dshape(shape)
    ph, pw = max(th - img.shape[0], 0), max(tw - img.shape[1], 0)
    margin = np.array([ph // 2, ph - ph // 2, pw // 2, pw - pw // 2], dtype=np.uint32)
    img = cv2.copyMakeBorder(img, int(margin[0]), int(margin[1]), int(margin[2]), int(margin[3]), border_mode, value=value)
    return img, margin


def normalize(img, mean, std):
    """uint8 HWC → float32 in [0,1], then (x - mean) / std; img_utils.py:181-187"""
    out = img.astype(np.float32) / 255.0
    out = out - mean
    return out / std
