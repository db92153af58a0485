"""ORACLE — test infrastructure only.

numpy restatement of the reference's training-time input pipeline for one sample
(TorchSeg model/bisenet/cityscapes.bisenet.R18/dataloader.py:11-33 `TrainPre.__call__`, built from
TorchSeg furnace/utils/img_utils.py: random_mirror :140-145, random_scale :118-125, normalize :181-187,
generate_random_crop_pos :44-60, random_crop_pad_to_shape :24-41 / pad_image_to_shape :63-78) and of the two OpenCV
routines it calls on uint8 data.

Third-party arithmetic: OpenCV (`cv2`, 4.13.0 in this image; the reference does not pin a version) —
`cv2.resize(..., INTER_LINEAR)` on 8-bit data is fixed point: 11-bit coefficients (INTER_RESIZE_COEF_SCALE = 2048),
horizontal pass in int32, vertical pass `(((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2`
(imgproc/src/resize.cpp, HResizeLinear / VResizeLinear<uchar,...>); `INTER_NEAREST` is `min(floor(dst*scale), size-1)`.
Both restatements are pinned bit-for-bit against cv2 itself (tests/test_cpu_data.py, IPP on and off) and the whole
pipeline against the LIVE reference TrainPre on seeded inputs (tests/golden/data_pipeline.json, tools/make_golden.py).
"""
import random

import numpy as np


def _coeffs(src, dst):
    """source index and fractional offset of every destination coordinate (resize.cpp: fx = (float)((dx+0.5)*scale-0.5))"""
    scale = 1.0 / (float(dst) / float(src))
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def resize_linear_u8(img, dw, dh):
    """cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR) for uint8 [H,W] / [H,W,C]"""
    H, W = img.shape[:2]
    sx, fx = _coeffs(W, dw)
    sy, fy = _coeffs(H, dh)
    fx = fx.copy()
    sx = sx.copy()
    lo = sx < 0
    fx[lo] = 0
    sx[lo] = 0
    hi = sx >= W - 1
    fx[hi] = 0
    sx[hi] = W - 1
    a0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(fx * np.float32(2048)).astype(np.int64)
    b0 = np.rint((np.float32(1) - fy) * np.float32(2048)).astype(np.int64)
    b1 = np.rint(fy * np.float32(2048)).astype(np.int64)
    sx1 = np.minimum(sx + 1, W - 1)
    src = img.astype(np.int64)
    if src.ndim == 2:
        src = src[:, :, None]
    hrow = src[:, sx, :] * a0[None, :, None] + src[:, sx1, :] * a1[None, :, None]
    y0 = np.clip(sy, 0, H - 1)
    y1 = np.clip(sy + 1, 0, H - 1)
    out = (((b0[:, None, None] * (hrow[y0] >> 4)) >> 16) + ((b1[:, None, None] * (hrow[y1] >> 4)) >> 16) + 2) >> 2
    out = np.clip(out, 0, 255).astype(np.uint8)
    return out if img.ndim == 3 else out[:, :, 0]


def resize_nearest(img, dw, dh):
    """cv2.resize(img, (dw, dh), interpolation=cv2.INTER_NEAREST)"""
    H, W = img.shape[:2]
    ifx = 1.0 / (float(dw) / float(W))
    ify = 1.0 / (float(dh) / float(H))
    xs = np.minimum(np.floor(np.arange(dw, dtype=np.float64) * ifx).astype(np.int64), W - 1)
    ys = np.minimum(np.floor(np.arange(dh, dtype=np.float64) * ify).astype(np.int64), H - 1)
    return img[ys][:, xs]


def draw_params(shape_hw, crop_size, scale_array, rng=random):
    """the random draws of TrainPre.__call__ in the reference's order (Python's `random` module): mirror, scale, crop"""
    H, W = shape_hw
    flip = rng.random() >= 0.5                                   # img_utils.py:141
    scale = rng.choice(scale_array) if scale_array is not None else 1   # :119
    sh, sw = (int(H * scale), int(W * scale)) if scale_array is not None else (H, W)
    ch, cw = crop_size
    pos_h = rng.randint(0, sh - ch + 1) if sh > ch else 0        # :54-58 (inclusive upper bound: may overshoot by one)
    pos_w = rng.randint(0, sw - cw + 1) if sw > cw else 0
    return dict(flip=bool(flip), scale=scale, sh=sh, sw=sw, pos_h=pos_h, pos_w=pos_w)


def _crop_pad(img, pos, crop_size, value):
    """random_crop_pad_to_shape (img_utils.py:24-41): crop, then centre the crop inside the target with a constant border"""
    ph, pw = pos
    ch, cw = crop_size
    c = img[ph:ph + ch, pw:pw + cw, ...]
    pad_h = max(ch - c.shape[0], 0)
    pad_w = max(cw - c.shape[1], 0)
    top, left = pad_h // 2, pad_w // 2
    out = np.full((c.shape[0] + pad_h, c.shape[1] + pad_w) + c.shape[2:], value, dtype=c.dtype)
    out[top:top + c.shape[0], left:left + c.shape[1], ...] = c
    return out


def train_pre(img_rgb, gt, params, crop_size, mean, std, gt_down_sampling=1):
    """img_rgb: uint8 [H,W,3] (after BaseDataset's `img[:, :, ::-1]`, BaseDataset.py:45), gt: uint8 [H,W].
    Returns (float32 [3,ch,cw], int64 [ch,cw]) exactly as BaseDataset.__getitem__ hands them to the loader (:49-51).
    gt_down_sampling > 1: the speed config (model/bisenet/cityscapes.bisenet.R18.speed/dataloader.py:28-30) resizes the
    cropped label to (cw // ds, ch // ds) with INTER_NEAREST."""
    if params["flip"]:
        img_rgb = img_rgb[:, ::-1]
        gt = gt[:, ::-1]
    if (params["sh"], params["sw"]) != img_rgb.shape[:2] or params["scale"] != 1:
        img_rgb = resize_linear_u8(np.ascontiguousarray(img_rgb), params["sw"], params["sh"])
        gt = resize_nearest(np.ascontiguousarray(gt), params["sw"], params["sh"])
    x = img_rgb.astype(np.float32) / 255.0                        # :183  (float32)
    x = x - mean                                                  # :184  (float64: mean / std are float64 arrays)
    x = x / std                                                   # :185
    pos = (params["pos_h"], params["pos_w"])
    p_img = _crop_pad(x, pos, crop_size, 0)
    p_gt = _crop_pad(gt, pos, crop_size, 255)
    if gt_down_sampling > 1:
        p_gt = resize_nearest(np.ascontiguousarray(p_gt), crop_size[1] // gt_down_sampling, crop_size[0] // gt_down_sampling)
    return np.ascontiguousarray(p_img.transpose(2, 0, 1)).astype(np.float32), np.ascontiguousarray(p_gt).astype(np.int64)


# --------------------------------------------------------------------------------------------------
# DFN border labels — TorchSeg model/dfn/cityscapes.dfn.R101_v1c/dataloader.py:15-29:
#   no255_gt = gt with 255 → 0; cgt = cv2.Canny(no255_gt, 5, 5, apertureSize=7); cgt = cv2.dilate(cgt, 7x7 rect); 255 → 1
# OpenCV's Canny for apertureSize = 7 (imgproc/src/canny.cpp): thresholds /16 then floor (5 → 0), dx / dy =
# Sobel(ksize 7, scale 1/16, BORDER_REPLICATE) as int16 (round half to even), magnitude |dx| + |dy| with a zero border,
# non-maximum suppression by the fixed-point tangent test (TG22 = round(tan 22.5° · 2^15)), then hysteresis (empty here:
# low == high). Pinned bit-for-bit against cv2 in tests/test_cpu_data.py.
# --------------------------------------------------------------------------------------------------
_SM7 = np.array([1, 6, 15, 20, 15, 6, 1], dtype=np.int64)
_DV7 = np.array([-1, -4, -5, 0, 5, 4, 1], dtype=np.int64)


def sobel7_over16(img):
    H, W = img.shape
    p = np.pad(img.astype(np.int64), 3, mode="edge")

    def sep(kx, ky):
        t = np.zeros((H + 6, W), dtype=np.int64)
        for i in range(7):
            t += kx[i] * p[:, i:i + W]
        o = np.zeros((H, W), dtype=np.int64)
        for i in range(7):
            o += ky[i] * t[i:i + H, :]
        return o

    def rnd(v):
        return np.clip(np.rint(v / 16.0), -32768, 32767).astype(np.int64)

    return rnd(sep(_DV7, _SM7)), rnd(sep(_SM7, _DV7))


def canny_ap7(img, low_t=5, high_t=5):
    """cv2.Canny(img, low_t, high_t, apertureSize=7) (L1 gradient) for uint8 [H,W]"""
    low = int(np.floor(low_t / 16.0))
    high = int(np.floor(high_t / 16.0))
    dx, dy = sobel7_over16(img)
    H, W = img.shape
    mp = np.pad(np.abs(dx) + np.abs(dy), 1)
    m = mp[1:-1, 1:-1]
    TG22 = int(0.4142135623730950488016887242097 * (1 << 15) + 0.5)
    x = np.abs(dx)
    y = np.abs(dy) << 15
    tg22x = x * TG22
    tg67x = tg22x + (x << 16)
    s = np.where((dx ^ dy) < 0, -1, 1)
    jj = np.arange(W)[None, :] + 1
    ii = np.arange(H)[:, None] + 1
    horiz = (y < tg22x) & (m > mp[1:-1, 0:-2]) & (m >= mp[1:-1, 2:])
    vert = (y >= tg22x) & (y > tg67x) & (m > mp[0:-2, 1:-1]) & (m >= mp[2:, 1:-1])
    diag = (y >= tg22x) & (y <= tg67x) & (m > mp[ii - 1, jj - s]) & (m > mp[ii + 1, jj + s])
    cand = (m > low) & (horiz | vert | diag)
    strong = cand & (m > high)
    weak = cand & ~strong
    if weak.any():                       # hysteresis: only when low < high (not the DFN call)
        out = strong.copy()
        stack = list(zip(*np.nonzero(strong)))
        while stack:
            i, j = stack.pop()
            for di in (-1, 0, 1):
                for dj in (-1, 0, 1):
                    a, b = i + di, j + dj
                    if 0 <= a < H and 0 <= b < W and weak[a, b] and not out[a, b]:
                        out[a, b] = True
                        stack.append((a, b))
        strong = out
    return (strong * 255).astype(np.uint8)


def dilate7(img):
    """cv2.dilate(img, cv2.getStructuringElement(cv2.MORPH_RECT, (7, 7))) for a non-negative uint8 map"""
    H, W = img.shape
    p = np.pad(img, 3)
    out = np.zeros_like(img)
    for i in range(7):
        for j in range(7):
            out = np.maximum(out, p[i:i + H, j:j + W])
    return out


def train_pre_dfn(img_rgb, gt, params, crop_size, mean, std):
    """DFN TrainPre.__call__ (dfn dataloader.py:15-44): as train_pre plus the border label 'aux_label' ∈ {0, 1, 255}"""
    if params["flip"]:
        img_rgb = img_rgb[:, ::-1]
        gt = gt[:, ::-1]
    img_rgb = resize_linear_u8(np.ascontiguousarray(img_rgb), params["sw"], params["sh"])
    gt = resize_nearest(np.ascontiguousarray(gt), params["sw"], params["sh"])
    no255 = gt.copy()
    no255[gt == 255] = 0
    cgt = dilate7(canny_ap7(no255, 5, 5))
    cgt[cgt == 255] = 1
    x = ((img_rgb.astype(np.float32) / 255.0) - mean) / std
    pos = (params["pos_h"], params["pos_w"])
    p_img = _crop_pad(x, pos, crop_size, 0)
    p_gt = _crop_pad(gt, pos, crop_size, 255)
    p_cgt = _crop_pad(cgt, pos, crop_size, 255)
    return (np.ascontiguousarray(p_img.transpose(2, 0, 1)).astype(np.float32), np.ascontiguousarray(p_gt).astype(np.int64),
            np.ascontiguousarray(p_cgt).astype(np.int64))
