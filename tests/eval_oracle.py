"""ORACLE — test infrastructure only: the OpenCV arithmetic of the evaluator (engine/evaluator.py).

numpy restatements of the three cv2.resize calls that `sliding_eval` / `scale_process` / `whole_eval` make, and of the
window cut + normalisation + padding that feeds the network, so that the device evaluator (tsb_eval_windows,
tsb_eval_accumulate, tsb_eval_resize_add) can be pinned bit for bit without calling cv2 inside a kernel test.
Pinned against cv2 itself (4.13 in this image) by tests/test_cpu_eval_oracle.py.

OpenCV facts restated (imgproc/src/resize.cpp):
- `cv2.resize(img, None, fx=s, fy=s)` takes dsize = (rint(W·s), rint(H·s)) and the coefficient scale 1/s, NOT src/dst.
- dsize == ssize is a plain copy.
- INTER_LINEAR with an exact integer scale of 2 in both directions (1/s == 2, or dsize exactly half of ssize) switches
  to INTER_AREA (resizeAreaFast).
  - uint8: `(a + b + c + d + 2) >> 2` over every full 2x2 block; a block cut by an odd border averages the pixels it
    has: rint((float)sum / count).
  - float: `0 + (((a00 + a01) + a10) + a11)` times 0.25 for channel counts other than 1 and 4.
- uint8 INTER_LINEAR is fixed point: 11-bit coefficients, int32 horizontal pass, vertical pass
  `(((b0·(S0>>4))>>16) + ((b1·(S1>>4))>>16) + 2) >> 2`.
- float INTER_LINEAR: f = (float)((d + 0.5)·scale − 0.5), s = floor(f), f −= s with scale = src/dst in double; in x
  only the borders clamp with f = 0; each pass rounds both products and the sum separately (no FMA); rows are clamped.
  For 1, 3 and 4 channels cv2 runs other vector code whose last bits differ (up to ~1.7e-5 relative); segmentation score
  maps have at least 2 channels, and the shipped lines have 19, 21 or 150.

Nothing under torchseg_b200/ imports this file.
"""
import numpy as np

EPS = np.finfo(np.float64).eps


def scaled_size(H, W, s):
    """dsize of cv2.resize(img, None, fx=s, fy=s): saturate_cast<int>(W·s), i.e. round half to even"""
    return int(np.rint(H * s)), int(np.rint(W * s))


def is_area_fast(scale_y, scale_x):
    """cv2's switch from INTER_LINEAR to INTER_AREA: both scales are (within DBL_EPSILON of) the integer 2"""
    return abs(scale_x - 2.0) < EPS and abs(scale_y - 2.0) < EPS


def _coef(dst, scale):
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    return s, f


def _clamp_x(s, f, src):
    s, f = s.copy(), f.copy()
    lo = s < 0
    f[lo], s[lo] = 0, 0
    hi = s >= src - 1
    f[hi], s[hi] = 0, src - 1
    return s, f


# -------------------------------------------------------------------------------------------------------------- uint8
def _linear_u8(img, dh, dw, scale_y, scale_x):
    H, W = img.shape[:2]
    sx, fx = _clamp_x(*_coef(dw, scale_x), W)
    sy, fy = _coef(dh, scale_y)
    a0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(fx * np.float32(2048)).astype(np.int64)
    b0 = np.rint((np.float32(1) - fy) * np.float32(2048)).astype(np.int64)
    b1 = np.rint(fy * np.float32(2048)).astype(np.int64)
    src = img.astype(np.int64)
    hrow = src[:, sx, :] * a0[None, :, None] + src[:, np.minimum(sx + 1, W - 1), :] * a1[None, :, None]
    y0, y1 = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
    out = (((b0[:, None, None] * (hrow[y0] >> 4)) >> 16) + ((b1[:, None, None] * (hrow[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def _area2_u8(img, dh, dw):
    H, W = img.shape[:2]
    src = img.astype(np.int64)
    out = np.empty((dh, dw, img.shape[2]), np.int64)
    fh, fw = min(H // 2, dh), min(W // 2, dw)
    out[:fh, :fw] = (src[0:2 * fh:2, 0:2 * fw:2] + src[0:2 * fh:2, 1:2 * fw:2] + src[1:2 * fh:2, 0:2 * fw:2]
                     + src[1:2 * fh:2, 1:2 * fw:2] + 2) >> 2
    for y in range(dh):                                   # blocks cut by an odd border: rint((float)sum / count)
        for x in range(dw):
            if y < fh and x < fw:
                continue
            blk = src[2 * y:2 * y + 2, 2 * x:2 * x + 2]
            cnt = blk.shape[0] * blk.shape[1]
            out[y, x] = np.rint(blk.sum(axis=(0, 1)).astype(np.float32) / np.float32(cnt))
    return np.clip(out, 0, 255).astype(np.uint8)


def resize_fx_u8(img, s):
    """cv2.resize(img, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR) for uint8 [H, W, C]"""
    H, W = img.shape[:2]
    dh, dw = scaled_size(H, W, s)
    if (dh, dw) == (H, W):
        return img.copy()
    scale = 1.0 / s
    if is_area_fast(scale, scale):
        return _area2_u8(img, dh, dw)
    return _linear_u8(img, dh, dw, scale, scale)


# -------------------------------------------------------------------------------------------------------------- float
def resize_f32(src, dh, dw):
    """cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR) for float32 [h, w, C], C not in {1, 3, 4}"""
    h, w = src.shape[:2]
    src = src.astype(np.float32)
    if (dh, dw) == (h, w):
        return src.copy()
    scale_y, scale_x = 1.0 / (dh / h), 1.0 / (dw / w)
    if is_area_fast(scale_y, scale_x):
        a00, a01 = src[0::2, 0::2][:dh, :dw], src[0::2, 1::2][:dh, :dw]
        a10, a11 = src[1::2, 0::2][:dh, :dw], src[1::2, 1::2][:dh, :dw]
        return (((a00 + a01) + a10) + a11) * np.float32(0.25)
    sx, fx = _clamp_x(*_coef(dw, scale_x), w)
    sy, fy = _coef(dh, scale_y)
    one = np.float32(1)
    hx = src[:, sx] * (one - fx)[None, :, None] + src[:, np.minimum(sx + 1, w - 1)] * fx[None, :, None]
    g = fy[:, None, None]
    return hx[np.clip(sy, 0, h - 1)] * (one - g) + hx[np.clip(sy + 1, 0, h - 1)] * g


# -------------------------------------------------------------------------------------------------------- windows
def normalize_lut(mean, std):
    """normalize() (utils/img_utils.py) of every uint8 value, as the float32 the network receives: [3, 256]"""
    v = np.arange(256, dtype=np.float32) / 255.0
    return ((v[None, :] - np.asarray(mean, np.float64)[:, None]) / np.asarray(std, np.float64)[:, None]).astype(np.float32)


def canvas(img, s, pad_shape, mean, std, pad_zero):
    """the normalised, padded [3, PH, PW] float32 image the windows are cut from.
    pad_zero=False: scale_process's sliding branch (uint8 padded with 0, then normalised: pad = normalize(0)).
    pad_zero=True: process_image(img, crop) (normalised, then padded with 0.0). s=None: no resize.
    Returns (canvas, margin[top, bottom, left, right])."""
    if img.shape[2] == 1:
        img = np.concatenate([img] * 3, axis=2)
    if s is not None:
        img = resize_fx_u8(img, s)
    H, W = img.shape[:2]
    th, tw = pad_shape
    ph, pw = max(th - H, 0), max(tw - W, 0)
    m = (ph // 2, ph - ph // 2, pw // 2, pw - pw // 2)
    lut = normalize_lut(mean, std)
    out = np.empty((3, H + ph, W + pw), np.float32)
    for c in range(3):
        out[c] = 0.0 if pad_zero else lut[c, 0]
        out[c, m[0]:m[0] + H, m[2]:m[2] + W] = lut[c][img[:, :, c]]
    return out, m


def windows(cv, corners, wh, ww, mirror=False):
    """[n, 3, wh, ww] crops of a canvas at (y, x) corners, optionally mirrored left-right"""
    out = np.stack([cv[:, y:y + wh, x:x + ww] for y, x in corners])
    return np.ascontiguousarray(out[..., ::-1] if mirror else out)
