"""CPU tests of the device evaluator's ground truth (tests/eval_oracle.py): the numpy restatements of every cv2 path the
host evaluator takes are bit-exact against cv2 itself, the window canvas equals the host evaluator's normalised and
padded image, and the three tsb_eval_* entry points reject bad arguments before touching a device."""
import ctypes

import numpy as np
import pytest

import eval_oracle as eo

MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
cv2 = pytest.importorskip("cv2")


def _cv_f32(src, dh, dw):
    out = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)
    return out[:, :, None] if out.ndim == 2 else out


@pytest.mark.parametrize("C", [2, 5, 19, 21, 150])
@pytest.mark.parametrize("dst", [(80, 120), (20, 30), (111, 159), (37, 53), (13, 41)])
def test_float_linear_bit_exact(C, dst):
    """float32 INTER_LINEAR of a [37, 53, C] score map: up, down, x3 and identity"""
    src = (np.random.default_rng(C).random((37, 53, C)) * 3).astype(np.float32)
    assert np.array_equal(eo.resize_f32(src, *dst), _cv_f32(src, *dst))


@pytest.mark.parametrize("C", [2, 5, 19, 21, 150])
def test_float_area_fast_bit_exact(C):
    """an exact 2x down-scale is INTER_AREA in cv2, not the linear formula"""
    src = np.random.default_rng(7).random((200, 260, C)).astype(np.float32)
    ref = _cv_f32(src, 100, 130)
    assert np.array_equal(eo.resize_f32(src, 100, 130), ref)
    assert eo.is_area_fast(2.0, 2.0) and not eo.is_area_fast(2.0, 1.9)


@pytest.mark.parametrize("C", [1, 3, 4])
def test_float_other_vector_paths_close(C):
    """1, 3 and 4 channels run other cv2 vector code: the restatement is within a few ulp, not bit-exact"""
    src = np.random.default_rng(C).random((37, 53, C)).astype(np.float32) * 3
    for dst in [(80, 120), (20, 30), (100, 26)]:
        ref = _cv_f32(src, *dst)
        assert np.allclose(eo.resize_f32(src, *dst), ref, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("hw", [(333, 271), (200, 260), (101, 99), (64, 65)])
@pytest.mark.parametrize("s", [0.5, 0.75, 1.0, 1.25, 1.5, 1.75])
def test_uint8_fx_bit_exact(hw, s):
    """cv2.resize(img, None, fx=s, fy=s) on uint8: coefficient scale 1/s, area-fast at s = 0.5 (odd borders included)"""
    img = np.random.default_rng(hw[0] + hw[1]).integers(0, 256, hw + (3,), dtype=np.uint8)
    ref = cv2.resize(img, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR)
    assert ref.shape[:2] == eo.scaled_size(*hw, s)
    assert np.array_equal(eo.resize_fx_u8(img, s), ref)


def test_uint8_fx_is_not_dsize_scale():
    """with fx, cv2's coefficient scale is 1/s; dsize / ssize (what the training pipeline uses) gives other pixels"""
    import oracle.data_ref as dr
    img = np.random.default_rng(1).integers(0, 256, (713, 517, 3), dtype=np.uint8)
    dh, dw = eo.scaled_size(713, 517, 1.75)
    assert not np.array_equal(dr.resize_linear_u8(img, dw, dh), cv2.resize(img, None, fx=1.75, fy=1.75))


def _host_evaluator(**kw):
    from torchseg_b200.engine.evaluator import Evaluator
    return Evaluator(dataset=None, class_num=5, image_mean=MEAN, image_std=STD, network=None, multi_scales=[1.0],
                     is_flip=False, devices=[0], **kw)


@pytest.mark.parametrize("s", [0.5, 0.75, 1.25])
def test_canvas_uint8_padding_matches_scale_process(s):
    """sliding branch: the uint8 frame is padded with 0, then normalised (pad pixels = normalize(0))"""
    from torchseg_b200.utils.img_utils import pad_image_to_shape
    ev = _host_evaluator()
    img = np.random.default_rng(2).integers(0, 256, (101, 57, 3), dtype=np.uint8)
    crop = 96
    scaled = cv2.resize(img, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR)
    padded, margin = pad_image_to_shape(scaled, crop, cv2.BORDER_CONSTANT, value=0)
    host = ev.process_image(padded).astype(np.float32)
    cv, m = eo.canvas(img, s, (crop, crop), MEAN, STD, pad_zero=False)
    assert tuple(m) == tuple(int(v) for v in margin)
    assert np.array_equal(cv, host)
    corners = ev.window_grid(cv.shape[1], cv.shape[2], crop, 2 / 3.0)
    ref = np.stack([host[:, y:y + crop, x:x + crop] for y, x in corners])
    assert np.array_equal(eo.windows(cv, corners, crop, crop), ref)
    assert np.array_equal(eo.windows(cv, corners, crop, crop, mirror=True), ref[..., ::-1])


@pytest.mark.parametrize("channels", [3, 1])
def test_canvas_zero_padding_matches_process_image(channels):
    """single-window branch and whole_eval(input_size=...): normalised first, then padded with 0.0; grey → 3 planes"""
    ev = _host_evaluator()
    img = np.random.default_rng(3).integers(0, 256, (70, 45, channels), dtype=np.uint8)
    host, margin = ev.process_image(img, (96, 80))
    cv, m = eo.canvas(img, None, (96, 80), MEAN, STD, pad_zero=True)
    assert tuple(m) == tuple(int(v) for v in margin)
    assert np.array_equal(cv, host.astype(np.float32))


def test_normalize_lut_matches_the_training_table():
    from torchseg_b200.utils.gpu_pipeline import normalize_lut
    assert np.array_equal(eo.normalize_lut(MEAN, STD), normalize_lut(MEAN, STD))


def test_eval_entry_points_validate_without_gpu():
    from torchseg_b200 import build, _lib
    build.build()
    lib = _lib.lib()
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255
    cases = [
        ("tsb_eval_windows", (None, 8, 8, 3, 1.0, 8, 8, 0, 0, A, 0, A, 1, 8, 8, 0, A, None), b"null pointer"),
        ("tsb_eval_windows", (A, 8, 8, 2, 1.0, 8, 8, 0, 0, A, 0, A, 1, 8, 8, 0, A, None), b"cin"),
        ("tsb_eval_windows", (A, 8, 8, 3, 0.5, 5, 4, 0, 0, A, 0, A, 1, 8, 8, 0, A, None), b"dsize"),
        ("tsb_eval_windows", (A, 7, 9, 3, 0.0, 4, 4, 0, 0, A, 0, A, 1, 8, 8, 0, A, None), b"dsize"),
        ("tsb_eval_windows", (A, 8, 8, 3, 1.0, 8, 8, 0, 0, A, 0, A, 0, 8, 8, 0, A, None), b"window"),
        ("tsb_eval_accumulate", (A, None, A, 0, 19, 8, 8, A, 8, 8, None), b"bad sizes"),
        ("tsb_eval_accumulate", (A, None, A, 1, 19, 8, 8, A, 0, 8, None), b"accumulator"),
        ("tsb_eval_accumulate", (None, None, A, 1, 19, 8, 8, A, 8, 8, None), b"null pointer"),
        ("tsb_eval_resize_add", (A, 19, 8, 8, 64, 4, A, 8, 8, None, None), b"strides"),
        ("tsb_eval_resize_add", (A, 19, 8, 8, 32, 8, A, 8, 8, None, None), b"strides"),
        ("tsb_eval_resize_add", (A, 0, 8, 8, 64, 8, A, 8, 8, None, None), b"bad sizes"),
        ("tsb_eval_resize_add", (A, 19, 8, 8, 64, 8, None, 8, 8, None, None), b"null pointer"),
    ]
    for name, args, msg in cases:
        rc = getattr(lib, name)(*args)
        err = lib.tsb_last_error()
        assert rc == -1 and msg in err and name.encode() in err, (name, args, rc, err)
