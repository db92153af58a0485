"""The device evaluator (Evaluator.sliding_eval_device / whole_eval_device on tsb_eval_windows, tsb_eval_accumulate,
tsb_eval_resize_add) against the host path it replaces: every kernel bit-exact against the numpy / cv2 restatement
(tests/eval_oracle.py) or the torch accumulation, and the end-to-end predictions identical to sliding_eval / whole_eval
for every pixel."""
import os

import numpy as np
import pytest
import torch

import eval_oracle as eo
from golden_cases import EVAL_KW, eval_image, eval_net

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
HERE = os.path.dirname(os.path.abspath(__file__))


def _lut(dev):
    return torch.from_numpy(eo.normalize_lut(MEAN, STD)).to(dev)


def _windows(cuda, img, s, pad_shape, pad_zero, corners, wh, ww, mirror=False):
    from torchseg_b200 import ops
    H, W = img.shape[:2]
    sh, sw = eo.scaled_size(H, W, s) if s is not None else (H, W)
    th, tw = pad_shape
    ph, pw = max(th - sh, 0), max(tw - sw, 0)
    src = torch.from_numpy(np.ascontiguousarray(img)).to(cuda)
    c = torch.tensor(corners, dtype=torch.int32, device=cuda)
    return ops.eval_windows(src, s, sh, sw, ph // 2, pw // 2, _lut(cuda), pad_zero, c, wh, ww, mirror).cpu().numpy()


@pytest.mark.parametrize("hw", [(333, 271), (200, 260)])
@pytest.mark.parametrize("s", [0.5, 0.75, 1.0, 1.25, 1.75])
@pytest.mark.parametrize("mirror", [False, True])
def test_windows_sliding_branch_exact(cuda, hw, s, mirror):
    img = np.random.default_rng(hw[0]).integers(0, 256, hw + (3,), dtype=np.uint8)
    crop = 160
    cv, _ = eo.canvas(img, s, (crop, crop), MEAN, STD, pad_zero=False)
    from torchseg_b200.engine.evaluator import Evaluator
    corners = Evaluator(None, 5, MEAN, STD, None, [s], False, [0]).window_grid(cv.shape[1], cv.shape[2], crop, 2 / 3.0)
    corners = corners[:5]                 # a batch that the default crop_batch (8) does not divide
    got = _windows(cuda, img, s, (crop, crop), False, corners, crop, crop, mirror)
    assert np.array_equal(got, eo.windows(cv, corners, crop, crop, mirror))


@pytest.mark.parametrize("channels", [3, 1])
@pytest.mark.parametrize("mirror", [False, True])
def test_windows_zero_padding_small_and_grey_exact(cuda, channels, mirror):
    """the single-window branch (small image, normalised then padded with 0.0) and whole_eval's grey frames"""
    img = np.random.default_rng(5).integers(0, 256, (70, 45, channels), dtype=np.uint8)
    cv, _ = eo.canvas(img, None, (96, 80), MEAN, STD, pad_zero=True)
    got = _windows(cuda, img, None, (96, 80), True, [(0, 0)], 96, 80, mirror)
    assert np.array_equal(got, eo.windows(cv, [(0, 0)], 96, 80, mirror))


@pytest.mark.parametrize("flip", [False, True])
def test_accumulate_matches_torch_accumulation(cuda, flip):
    """overlapping windows summed in window order, exp(lp + mirror(lp_flip)) — today's scale_process loop on the device"""
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(9)
    C, crop, PH, PW = 19, 64, 100, 150
    corners = [(0, 0), (0, 43), (0, 86), (36, 0), (36, 43), (36, 86), (10, 20)]
    lp = torch.log_softmax(torch.randn(len(corners), C, crop, crop, generator=g) * 3, 1).to(cuda)
    lpf = torch.log_softmax(torch.randn(len(corners), C, crop, crop, generator=g) * 3, 1).to(cuda) if flip else None
    ref = torch.zeros((C, PH, PW), dtype=torch.float32, device=cuda)
    got = torch.zeros_like(ref)
    for b0 in range(0, len(corners), 3):                  # chunks of 3 windows, like crop_batch = 3
        idx = slice(b0, b0 + 3)
        sc = lp[idx] + lpf[idx].flip(-1) if flip else lp[idx]
        sc = torch.exp(sc.float())
        for (y, x), s in zip(corners[idx], sc):
            ref[:, y:y + crop, x:x + crop] += s
        c = torch.tensor(corners[idx], dtype=torch.int32, device=cuda)
        ops.eval_accumulate(lp[idx].contiguous(), lpf[idx].contiguous() if flip else None, c, got)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("C", [2, 5, 19, 21, 150])
@pytest.mark.parametrize("dst", [(80, 120), (20, 30), (111, 159), (37, 53), (18, 26)])
def test_resize_add_matches_cv2(cuda, C, dst):
    """a margin-cropped strided view, resized like cv2 (linear, x3, identity, exact 2x down = area), added in fp64"""
    from torchseg_b200 import ops
    rng = np.random.default_rng(C)
    buf = (rng.random((C, 45, 60)) * 3).astype(np.float32)
    view = buf[:, 3:3 + 37, 5:5 + 53] if dst != (18, 26) else buf[:, 3:39, 5:57]
    ref = cv2.resize(np.ascontiguousarray(view.transpose(1, 2, 0)), (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    ref = ref.transpose(2, 0, 1)
    prev = rng.random((C,) + dst)
    b = torch.from_numpy(buf).to(cuda)
    v = b[:, 3:3 + view.shape[1], 5:5 + view.shape[2]]
    total = torch.from_numpy(prev).to(cuda)
    ops.eval_resize_add(v, total)
    assert np.array_equal(total.cpu().numpy(), prev + ref.astype(np.float64))
    pred = torch.empty(dst, dtype=torch.int64, device=cuda)
    total = torch.from_numpy(prev).to(cuda)
    ops.eval_resize_add(v, total, pred)
    assert np.array_equal(pred.cpu().numpy(), (prev + ref.astype(np.float64)).argmax(0))
    assert np.array_equal(total.cpu().numpy(), prev)          # the last scale does not store the total


def test_resize_add_multi_scale_sum_and_first_index_ties(cuda):
    from torchseg_b200 import ops
    rng = np.random.default_rng(4)
    C, H, W = 6, 40, 50
    total = torch.zeros((C, H, W), dtype=torch.float64, device=cuda)
    ref = np.zeros((H, W, C))
    for h, w in [(20, 25), (30, 37), (40, 50), (70, 88)]:
        sc = rng.random((h, w, C)).astype(np.float32)
        ref += cv2.resize(sc, (W, H), interpolation=cv2.INTER_LINEAR)
        ops.eval_resize_add(torch.from_numpy(sc.transpose(2, 0, 1).copy()).to(cuda), total)
    assert np.array_equal(total.cpu().numpy(), ref.transpose(2, 0, 1))
    # ties: integer scores, identity size → equal maxima; numpy takes the first
    sc = rng.integers(0, 3, (C, H, W)).astype(np.float32)
    pred = torch.empty((H, W), dtype=torch.int64, device=cuda)
    ops.eval_resize_add(torch.from_numpy(sc).to(cuda), torch.zeros((C, H, W), dtype=torch.float64, device=cuda), pred)
    assert np.array_equal(pred.cpu().numpy(), sc.astype(np.float64).argmax(0))


# ---------------------------------------------------------------------------------------------------------- end to end
def _bisenet(cuda):
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    BN = torch.nn.BatchNorm2d
    torch.manual_seed(31)
    model = BiSeNet(19, False, None, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = torch.Generator().manual_seed(32)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) * 1.5 + 0.5)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    return model


def _evaluator(net, class_num, scales, flip, crop_batch):
    from torchseg_b200.engine.evaluator import Evaluator
    ev = Evaluator(dataset=None, class_num=class_num, image_mean=MEAN, image_std=STD, network=None, multi_scales=scales,
                   is_flip=flip, devices=[0], crop_batch=crop_batch)
    ev.val_func = net
    return ev


def test_sliding_eval_device_bisenet_ms_flip_every_pixel(cuda):
    """libtsb BiSeNet-R18, scales [0.5, 0.75, 1.0, 1.25] with flip on an odd frame: identical predictions, identical
    confusion matrix, identical bits on a second run"""
    from torchseg_b200.seg_opr.metric import hist_info, hist_info_torch
    ev = _evaluator(_bisenet(cuda), 19, [0.5, 0.75, 1.0, 1.25], True, 3)
    img = np.random.default_rng(33).integers(0, 256, (301, 427, 3), dtype=np.uint8)
    host = ev.sliding_eval(img, 192, 2 / 3.0, cuda)
    dev = ev.sliding_eval_device(img, 192, 2 / 3.0, cuda)
    assert dev.device.type == "cuda" and dev.dtype == torch.int64
    assert np.array_equal(dev.cpu().numpy(), host)
    gt = np.random.default_rng(34).integers(0, 21, host.shape)
    gt[:20] = 255
    conf, lab, ok = hist_info_torch(19, dev, torch.from_numpy(gt).to(cuda))
    rconf, rlab, rok = hist_info(19, host, gt)
    assert np.array_equal(conf.cpu().numpy(), rconf) and int(lab) == rlab and int(ok) == rok
    assert torch.equal(ev.sliding_eval_device(img, 192, 2 / 3.0, cuda), dev)


def test_sliding_eval_device_pspnet_150_classes(cuda):
    import torchseg_b200
    from torchseg_b200.networks import PSPNet
    torch.manual_seed(41)
    net = PSPNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1))
    net.to(cuda)
    torchseg_b200.prepare_model(net)
    ev = _evaluator(net, 150, [0.75, 1.0], False, 2)
    img = np.random.default_rng(42).integers(0, 256, (181, 243, 3), dtype=np.uint8)
    host = ev.sliding_eval(img, 160, 2 / 3.0, cuda)
    assert np.array_equal(ev.sliding_eval_device(img, 160, 2 / 3.0, cuda).cpu().numpy(), host)


@pytest.mark.parametrize("output_size,input_size", [(None, None), ((75, 105), (160, 224)), ((300, 420), None),
                                                    ((75, 105), None), ((150, 210), (150, 224))])
def test_whole_eval_device(cuda, output_size, input_size):
    """with and without padding to input_size and resizing to output_size; (75, 105) is an exact 2x down-scale (area)"""
    ev = _evaluator(eval_net().to(cuda), 5, [1.0], True, 3)
    img = eval_image()
    host = ev.whole_eval(img, output_size, input_size, cuda)
    assert np.array_equal(ev.whole_eval_device(img, output_size, input_size, cuda).cpu().numpy(), host)


def test_whole_eval_device_grey(cuda):
    ev = _evaluator(eval_net().to(cuda), 5, [1.0], True, 3)
    img = eval_image()[:, :, :1]
    assert np.array_equal(ev.whole_eval_device(img, None, None, cuda).cpu().numpy(), ev.whole_eval(img, None, None, cuda))


def test_golden_eval_case_on_the_device(cuda):
    """the live-reference-pinned evaluator case (tests/golden/live_reference.npz): the device path equals the host path
    run on the same GPU, and agrees with the reference's CPU predictions as closely as the CPU test requires"""
    from torchseg_b200.engine.evaluator import Evaluator
    live = np.load(os.path.join(HERE, "golden", "live_reference.npz"))
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False                # fp32 convolutions, like the reference's CPU run
    try:
        _golden_case(cuda, live)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _golden_case(cuda, live):
    from torchseg_b200.engine.evaluator import Evaluator
    ev = Evaluator(crop_batch=3, **EVAL_KW)
    ev.val_func = eval_net().to(cuda)
    img = eval_image()
    dev = ev.sliding_eval_device(img, 96, 2 / 3.0, cuda).cpu().numpy()
    assert np.array_equal(dev, ev.sliding_eval(img, 96, 2 / 3.0, cuda))
    assert (live["eval_sliding"] == dev).mean() > 0.999
    small = ev.sliding_eval_device(img[:80, :70], 96, 2 / 3.0, cuda).cpu().numpy()
    assert np.array_equal(small, ev.sliding_eval(img[:80, :70], 96, 2 / 3.0, cuda))
    assert (live["eval_small"] == small).mean() > 0.999
    whole = ev.whole_eval_device(img, (75, 105), (160, 224), cuda).cpu().numpy()
    assert (live["eval_whole"] == whole).mean() > 0.999
    grey = ev.whole_eval_device(img[:, :, :1], None, None, cuda).cpu().numpy()
    assert (live["eval_grey"] == grey).mean() > 0.999
