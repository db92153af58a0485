"""Bit-exact checks of the wgmma convolution kernels on small-integer operands.

Every product and every fp32 partial sum below is an exactly representable number, so any summation order gives the
same fp32 result and the kernels must match a float64 reference bit for bit. A pipeline stage released to the producer
while its MMAs are still reading it, or an epilogue that reads accumulators of the wrong tile, shows up here as a wrong
value rather than as noise inside a tolerance."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv import FULL_SIZE

pytestmark = pytest.mark.gpu

# (N, C, H, W, K, R, stride, pad, dil)
EXTRA = [
    (1, 64, 8, 128, 64, 3, 1, 1, 1),     # 8 row tiles: one tile per CTA
    (3, 64, 132, 128, 64, 3, 1, 1, 1),   # 396 row tiles over 132 CTAs: three (odd) tiles per CTA
    (4, 128, 60, 60, 192, 3, 1, 2, 2),   # dilated 3x3, Q = 60: the nine-tap wgrad kernel
    (2, 64, 8, 8, 64, 3, 1, 2, 2),       # dilated 3x3, Q = 8: too narrow for the nine-tap and row kernels, generic wgrad
]


def _ints(shape, lo, hi, g, dev):
    return torch.randint(lo, hi + 1, shape, device=dev, generator=g).double()


@pytest.mark.parametrize("case", FULL_SIZE + EXTRA, ids=[str(c) for c in FULL_SIZE + EXTRA])
def test_conv_exact_small_integers(cuda, case):
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(21)
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    # |x|, |gy| <= 2, w in quarters of [-2, 2]: fprop / dgrad sums stay below 2^13 in steps of 1/4, wgrad sums (at most
    # 2^20 pixels x 4) below 2^23: every partial sum is exact in fp32
    x = _ints((N, C, H, W), -2, 2, g, cuda)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    y_ref = F.conv2d(xr, wr, None, stride, pad, dil)
    y_ref.backward(gy)

    xd = ops.to_nhwc(x.to(torch.bfloat16))
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wb = torch.empty((K, R, R, C), dtype=torch.bfloat16, device=cuda)
    wt = torch.empty((C, R, R, K), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), ops.ptr(wt), ops.stream())

    y = ops.conv_fprop(xd, wb, K, R, stride, pad, dil, out_dtype=torch.float32)
    assert torch.equal(y, y_ref.float()), "fprop differs"

    gyd = ops.to_nhwc(gy.to(torch.bfloat16))
    dx = ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil)
    assert torch.equal(dx, xr.grad.float().to(torch.bfloat16)), "dgrad differs"

    dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw)
    assert torch.equal(dw.permute(0, 3, 1, 2), wr.grad.float()), "wgrad differs"


@pytest.mark.parametrize("case", FULL_SIZE + EXTRA, ids=[str(c) for c in FULL_SIZE + EXTRA])
def test_conv_statistics_exact(cuda, case):
    """BN Σ / Σ² of a bf16-output launch equal the sums of that output. Three ±1 weights per output channel and
    x in {-1, 0, 1} keep |y| <= 3, so every y, y² and partial sum is a small integer."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(22)
    x = _ints((N, C, H, W), -1, 1, g, cuda)
    w = torch.zeros((K, R * R * C), device=cuda)
    pos = torch.stack([torch.randperm(R * R * C, device=cuda, generator=g)[:3] for _ in range(K)])
    w.scatter_(1, pos, _ints((K, 3), 0, 1, g, cuda).float() * 2 - 1)
    wb = w.view(K, R, R, C).to(torch.bfloat16)
    stats = torch.zeros(2, K, device=cuda)
    y = ops.conv_fprop(ops.to_nhwc(x.to(torch.bfloat16)), wb, K, R, stride, pad, dil, stats=stats).double()
    s1, s2 = y.sum(dim=(0, 2, 3)), (y * y).sum(dim=(0, 2, 3))
    assert float(s2.max()) < 2 ** 24
    assert torch.equal(stats[0].double(), s1), "Σ differs"
    assert torch.equal(stats[1].double(), s2), "Σ² differs"


# (N, C, H, W, K, R, stride, pad, dil, ycs): one shape per kernel family of the fused inference conv
FUSED = [
    (2, 64, 16, 16, 64, 1, 1, 0, 1, 72),     # 1x1: flat GEMM over all pixels
    (1, 64, 8, 128, 64, 3, 1, 1, 1, 72),     # Q >= 96: row tiles
    (2, 128, 20, 24, 64, 3, 1, 1, 1, 80),    # generic tiles
    (2, 64, 32, 32, 128, 3, 2, 1, 1, 136),   # stride 2
    (2, 64, 16, 16, 64, 3, 1, 2, 2, 72),     # dilation 2
    (2, 128, 16, 16, 19, 1, 1, 0, 1, 32),    # 19-class classifier: 24 channels stored, ycs = 32
]
_SENT16, _SENT32 = 0x7FA5, 0x7FA5A5A5   # NaN bit patterns no epilogue computes


@pytest.mark.parametrize("case", FUSED, ids=[str(c) for c in FUSED])
def test_conv_fprop_fused_exact(cuda, case):
    """tsb_conv2d_fprop_fused (folded-BN inference conv): y = relu?(conv + bias (+ res)) equals float64 bit for bit for
    every combination of bias, residual and ReLU, with bf16 and f32 outputs. x is a channel slice whose pad channels
    hold NaN; output channels past the stored K_store = ceil8(K) keep their bits"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil, ycs = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    kst = min((K + 7) // 8 * 8, ycs)
    g = torch.Generator(device="cuda").manual_seed(23)
    x = _ints((N, C, H, W), -2, 2, g, cuda)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    bias = _ints((K,), -8, 8, g, cuda) / 4
    res = _ints((N, P, Q, K), -8, 8, g, cuda)
    conv = F.conv2d(x, w, None, stride, pad, dil).permute(0, 2, 3, 1)
    xcs = C + 64
    xb = torch.full((N, H, W, xcs), float("nan"), dtype=torch.bfloat16, device=cuda)
    xb[..., :C] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wb = torch.empty((K, R, R, C), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), None, ops.stream())
    resb = torch.zeros((N, P, Q, ycs), dtype=torch.bfloat16, device=cuda)   # laid out like y; its pad channels are 0
    resb[..., :K] = res.to(torch.bfloat16)
    bias_f = bias.float()
    shp = ops.make_shape(N, H, W, C, K, R, stride, pad, dil)
    for ydt, tag, bits, sent in ((torch.float32, 0, torch.int32, _SENT32), (torch.bfloat16, 1, torch.int16, _SENT16)):
        for use_bias in (False, True):
            for use_res in ((False, True) if ydt == torch.bfloat16 else (False,)):
                for relu in (0, 1):
                    y = torch.full((N, P, Q, ycs), sent, dtype=bits, device=cuda).view(ydt)
                    ops.call("tsb_conv2d_fprop_fused", ctypes.byref(shp), ops.ptr(xb), xcs, ops.ptr(wb),
                             ops.ptr(bias_f) if use_bias else None, ops.ptr(resb) if use_res else None,
                             ycs if use_res else 0, relu, ops.ptr(y), tag, ycs, ops.stream())
                    ref = conv + (bias if use_bias else 0) + (res if use_res else 0)
                    ref = ref.clamp_min(0) if relu else ref
                    what = "ydtype %s bias %d res %d relu %d" % (ydt, use_bias, use_res, relu)
                    assert torch.equal(y[..., :K], ref.to(ydt)), what
                    assert bool((y[..., K:kst] == 0).all()), what + ": stored pad channels are not zero"
                    assert bool((y.view(bits)[..., kst:] == sent).all()), what + ": wrote past K_store"


@pytest.mark.parametrize("R", [7, 3])
def test_conv_stem_fprop_fused_exact(cuda, R):
    """tsb_conv_stem_fprop_fused (7x7/2 pad 3 or 3x3/2 pad 1 on the space-to-depth image, folded BN) against F.conv2d
    on an integer image, with and without bias and ReLU; output channels past K keep their bits"""
    from torchseg_b200 import ops
    N, H, W, K = 2, 64, 96, 64
    g = torch.Generator(device="cuda").manual_seed(24 + R)
    img = _ints((N, 3, H, W), -2, 2, g, cuda)
    w = _ints((K, 3, R, R), -2, 2, g, cuda) / 4
    bias = _ints((K,), -8, 8, g, cuda) / 4
    imgf = img.float().contiguous()
    xs2d = torch.empty((N, H // 2, W // 2 + 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_image_s2d", ops.ptr(imgf), N, H, W, ops.ptr(xs2d), ops.stream())
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wp = torch.empty((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_stem_weight", ops.ptr(wk), K, R, ops.ptr(wp), ops.stream())
    bias_f = bias.float()
    ycs = K + 8
    for use_bias in (False, True):
        for relu in (0, 1):
            y = torch.full((N, H // 2, W // 2, ycs), _SENT16, dtype=torch.int16, device=cuda).view(torch.bfloat16)
            ops.call("tsb_conv_stem_fprop_fused", ops.ptr(xs2d), N, H, W, ops.ptr(wp), K,
                     ops.ptr(bias_f) if use_bias else None, relu, ops.ptr(y), ycs, ops.stream())
            ref = F.conv2d(img, w, bias if use_bias else None, 2, (R - 1) // 2).permute(0, 2, 3, 1)
            ref = ref.clamp_min(0) if relu else ref
            assert torch.equal(y[..., :K], ref.to(torch.bfloat16)), "bias %d relu %d" % (use_bias, relu)
            assert bool((y.view(torch.int16)[..., K:] == _SENT16).all()), "wrote past K"
