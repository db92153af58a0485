"""Bit-exact checks of the wgmma convolution kernels on small-integer operands.

Every product and every fp32 partial sum below is an exactly representable number, so any summation order gives the
same fp32 result and the kernels must match a float64 reference bit for bit. A pipeline stage released to the producer
while its MMAs are still reading it, or an epilogue that reads accumulators of the wrong tile, shows up here as a wrong
value rather than as noise inside a tolerance. Each case asserts the bound that keeps it inside the exact range.

Layouts: the "sliced" cases hand every kernel operand as a channel slice of a wider NHWC buffer, at a 16-byte channel
offset, with NaN in every channel the kernel must not read, and write into buffers prefilled with NaN bit patterns no
epilogue computes, so a read or a write outside the slice shows up as a NaN or as a changed sentinel."""
import ctypes
import re

import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv import CASES, FULL_SIZE

pytestmark = pytest.mark.gpu

# (N, C, H, W, K, R, stride, pad, dil)
EXTRA = [
    (1, 64, 8, 128, 64, 3, 1, 1, 1),     # 8 row tiles: one tile per CTA
    (3, 64, 132, 128, 64, 3, 1, 1, 1),   # 396 row tiles over 132 CTAs: three (odd) tiles per CTA
    (4, 128, 60, 60, 192, 3, 1, 2, 2),   # dilated 3x3, Q = 60: the nine-tap wgrad kernel
    (2, 64, 8, 8, 64, 3, 1, 2, 2),       # dilated 3x3, Q = 8: too narrow for the nine-tap and row kernels, generic wgrad
    # edge shapes
    (2, 64, 9, 1, 64, 3, 1, 1, 1),       # Q = 1: 1 x 128 pixel tiles (TW = 1)
    (2, 64, 10, 2, 64, 3, 1, 1, 1),      # Q = 2
    (2, 64, 9, 3, 64, 3, 1, 1, 1),       # Q = 3: TW = 4, one ragged column per tile
    (3, 64, 7, 5, 128, 3, 1, 1, 1),      # Q = 5: TW = 8
    (2, 64, 12, 20, 64, 3, 1, 0, 1),     # pad 0: P != H, the nine-tap wgrad kernel refuses it
    (1, 64, 6, 300, 64, 1, 2, 0, 1),     # 1x1 stride 2, Q = 150: long rows on the generic wgrad kernel (the row kernel
                                         # serves every long-row R > 1 shape: its groups never span more than 8 pixels)
    (2, 64, 15, 21, 64, 3, 2, 1, 1),     # stride 2, odd H and W: parity views of unequal size
    (2, 64, 15, 21, 128, 1, 2, 0, 1),    # 1x1 stride 2, odd H and W: dgrad parity classes without taps
    (2, 64, 12, 12, 192, 3, 1, 1, 1),    # K = 192: two N tiles, the second half empty
    (2, 128, 12, 20, 64, 3, 1, 1, 1),    # fprop igemm_v2<64, false> (3x3 with streamed weights)
    (2, 1024, 8, 8, 64, 1, 1, 0, 1),     # fprop igemm_v2<64, false> on a 1x1 (16 K-chunks do not fit resident)
    (2, 128, 16, 16, 64, 3, 2, 1, 1),    # dgrad igemm_v2<128, true> on a 3x3 (stride-2 parity classes of <= 4 taps)
]
ALL = list(dict.fromkeys(CASES + FULL_SIZE + EXTRA))
# full-size shapes run dense only (runtime); every other shape also as channel slices
LAYOUTS = [(c, "dense") for c in ALL] + [(c, "sliced") for c in ALL if c not in FULL_SIZE]
_SENT16, _SENT32 = 0x7FA5, 0x7FA5A5A5   # NaN bit patterns no epilogue computes
_OFF = 8                                # channel offset of a slice: 16 bytes of bf16, the least tsb_aligned16 admits


def _ints(shape, lo, hi, g, dev):
    return torch.randint(lo, hi + 1, shape, device=dev, generator=g).double()


def _ceil(v, m):
    return (v + m - 1) // m * m


def _exact_range(terms, max_term, step):
    """a sum of `terms` products of magnitude <= max_term on a grid of `step` never leaves the fp32 integers of that
    grid: every partial sum is exact"""
    assert terms * max_term / step < 2 ** 24, "case leaves the exact fp32 range"


def _slice_in(t, off, cs, fill=float("nan")):
    """[N,C,H,W] values → bf16 channel slice [off, off + C) of a cs-wide NHWC buffer whose other channels hold `fill`:
    returns (buffer, logical NCHW view)"""
    N, C, H, W = t.shape
    buf = torch.full((N, H, W, cs), fill, dtype=torch.bfloat16, device=t.device)
    buf[..., off:off + C] = t.permute(0, 2, 3, 1).to(torch.bfloat16)
    return buf, buf[..., off:off + C].permute(0, 3, 1, 2)


def _sentinel(N, H, W, cs, dtype, dev):
    bits, sent = (torch.int32, _SENT32) if dtype == torch.float32 else (torch.int16, _SENT16)
    return torch.full((N, H, W, cs), sent, dtype=bits, device=dev).view(dtype)


def _untouched(buf, lo, hi):
    """channels outside [lo, hi) of a sentinel buffer still hold the sentinel bits"""
    bits, sent = (torch.int32, _SENT32) if buf.dtype == torch.float32 else (torch.int16, _SENT16)
    b = buf.view(bits)
    return bool((b[..., :lo] == sent).all()) and bool((b[..., hi:] == sent).all())


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _pack(ops, w, want_t=True):
    K, C, R, _ = w.shape
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wb = torch.empty((K, R, R, C), dtype=torch.bfloat16, device=w.device)
    wt = torch.empty((C, R, R, K), dtype=torch.bfloat16, device=w.device) if want_t else None
    ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), ops.ptr(wt), ops.stream())
    return wb, wt


def _wgrad_twice(ops, x, dy, case):
    """two identical weight-gradient calls: the split partial sums are added in a fixed order, so the bits agree"""
    N, C, H, W, K, R, stride, pad, dil = case
    out = []
    for _ in range(2):
        dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=x.device)
        ops.conv_wgrad(x, dy, K, R, stride, pad, dil, dw)
        out.append(dw)
    assert bool(torch.isfinite(out[0]).all()), "wgrad read a NaN pad channel"
    assert _same_bits(out[0], out[1]), "wgrad is not bit-reproducible"


@pytest.mark.parametrize("case,layout", LAYOUTS, ids=[str(c) + ("" if lay == "dense" else "-sliced") for c, lay in LAYOUTS])
def test_conv_exact_small_integers(cuda, case, layout):
    """fprop (fp32 output), dgrad and wgrad against float64 autograd. Sliced: x and dy sit at channel offset 8 of buffers
    24 / 16 channels wider whose other channels are NaN; y and dx land at offset 8 of sentinel buffers, and exactly the
    channels [0, ceil8(K)) of y (zeros past K) and [0, C) of dx change. The weight gradient of random operands is
    computed twice and must repeat bit for bit."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    sliced = layout == "sliced"
    g = torch.Generator(device="cuda").manual_seed(21)
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    # |x|, |gy| <= 2, w in quarters of [-2, 2]
    _exact_range(C * R * R, 4, 0.25)    # fprop
    _exact_range(K * R * R, 4, 0.25)    # dgrad
    _exact_range(N * P * Q, 4, 1)       # wgrad
    x = _ints((N, C, H, W), -2, 2, g, cuda)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    y_ref = F.conv2d(xr, wr, None, stride, pad, dil)
    y_ref.backward(gy)
    wb, wt = _pack(ops, w)
    kst = _ceil(K, 8)

    if sliced:
        xbuf, xd = _slice_in(x, _OFF, C + 24)
        dybuf, gyd = _slice_in(gy, _OFF, K + 16)
        ybuf = _sentinel(N, P, Q, kst + 16, torch.float32, cuda)
        ops.conv_fprop(xd, wb, K, R, stride, pad, dil, out=ybuf[..., _OFF:_OFF + K].permute(0, 3, 1, 2))
        assert torch.equal(ybuf[..., _OFF:_OFF + K], y_ref.permute(0, 2, 3, 1).float()), "fprop differs"
        assert bool((ybuf[..., _OFF + K:_OFF + kst] == 0).all()), "fprop: stored pad channels are not zero"
        assert _untouched(ybuf, _OFF, _OFF + kst), "fprop wrote outside its channels"
        dxbuf = _sentinel(N, H, W, C + 16, torch.bfloat16, cuda)
        ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dxbuf[..., _OFF:_OFF + C].permute(0, 3, 1, 2))
        assert torch.equal(dxbuf[..., _OFF:_OFF + C], xr.grad.permute(0, 2, 3, 1).float().to(torch.bfloat16)), "dgrad differs"
        assert _untouched(dxbuf, _OFF, _OFF + C), "dgrad wrote outside its channels"
    else:
        xd = ops.to_nhwc(x.to(torch.bfloat16))
        gyd = ops.to_nhwc(gy.to(torch.bfloat16))
        y = ops.conv_fprop(xd, wb, K, R, stride, pad, dil, out_dtype=torch.float32)
        assert torch.equal(y, y_ref.float()), "fprop differs"
        dx = ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil)
        assert torch.equal(dx, xr.grad.float().to(torch.bfloat16)), "dgrad differs"

    dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw)
    assert torch.equal(dw.permute(0, 3, 1, 2), wr.grad.float()), "wgrad differs"

    xd.copy_(torch.randn(N, C, H, W, device=cuda, generator=g))
    gyd.copy_(torch.randn(N, K, P, Q, device=cuda, generator=g))
    _wgrad_twice(ops, xd, gyd, case)


def _stats_operands(N, C, H, W, K, R, g, dev):
    """x in {-1, 0, 1} and three ±1 weights per output channel: |y| <= 3"""
    x = _ints((N, C, H, W), -1, 1, g, dev)
    w = torch.zeros((K, R * R * C), device=dev, dtype=torch.float64)
    pos = torch.stack([torch.randperm(R * R * C, device=dev, generator=g)[:3] for _ in range(K)])
    w.scatter_(1, pos, _ints((K, 3), 0, 1, g, dev) * 2 - 1)
    return x, w.view(K, R, R, C).permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", ALL, ids=[str(c) for c in ALL])
def test_conv_statistics_exact(cuda, case):
    """BN Σ / Σ² of a bf16-output launch equal the sums of that output, and repeat bit for bit on random data. Three ±1
    weights per output channel and x in {-1, 0, 1} keep |y| <= 3, so every y, y² and partial sum is a small integer."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(22)
    x, w = _stats_operands(N, C, H, W, K, R, g, cuda)
    wb, _ = _pack(ops, w, want_t=False)
    stats = torch.zeros(2, K, device=cuda)
    xd = ops.to_nhwc(x.to(torch.bfloat16))
    y = ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=stats).double()
    s1, s2 = y.sum(dim=(0, 2, 3)), (y * y).sum(dim=(0, 2, 3))
    _exact_range(y[0, 0].numel() * N, 9, 1)
    assert torch.equal(stats[0].double(), s1), "Σ differs"
    assert torch.equal(stats[1].double(), s2), "Σ² differs"
    _stats_twice(ops, lambda st: ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=st), xd, K, g)


def _stats_twice(ops, run, xd, K, g):
    """the statistics of random data, computed twice: per-CTA partials are added in CTA order, so the bits agree"""
    xd.copy_(torch.randn(xd.shape, device=xd.device, generator=g))
    out = []
    for _ in range(2):
        st = torch.zeros(2, K, device=xd.device)
        run(st)
        out.append(st)
    assert bool(torch.isfinite(out[0]).all()), "statistics are not finite"
    assert _same_bits(out[0], out[1]), "statistics are not bit-reproducible"


# (N, C, H, W, K, R, stride, pad, dil, ycs): one shape per kernel family of the fused inference conv
FUSED = [
    (2, 64, 16, 16, 64, 1, 1, 0, 1, 72),     # 1x1: flat GEMM over all pixels
    (1, 64, 8, 128, 64, 3, 1, 1, 1, 72),     # Q >= 96: row tiles
    (2, 128, 20, 24, 64, 3, 1, 1, 1, 80),    # generic tiles
    (2, 64, 32, 32, 128, 3, 2, 1, 1, 136),   # stride 2
    (2, 64, 16, 16, 64, 3, 1, 2, 2, 72),     # dilation 2
    (2, 128, 16, 16, 19, 1, 1, 0, 1, 32),    # 19-class classifier: 24 channels stored, ycs = 32
]


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


# ------------------------------------------------------------------------------------------------------ epilogue modes
# (K, y channel offset, ycs): one N tile of 64 (K = 8, 19, 64), two of 128 with the second partly (150) or half (192)
# real; K = 19 into the fp32 ocs = 32 buffer of the classifier heads
EPILOGUE = [(8, _OFF, 24), (19, 0, 32), (64, _OFF, 80), (150, _OFF, 168), (192, 0, 200)]


@pytest.mark.parametrize("K,yoff,ycs", EPILOGUE, ids=["K%d" % e[0] for e in EPILOGUE])
def test_conv_fprop_epilogue_exact(cuda, K, yoff, ycs):
    """training fprop (tsb_conv2d_fprop) for bias x {bf16, fp32} output x statistics (bf16 only) on a channel slice with
    NaN pads: y equals float64, channels [K, ceil8(K)) are zeros, nothing else of the sentinel buffer changes, Σ / Σ²
    cover exactly the K real channels. |y| <= 3 + 2 in quarters: y, y² and every partial sum are exact."""
    from torchseg_b200 import ops
    N, C, H, W, R = 2, 128, 12, 20, 3
    g = torch.Generator(device="cuda").manual_seed(30 + K)
    x, w = _stats_operands(N, C, H, W, K, R, g, cuda)
    bias = _ints((K,), -8, 8, g, cuda) / 4
    _exact_range(N * H * W, 25, 1 / 16)
    conv = F.conv2d(x, w, None, 1, 1).permute(0, 2, 3, 1)
    wb, _ = _pack(ops, w, want_t=False)
    _, xd = _slice_in(x, _OFF, C + 24)
    bias_f = bias.float()
    kst = _ceil(K, 8)
    for ydt in (torch.float32, torch.bfloat16):
        for use_bias in (False, True):
            for use_stats in ((False, True) if ydt == torch.bfloat16 else (False,)):
                what = "ydtype %s bias %d stats %d" % (ydt, use_bias, use_stats)
                ybuf = _sentinel(N, H, W, ycs, ydt, cuda)
                stats = torch.zeros(2, K, device=cuda) if use_stats else None
                ops.conv_fprop(xd, wb, K, R, 1, 1, 1, bias=bias_f if use_bias else None, stats=stats,
                               out=ybuf[..., yoff:yoff + K].permute(0, 3, 1, 2))
                ref = conv + (bias if use_bias else 0)
                assert torch.equal(ybuf[..., yoff:yoff + K], ref.to(ydt)), what
                assert bool((ybuf[..., yoff + K:yoff + kst] == 0).all()), what + ": stored pad channels are not zero"
                assert _untouched(ybuf, yoff, yoff + kst), what + ": wrote outside its channels"
                if use_stats:
                    assert torch.equal(stats[0].double(), ref.sum(dim=(0, 1, 2))), what + ": Σ differs"
                    assert torch.equal(stats[1].double(), (ref * ref).sum(dim=(0, 1, 2))), what + ": Σ² differs"
    _stats_twice(ops, lambda st: ops.conv_fprop(xd, wb, K, R, 1, 1, 1, bias=bias_f, stats=st), xd, K, g)


# (N, C, H, W, K, R, stride, pad, dil)
ACCUMULATE = [
    (2, 64, 16, 16, 64, 3, 1, 1, 1),     # stride 1 (GradShare forks of a BasicBlock)
    (2, 64, 15, 21, 128, 3, 2, 1, 1),    # stride 2, 3x3: four parity classes with taps
    (2, 64, 15, 21, 128, 1, 2, 0, 1),    # stride 2, 1x1: three parity classes have no tap and must keep the base
    (2, 128, 16, 16, 64, 1, 1, 0, 1),    # flat 1x1
]


@pytest.mark.parametrize("case", ACCUMULATE, ids=[str(c) for c in ACCUMULATE])
def test_conv_dgrad_accumulate_exact(cuda, case):
    """dgrad with accumulate = 1 adds onto an integer base (dx = base + conv_transpose) bit for bit, and changes no
    channel outside the slice; the same launch without accumulate writes exact zeros where no tap reaches (the odd
    positions of a 1x1 stride-2 conv). The base (multiples of 4 up to 1024, exact in bf16) puts most sums past bf16's 8
    significant bits, so the one rounding of the fp32 sum to bf16 is checked too."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(31)
    _exact_range(K * R * R + 1, 1024, 0.25)
    x = torch.zeros((N, C, H, W), dtype=torch.float64, device=cuda, requires_grad=True)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    base = _ints((N, C, H, W), -256, 256, g, cuda) * 4
    F.conv2d(x, w, None, stride, pad, dil).backward(gy)
    dx_ref = x.grad
    _, wt = _pack(ops, w)
    _, gyd = _slice_in(gy, _OFF, K + 16)
    dxbuf = _sentinel(N, H, W, C + 16, torch.bfloat16, cuda)
    dxbuf[..., _OFF:_OFF + C] = base.permute(0, 2, 3, 1).to(torch.bfloat16)
    dx = dxbuf[..., _OFF:_OFF + C].permute(0, 3, 1, 2)
    ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dx, accumulate=True)
    ref = (base + dx_ref).float().to(torch.bfloat16)
    assert float((ref.double() != base + dx_ref).double().mean()) > 0.1, "case does not exercise the bf16 rounding"
    assert torch.equal(dx, ref), "accumulated dgrad differs"
    assert _untouched(dxbuf, _OFF, _OFF + C), "dgrad wrote outside its channels"
    ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dx)
    assert torch.equal(dx, dx_ref.float().to(torch.bfloat16)), "dgrad differs"
    if stride == 2 and R == 1:
        assert bool((dx[:, :, 1::2, :] == 0).all()) and bool((dx[:, :, :, 1::2] == 0).all()), "tap-less positions not zero"


# (N, C, H, W, K, R, stride, pad, dil, dx channel offset, dxcs): dgrad output widths that are not a multiple of 64
PARTIAL_N = [
    (2, 72, 10, 12, 64, 3, 1, 1, 1, _OFF, 96),       # one 128-wide N tile, 72 columns real
    (2, 200, 10, 12, 128, 1, 1, 0, 1, _OFF, 216),    # two N tiles, 72 columns of the second real
    (1, 3600, 60, 60, 512, 1, 1, 0, 1, 0, 3648),     # PSANet dS = dout · x^T: L = 3600 into the 3648-wide softmax buffer
]


@pytest.mark.parametrize("case", PARTIAL_N, ids=[str(c) for c in PARTIAL_N])
def test_conv_dgrad_partial_n_tile_exact(cuda, case):
    """dgrad with C % 64 != 0 (ncols = C, a partly empty last N tile) writes exactly channels [0, C) of the slice"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil, off, dxcs = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(32)
    _exact_range(K * R * R, 4, 0.25)
    x = torch.zeros((N, C, H, W), dtype=torch.float64, device=cuda, requires_grad=True)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    F.conv2d(x, w, None, stride, pad, dil).backward(gy)
    _, wt = _pack(ops, w)
    _, gyd = _slice_in(gy, 0, K + 64)
    dxbuf = _sentinel(N, H, W, dxcs, torch.bfloat16, cuda)
    ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dxbuf[..., off:off + C].permute(0, 3, 1, 2))
    assert torch.equal(dxbuf[..., off:off + C], x.grad.permute(0, 2, 3, 1).float().to(torch.bfloat16)), "dgrad differs"
    assert _untouched(dxbuf, off, off + C), "dgrad wrote outside its channels"


# geometries of the narrow-K weight gradient: (N, C, H, W, R, stride, pad, dil)
NARROW_GEOM = [
    (2, 128, 16, 16, 1, 1, 0, 1),    # 1x1 classifier head (flat GEMM, generic kernel)
    (2, 64, 12, 20, 3, 1, 1, 1),     # 3x3, Q = 20: nine-tap kernel when K % 8 == 0, else generic
    (1, 64, 6, 200, 3, 2, 1, 1),     # 3x3 stride 2, Q = 100: row kernel
]
NARROW = [g[:4] + (K,) + g[4:] for g in NARROW_GEOM for K in (8, 19, 150, 192)]


@pytest.mark.parametrize("case", NARROW, ids=[str(c) for c in NARROW])
def test_conv_wgrad_narrow_k_exact(cuda, case):
    """wgrad with K < 64 or K % 64 != 0 from a dy buffer 64 channels wider whose pad channels hold NaN (ConvFn runs the
    classifier's K = 19 on dy[:, :19] of a 64-wide buffer): exact, and bit-reproducible on random data"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(33)
    _exact_range(N * P * Q, 4, 1)
    x = _ints((N, C, H, W), -2, 2, g, cuda)
    w = torch.zeros((K, C, R, R), dtype=torch.float64, device=cuda, requires_grad=True)
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    F.conv2d(x, w, None, stride, pad, dil).backward(gy)
    xd = ops.to_nhwc(x.to(torch.bfloat16))
    _, gyd = _slice_in(gy, 0, _ceil(K, 8) + 64)
    dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw)
    assert torch.equal(dw.permute(0, 3, 1, 2), w.grad.float()), "wgrad differs"
    xd.copy_(torch.randn(N, C, H, W, device=cuda, generator=g))
    gyd.copy_(torch.randn(N, K, P, Q, device=cuda, generator=g))
    _wgrad_twice(ops, xd, gyd, case)


# ---------------------------------------------------------------------------------------------------------------- stem
# (R, K, y channel offset, ycs, H, W): K = 8 is the X39 stem; K = 64 at offset 64 of a 128-wide buffer is the second
# stem of StemPairFn; K = 128 is StemPairFn's fused weight gradient; 57 x 75 and 45 x 34 are odd images
STEM = [
    (3, 8, 0, 16, 48, 80),
    (7, 8, 0, 16, 45, 34),
    (3, 64, 0, 72, 57, 75),
    (7, 64, 64, 128, 64, 96),
    (3, 64, 64, 128, 32, 64),
    (7, 128, 0, 136, 48, 80),
]


@pytest.mark.parametrize("R,K,yoff,ycs,H,W", STEM, ids=["R%d-K%d-off%d-%dx%d" % (s[0], s[1], s[2], s[4], s[5]) for s in STEM])
def test_conv_stem_train_exact(cuda, R, K, yoff, ycs, H, W):
    """tsb_conv_stem_fprop with statistics into a channel slice of a sentinel buffer, and tsb_conv_stem_wgrad +
    tsb_unpack_stem_wgrad from a dy slice with NaN pads (dycs > K), against float64 F.conv2d / autograd on the image
    through tsb_pack_image_s2d; statistics and weight gradient repeat bit for bit on random data"""
    from torchseg_b200 import ops
    N = 2
    g = torch.Generator(device="cuda").manual_seed(34 + R + K)
    img, w = _stats_operands(N, 3, H, W, K, R, g, cuda)
    wr = w.clone().requires_grad_(True)
    y_ref = F.conv2d(img, wr, None, 2, (R - 1) // 2)
    P, Q = y_ref.shape[2:]
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    y_ref.backward(gy)
    _exact_range(N * P * Q, 9, 1)
    xs = ops.pack_image_s2d(img.float().contiguous())
    He, We = 2 * P, 2 * Q
    assert tuple(xs.shape) == (N, 16, He // 2, We // 2 + 4)
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wp = torch.empty((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_stem_weight", ops.ptr(wk), K, R, ops.ptr(wp), ops.stream())

    def fprop(stats):
        ybuf = _sentinel(N, P, Q, ycs, torch.bfloat16, cuda)
        ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, He, We, ops.ptr(wp), K, ops.ptr(ybuf[..., yoff:]), ycs,
                 ops.ptr(stats[0]), ops.ptr(stats[1]), *ops.det_ws(), ops.stream())
        return ybuf

    stats = torch.zeros(2, K, device=cuda)
    ybuf = fprop(stats)
    ref = y_ref.detach().permute(0, 2, 3, 1)
    assert torch.equal(ybuf[..., yoff:yoff + K], ref.to(torch.bfloat16)), "stem fprop differs"
    assert _untouched(ybuf, yoff, yoff + K), "stem fprop wrote outside its channels"
    assert torch.equal(stats[0].double(), ref.sum(dim=(0, 1, 2))), "Σ differs"
    assert torch.equal(stats[1].double(), (ref * ref).sum(dim=(0, 1, 2))), "Σ² differs"

    dycs = K + 16
    dybuf, gyd = _slice_in(gy, 0, dycs)

    def wgrad():
        dwp = torch.zeros((K, 4, 64), device=cuda)
        ops.call("tsb_conv_stem_wgrad", ops.ptr(xs), N, He, We, ops.ptr(dybuf), dycs, K, ops.ptr(dwp), *ops.det_ws(),
                 ops.stream())
        return dwp

    dw = torch.zeros((K, R, R, 3), device=cuda)
    ops.call("tsb_unpack_stem_wgrad", ops.ptr(wgrad()), K, R, ops.ptr(dw), ops.stream())
    assert torch.equal(dw.permute(0, 3, 1, 2), wr.grad.float()), "stem wgrad differs"

    xs.copy_(torch.randn(xs.shape, device=cuda, generator=g))
    gyd.copy_(torch.randn(gyd.shape, device=cuda, generator=g))
    s = [torch.zeros(2, K, device=cuda) for _ in range(2)]
    fprop(s[0])
    fprop(s[1])
    assert bool(torch.isfinite(s[0]).all()) and _same_bits(s[0], s[1]), "stem statistics are not bit-reproducible"
    d1, d2 = wgrad(), wgrad()
    assert bool(torch.isfinite(d1).all()) and _same_bits(d1, d2), "stem wgrad is not bit-reproducible"


# --------------------------------------------------------------------------------------------------- dispatch coverage
def _route(case):
    """the kernels a case is meant to run, restated from the host dispatch: fprop / dgrad (conv_v2.cu launch) take
    BN = 64 when the output has <= 64 columns, else 128, and keep the weights resident when ntaps x (GEMM-K / 64) tiles
    of BN x 64 bf16 fit in 112 KiB; dgrad of stride 2 launches one kernel per output parity class (taps of that class
    only). wgrad (conv_igemm.cu) tries the nine-tap kernel (3x3, stride 1, pad == dil <= 8, C % 64, K % 8, tile width
    >= 16 i.e. Q > 8), then the row kernel (R > 1, Q >= 64), else the generic kernel. Returns (fprop set, dgrad set,
    wgrad name, fprop tile mode)."""
    N, C, H, W, K, R, stride, pad, dil = case
    Q = (W + 2 * pad - dil * (R - 1) - 1) // stride + 1
    flat = R == 1 and stride == 1 and pad == 0

    def v2(ncols, ntaps, kchunks):
        bn = 64 if ncols <= 64 else 128
        return "igemm_v2_kernel<%d, %s>" % (bn, "true" if ntaps * kchunks * bn * 128 <= 112 * 1024 else "false")

    fprop = {v2(_ceil(K, 8), R * R, C // 64)}
    if stride == 1:
        dgrad = {v2(C, R * R, K // 64)}
    else:
        dgrad = set()
        for ph in (0, 1):
            for pw in (0, 1):
                if (H - ph + 1) // 2 <= 0 or (W - pw + 1) // 2 <= 0:
                    continue
                nh = sum((ph + pad - r * dil) % 2 == 0 for r in range(R))
                nw = sum((pw + pad - s * dil) % 2 == 0 for s in range(R))
                dgrad.add(v2(C, nh * nw, K // 64))
    if not flat and R == 3 and stride == 1 and pad == dil <= 8 and C % 64 == 0 and K % 8 == 0 and Q > 8:
        wgrad = "wgrad_taps_kernel"
    elif not flat and R > 1 and Q >= 64:
        wgrad = "wgrad_rows_kernel"
    else:
        wgrad = "wgrad_mnmajor_kernel"
    tile = "flat" if flat else ("rows" if Q >= 96 else "generic")
    return fprop, dgrad, wgrad, tile


_KERNEL_RE = re.compile(r"(igemm_v2_kernel<\d+, (?:true|false)>|wgrad_(?:taps|rows|mnmajor)_kernel)")


def _kernels_of(fn):
    """the conv kernels fn launches, by name. In a long process the profiler occasionally returns a trace without any
    of the kernels the library launched inside its window (seen: one full-size case, all three ops, in a whole-suite
    run); such a lost trace is told apart by the library's own launch counter and measured again, at most twice. A
    call that launches nothing still reports nothing."""
    from torch.profiler import ProfilerActivity, profile
    from torchseg_b200 import _lib
    for _ in range(3):
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        got = {m.group(1) for m in (_KERNEL_RE.search(e.name) for e in prof.events()) if m}
        if got or _lib.launch_count() == n0:
            return got
    return got


def test_conv_dispatch_coverage(cuda):
    """every case of the exact tests runs the kernels _route assigns it (seen by torch.profiler), and the table reaches
    all four igemm_v2_kernel<BN, RES> variants and all three wgrad kernels. A retuned threshold that moves a case onto
    another kernel fails here, by name, instead of silently changing what the exact tests cover."""
    from torchseg_b200 import ops
    seen_v2, seen_wg, wrong, table = set(), set(), [], []
    for case in ALL:
        N, C, H, W, K, R, stride, pad, dil = case
        P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
        fprop, dgrad, wgrad, tile = _route(case)
        xd = ops.nhwc_zeros(N, C, H, W, device=cuda)
        gyd = ops.nhwc_zeros(N, K, P, Q, device=cuda)
        wb = torch.zeros((K, R, R, C), dtype=torch.bfloat16, device=cuda)
        wt = torch.zeros((C, R, R, K), dtype=torch.bfloat16, device=cuda)
        dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
        got_f = _kernels_of(lambda: ops.conv_fprop(xd, wb, K, R, stride, pad, dil))
        got_d = _kernels_of(lambda: ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil))
        got_w = _kernels_of(lambda: ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw))
        table.append("%-42s %-7s fprop %-28s dgrad %-58s wgrad %s" % (case, tile, ",".join(sorted(got_f)),
                                                                        ",".join(sorted(got_d)), ",".join(sorted(got_w))))
        for op, want, got in (("fprop", fprop, got_f), ("dgrad", dgrad, got_d), ("wgrad", {wgrad}, got_w)):
            if got != want:
                wrong.append("%s %s: expected %s, ran %s" % (case, op, sorted(want), sorted(got)))
        seen_v2 |= fprop | dgrad
        seen_wg.add(wgrad)
    print("\n" + "\n".join(table))
    assert not wrong, "\n".join(wrong)
    assert seen_v2 == {"igemm_v2_kernel<%d, %s>" % (bn, res) for bn in (64, 128) for res in ("true", "false")}, seen_v2
    assert seen_wg == {"wgrad_taps_kernel", "wgrad_rows_kernel", "wgrad_mnmajor_kernel"}, seen_wg


# -------------------------------------------------------------------------------------------------- entry-point checks
def test_conv_entry_points_refuse_narrow_layouts(cuda):
    """a channel stride below the channel count is refused before any launch (xcs < C for wgrad, ycs < K for fprop and
    the stem, dycs < K for the stem wgrad), not clamped or read across pixels. Every buffer is sized for the full
    channel count, so no call below could reach outside it even if it ran."""
    from torchseg_b200 import ops
    N, C, H, W, K = 1, 64, 8, 8, 64
    x = torch.zeros((N, H, W, C), dtype=torch.bfloat16, device=cuda)
    dy = torch.zeros((N, H, W, K), dtype=torch.bfloat16, device=cuda)
    y = torch.zeros((N, H, W, K), dtype=torch.bfloat16, device=cuda)
    wb = torch.zeros((K, 3, 3, C), dtype=torch.bfloat16, device=cuda)
    dw = torch.zeros((K, 3, 3, C), dtype=torch.float32, device=cuda)
    shp = ops.make_shape(N, H, W, C, K, 3, 1, 1, 1)
    with pytest.raises(RuntimeError, match="tsb_conv2d_wgrad: layout"):
        ops.call("tsb_conv2d_wgrad", ctypes.byref(shp), ops.ptr(x), C - 8, ops.ptr(dy), K, ops.ptr(dw), *ops.det_ws(),
                 ops.stream())
    with pytest.raises(RuntimeError, match="at least K"):
        ops.call("tsb_conv2d_fprop", ctypes.byref(shp), ops.ptr(x), C, ops.ptr(wb), None, ops.ptr(y), 1, K - 8,
                 None, None, None, 0, ops.stream())
    with pytest.raises(RuntimeError, match="at least K"):
        ops.call("tsb_conv2d_fprop_fused", ctypes.byref(shp), ops.ptr(x), C, ops.ptr(wb), None, None, 0, 0, ops.ptr(y),
                 1, K - 8, ops.stream())
    xs = torch.zeros((N, H, W + 4, 16), dtype=torch.bfloat16, device=cuda)    # s2d image of a 2H x 2W input
    wp = torch.zeros((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    dwp = torch.zeros((K, 4, 64), device=cuda)
    with pytest.raises(RuntimeError, match="ycs >= K"):
        ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, 2 * H, 2 * W, ops.ptr(wp), K, ops.ptr(y), K - 8, None, None,
                 *ops.det_ws(), ops.stream())
    with pytest.raises(RuntimeError, match="dycs >= K"):
        ops.call("tsb_conv_stem_wgrad", ops.ptr(xs), N, 2 * H, 2 * W, ops.ptr(dy), K - 8, K, ops.ptr(dwp), *ops.det_ws(),
                 ops.stream())
