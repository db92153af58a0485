"""GPU parity tests of the wgmma implicit-GEMM convolution (fprop / dgrad / wgrad / stem) against
F.conv2d autograd in fp32 on bf16-rounded operands. Tolerance 1e-2 of the output scale (bf16 path)."""
import pytest
import torch
import torch.nn.functional as F

from util import rel_err, bf16_round

pytestmark = pytest.mark.gpu

# (N, C, H, W, K, R, stride, pad, dil)
CASES = [
    (2, 64, 32, 32, 64, 3, 1, 1, 1),       # layer1-like
    (2, 64, 32, 32, 128, 3, 2, 1, 1),      # layer2.0.conv1
    (2, 128, 16, 16, 128, 3, 1, 1, 1),
    (1, 256, 20, 28, 256, 3, 1, 2, 2),     # dilated, ragged spatial size (PSP layer3)
    (2, 512, 8, 8, 128, 3, 1, 1, 1),       # ARM conv on a small map
    (2, 64, 32, 32, 128, 1, 2, 0, 1),      # 1x1 stride-2 downsample
    (2, 256, 16, 16, 256, 1, 1, 0, 1),     # FFM 1x1 (flat GEMM path)
    (3, 64, 17, 23, 64, 3, 2, 1, 1),       # odd sizes, stride 2
    (2, 128, 12, 12, 256, 3, 1, 4, 4),     # dilation 4
    (4, 512, 1, 1, 128, 1, 1, 0, 1),       # global-context conv on a 1x1 map
    (1, 64, 6, 160, 64, 3, 1, 1, 1),       # long rows → row tiles (3 taps share one halo load)
    (2, 128, 5, 200, 128, 3, 1, 2, 2),     # row tiles + dilation 2, ragged width
    (1, 64, 7, 260, 128, 3, 2, 1, 1),      # row tiles, stride 2 (parity views), Q = 130
    (1, 64, 3, 300, 64, 3, 1, 4, 4),       # row tiles + dilation 4 (span 8)
    (1, 128, 4, 256, 64, 1, 1, 0, 1),      # 1x1 → flat GEMM, resident weights
    # >= 2 tiles per CTA with streamed weights, odd tails
    (8, 128, 64, 128, 128, 3, 1, 1, 1),    # 512 row tiles over 132 CTAs (3 or 4 each)
    (4, 128, 40, 136, 256, 3, 1, 2, 2),    # two N tiles, dilation 2, ragged width (2 tiles per row)
    (4, 1024, 48, 128, 256, 1, 1, 0, 1),   # 1x1 with streamed weights (flat GEMM), 4 stages
]


def _ref(x, w, stride, pad, dil, gy):
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    y = F.conv2d(xr, wr, None, stride, pad, dil)
    y.backward(gy)
    return y.detach(), xr.grad, wr.grad


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_conv_fprop_dgrad_wgrad(cuda, case):
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator().manual_seed(hash(case) % 1000)
    x = bf16_round(torch.randn(N, C, H, W, generator=g))
    w = bf16_round(torch.randn(K, C, R, R, generator=g) / (C * R * R) ** 0.5)
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    gy = bf16_round(torch.randn(N, K, P, Q, generator=g))
    y_ref, dx_ref, dw_ref = _ref(x, w, stride, pad, dil, gy)

    xd = ops.to_nhwc(x.to(cuda))
    wk = w.to(cuda).permute(0, 2, 3, 1).contiguous()              # KRSC fp32
    wb = torch.empty((K, R, R, C), dtype=torch.bfloat16, device=cuda)
    wt = torch.empty((C, R, R, K), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), ops.ptr(wt), ops.stream())
    stats = torch.zeros(2, K, device=cuda)
    y = ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=stats)
    torch.cuda.synchronize()
    e = rel_err(y, y_ref)
    assert e < 1e-2, "fprop rel err %g" % e
    yb = y.float()
    assert rel_err(stats[0], yb.sum(dim=(0, 2, 3))) < 1e-3
    assert rel_err(stats[1], (yb * yb).sum(dim=(0, 2, 3))) < 1e-3

    gyd = ops.to_nhwc(gy.to(cuda))
    dx = ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil)
    torch.cuda.synchronize()
    e = rel_err(dx, dx_ref)
    assert e < 1e-2, "dgrad rel err %g" % e

    dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw)
    torch.cuda.synchronize()
    e = rel_err(dw.permute(0, 3, 1, 2), dw_ref)
    assert e < 1e-2, "wgrad rel err %g" % e


def test_conv_classifier_fp32_bias(cuda):
    """1x1 classifier 256→19 with bias, fp32 NHWC output with channel stride 32 (head logits)"""
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(1)
    N, C, H, W, K = 2, 256, 16, 16, 19
    x = bf16_round(torch.randn(N, C, H, W, generator=g))
    w = bf16_round(torch.randn(K, C, 1, 1, generator=g) / 16)
    b = torch.randn(K, generator=g)
    y_ref = F.conv2d(x, w, b)
    xd = ops.to_nhwc(x.to(cuda))
    wb = w.to(cuda).permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    y = ops.conv_fprop(xd, wb, K, 1, 1, 0, 1, bias=b.to(cuda), out_dtype=torch.float32, ocs=32)
    assert ops.cs_of(y) == 32
    assert rel_err(y, y_ref) < 1e-2


def test_conv_dgrad_accumulate(cuda):
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(2)
    N, C, H, W, K = 2, 64, 16, 16, 64
    w = bf16_round(torch.randn(K, C, 3, 3, generator=g) / 24)
    gy = bf16_round(torch.randn(N, K, H, W, generator=g))
    base = bf16_round(torch.randn(N, C, H, W, generator=g))
    ref = F.conv_transpose2d(gy, w, None, 1, 1) + base
    wk = w.to(cuda).permute(0, 2, 3, 1).contiguous()
    wt = torch.empty((C, 3, 3, K), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, 3, 3, C, None, ops.ptr(wt), ops.stream())
    out = ops.to_nhwc(base.to(cuda))
    ops.conv_dgrad(ops.to_nhwc(gy.to(cuda)), wt, (N, C, H, W), K, 3, 1, 1, 1, out=out, accumulate=True)
    assert rel_err(out, ref) < 1e-2


@pytest.mark.parametrize("HW,R", [((64, 64), 7), ((32, 96), 7), ((48, 80), 3)])
def test_stem_7x7(cuda, HW, R):
    """7x7/2 (pad 3) and 3x3/2 (pad 1, v1c deep stem) C_in=3 stems through the space-to-depth pack (fprop + wgrad)"""
    from torchseg_b200 import ops
    H, W = HW
    g = torch.Generator().manual_seed(3)
    N, K = 2, 64
    img = torch.randn(N, 3, H, W, generator=g)
    w = bf16_round(torch.randn(K, 3, R, R, generator=g) / 12)
    img_b = bf16_round(img)
    gy = bf16_round(torch.randn(N, K, H // 2, W // 2, generator=g))
    wr = w.clone().requires_grad_(True)
    y_ref = F.conv2d(img_b, wr, None, 2, (R - 1) // 2)
    y_ref.backward(gy)
    xs = ops.pack_image_s2d(img.to(cuda))
    wk = w.to(cuda).permute(0, 2, 3, 1).contiguous()
    wp = torch.empty((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_stem_weight", ops.ptr(wk), K, R, ops.ptr(wp), ops.stream())
    y = ops.nhwc_empty(N, K, H // 2, W // 2)
    stats = torch.zeros(2, K, device=cuda)
    ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, H, W, ops.ptr(wp), K, ops.ptr(y), K, ops.ptr(stats[0]), ops.ptr(stats[1]),
             *ops.det_ws(), ops.stream())
    torch.cuda.synchronize()
    assert rel_err(y, y_ref) < 1e-2
    dwp = torch.zeros((K, 4, 64), device=cuda)
    ops.call("tsb_conv_stem_wgrad", ops.ptr(xs), N, H, W, ops.ptr(ops.to_nhwc(gy.to(cuda))), K, K, ops.ptr(dwp), *ops.det_ws(), ops.stream())
    dw = torch.zeros((K, R, R, 3), device=cuda)
    ops.call("tsb_unpack_stem_wgrad", ops.ptr(dwp), K, R, ops.ptr(dw), ops.stream())
    torch.cuda.synchronize()
    assert rel_err(dw.permute(0, 3, 1, 2), wr.grad) < 1e-2


def test_conv_full_size_linearity(cuda):
    """BASELINE-size layer (16 x 64 x 256 x 256, 3x3): size-independent property conv(a)+conv(b) == conv(a+b)
    on exactly representable inputs, and agreement with cuDNN on a random crop of the output."""
    from torchseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    N, C, H, W, K = 16, 64, 256, 256, 64
    a = torch.randint(-4, 5, (N, H, W, C), device=cuda, generator=g).to(torch.bfloat16).permute(0, 3, 1, 2)
    b = torch.randint(-4, 5, (N, H, W, C), device=cuda, generator=g).to(torch.bfloat16).permute(0, 3, 1, 2)
    w = (torch.randint(-2, 3, (K, 3, 3, C), device=cuda, generator=g).float() / 4)
    wb = w.to(torch.bfloat16)
    f32 = torch.float32
    ya = ops.conv_fprop(a, wb, K, 3, 1, 1, 1, out_dtype=f32)
    yb = ops.conv_fprop(b, wb, K, 3, 1, 1, 1, out_dtype=f32)
    yab = ops.conv_fprop((a + b), wb, K, 3, 1, 1, 1, out_dtype=f32)
    assert torch.equal(ya + yb, yab)  # all partial sums are small integers / 4: exact in fp32
    ref = F.conv2d(a[:2].float(), w.permute(0, 3, 1, 2), None, 1, 1)
    assert torch.equal(ya[:2], ref)


# BASELINE.json configs[1] layer shapes (batch 16 @ 1024 x 1024 input): the tile choices that only exist at this size —
# row tiles, persistent CTAs with resident / streamed weights, the nine-tap wgrad kernel, stride-2 parity views
FULL_SIZE = [
    (16, 64, 256, 256, 64, 3, 1, 1, 1),     # layer1 (resident weights, row tiles; nine-tap wgrad, K = 64)
    (16, 64, 256, 256, 128, 3, 2, 1, 1),    # layer2.0.conv1 (stride 2)
    (16, 128, 128, 128, 128, 3, 1, 1, 1),   # layer2 (streamed weights)
    (16, 256, 64, 64, 256, 3, 1, 1, 1),     # layer3
    (16, 512, 32, 32, 512, 3, 1, 1, 1),     # layer4 (TW = 32, TH = 2 tiles in the nine-tap wgrad)
    (16, 128, 128, 128, 256, 3, 1, 1, 1),   # aux head 3x3
    (16, 256, 128, 128, 256, 1, 1, 0, 1),   # FFM 1x1 (flat GEMM)
    (16, 512, 32, 32, 128, 3, 1, 1, 1),     # ARM 3x3
]


@pytest.mark.parametrize("case", FULL_SIZE, ids=[str(c) for c in FULL_SIZE])
def test_conv_full_size_vs_cudnn(cuda, case):
    """fprop / dgrad / wgrad of the BASELINE-size layers against cuDNN in strict fp32 on the same bf16-rounded operands
    (computed on the GPU). Tolerance 1e-2 of the output scale (bf16 output rounding; fp32 accumulation both sides)."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(11)
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        x = torch.randn(N, C, H, W, device=cuda, generator=g).to(torch.bfloat16)
        w = (torch.randn(K, C, R, R, device=cuda, generator=g) / (C * R * R) ** 0.5).to(torch.bfloat16)
        P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
        gy = torch.randn(N, K, P, Q, device=cuda, generator=g).to(torch.bfloat16)
        xr = x.float().requires_grad_(True)
        wr = w.float().requires_grad_(True)
        y_ref = F.conv2d(xr, wr, None, stride, pad, dil)
        y_ref.backward(gy.float())
        xd = ops.to_nhwc(x)
        wk = w.float().permute(0, 2, 3, 1).contiguous()
        wb = torch.empty((K, R, R, C), dtype=torch.bfloat16, device=cuda)
        wt = torch.empty((C, R, R, K), dtype=torch.bfloat16, device=cuda)
        ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), ops.ptr(wt), ops.stream())
        stats = torch.zeros(2, K, device=cuda)
        y = ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=stats)
        assert rel_err(y, y_ref) < 1e-2
        yb = y.float()
        assert rel_err(stats[0], yb.sum(dim=(0, 2, 3))) < 1e-3 and rel_err(stats[1], (yb * yb).sum(dim=(0, 2, 3))) < 1e-3
        gyd = ops.to_nhwc(gy)
        dx = ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil)
        assert rel_err(dx, xr.grad) < 1e-2
        dw = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
        ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, dw)
        e = rel_err(dw.permute(0, 3, 1, 2), wr.grad)
        assert e < 2e-3, "wgrad rel err %g (fp32 accumulation of bf16 products: only the summation order differs)" % e
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("HW,R", [((57, 75), 3), ((45, 34), 7)])
def test_stem_odd_image_size(cuda, HW, R):
    """odd input sizes (BASELINE configs[2] 713, configs[4] 473): the space-to-depth pack pads one zero row / column, which
    is the stem's own zero padding — output identical to F.conv2d on the odd image"""
    from torchseg_b200 import ops
    H, W = HW
    g = torch.Generator().manual_seed(13)
    N, K = 2, 64
    img = torch.randn(N, 3, H, W, generator=g)
    w = bf16_round(torch.randn(K, 3, R, R, generator=g) / 12)
    y_ref = F.conv2d(bf16_round(img), w, None, 2, (R - 1) // 2)
    xs = ops.pack_image_s2d(img.to(cuda))
    He, We = H + (H & 1), W + (W & 1)
    assert tuple(xs.shape) == (N, 16, He // 2, We // 2 + 4) and tuple(y_ref.shape[2:]) == (He // 2, We // 2)
    wk = w.to(cuda).permute(0, 2, 3, 1).contiguous()
    wp = torch.empty((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_stem_weight", ops.ptr(wk), K, R, ops.ptr(wp), ops.stream())
    y = ops.nhwc_empty(N, K, He // 2, We // 2)
    ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, He, We, ops.ptr(wp), K, ops.ptr(y), K, None, None, *ops.det_ws(), ops.stream())
    torch.cuda.synchronize()
    assert rel_err(y, y_ref) < 1e-2


@pytest.mark.parametrize("case", [(2, 64, 32, 32, 64, 3, 1, 1, 1), (1, 64, 7, 260, 128, 3, 2, 1, 1),
                                  (2, 256, 16, 16, 256, 1, 1, 0, 1)], ids=["taps", "rows", "generic"])
def test_wgrad_without_workspace_adds_in_place(cuda, case):
    """with no reduction workspace the weight gradient runs as one pixel split that adds straight into dW. On integer
    operands (|x|, |dy| <= 2, an integer base: every partial sum is an exact fp32 integer) it equals the split path and
    float64 exactly, and it accumulates onto what dW already holds"""
    import ctypes
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(14)
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    assert (N * P * Q * 4 + 64) < 2 ** 24
    x = torch.randint(-2, 3, (N, C, H, W), device=cuda, generator=g).double()
    gy = torch.randint(-2, 3, (N, K, P, Q), device=cuda, generator=g).double()
    w = torch.zeros((K, C, R, R), dtype=torch.float64, device=cuda, requires_grad=True)
    F.conv2d(x, w, None, stride, pad, dil).backward(gy)
    xd, gyd = ops.to_nhwc(x), ops.to_nhwc(gy)
    ref = torch.zeros((K, R, R, C), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(xd, gyd, K, R, stride, pad, dil, ref)
    assert torch.equal(ref.permute(0, 3, 1, 2), w.grad.float()), "split wgrad differs"
    base = torch.randint(-64, 65, (K, R, R, C), device=cuda, generator=g).float()
    dw = base.clone()
    shp = ops.make_shape(N, H, W, C, K, R, stride, pad, dil)
    ops.call("tsb_conv2d_wgrad", ctypes.byref(shp), ops.ptr(xd), ops.cs_of(xd), ops.ptr(gyd), ops.cs_of(gyd), ops.ptr(dw),
             None, 0, ops.stream())
    assert torch.equal(dw, base + ref), "in-place wgrad differs"


def test_conv_statistics_need_a_workspace(cuda):
    """per-CTA statistics without a workspace are refused, not summed into a buffer the caller does not own"""
    import ctypes
    from torchseg_b200 import ops
    N, C, H, W, K = 1, 64, 8, 8, 64
    x = ops.to_nhwc(torch.randn(N, C, H, W, device=cuda))
    wb = torch.zeros((K, 3, 3, C), dtype=torch.bfloat16, device=cuda)
    y = ops.nhwc_empty(N, K, H, W)
    stats = torch.zeros(2, K, device=cuda)
    shp = ops.make_shape(N, H, W, C, K, 3, 1, 1, 1)
    with pytest.raises(RuntimeError, match="workspace"):
        ops.call("tsb_conv2d_fprop", ctypes.byref(shp), ops.ptr(x), ops.cs_of(x), ops.ptr(wb), None, ops.ptr(y), 1, K,
                 ops.ptr(stats[0]), ops.ptr(stats[1]), None, 0, ops.stream())
