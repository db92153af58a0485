"""Bit-exact checks of the 64-column wgmma convolutions (igemm_v2_kernel<64, *>) at the edges of their tiling.

These kernels put the pixels on the wgmma N side: a CTA work unit is a pair of its 128-pixel m-tiles (CTA b of G takes
the tiles b, b + G, b + 2G, ...), one per consumer warpgroup, and the epilogue transposes the accumulators to
pixel-major rows through shared memory. The cases below put the last pair half-empty (odd tile counts per CTA), let a
pair straddle two images or end the batch, run the
stride-2 dgrad parity classes of odd maps, the K = 19 fp32 logits at channel stride 32, the accumulating dgrad, channel
slices with NaN input pads and sentinel output pads, and the stem at an odd output size. Operands are small integers,
so every result is exact and must match float64 bit for bit (the method of test_gpu_conv_exact.py); every case also
asserts that it ran a BN = 64 kernel and no other."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv_exact import (_OFF, _ceil, _exact_range, _ints, _kernels_of, _pack, _same_bits, _sentinel,
                                 _slice_in, _stats_operands, _untouched)

pytestmark = pytest.mark.gpu

_N64 = {"igemm_v2_kernel<64, true>", "igemm_v2_kernel<64, false>"}


def _run_n64(fn):
    """run fn under the profiler: it must launch 64-column kernels only"""
    got = _kernels_of(fn)
    assert got and got <= _N64, "expected igemm_v2_kernel<64, *>, ran %s" % sorted(got)


def _m_tiles(N, P, Q, flat):
    """128-pixel m-tiles of a launch, restated from the host tiling: flat GEMM, row tiles (Q >= 96) or TW x TH tiles"""
    if flat:
        return (N * P * Q + 127) // 128
    if Q >= 96:
        return N * P * ((Q + 127) // 128)
    tw = min(16, 1 << (Q - 1).bit_length())
    th = 128 // tw
    return N * ((P + th - 1) // th) * ((Q + tw - 1) // tw)


# (N, C, H, W, K, R, stride, pad, dil): fprop and dgrad both have <= 64 output columns
FPROP = [
    (1, 64, 3, 128, 64, 3, 1, 1, 1),     # row tiles, 3 m-tiles: one per CTA, every pair half-empty
    (3, 64, 5, 100, 64, 3, 1, 1, 1),     # row tiles, 5 per image, 15 CTAs
    (2, 64, 140, 128, 64, 3, 1, 1, 1),   # 280 row tiles over 132 CTAs: pairs (b, b + 132) straddle the two images,
                                         # CTAs 0-15 end on a half-empty pair
    (2, 64, 3, 200, 64, 3, 1, 1, 1),     # row tiles of 128 + 72 pixels: ragged second tile of every row
    (1, 64, 17, 45, 64, 3, 1, 1, 1),     # generic 16 x 8 tiles, 9 m-tiles
    (1, 128, 7, 37, 64, 1, 1, 0, 1),     # flat 1x1 over 259 pixels: 3 m-tiles, the last ragged
    (1, 192, 19, 13, 64, 3, 1, 1, 1),    # streamed weights (9 taps x 3 K-chunks), 3 generic m-tiles
    (1, 64, 15, 21, 64, 3, 2, 1, 1),     # stride 2 fprop (parity views), 8 x 11 output: one m-tile
    (3, 64, 7, 9, 40, 3, 1, 2, 2),       # K = 40: part of the tile's channels real, dilation 2, 3 m-tiles
]


@pytest.mark.parametrize("case", FPROP, ids=[str(c) for c in FPROP])
def test_n64_fprop_exact(cuda, case):
    """fprop into channel slices of sentinel buffers from an x slice with NaN pads: bf16 output with BN statistics and
    fp32 output with a bias, both equal float64; nothing outside channels [0, ceil8(K)) of the slice changes"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(40)
    x, w = _stats_operands(N, C, H, W, K, R, g, cuda)
    bias = _ints((K,), -8, 8, g, cuda) / 4
    _exact_range(N * P * Q, 25, 1 / 16)
    conv = F.conv2d(x, w, None, stride, pad, dil).permute(0, 2, 3, 1)
    wb, _ = _pack(ops, w, want_t=False)
    _, xd = _slice_in(x, _OFF, C + 24)
    kst = _ceil(K, 8)
    ycs = kst + 16

    y16 = _sentinel(N, P, Q, ycs, torch.bfloat16, cuda)
    stats = torch.zeros(2, K, device=cuda)
    _run_n64(lambda: ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=stats,
                                    out=y16[..., _OFF:_OFF + K].permute(0, 3, 1, 2)))
    assert torch.equal(y16[..., _OFF:_OFF + K], conv.to(torch.bfloat16)), "bf16 fprop differs"
    assert bool((y16[..., _OFF + K:_OFF + kst] == 0).all()), "stored pad channels are not zero"
    assert _untouched(y16, _OFF, _OFF + kst), "bf16 fprop wrote outside its channels"
    assert torch.equal(stats[0].double(), conv.sum(dim=(0, 1, 2))), "Σ differs"
    assert torch.equal(stats[1].double(), (conv * conv).sum(dim=(0, 1, 2))), "Σ² differs"

    y32 = _sentinel(N, P, Q, ycs, torch.float32, cuda)
    _run_n64(lambda: ops.conv_fprop(xd, wb, K, R, stride, pad, dil, bias=bias.float(),
                                    out=y32[..., _OFF:_OFF + K].permute(0, 3, 1, 2)))
    assert torch.equal(y32[..., _OFF:_OFF + K], (conv + bias).float()), "fp32 fprop differs"
    assert _untouched(y32, _OFF, _OFF + kst), "fp32 fprop wrote outside its channels"


def test_n64_classifier_logits_exact(cuda):
    """the 19-class classifier: 1x1 with bias into fp32 logits at channel stride 32, over an odd number of m-tiles"""
    from torchseg_b200 import ops
    N, C, H, W, K = 1, 256, 11, 33, 19
    assert _m_tiles(N, H, W, True) % 2 == 1
    g = torch.Generator(device="cuda").manual_seed(41)
    x = _ints((N, C, H, W), -2, 2, g, cuda)
    w = _ints((K, C, 1, 1), -2, 2, g, cuda) / 4
    bias = _ints((K,), -8, 8, g, cuda) / 4
    _exact_range(C + 1, 4, 0.25)
    ref = (F.conv2d(x, w, None) + bias.view(1, K, 1, 1)).permute(0, 2, 3, 1)
    wb, _ = _pack(ops, w, want_t=False)
    xd = ops.to_nhwc(x.to(torch.bfloat16))
    y = _sentinel(N, H, W, 32, torch.float32, cuda)
    _run_n64(lambda: ops.conv_fprop(xd, wb, K, 1, 1, 0, 1, bias=bias.float(), out=y[..., :K].permute(0, 3, 1, 2)))
    assert torch.equal(y[..., :K], ref.float()), "logits differ"
    assert bool((y[..., K:24] == 0).all()), "stored pad channels are not zero"
    assert _untouched(y, 0, 24), "wrote past K_store"


# (N, C, H, W, K, R, stride, pad, dil): dgrad into C = 64 channels
DGRAD = [
    (1, 64, 3, 128, 64, 3, 1, 1, 1),     # row tiles, odd m-tile count
    (3, 64, 5, 100, 128, 3, 1, 1, 1),    # 15 row tiles; two K-chunks
    (2, 64, 140, 128, 64, 3, 1, 1, 1),   # 280 row tiles: pairs straddle the images, CTAs 0-15 end half-empty
    (2, 64, 15, 21, 64, 3, 2, 1, 1),     # stride 2, odd H and W: four parity classes of unequal size
    (1, 64, 13, 19, 128, 1, 2, 0, 1),    # 1x1 stride 2: three parity classes have no tap
    (2, 64, 9, 260, 128, 3, 2, 1, 1),    # stride 2 with row tiles in the parity classes (Wl = 130)
    (1, 64, 7, 37, 384, 1, 1, 0, 1),     # flat 1x1, six K-chunks, 259 pixels
]


@pytest.mark.parametrize("case", DGRAD, ids=[str(c) for c in DGRAD])
def test_n64_dgrad_exact(cuda, case):
    """dgrad from a dy slice with NaN pads into a dx slice of a sentinel buffer, plain and accumulating onto an integer
    base, against float64 autograd; the accumulating launch adds the base before the one rounding to bf16"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(42)
    _exact_range(K * R * R + 1, 1024, 0.25)
    x = torch.zeros((N, C, H, W), dtype=torch.float64, device=cuda, requires_grad=True)
    w = _ints((K, C, R, R), -2, 2, g, cuda) / 4
    gy = _ints((N, K, P, Q), -2, 2, g, cuda)
    F.conv2d(x, w, None, stride, pad, dil).backward(gy)
    dx_ref = x.grad.permute(0, 2, 3, 1)
    _, wt = _pack(ops, w)
    _, gyd = _slice_in(gy, _OFF, K + 16)
    dxbuf = _sentinel(N, H, W, C + 16, torch.bfloat16, cuda)
    dx = dxbuf[..., _OFF:_OFF + C].permute(0, 3, 1, 2)
    _run_n64(lambda: ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dx))
    assert torch.equal(dxbuf[..., _OFF:_OFF + C], dx_ref.float().to(torch.bfloat16)), "dgrad differs"
    assert _untouched(dxbuf, _OFF, _OFF + C), "dgrad wrote outside its channels"

    base = _ints((N, H, W, C), -256, 256, g, cuda) * 4
    dxbuf[..., _OFF:_OFF + C] = base.to(torch.bfloat16)
    _run_n64(lambda: ops.conv_dgrad(gyd, wt, (N, C, H, W), K, R, stride, pad, dil, out=dx, accumulate=True))
    assert torch.equal(dxbuf[..., _OFF:_OFF + C], (base + dx_ref).float().to(torch.bfloat16)), "accumulated dgrad differs"
    assert _untouched(dxbuf, _OFF, _OFF + C), "accumulating dgrad wrote outside its channels"


@pytest.mark.parametrize("R", [7, 3])
def test_n64_stem_odd_exact(cuda, R):
    """the stem (tsb_conv_stem_fprop) at a 70 x 90 image, a 35 x 45 output of an odd number of m-tiles, into a channel
    slice of a sentinel buffer, with BN statistics"""
    from torchseg_b200 import ops
    N, H, W, K, yoff, ycs = 1, 70, 90, 64, _OFF, 80
    g = torch.Generator(device="cuda").manual_seed(43 + R)
    img, w = _stats_operands(N, 3, H, W, K, R, g, cuda)
    ref = F.conv2d(img, w, None, 2, (R - 1) // 2).permute(0, 2, 3, 1)
    P, Q = ref.shape[1:3]
    assert _m_tiles(N, P, Q, False) % 2 == 1
    _exact_range(N * P * Q, 9, 1)
    xs = ops.pack_image_s2d(img.float().contiguous())
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wp = torch.empty((K, 4, 4, 16), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_stem_weight", ops.ptr(wk), K, R, ops.ptr(wp), ops.stream())
    y = _sentinel(N, P, Q, ycs, torch.bfloat16, cuda)
    stats = torch.zeros(2, K, device=cuda)
    _run_n64(lambda: ops.call("tsb_conv_stem_fprop", ops.ptr(xs), N, 2 * P, 2 * Q, ops.ptr(wp), K,
                              ops.ptr(y[..., yoff:]), ycs, ops.ptr(stats[0]), ops.ptr(stats[1]), *ops.det_ws(),
                              ops.stream()))
    assert torch.equal(y[..., yoff:yoff + K], ref.to(torch.bfloat16)), "stem fprop differs"
    assert _untouched(y, yoff, yoff + K), "stem fprop wrote outside its channels"
    assert torch.equal(stats[0].double(), ref.sum(dim=(0, 1, 2))), "Σ differs"
    assert torch.equal(stats[1].double(), (ref * ref).sum(dim=(0, 1, 2))), "Σ² differs"


@pytest.mark.parametrize("case", [FPROP[2], FPROP[6], FPROP[7]], ids=str)
def test_n64_repeatable(cuda, case):
    """random data: two identical fprop launches with statistics, and two accumulating dgrad launches onto the same
    base, give the same bits (the statistics are summed in a fixed order, with no float atomics)"""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    P, Q = ops.conv_out_size(H, R, stride, pad, dil), ops.conv_out_size(W, R, stride, pad, dil)
    g = torch.Generator(device="cuda").manual_seed(44)
    xd = ops.to_nhwc(torch.randn(N, C, H, W, device=cuda, generator=g).to(torch.bfloat16))
    w = torch.randn(K, C, R, R, device=cuda, generator=g, dtype=torch.float64) / (C * R * R) ** 0.5
    wb, _ = _pack(ops, w, want_t=False)
    ys, sts = [], []
    for _ in range(2):
        st = torch.zeros(2, K, device=cuda)
        ys.append(ops.conv_fprop(xd, wb, K, R, stride, pad, dil, stats=st))
        sts.append(st)
    assert bool(torch.isfinite(sts[0]).all()), "statistics are not finite"
    assert torch.equal(ys[0].view(torch.int16), ys[1].view(torch.int16)), "fprop output is not bit-reproducible"
    assert _same_bits(sts[0], sts[1]), "statistics are not bit-reproducible"

    Kd = 128
    wd = torch.randn(Kd, C, R, R, device=cuda, generator=g, dtype=torch.float64) / (Kd * R * R) ** 0.5
    _, wt = _pack(ops, wd)
    gyd = ops.to_nhwc(torch.randn(N, Kd, P, Q, device=cuda, generator=g).to(torch.bfloat16))
    base = ops.to_nhwc(torch.randn(N, C, H, W, device=cuda, generator=g).to(torch.bfloat16))
    dxs = []
    for _ in range(2):
        dx = base.clone()
        ops.conv_dgrad(gyd, wt, (N, C, H, W), Kd, R, stride, pad, dil, out=dx, accumulate=True)
        dxs.append(dx)
    assert torch.equal(dxs[0].view(torch.int16), dxs[1].view(torch.int16)), "dgrad is not bit-reproducible"


@pytest.mark.parametrize("case", [FPROP[2], FPROP[4], FPROP[6]], ids=str)
def test_n64_same_order_as_n128(cuda, case):
    """random data: a 64-column launch and a 72-column launch (BN = 128) whose first 64 filters are the same give the
    same bits for those 64 output channels and their Σ / Σ². Both tile widths give a CTA the same m-tiles and sum
    every channel in the same order, so the statistics do not depend on which kernel ran."""
    from torchseg_b200 import ops
    N, C, H, W, K, R, stride, pad, dil = case
    g = torch.Generator(device="cuda").manual_seed(45)
    xd = ops.to_nhwc(torch.randn(N, C, H, W, device=cuda, generator=g).to(torch.bfloat16))
    w = torch.randn(72, C, R, R, device=cuda, generator=g, dtype=torch.float64) / (C * R * R) ** 0.5
    out = []
    for k, kernels in ((64, _N64), (72, {"igemm_v2_kernel<128, true>", "igemm_v2_kernel<128, false>"})):
        wb, _ = _pack(ops, w[:k], want_t=False)
        st = torch.zeros(2, k, device=cuda)
        box = []
        got = _kernels_of(lambda: box.append(ops.conv_fprop(xd, wb, k, R, stride, pad, dil, stats=st)))
        assert got and got <= kernels, sorted(got)
        out.append((box[0][:, :64].contiguous(), st[:, :64].contiguous()))
    assert torch.equal(out[0][0].view(torch.int16), out[1][0].view(torch.int16)), "outputs differ"
    assert _same_bits(out[0][1], out[1][1]), "statistics differ"
