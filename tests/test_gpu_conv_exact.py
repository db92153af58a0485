"""Bit-exact checks of the wgmma convolution kernels on small-integer operands.

Every product and every fp32 partial sum below is an exactly representable number, so any summation order gives the
same fp32 result and the kernels must match a float64 reference bit for bit. A pipeline stage released to the producer
while its MMAs are still reading it, or an epilogue that reads accumulators of the wrong tile, shows up here as a wrong
value rather than as noise inside a tolerance."""
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
