"""The ordered slot sum (tsb_det_reduce) bit for bit against a float32 sequential chain in numpy:
out[i] += ((0 + slot[0][i]) + slot[1][i]) + ... in slot order, on both of its kernels (the column kernel for small n,
the grid-wide kernel for large n), and through the entry points whose Σ / Σ² pairs now run as one launch over 2C
outputs. Every slot count from one to the 8 x 132 CTAs of a BatchNorm reduction, strides n and 2n, ±0 and subnormal
slot values, and a non-zero `out` so that the final add is checked too."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NPARTS = [1, 31, 32, 33, 132, 257, 1056]
# 5280 = 8 outputs x 5 x 132 CTAs, the largest n of the column kernel on a 132-SM H100 (nparts > 32); 5288 is past
# it; 36864 is the weight gradient of a 3 x 3, 64 -> 64 convolution
NS = [8, 19, 64, 128, 1024, 5280, 5288, 36864]


def _lib():
    from torchseg_b200 import _lib
    h = _lib.lib()
    h.tsb_det_reduce.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_longlong,
                                 ctypes.c_void_p]
    return h


def _chain(slots, out0):
    """float32 chain in slot order, then added to out0 (numpy keeps subnormals and rounds every add to float32)"""
    s = np.zeros(slots.shape[1:], dtype=np.float32)
    for b in range(slots.shape[0]):
        s = s + slots[b]
    return out0 + s


def _special(t, g):
    """put +0, -0 and subnormals of both signs into a random float32 tensor"""
    flat = t.view(-1)
    k = max(1, flat.numel() // 16)
    for v in (0.0, -0.0, 1e-40, -3e-42, 1.2e-38):
        idx = torch.randint(0, flat.numel(), (k,), device=t.device, generator=g)
        flat[idx] = v
    return t


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("stride_mul", [1, 2])
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("nparts", NPARTS)
def test_det_reduce_bits(cuda, nparts, n, stride_mul):
    h = _lib()
    stride = n * stride_mul
    g = torch.Generator(device=cuda).manual_seed(nparts * 7919 + n * 2 + stride_mul)
    parts = torch.randn(nparts * stride, device=cuda, generator=g) * torch.exp2(
        torch.randint(-20, 20, (nparts * stride,), device=cuda, generator=g).float())
    _special(parts, g)
    out = _special(torch.randn(n, device=cuda, generator=g), g)
    want = _chain(parts.view(nparts, stride)[:, :n].cpu().numpy(), out.cpu().numpy())
    rc = h.tsb_det_reduce(out.data_ptr(), parts.data_ptr(), nparts, n, stride, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, h.tsb_last_error().decode()
    got = out.cpu().numpy()
    assert np.array_equal(_bits(got), _bits(want)), "%d outputs differ" % int((_bits(got) != _bits(want)).sum())


def _stats_check(ws, C, out_a, out_b, a0, b0):
    """out_a / out_b equal the float32 chains over the [slot][2][C] workspace (slots the launch did not write are +0,
    which leaves a chain that started at +0 unchanged)"""
    slots = ws.view(-1, 2, C).cpu().numpy()
    for got, start, half in ((out_a, a0, 0), (out_b, b0, 1)):
        want = _chain(slots[:, half, :], start)
        assert np.array_equal(_bits(got.cpu().numpy()), _bits(want)), "half %d differs" % half


def _outs(C, adjacent, dev, g):
    """the two outputs as the rows of one [2, C] tensor (one merged launch) or as two separate tensors (two launches),
    starting from non-zero values"""
    if adjacent:
        t = torch.randn(2, C, device=dev, generator=g)
        a, b = t[0], t[1]
    else:
        a = torch.randn(C + 64, device=dev, generator=g)[:C]
        b = torch.randn(C + 64, device=dev, generator=g)[64:]
    return a, b, a.cpu().numpy().copy(), b.cpu().numpy().copy()


@pytest.mark.parametrize("adjacent", [True, False], ids=["pair", "apart"])
@pytest.mark.parametrize("C,npix", [(64, 600_000), (512, 40_000)])
def test_bn_stats_sums_its_slots(cuda, C, npix, adjacent):
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C + adjacent)
    x = torch.randn(npix, C, device=cuda, generator=g).to(torch.bfloat16)
    ws = torch.zeros(1100 * 2 * C, device=cuda)
    a, b, a0, b0 = _outs(C, adjacent, cuda, g)
    ops.call("tsb_bn_stats", ops.ptr(x), C, npix, C, ops.ptr(a), ops.ptr(b), ops.ptr(ws), ws.numel(), ops.stream())
    assert int((ws.view(-1, 2, C)[:, 0].abs().sum(1) > 0).sum()) > 32, "too few slots to exercise the chain"
    _stats_check(ws, C, a, b, a0, b0)


@pytest.mark.parametrize("adjacent", [True, False], ids=["pair", "apart"])
@pytest.mark.parametrize("C,npix", [(64, 600_000), (256, 80_000)])
def test_bn_bwd_reduce_sums_its_slots(cuda, C, npix, adjacent):
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(10 + C + adjacent)
    dy = torch.randn(npix, C, device=cuda, generator=g).to(torch.bfloat16)
    x = torch.randn(npix, C, device=cuda, generator=g).to(torch.bfloat16)
    mean = torch.randn(C, device=cuda, generator=g) * 0.1
    invstd = torch.rand(C, device=cuda, generator=g) + 0.5
    ws = torch.zeros(1100 * 2 * C, device=cuda)
    a, b, a0, b0 = _outs(C, adjacent, cuda, g)
    ops.call("tsb_bn_bwd_reduce", ops.ptr(dy), C, None, 0, ops.ptr(x), C, ops.ptr(mean), ops.ptr(invstd), 0, npix, C,
             ops.ptr(a), ops.ptr(b), None, None, ops.ptr(ws), ws.numel(), ops.stream())
    _stats_check(ws, C, a, b, a0, b0)


@pytest.mark.parametrize("adjacent", [True, False], ids=["pair", "apart"])
@pytest.mark.parametrize("K", [64, 128])
def test_conv_fprop_statistics_sum_their_slots(cuda, K, adjacent):
    from torchseg_b200 import ops, _lib
    N, C, H, W, R = 4, 64, 64, 64, 3
    g = torch.Generator(device=cuda).manual_seed(20 + K + adjacent)
    x = torch.randn(N, H, W, C, device=cuda, generator=g).to(torch.bfloat16)
    wk = torch.randn(K, R, R, C, device=cuda, generator=g) * 0.05
    wb = torch.empty(K, R, R, C, dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, R, R, C, ops.ptr(wb), None, ops.stream())
    y = torch.empty(N, H, W, K, dtype=torch.bfloat16, device=cuda)
    shp = ops.make_shape(N, H, W, C, K, R, 1, 1, 1)
    ws = torch.zeros(300 * 2 * K, device=cuda)
    a, b, a0, b0 = _outs(K, adjacent, cuda, g)
    ops.call("tsb_conv2d_fprop", ctypes.byref(shp), ops.ptr(x), C, ops.ptr(wb), None, ops.ptr(y), _lib.BF16, K,
             ops.ptr(a), ops.ptr(b), ops.ptr(ws), ws.numel(), ops.stream())
    _stats_check(ws, K, a, b, a0, b0)
