"""Exact checks of the memory-bound NHWC kernels (resize_pool.cu, bn.cu, pack_opt.cu, psa.cu) through the C ABI.

Rules used throughout:
- Operands are small integers and dyadic scales, so every fp32 product and partial sum is exact and the result must
  equal the float64 reference rounded to the output dtype (torch.equal). Where an op cannot be exact (expf in the
  soft-max, __expf in the sigmoid, a non-dyadic bilinear weight), every element must lie within 1 ulp of the output
  dtype around the float64 reference.
- Every activation is a channel slice [8, 8 + C) of a wider buffer. Input pad channels hold NaN, so a read of them
  poisons the result; output pad channels hold a NaN bit pattern that must come back bit-identical; regions a kernel
  must write as zeros are pre-filled with NaN.
- The grid-stride (VecWalk) kernels run at least one shape that takes three or more trips of the grid and does not
  end on an even trip, so VecWalk::next() and the kU = 2 tail of the BN kernels run.
- Channel counts C8 = C / 8 in {1, 3, 12, 48, 256, 257, 512} reach the hoisted and non-hoisted parameter paths, one
  pixel lane per channel group, and a second pass over channel groups.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
_BITS = {BF: torch.int16, F32: torch.int32}
SENT = {BF: 0x7FA5, F32: 0x7FA5A5A5}   # NaN bit patterns no kernel computes
OFF = 8                                # channel offset of every slice (16 bytes of bf16, 32 of fp32)
C8S = [1, 3, 12, 48, 256, 257, 512]


def _tsb(dt):
    return 1 if dt == BF else 0


def _trip():
    """16-byte vectors one trip of a tsb_grid_for(., 256, 8) grid covers"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256


def _multi_trip(per):
    """smallest n with n * per >= 3 trips and n * per not a whole number of double trips (the kU = 2 tail runs)"""
    T = _trip()
    n = -(-3 * T // per)
    while (n * per) % (2 * T) == 0:
        n += 1
    return n


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, tuple(shape), generator=g, device="cuda").double()


def _pick(shape, values, g):
    v = torch.tensor(values, dtype=torch.float64, device="cuda")
    return v[torch.randint(0, len(values), tuple(shape), generator=g, device="cuda")]


class Slab:
    """channels [OFF, OFF + C) of a buffer [*pix, cs]; the rest is NaN (inputs) or the sentinel pattern (outputs)"""

    def __init__(self, pix, C, cs, dtype, vals=None, out=False):
        assert cs >= OFF + C, "the slice must fit the channel stride"
        shape = tuple(pix) + (cs,)
        if out:
            self.buf = torch.full(shape, SENT[dtype], dtype=_BITS[dtype], device="cuda").view(dtype)
        else:
            self.buf = torch.full(shape, float("nan"), dtype=dtype, device="cuda")
        self.C, self.cs, self.dtype = C, cs, dtype
        if vals is not None:
            self.buf[..., OFF:OFF + C] = vals.to(dtype)

    @property
    def ptr(self):
        return self.buf.data_ptr() + OFF * self.buf.element_size()

    @property
    def v(self):
        return self.buf[..., OFF:OFF + self.C]

    def assert_pad(self, what, upto=None):
        """channels outside [OFF, OFF + upto) still hold the sentinel bits"""
        end = OFF + (self.C if upto is None else upto)
        bits = self.buf.view(_BITS[self.dtype])
        assert bool((bits[..., :OFF] == SENT[self.dtype]).all()), "%s: wrote below the channel slice" % what
        assert bool((bits[..., end:] == SENT[self.dtype]).all()), "%s: wrote past the channel slice" % what


def _eq(out, ref, what):
    """out equals the float64 reference rounded to out's dtype, bit for bit"""
    want = ref.to(out.dtype)
    if not torch.equal(out, want):
        bad = (out.double() != want.double()) | torch.isnan(out)
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %s want %s" % (
            what, int(bad.sum()), out.numel(), idx, [float(out[tuple(i)]) for i in idx],
            [float(want[tuple(i)]) for i in idx]))


def _ulp(ref, dtype):
    """spacing of `dtype` at |ref| (ref float64): 2^(e - p) for |ref| in [2^(e-1), 2^e), p significand bits"""
    p = 8 if dtype == BF else 24
    _, e = torch.frexp(ref.abs())
    u = torch.ldexp(torch.ones_like(ref), e - p)
    return torch.where(ref == 0, torch.full_like(ref, 2.0 ** (-126 - p + 1)), u)


def _ulp1(out, ref, what):
    err = (out.double() - ref).abs()
    bad = ~(err <= _ulp(ref, out.dtype))
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError("%s: %d elements further than 1 ulp, first at %s: got %s want %s" % (
            what, int(bad.sum()), idx, [float(out[tuple(i)]) for i in idx], [float(ref[tuple(i)]) for i in idx]))


def _call(name, *args):
    from torchseg_b200 import ops
    ops.call(name, *args, ops.stream())


def _ws():
    from torchseg_b200 import ops
    return ops.det_ws()


# ------------------------------------------------------------------------------------------------ bilinear resize
def _lerp_matrix(n_in, n_out):
    """[n_out, n_in] float64 matrix of the kernel's fp32 lerp weights (area_scale / make_lerp in resize_pool.cu)"""
    if n_out > 1:
        sc = torch.tensor(float(n_in - 1), dtype=F32) / torch.tensor(float(n_out - 1), dtype=F32)
    else:
        sc = torch.tensor(0.0, dtype=F32)
    src = sc * torch.arange(n_out, dtype=F32)
    i0 = src.to(torch.int64).clamp(max=n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = src - i0.to(F32)
    l0 = torch.tensor(1.0, dtype=F32) - l1
    M = torch.zeros(n_out, n_in, dtype=torch.float64)
    r = torch.arange(n_out)
    M.index_put_((r, i0), l0.double(), accumulate=True)
    M.index_put_((r, i1), l1.double(), accumulate=True)
    return M.cuda()


def _dyadic(n_in, n_out):
    """(n_in - 1) / (n_out - 1) a power of two (or a 1-pixel side): every weight is exact"""
    if n_in == 1 or n_out == 1:
        return True
    num, den = n_in - 1, n_out - 1
    while num % 2 == 0 and den % 2 == 0:
        num, den = num // 2, den // 2
    return (num & (num - 1)) == 0 and (den & (den - 1)) == 0


def _bilinear_fwd_cases():
    pairs = [(BF, BF), (BF, F32), (F32, BF), (F32, F32)]
    out = []
    for it, ot in pairs:
        out.append((2, 24, 9, 9, 33, 33, it, ot, 40, 32))       # x4 up
        out.append((1, 16, 17, 17, 129, 129, it, ot, 24, 80))   # x8 up
        out.append((2, 32, 33, 33, 17, 17, it, ot, 48, 40))     # down by 2
        out.append((2, 64, 1, 1, 7, 9, it, ot, 72, 128))        # 1x1 -> HxW
        out.append((2, 19, 9, 9, 33, 33, it, ot, 32, 27))       # C % 8 != 0: scalar path
    for it in (BF, F32):   # non-dyadic weights: 1 ulp of a bf16 output
        out.append((2, 16, 16, 20, 128, 160, it, BF, 24, 32))   # x8-ish ragged
        out.append((2, 32, 40, 30, 13, 11, it, BF, 40, 48))     # down, ragged
        out.append((1, 16, 16, 20, 128, 160, it, BF, 28, 24))   # C % 8 == 0, ics % 8 != 0: scalar path
    out.append(("multi", 8, 9, 9, 129, 129, BF, BF, 16, 24))    # several grid trips
    return out


_DTN = {BF: "bf", F32: "f32"}


def _case_id(c):
    return "N%sC%dH%dW%d-H%dW%d-%s-%s-ics%docs%d" % (c[0], c[1], c[2], c[3], c[4], c[5], _DTN[c[6]], _DTN[c[7]], c[8],
                                                     c[9])


@pytest.mark.parametrize("case", _bilinear_fwd_cases(), ids=[_case_id(c) for c in _bilinear_fwd_cases()])
def test_bilinear_fwd(cuda, case):
    N, C, Hi, Wi, Ho, Wo, it, ot, ics, ocs = case
    if N == "multi":
        N = _multi_trip(Ho * Wo * (C // 8))
    exact = _dyadic(Hi, Ho) and _dyadic(Wi, Wo)
    g = torch.Generator(device="cuda").manual_seed(Hi * 1000 + Ho + C)
    # non-negative operands where a weight is inexact: no cancellation, so fp32 keeps the result well inside 1 bf16 ulp
    x = _ints((N, Hi, Wi, C), -8 if exact else 0, 8, g)
    xs = Slab((N, Hi, Wi), C, ics, it, x)
    ys = Slab((N, Ho, Wo), C, ocs, ot, out=True)
    _call("tsb_bilinear_fwd", xs.ptr, _tsb(it), ics, ys.ptr, _tsb(ot), ocs, N, C, Hi, Wi, Ho, Wo)
    ref = torch.einsum("yi,xj,nijc->nyxc", _lerp_matrix(Hi, Ho), _lerp_matrix(Wi, Wo), xs.v.double())
    if exact:
        _eq(ys.v, ref, "bilinear fwd")
    else:
        _ulp1(ys.v, ref, "bilinear fwd")
    ys.assert_pad("bilinear fwd")


def _bilinear_bwd_cases():
    out = []
    for ot, it in [(BF, BF), (BF, F32), (F32, BF), (F32, F32)]:
        for acc in (0, 1):
            out.append((1, 16, 9, 9, 65, 65, ot, it, 32, 24, acc))     # x8 up: > 12 candidate columns per input pixel
            out.append((2, 24, 33, 33, 17, 17, ot, it, 40, 48, acc))   # down by 2
            out.append((2, 8, 9, 17, 33, 33, ot, it, 16, 64, acc))     # x4 / x2 up
    out.append(("multi", 8, 129, 129, 65, 65, BF, BF, 16, 24, 1))      # several grid trips
    return out


@pytest.mark.parametrize("case", _bilinear_bwd_cases(),
                         ids=[_case_id(c) + "-acc%d" % c[10] for c in _bilinear_bwd_cases()])
def test_bilinear_bwd(cuda, case):
    N, C, Hi, Wi, Ho, Wo, ot, it, ocs, ics, acc = case
    if N == "multi":
        N = _multi_trip(Hi * Wi * (C // 8))
    g = torch.Generator(device="cuda").manual_seed(Hi * 1000 + Ho + C + acc)
    dy = _ints((N, Ho, Wo, C), -8, 8, g)
    old = _ints((N, Hi, Wi, C), -8, 8, g)
    dys = Slab((N, Ho, Wo), C, ocs, ot, dy)
    dxs = Slab((N, Hi, Wi), C, ics, it, old if acc else None, out=True)
    _call("tsb_bilinear_bwd", dys.ptr, _tsb(ot), ocs, dxs.ptr, _tsb(it), ics, N, C, Hi, Wi, Ho, Wo, acc)
    ref = torch.einsum("yi,xj,nyxc->nijc", _lerp_matrix(Hi, Ho), _lerp_matrix(Wi, Wo), dys.v.double())
    if acc:
        ref = ref + old.to(it).double()
    _eq(dxs.v, ref, "bilinear bwd")
    dxs.assert_pad("bilinear bwd")


# ------------------------------------------------------------------------------------------------ pooling
def _bins(n, S):
    return [((i * n) // S, -(-((i + 1) * n) // S)) for i in range(S)]


# (N, C, H, W, S): every bin area is a power of two, so the per-bin 1/area is exact
POOL_CASES = [(2, 24, 16, 16, 1), (2, 24, 16, 8, 2), (2, 24, 10, 10, 3), (2, 24, 20, 20, 6), (2, 24, 3, 3, 3),
              (3, 24, 6, 6, 6), (2, 2056, 20, 20, 6), (2, 2056, 8, 8, 1), (2, 2056, 10, 10, 3),
              ("multi", 24, 512, 512, 2), ("multi", 24, 512, 512, 1)]


@pytest.mark.parametrize("case", POOL_CASES, ids=["N%sC%dH%dW%dS%d" % c for c in POOL_CASES])
def test_adaptive_avgpool(cuda, case):
    N, C, H, W, S = case
    if N == "multi":
        N = _multi_trip(H * W * (C // 8))
    cs = C + 16
    g = torch.Generator(device="cuda").manual_seed(C * 100 + H + S)
    x = _ints((N, H, W, C), -8, 8, g)
    xs = Slab((N, H, W), C, cs, BF, x)
    out = torch.full((N, S, S, C), float("nan"), dtype=F32, device="cuda")
    _call("tsb_adaptive_avgpool_fwd", xs.ptr, cs, N, C, H, W, S, out.data_ptr(), *_ws())
    ref = torch.empty((N, S, S, C), dtype=torch.float64, device="cuda")
    for i, (h0, h1) in enumerate(_bins(H, S)):
        for j, (w0, w1) in enumerate(_bins(W, S)):
            ref[:, i, j] = x[:, h0:h1, w0:w1].mean(dim=(1, 2))
    _eq(out, ref, "adaptive avgpool fwd")

    dout = _ints((N, S, S, C), -8, 8, g).float()
    old = _ints((N, H, W, C), -8, 8, g)
    dref = torch.zeros((N, H, W, C), dtype=torch.float64, device="cuda")
    for i, (h0, h1) in enumerate(_bins(H, S)):
        for j, (w0, w1) in enumerate(_bins(W, S)):
            dref[:, h0:h1, w0:w1] += (dout[:, i, j].double() / ((h1 - h0) * (w1 - w0)))[:, None, None]
    for acc in (0, 1):
        dxs = Slab((N, H, W), C, cs, BF, old if acc else None, out=True)
        _call("tsb_adaptive_avgpool_bwd", dout.data_ptr(), N, C, H, W, S, dxs.ptr, cs, acc)
        _eq(dxs.v, dref + old if acc else dref, "adaptive avgpool bwd accumulate=%d" % acc)
        dxs.assert_pad("adaptive avgpool bwd")


# (N, C, H, W, lo, hi): all-negative inputs (the padding must act as -inf), many ties, odd sizes, H = 1
MAXPOOL_CASES = [(2, 24, 7, 9, -8, -1), (2, 24, 9, 7, -1, 0), (2, 16, 1, 5, -3, -1), (1, 8, 1, 1, -2, -1),
                 (2, 96, 13, 11, -2, 1), (1, 2056, 5, 6, -1, 0), ("multi", 8, 257, 255, -2, 0)]


@pytest.mark.parametrize("case", MAXPOOL_CASES, ids=["N%sC%dH%dW%d[%d,%d]" % c for c in MAXPOOL_CASES])
def test_maxpool3x3s2(cuda, case):
    N, C, H, W, lo, hi = case
    P, Q = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if N == "multi":
        N = _multi_trip(P * Q * (C // 8))
    ics, ocs, dcs = C + 8, C + 24, C + 16
    g = torch.Generator(device="cuda").manual_seed(C * 100 + H * 10 + W)
    x = _ints((N, H, W, C), lo, hi, g)
    xs = Slab((N, H, W), C, ics, BF, x)
    ys = Slab((N, P, Q), C, ocs, BF, out=True)
    am = torch.full((N, P, Q, C), 255, dtype=torch.uint8, device="cuda")
    _call("tsb_maxpool3x3s2_fwd", xs.ptr, ics, ys.ptr, ocs, am.data_ptr(), N, C, H, W)
    ref, flat = F.max_pool2d(x.permute(0, 3, 1, 2).contiguous(), 3, 2, 1, return_indices=True)   # first maximum in scan order
    _eq(ys.v, ref.permute(0, 2, 3, 1), "maxpool fwd")
    ys.assert_pad("maxpool fwd")
    p = torch.arange(P, device="cuda").view(1, 1, P, 1)
    q = torch.arange(Q, device="cuda").view(1, 1, 1, Q)
    code = (flat // W - (2 * p - 1)) * 3 + (flat % W - (2 * q - 1))
    assert torch.equal(am, code.permute(0, 2, 3, 1).to(torch.uint8)), "maxpool argmax differs from ATen's first maximum"

    dy = _ints((N, P, Q, C), -8, 8, g)
    dys = Slab((N, P, Q), C, ocs, BF, dy)
    dxs = Slab((N, H, W), C, dcs, BF, out=True)
    _call("tsb_maxpool3x3s2_bwd", am.data_ptr(), dys.ptr, ocs, dxs.ptr, dcs, N, C, H, W)
    dref = torch.zeros((N * C, H * W), dtype=torch.float64, device="cuda")
    dref.scatter_add_(1, flat.reshape(N * C, P * Q), dy.permute(0, 3, 1, 2).reshape(N * C, P * Q))
    _eq(dxs.v, dref.view(N, C, H, W).permute(0, 2, 3, 1), "maxpool bwd")
    dxs.assert_pad("maxpool bwd")


# ------------------------------------------------------------------------------------------------ BatchNorm
def _bn_npix(C8):
    return _multi_trip(C8)


def _bn_params(C, g):
    """dyadic per-channel vectors: every fma / product below is exact in fp32"""
    return dict(mean=_pick((C,), [-1.0, -0.5, -0.25, 0.0, 0.25, 0.75, 1.0], g),
                invstd=_pick((C,), [0.5, 1.0, 2.0], g),
                scale=_pick((C,), [-1.0, -0.5, -0.125, 0.125, 0.375, 0.5, 1.0], g),
                shift=_pick((C,), [-1.0, -0.25, 0.0, 0.25, 0.5], g),
                gamma=_pick((C,), [0.5, 1.0, 2.0, -1.0], g))


def _f(t):
    return t.float().contiguous()


@pytest.mark.parametrize("C8", C8S)
def test_bn_stats_and_apply(cuda, C8):
    C = 8 * C8
    npix = _bn_npix(C8)
    cs = C + 64
    g = torch.Generator(device="cuda").manual_seed(C8)
    x = _ints((npix, C), -2, 2, g)   # Σx² < 2^24: exact
    r = _ints((npix, C), -8, 8, g)
    xs, rs = Slab((npix,), C, cs, BF, x), Slab((npix,), C, C + 8, BF, r)
    s = torch.zeros(2, C, device="cuda")
    _call("tsb_bn_stats", xs.ptr, cs, npix, C, s[0].data_ptr(), s[1].data_ptr(), *_ws())
    _eq(s[0], x.sum(0), "bn_stats sum")
    _eq(s[1], (x * x).sum(0), "bn_stats sumsq")

    prm = _bn_params(C, g)
    sc, sh = _f(prm["scale"]), _f(prm["shift"])
    for relu in (0, 1):
        for res in (False, True):
            ys = Slab((npix,), C, C + 16, BF, out=True)
            _call("tsb_bn_apply", xs.ptr, cs, sc.data_ptr(), sh.data_ptr(), rs.ptr if res else None, C + 8 if res else 0,
                  relu, ys.ptr, C + 16, npix, C)
            ref = x * prm["scale"] + prm["shift"] + (r if res else 0)
            _eq(ys.v, ref.clamp_min(0) if relu else ref, "bn_apply relu=%d res=%d" % (relu, res))
            ys.assert_pad("bn_apply")


def test_bn_finalize_exact(cuda):
    """dyadic mean and variance with eps = 0 and 5 samples: mean, invstd, scale, shift and both running statistics are
    exact in fp32"""
    C = 24
    g = torch.Generator(device="cuda").manual_seed(5)
    cnt = 5.0
    m = _pick((C,), [-1.5, -0.25, 0.0, 0.5, 2.0], g)
    var = _pick((C,), [0.25, 1.0, 4.0, 16.0], g)
    gamma, beta = _pick((C,), [0.5, 1.0, -2.0], g), _pick((C,), [-1.0, 0.0, 0.25], g)
    rm0, rv0 = _pick((C,), [0.0, 1.0, -0.5], g), _pick((C,), [1.0, 0.5, 2.0], g)
    ssum, ssq = _f(m * cnt), _f((var + m * m) * cnt)
    outs = [torch.full((C,), float("nan"), device="cuda") for _ in range(4)]
    rm, rv, gf, bf = _f(rm0), _f(rv0), _f(gamma), _f(beta)
    _call("tsb_bn_finalize", ssum.data_ptr(), ssq.data_ptr(), cnt, C, gf.data_ptr(), bf.data_ptr(), 0.0, 0.25,
          *[o.data_ptr() for o in outs], rm.data_ptr(), rv.data_ptr())
    istd = var.rsqrt()
    _eq(outs[0], m, "mean")
    _eq(outs[1], istd, "invstd")
    _eq(outs[2], gamma * istd, "scale")
    _eq(outs[3], beta - m * gamma * istd, "shift")
    _eq(rm, 0.75 * rm0 + 0.25 * m, "running_mean")
    _eq(rv, 0.75 * rv0 + 0.25 * var * cnt / (cnt - 1), "running_var")


@pytest.mark.parametrize("C8", C8S)
def test_bn_backward(cuda, C8):
    C = 8 * C8
    npix = _bn_npix(C8)
    g = torch.Generator(device="cuda").manual_seed(100 + C8)
    x, dy = _ints((npix, C), -2, 2, g), _ints((npix, C), -2, 2, g)
    prm = _bn_params(C, g)
    m, istd, sc, sh, ga = _f(prm["mean"]), _f(prm["invstd"]), _f(prm["scale"]), _f(prm["shift"]), _f(prm["gamma"])
    xs, dys = Slab((npix,), C, C + 8, BF, x), Slab((npix,), C, C + 64, BF, dy)
    # y of a layer without residual: the mode-1 mask (y > 0) and the mode-2 mask (x·scale + shift > 0) agree
    ys = Slab((npix,), C, C + 16, BF, out=True)
    _call("tsb_bn_apply", xs.ptr, C + 8, sc.data_ptr(), sh.data_ptr(), None, 0, 1, ys.ptr, C + 16, npix, C)
    mask = (x * prm["scale"] + prm["shift"]) > 0
    xhat = (x - prm["mean"]) * prm["invstd"]
    count = 64.0   # the count only scales the reductions: a power of two keeps every coefficient dyadic
    # sums handed to the apply pass: small dyadic values, independent of this data, so its coefficients stay exact
    s1, s2 = _pick((C,), [-4.0, -1.0, 0.0, 2.0, 8.0], g), _pick((C,), [-2.0, 0.5, 0.0, 3.0], g)
    dg0, db0 = _pick((C,), [0.5, -1.0, 3.0], g), _pick((C,), [-0.25, 2.0, 1.0], g)
    results = {}
    for relu, mode in ((0, 0), (1, 1), (1, 2)):
        dz = torch.where(mask, dy, torch.zeros_like(dy)) if relu else dy
        y_ptr, ycs = (ys.ptr, C + 16) if mode == 1 else (None, 0)
        sums = torch.zeros(2, C, device="cuda")
        _call("tsb_bn_bwd_reduce", dys.ptr, C + 64, y_ptr, ycs, xs.ptr, C + 8, m.data_ptr(), istd.data_ptr(), relu, npix,
              C, sums[0].data_ptr(), sums[1].data_ptr(), sc.data_ptr() if mode == 2 else None,
              sh.data_ptr() if mode == 2 else None, *_ws())
        _eq(sums[0], dz.sum(0), "bn_bwd_reduce sum_dz mode %d" % mode)
        _eq(sums[1], (dz * xhat).sum(0), "bn_bwd_reduce sum_dz_xhat mode %d" % mode)

        dxs = Slab((npix,), C, C + 24, BF, out=True)
        drs = Slab((npix,), C, C + 8, BF, out=True)
        dga, dba = _f(dg0), _f(db0)
        S1, S2 = _f(s1), _f(s2)
        _call("tsb_bn_bwd_apply", dys.ptr, C + 64, y_ptr, ycs, xs.ptr, C + 8, m.data_ptr(), istd.data_ptr(),
              ga.data_ptr(), S1.data_ptr(), S2.data_ptr(), count, relu, dxs.ptr, C + 24, drs.ptr, C + 8, npix, C,
              dga.data_ptr(), dba.data_ptr(), sc.data_ptr() if mode == 2 else None, sh.data_ptr() if mode == 2 else None)
        ref = prm["gamma"] * prm["invstd"] * (dz - s1 / count - xhat * s2 / count)
        _eq(dxs.v, ref, "bn_bwd_apply dx mode %d" % mode)
        _eq(drs.v, dz, "bn_bwd_apply dres mode %d" % mode)
        _eq(dga, dg0 + s2, "dgamma_acc")
        _eq(dba, db0 + s1, "dbeta_acc")
        dxs.assert_pad("bn_bwd_apply dx")
        drs.assert_pad("bn_bwd_apply dres")
        results[mode] = (sums.clone(), dxs.v.clone())
    assert torch.equal(results[1][0], results[2][0]) and torch.equal(results[1][1], results[2][1]), \
        "relu mask from y and from x*scale+shift differ"


# ------------------------------------------------------------------------------------------------ channel attention
def _chan_cases():
    out = []
    for C in (24, 384, 2048):
        for base in (0.0, 1.0):
            for add in (False, True):
                out.append((3, 7 * 13, C, base, add))
    out.append(("multi", 0, 24, 1.0, True))
    return out


@pytest.mark.parametrize("case", _chan_cases(), ids=["N%sHW%dC%d-base%g-add%d" % c for c in _chan_cases()])
def test_chan_scale(cuda, case):
    N, HW, C, base, add = case
    if N == "multi":
        N = 3
        HW = _multi_trip(N * (C // 8)) | 1
    g = torch.Generator(device="cuda").manual_seed(C + int(base) * 7 + add)
    # a = ±100 and 0 give sigmoid = 1, 0 and 1/2 exactly (even through __expf), different for every image n
    a = _pick((N, C), [-100.0, 0.0, 100.0], g)
    sig = torch.sigmoid(a).round(decimals=3)
    x, r, dy = _ints((N, HW, C), -8, 8, g), _ints((N, HW, C), -8, 8, g), _ints((N, HW, C), -8, 8, g)
    xs, rs, dys = Slab((N, HW), C, C + 8, BF, x), Slab((N, HW), C, C + 16, BF, r), Slab((N, HW), C, C + 64, BF, dy)
    af = _f(a)
    ys = Slab((N, HW), C, C + 24, BF, out=True)
    _call("tsb_chan_scale_fwd", xs.ptr, C + 8, af.data_ptr(), base, rs.ptr if add else None, C + 16 if add else 0, ys.ptr,
          C + 24, N, HW, C)
    _eq(ys.v, x * (base + sig[:, None]) + (r if add else 0), "chan_scale fwd")
    ys.assert_pad("chan_scale fwd")

    dxs = Slab((N, HW), C, C + 8, BF, out=True)
    da0 = _pick((N, C), [0.0, 0.5, -3.0], g)
    da = _f(da0)
    _call("tsb_chan_scale_bwd", dys.ptr, C + 64, xs.ptr, C + 8, af.data_ptr(), base, dxs.ptr, C + 8, da.data_ptr(), N, HW,
          C, *_ws())
    _eq(dxs.v, dy * (base + sig[:, None]), "chan_scale bwd dx")
    _eq(da, da0 + (dy * x).sum(1) * sig * (1 - sig), "chan_scale bwd da")
    dxs.assert_pad("chan_scale bwd")

    if case[0] != "multi" and C == 24:   # general logits: __expf is not exact, so 1 ulp of the bf16 output
        a2 = (torch.randn((N, C), generator=g, device="cuda") * 3).contiguous()
        xp, rp = Slab((N, HW), C, C + 8, BF, x.abs()), Slab((N, HW), C, C + 16, BF, r.abs())
        y2 = Slab((N, HW), C, C + 24, BF, out=True)
        _call("tsb_chan_scale_fwd", xp.ptr, C + 8, a2.data_ptr(), base, rp.ptr if add else None,
              C + 16 if add else 0, y2.ptr, C + 24, N, HW, C)
        _ulp1(y2.v, x.abs() * (base + torch.sigmoid(a2.double())[:, None]) + (r.abs() if add else 0),
              "chan_scale fwd, general logits")


# ------------------------------------------------------------------------------------------------ elementwise glue
@pytest.mark.parametrize("sdt,ddt", [(BF, BF), (BF, F32), (F32, BF), (F32, F32)], ids=["bf-bf", "bf-f32", "f32-bf", "f32-f32"])
def test_cast_scale(cuda, sdt, ddt):
    g = torch.Generator(device="cuda").manual_seed(3)
    for C, npix in ((24, 1001), (24, _multi_trip(3)), (2056, 37)):
        src = torch.randn((npix, C), generator=g, device="cuda").double() * 100
        ss = Slab((npix,), C, C + 8, sdt, src)
        for scale in (None, -0.25):
            ds = Slab((npix,), C, C + 16, ddt, out=True)
            sv = torch.tensor([scale], device="cuda") if scale is not None else None
            _call("tsb_cast_scale", ss.ptr, _tsb(sdt), C + 8, ds.ptr, _tsb(ddt), C + 16, npix, C,
                  sv.data_ptr() if sv is not None else None)
            _eq(ds.v, ss.v.double() * (1.0 if scale is None else scale), "cast_scale")
            ds.assert_pad("cast_scale")


@pytest.mark.parametrize("K", [1, 19, 150])
@pytest.mark.parametrize("sdt", [BF, F32], ids=["bf", "f32"])
def test_cast_pad(cuda, K, sdt):
    Kp = (K + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(K)
    for npix in (333, _multi_trip(Kp // 8)):
        scs = K + 3   # not a multiple of 8
        src = torch.randn((npix, K), generator=g, device="cuda").double()
        sbuf = torch.full((npix, scs), float("nan"), dtype=sdt, device="cuda")
        sbuf[:, :K] = src.to(sdt)
        ds = Slab((npix,), Kp, Kp + 16, BF, out=True)
        ds.v.fill_(float("nan"))   # [K, Kp) must come back as zeros
        _call("tsb_cast_pad", sbuf.data_ptr(), _tsb(sdt), scs, K, ds.ptr, Kp + 16, Kp, npix)
        _eq(ds.v[:, :K], sbuf[:, :K].float(), "cast_pad values")
        assert bool((ds.v[:, K:] == 0).all()), "cast_pad did not zero channels [K, Kp)"
        ds.assert_pad("cast_pad")


@pytest.mark.parametrize("C", [24, 2056])
def test_add_relu_and_relu_bwd(cuda, C):
    g = torch.Generator(device="cuda").manual_seed(C)
    for npix in (517, _multi_trip(C // 8)):
        a, b = _ints((npix, C), -8, 8, g), _ints((npix, C), -8, 8, g)
        a[::7] = -b[::7]          # a + b == 0 exactly
        a[1::7] = -0.0
        b[1::7] = -0.0            # -0 + -0 == -0
        As, Bs = Slab((npix,), C, C + 8, BF, a), Slab((npix,), C, C + 16, BF, b)
        for name, ref in (("tsb_add", a + b), ("tsb_add_relu", (a + b).clamp_min(0))):
            ys = Slab((npix,), C, C + 24, BF, out=True)
            _call(name, As.ptr, C + 8, Bs.ptr, C + 16, ys.ptr, C + 24, npix, C)
            _eq(ys.v, ref, name)
            ys.assert_pad(name)
        # relu_bwd: y = relu output with +0, -0 and negative entries; dx = dy where y > 0
        y = a + b
        y[2::7] = -0.0
        Ys = Slab((npix,), C, C + 8, BF, y)
        dxs = Slab((npix,), C, C + 16, BF, out=True)
        _call("tsb_relu_bwd", Bs.ptr, C + 16, Ys.ptr, C + 8, dxs.ptr, C + 16, npix, C)
        _eq(dxs.v, torch.where(y > 0, b, torch.zeros_like(b)), "relu_bwd")
        dxs.assert_pad("relu_bwd")


@pytest.mark.parametrize("K", [1, 19, 150])
def test_bias_grad(cuda, K):
    npix = 200003   # a few hundred workspace slots
    dycs = K + 5
    g = torch.Generator(device="cuda").manual_seed(K)
    dy = _ints((npix, K), -8, 8, g)
    buf = torch.full((npix, dycs), float("nan"), dtype=BF, device="cuda")
    buf[:, :K] = dy.to(BF)
    db0 = _pick((K,), [0.5, -2.0, 0.0], g)
    outs = []
    for _ in range(2):
        db = _f(db0)
        _call("tsb_bias_grad", buf.data_ptr(), dycs, npix, K, db.data_ptr(), *_ws())
        outs.append(db)
    _eq(outs[0], db0 + dy.sum(0), "bias_grad")
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "bias_grad is not reproducible"


# ------------------------------------------------------------------------------------------------ PSANet helpers
@pytest.mark.parametrize("C,Cp", [(8, 8), (8, 64), (3600, 3648), (8192, 8192)])
@pytest.mark.parametrize("idt", [BF, F32], ids=["bf", "f32"])
def test_softmax_rows(cuda, C, Cp, idt):
    rows = 37
    ics, ocs = C + 24, Cp + 16
    g = torch.Generator(device="cuda").manual_seed(C + Cp)
    logits = torch.randn((rows, C), generator=g, device="cuda").double() * 3
    xs = Slab((rows,), C, ics, idt, logits)
    ys = Slab((rows,), Cp, ocs, BF, out=True)
    ys.v.fill_(float("nan"))   # [C, Cp) must come back as zeros
    _call("tsb_softmax_rows_fwd", xs.ptr, _tsb(idt), ics, ys.ptr, ocs, rows, C, Cp)
    ref = torch.softmax(xs.v.double(), dim=1)
    _ulp1(ys.v[:, :C], ref, "softmax fwd")
    assert bool((ys.v[:, C:] == 0).all()), "softmax did not zero channels [C, Cp)"
    ys.assert_pad("softmax fwd")
    row_err = (ys.v[:, :C].double().sum(1) - 1).abs()
    assert bool((row_err <= _ulp(ref, BF).sum(1)).all()), "softmax rows do not sum to 1 within bf16 rounding"

    # backward on operands that make Σ S·dS exact: S = k / 2^14 (k <= 32), dS small integers
    S = torch.randint(0, 33, (rows, C), generator=g, device="cuda").double() / 2 ** 14
    dS = _ints((rows, C), -8, 8, g)
    Ss, dSs = Slab((rows,), C, C + 8, BF, S), Slab((rows,), C, C + 40, BF, dS)
    dAs = Slab((rows,), Cp, ocs, BF, out=True)
    dAs.v.fill_(float("nan"))
    _call("tsb_softmax_rows_bwd", Ss.ptr, C + 8, dSs.ptr, C + 40, dAs.ptr, ocs, rows, C, Cp)
    dref = S * (dS - (S * dS).sum(1, keepdim=True))
    _ulp1(dAs.v[:, :C], dref, "softmax bwd")
    assert bool((dAs.v[:, C:] == 0).all()), "softmax bwd did not zero channels [C, Cp)"
    dAs.assert_pad("softmax bwd")


@pytest.mark.parametrize("R,Cc,Rp", [(45, 70, 64), (100, 33, 128), (1, 5, 8), (64, 64, 96)])
@pytest.mark.parametrize("idt", [BF, F32], ids=["bf", "f32"])
def test_transpose_pad(cuda, R, Cc, Rp, idt):
    ics, ocs = Cc + 11, Rp + 16
    g = torch.Generator(device="cuda").manual_seed(R * 100 + Cc)
    src = torch.randn((R, Cc), generator=g, device="cuda").double()
    inb = torch.full((R, ics), float("nan"), dtype=idt, device="cuda")
    inb[:, :Cc] = src.to(idt)
    out = Slab((Cc,), Rp, ocs, BF, out=True)
    out.v.fill_(float("nan"))   # [R, Rp) must come back as zeros
    _call("tsb_transpose_pad", inb.data_ptr(), _tsb(idt), ics, out.ptr, ocs, R, Cc, Rp)
    assert torch.equal(out.v[:, :R], inb[:, :Cc].t().to(BF)), "transpose_pad values"
    assert bool((out.v[:, R:] == 0).all()), "transpose_pad did not zero columns [R, Rp)"
    out.assert_pad("transpose_pad")


# ------------------------------------------------------------------------------------------------ weight packing, SGD
def test_pack_wt_multi_matches_pack_weight(cuda):
    shapes = [(19, 3, 3, 40), (64, 1, 1, 2048), (150, 3, 3, 72), (5, 1, 1, 8)]
    g = torch.Generator(device="cuda").manual_seed(9)
    descs, starts, refs, off, nb = [], [], [], 8, 0
    total = sum(K * R * S * C for K, R, S, C in shapes) + 64 * len(shapes) + 8
    wb_flat = torch.full((total,), float("nan"), dtype=BF, device="cuda")
    wt_flat = torch.full((total,), SENT[BF], dtype=torch.int16, device="cuda").view(BF)
    for K, R, S, C in shapes:
        w = torch.randn((K, R, S, C), generator=g, device="cuda")
        n = w.numel()
        wt_ref = torch.empty((C, R, S, K), dtype=BF, device="cuda")
        _call("tsb_pack_weight", w.data_ptr(), K, R, S, C, None, wt_ref.data_ptr())
        wb_flat[off:off + n] = w.to(BF).flatten()
        tk, tc = (K + 31) // 32, (C + 31) // 32
        descs.append((off, K, R * S, C, tk, tc, 0))
        starts.append(nb)
        nb += R * S * tk * tc
        refs.append((off, n, wt_ref))
        off += n + 37   # odd gaps: the bytes between tensors must stay untouched
    dt = np.dtype([("off", "<i8"), ("K", "<i4"), ("RS", "<i4"), ("C", "<i4"), ("tk", "<i4"), ("tc", "<i4"), ("pad", "<i4")])
    assert dt.itemsize == 32
    desc = torch.from_numpy(np.array(descs, dtype=dt).view(np.uint8).copy()).cuda()
    bstart = torch.tensor(starts, dtype=torch.int32, device="cuda")
    _call("tsb_pack_wt_multi", wb_flat.data_ptr(), wt_flat.data_ptr(), desc.data_ptr(), bstart.data_ptr(), len(shapes), nb)
    touched = torch.zeros(total, dtype=torch.bool, device="cuda")
    for o, n, wt_ref in refs:
        assert torch.equal(wt_flat[o:o + n].view(torch.int16), wt_ref.flatten().view(torch.int16)), "pack_wt_multi"
        touched[o:o + n] = True
    assert bool((wt_flat.view(torch.int16)[~touched] == SENT[BF]).all()), "pack_wt_multi wrote between tensors"


def test_sgd_flat_pack_matches_sgd_flat(cuda):
    n = 1000003   # n % 4 != 0
    g = torch.Generator(device="cuda").manual_seed(4)
    seg_end = torch.tensor([12345, 500001, 777777, n], dtype=torch.int64, device="cuda")   # odd segment ends
    seg_lr = torch.tensor([0.01, 0.1, 0.003, 0.05], device="cuda")
    seg_wd = torch.tensor([1e-4, 0.0, 5e-4, 1e-4], device="cuda")
    p0 = torch.randn(n, generator=g, device="cuda")
    pa, pb = p0.clone(), p0.clone()
    ma, mb = torch.full_like(p0, float("nan")), torch.full_like(p0, float("nan"))   # first_step never reads mom
    pbf = torch.full((n + 8,), SENT[BF], dtype=torch.int16, device="cuda").view(BF)
    for first in (1, 0, 0):
        grad = torch.randn(n, generator=g, device="cuda")
        _call("tsb_sgd_flat", pa.data_ptr(), grad.data_ptr(), ma.data_ptr(), n, seg_end.data_ptr(), seg_lr.data_ptr(),
              seg_wd.data_ptr(), 4, 0.9, 0.5, first)
        _call("tsb_sgd_flat_pack", pb.data_ptr(), grad.data_ptr(), mb.data_ptr(), n, seg_end.data_ptr(),
              seg_lr.data_ptr(), seg_wd.data_ptr(), 4, 0.9, 0.5, first, pbf.data_ptr())
        assert torch.equal(pa.view(torch.int32), pb.view(torch.int32)), "param differs (first_step=%d)" % first
        assert torch.equal(ma.view(torch.int32), mb.view(torch.int32)), "momentum differs (first_step=%d)" % first
        assert torch.equal(pbf[:n].view(torch.int16), pb.to(BF).view(torch.int16)), "bf16 copy differs"
        assert bool((pbf[n:].view(torch.int16) == SENT[BF]).all()), "bf16 copy written past n"
