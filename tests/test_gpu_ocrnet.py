"""OCRNet on the H100: the cross form of the fused attention kernels (tsb_cross_attention_{fwd,bwd}) against float64
autograd of the materialised softmax(scale · q kᵀ) v with Nq queries and Nk keys, bit-equality with tsb_attention_*
at Nq = Nk, exact cases, channel slices, bounds and determinism; the soft-max over the pixels of each image
(tsb_spatial_softmax_{fwd,bwd}) against float64; ops.SpatialGatherFn against float64; the object attention block and
the OCR module teacher-forced against the bf16-emulating oracle; and the whole training and eval step against the
oracle (tests/ocrnet_oracle.py on the blocks of oracle/torch_ref.py, pinned to the live reference composition by
tests/test_cpu_ocrnet.py) and its bf16-storage emulation."""
import pytest
import torch

from util import norm_err, bf16_round
from net_checks import (check_train_reproducible, check_graphed_matches_eager,
                        check_eval_vs_oracle_and_sliding)

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d
D = 256
SCALE = D ** -0.5


# ------------------------------------------------------------------------------------------------- cross attention
def _rows(B, N, cs, dev, fill=0.0):
    return torch.full((B, N, cs), fill, dtype=torch.bfloat16, device=dev)


def _xfwd(q, k, v, o=None, lse=True, scale=SCALE):
    from torchseg_b200._lib import call, ptr, stream
    B, Nq = q.shape[:2]
    Nk = k.shape[1]
    o = _rows(B, Nq, D, q.device) if o is None else o
    lse_t = torch.empty((B, Nq), dtype=torch.float32, device=q.device) if lse else None
    call("tsb_cross_attention_fwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(lse_t), B, Nq, Nk, D, D, float(scale), stream())
    return o, lse_t


def _xbwd(q, k, v, o, do, lse, dq=None, dk=None, dv=None, scale=SCALE):
    from torchseg_b200._lib import call, ptr, stream
    B, Nq = q.shape[:2]
    Nk = k.shape[1]
    dev = q.device
    dq = _rows(B, Nq, D, dev) if dq is None else dq
    dk = _rows(B, Nk, D, dev) if dk is None else dk
    dv = _rows(B, Nk, D, dev) if dv is None else dv
    delta = torch.empty((B, Nq), dtype=torch.float32, device=dev)
    call("tsb_cross_attention_bwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(do), do.stride(1), ptr(lse), ptr(delta), ptr(dq), dq.stride(1), ptr(dk), dk.stride(1), ptr(dv),
         dv.stride(1), B, Nq, Nk, D, D, float(scale), stream())
    return dq, dk, dv


def _ref64(q, k, v, do):
    """float64 autograd of the materialised form on the same bf16 inputs: (o, lse, dq, dk, dv)"""
    q64, k64, v64 = (t[..., :D].double().requires_grad_(True) for t in (q, k, v))
    s = torch.matmul(q64, k64.transpose(1, 2)) * SCALE
    o = torch.matmul(torch.softmax(s, -1), v64)
    lse = torch.logsumexp(s, -1)
    o.backward(do[..., :D].double())
    return o.detach(), lse.detach(), q64.grad, k64.grad, v64.grad


def _rand(B, N, dev, g, cs=D, mul=1.0):
    t = _rows(B, N, cs, dev, float("nan"))
    t[..., :D] = (torch.randn(B, N, D, device=dev, generator=g) * mul).to(torch.bfloat16)
    return t


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Nq,Nk", [(1, 1), (37, 19), (100, 1000), (9409, 19), (9409, 150)])
def test_cross_attention_vs_float64(cuda, B, Nq, Nk):
    g = torch.Generator(device=cuda).manual_seed(Nq * 13 + Nk * 7 + B)
    q, do = _rand(B, Nq, cuda, g), _rand(B, Nq, cuda, g)
    k, v = _rand(B, Nk, cuda, g), _rand(B, Nk, cuda, g)
    o, lse = _xfwd(q, k, v)
    dq, dk, dv = _xbwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    ro, rlse, rdq, rdk, rdv = _ref64(q, k, v, do)
    assert norm_err(o, ro) < 6e-3, norm_err(o, ro)
    assert float((lse.double() - rlse).abs().max()) < 2e-4 * max(1.0, float(rlse.abs().max()))
    if Nk == 1:
        # one key: P = 1, so o = v and dv = Σ_i dout_i; dS = dout·v − dout·o is 0 up to the fp32 summation order
        assert torch.equal(o, v[..., :D].expand(B, Nq, D))
        assert float(dq.float().abs().max()) < 1e-4 and float(dk.float().abs().max()) < 1e-4
        assert norm_err(dv, rdv) < 1e-2
        return
    for name, a, b in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        assert norm_err(a, b) < 1.5e-2, (name, norm_err(a, b))


@pytest.mark.parametrize("N", [19, 333])
def test_cross_attention_equal_counts_match_self_attention_bitwise(cuda, N):
    from torchseg_b200._lib import call, ptr, stream
    B = 2
    g = torch.Generator(device=cuda).manual_seed(N)
    q, k, v, do = (_rand(B, N, cuda, g) for _ in range(4))
    o, lse = _xfwd(q, k, v)
    grads = _xbwd(q, k, v, o, do, lse)
    o2 = _rows(B, N, D, cuda)
    lse2 = torch.empty((B, N), dtype=torch.float32, device=cuda)
    call("tsb_attention_fwd", ptr(q), D, ptr(k), D, ptr(v), D, ptr(o2), D, ptr(lse2), B, N, D, D, SCALE, stream())
    g2 = [_rows(B, N, D, cuda) for _ in range(3)]
    delta = torch.empty((B, N), dtype=torch.float32, device=cuda)
    call("tsb_attention_bwd", ptr(q), D, ptr(k), D, ptr(v), D, ptr(o2), D, ptr(do), D, ptr(lse2), ptr(delta),
         ptr(g2[0]), D, ptr(g2[1]), D, ptr(g2[2]), D, 0, B, N, D, D, SCALE, stream())
    torch.cuda.synchronize()
    assert torch.equal(o, o2) and torch.equal(lse, lse2)
    for a, b in zip(grads, g2):
        assert torch.equal(a, b)


@pytest.mark.parametrize("Nq,Nk", [(100, 19), (9409, 150)])
def test_cross_attention_one_hot_exact(cuda, Nq, Nk):
    """query i picks key perm(i mod Nk): q_i = 48·e_{i mod Nk}, k_perm(j) = 48·e_j, so every other weight underflows to
    0 in fp32; o = v[perm(i mod Nk)] and dq = dk = 0 exactly (small-integer v, dout)"""
    B = 2
    perm = torch.randperm(Nk, generator=torch.Generator().manual_seed(Nk)).to(cuda)
    eye = torch.eye(D, device=cuda)[:Nk] * 48
    sel = torch.arange(Nq, device=cuda) % Nk
    q = _rows(B, Nq, D, cuda)
    k = _rows(B, Nk, D, cuda)
    q[:] = eye[sel].to(torch.bfloat16)
    k[:, perm] = eye.to(torch.bfloat16)
    g = torch.Generator(device=cuda).manual_seed(3)
    v = torch.randint(-4, 5, (B, Nk, D), device=cuda, generator=g).to(torch.bfloat16)
    do = torch.randint(-4, 5, (B, Nq, D), device=cuda, generator=g).to(torch.bfloat16)
    o, lse = _xfwd(q, k, v)
    dq, dk, dv = _xbwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    assert torch.equal(o, v[:, perm[sel]])
    ref_dv = torch.zeros(B, Nk, D, dtype=torch.float64, device=cuda)
    ref_dv.index_add_(1, perm[sel], do.double())
    assert torch.equal(dv.double(), ref_dv)   # small integers: exact in fp32 and bf16
    assert int(dq.float().abs().max()) == 0 and int(dk.float().abs().max()) == 0


@pytest.mark.parametrize("Nq,Nk", [(37, 64), (1000, 128)])
def test_cross_attention_uniform_exact(cuda, Nq, Nk):
    """k = 0: every weight is 1/Nk, and with small-integer v the output is the exact mean over the keys"""
    B = 2
    g = torch.Generator(device=cuda).manual_seed(Nq)
    q = _rand(B, Nq, cuda, g)
    k = _rows(B, Nk, D, cuda)
    v = torch.randint(-8, 9, (B, Nk, D), device=cuda, generator=g).to(torch.bfloat16)
    o, _ = _xfwd(q, k, v)
    torch.cuda.synchronize()
    ref = (v.double().sum(1, keepdim=True) / Nk).expand(B, Nq, D).float().to(torch.bfloat16)
    assert torch.equal(o, ref)


def test_cross_attention_channel_slices_and_bounds(cuda):
    """inputs as channel slices of wider buffers whose other channels are NaN give the dense results bit for bit; the
    outputs' other channels and the rows past B·Nq (o, dq) or B·Nk (dk, dv) keep their sentinel"""
    B, Nq, Nk = 2, 333, 19
    g = torch.Generator(device=cuda).manual_seed(4)
    q, k, v, do = _rand(B, Nq, cuda, g), _rand(B, Nk, cuda, g), _rand(B, Nk, cuda, g), _rand(B, Nq, cuda, g)
    o0, lse0 = _xfwd(q, k, v)
    grads0 = _xbwd(q, k, v, o0, do, lse0)
    wide = []
    for t, cs in zip((q, k, v, do), (264, 512, 320, 272)):
        w = _rows(B, t.shape[1], cs, cuda, float("nan"))
        w[..., :D] = t
        wide.append(w)
    sentinel = -3.5

    def out_buf(N, cs):
        buf = torch.full((B * N + 64, cs), sentinel, dtype=torch.bfloat16, device=cuda)
        return buf, buf[:B * N].view(B, N, cs)

    ob, o = out_buf(Nq, 288)
    o, lse = _xfwd(*wide[:3], o=o)
    bufs = [out_buf(Nq, 264), out_buf(Nk, 296), out_buf(Nk, 512)]
    _xbwd(*wide[:3], o, wide[3], lse, dq=bufs[0][1], dk=bufs[1][1], dv=bufs[2][1])
    torch.cuda.synchronize()
    assert torch.equal(o[..., :D], o0) and torch.equal(lse, lse0)
    for (buf, view), ref, N in zip([(ob, o)] + bufs, (o0,) + tuple(grads0), (Nq, Nq, Nk, Nk)):
        assert torch.equal(view[..., :D], ref)
        assert bool((buf[B * N:] == sentinel).all()) and bool((buf[:, D:] == sentinel).all())


def test_cross_attention_deterministic_and_batch_independent(cuda):
    Nq, Nk = 1500, 150
    g = torch.Generator(device=cuda).manual_seed(6)
    q, do = _rand(3, Nq, cuda, g), _rand(3, Nq, cuda, g)
    k, v = _rand(3, Nk, cuda, g), _rand(3, Nk, cuda, g)
    runs = []
    for _ in range(3):
        o, lse = _xfwd(q, k, v)
        runs.append((o, lse) + _xbwd(q, k, v, o, do, lse))
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)
    for b in range(3):
        sl = [t[b:b + 1].contiguous() for t in (q, k, v, do)]
        o1, lse1 = _xfwd(*sl[:3])
        one = (o1, lse1) + _xbwd(*sl[:3], o1, sl[3], lse1)
        for a, c in zip(runs[0], one):
            assert torch.equal(a[b:b + 1], c)


# ----------------------------------------------------------------------------------------------- spatial soft-max
def _logits(B, N, K, lcs, dev, g, offset=0.0, scale=3.0):
    """fp32 rows [B·N][lcs], K valid channels, NaN in the others; per (image, class) offsets up to ±`offset`"""
    t = torch.full((B, N, lcs), float("nan"), dtype=torch.float32, device=dev)
    off = (torch.rand(B, 1, K, device=dev, generator=g) * 2 - 1) * offset
    t[..., :K] = torch.randn(B, N, K, device=dev, generator=g) * scale + off
    return t


def _ssm_fwd(l, K):
    from torchseg_b200._lib import call, det_ws, ptr, stream
    B, N, lcs = l.shape
    Kp = (K + 63) // 64 * 64
    P = torch.full((B, N, Kp), float("nan"), dtype=torch.bfloat16, device=l.device)
    stats = torch.empty((B, 2, K), dtype=torch.float32, device=l.device)
    call("tsb_spatial_softmax_fwd", ptr(l), lcs, ptr(P), ptr(stats), B, N, K, *det_ws(), stream())
    return P, stats


def _ssm_bwd(l, stats, dP, K, dl=None):
    from torchseg_b200._lib import call, det_ws, ptr, stream
    B, N, lcs = l.shape
    dl = torch.full((B, N, lcs), -7.0, dtype=torch.float32, device=l.device) if dl is None else dl
    call("tsb_spatial_softmax_bwd", ptr(l), lcs, ptr(stats), ptr(dP), dP.shape[2], ptr(dl), dl.shape[2], B, N, K,
         *det_ws(), stream())
    return dl


@pytest.mark.parametrize("K", [19, 150])
@pytest.mark.parametrize("N", [1, 37, 9409])
def test_spatial_softmax_vs_float64(cuda, K, N):
    B = 3
    g = torch.Generator(device=cuda).manual_seed(K * 31 + N)
    lcs = (K + 31) // 32 * 32
    l = _logits(B, N, K, lcs, cuda, g, offset=1e3)
    Kp = (K + 63) // 64 * 64
    dP = torch.full((B, N, Kp), float("nan"), dtype=torch.float32, device=cuda)
    dP[..., :K] = torch.randn(B, N, K, device=cuda, generator=g)
    P, stats = _ssm_fwd(l, K)
    dl = _ssm_bwd(l, stats, dP, K)
    torch.cuda.synchronize()
    l64 = l[..., :K].double().requires_grad_(True)
    p64 = torch.softmax(l64, dim=1)
    p64.backward(dP[..., :K].double())
    assert torch.equal(P[..., K:], torch.zeros_like(P[..., K:]))
    assert float((P[..., :K].double() - p64.detach()).abs().max()) <= float(p64.detach().abs().max()) * 2 ** -8
    assert norm_err(P[..., :K], p64.detach()) < 4e-3
    assert torch.allclose(stats[:, 0].double(), l64.detach().max(1).values)
    assert norm_err(dl[..., :K], l64.grad) < 1e-5 if N > 1 else float(dl[..., :K].abs().max()) < 1e-6
    assert bool((dl[..., K:] == -7.0).all())


@pytest.mark.parametrize("N", [64, 4096, 8192])
def test_spatial_softmax_constant_logits_exact(cuda, N):
    K = 19
    l = torch.full((2, N, 32), float("nan"), dtype=torch.float32, device=cuda)
    l[..., :K] = 2.75
    P, stats = _ssm_fwd(l, K)
    torch.cuda.synchronize()
    assert bool((P[..., :K] == 1.0 / N).all()) and bool((P[..., K:] == 0).all())
    assert bool((stats[:, 1] == N).all())


def test_spatial_softmax_reproducible_and_batch_independent(cuda):
    B, N, K = 3, 9409, 150
    g = torch.Generator(device=cuda).manual_seed(12)
    l = _logits(B, N, K, 160, cuda, g, offset=30.0)
    dP = torch.randn(B, N, 192, device=cuda, generator=g)
    runs = []
    for _ in range(3):
        P, stats = _ssm_fwd(l, K)
        runs.append((P, stats, _ssm_bwd(l, stats, dP, K)))
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                               b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))
    for b in range(B):
        P1, s1 = _ssm_fwd(l[b:b + 1].contiguous(), K)
        d1 = _ssm_bwd(l[b:b + 1].contiguous(), s1, dP[b:b + 1].contiguous(), K)
        assert torch.equal(P1, runs[0][0][b:b + 1]) and torch.equal(s1, runs[0][1][b:b + 1])
        assert torch.equal(d1.view(torch.int32), runs[0][2][b:b + 1].view(torch.int32))


# ---------------------------------------------------------------------------------------------------- module level
@pytest.mark.parametrize("K", [19, 150])
def test_spatial_gather_fn_vs_float64(cuda, K):
    from torchseg_b200 import ops
    B, C, h, w = 2, 512, 13, 11
    g = torch.Generator(device=cuda).manual_seed(K)
    f = ops.to_nhwc(torch.randn(B, C, h, w, device=cuda, generator=g)).requires_grad_(True)
    lcs = (K + 31) // 32 * 32
    lbuf = ops.nhwc_zeros(B, K, h, w, dtype=torch.float32, device=cuda, cs=lcs)
    with torch.no_grad():
        lbuf.copy_(torch.randn(B, K, h, w, device=cuda, generator=g) * 3)
    logits = lbuf.requires_grad_(True)
    ctx = ops.SpatialGatherFn.apply(f, logits, K)
    assert tuple(ctx.shape) == (B, C, K, 1) and ctx.dtype == torch.bfloat16
    gy = torch.randn(B, C, K, 1, device=cuda, generator=g)
    ctx.backward(ops.to_nhwc(gy))
    torch.cuda.synchronize()
    f64 = f.detach().double().requires_grad_(True)
    l64 = logits.detach().double().requires_grad_(True)
    P = torch.softmax(l64.reshape(B, K, -1), dim=2)
    ref = torch.matmul(P, f64.reshape(B, C, -1).transpose(1, 2)).transpose(1, 2).unsqueeze(3)
    ref.backward(gy.double())
    assert norm_err(ctx, ref.detach()) < 6e-3, norm_err(ctx, ref.detach())
    assert norm_err(f.grad, f64.grad) < 1e-2, norm_err(f.grad, f64.grad)
    assert norm_err(logits.grad, l64.grad) < 1.5e-2, norm_err(logits.grad, l64.grad)


def _close(a, emu, ref32, tol, slack):
    """a within tol of the emulating oracle, or no farther from the fp32 oracle than 1.5x the emulation is (+slack)"""
    return norm_err(a, emu) < tol or norm_err(a, ref32) <= 1.5 * norm_err(emu, ref32) + slack


def _teacher_forced(cuda, mod, fn, prefix, x, proxy, gy):
    """module(x, proxy) vs the bf16-emulating oracle: output, both input gradients and parameter gradients (norm),
    each within 1e-2 / 2e-2 of the emulation or within 1.5x the distance between the fp32 oracle and its emulation.
    The OCR block is sensitive to bf16 storage itself: f_object's and f_down's BatchNorm normalise over the B·K region
    proxies, which are soft averages over many pixels and differ little, so their bf16 rounding is amplified (the fp32
    oracle and its emulation differ by ~1.4 % in the block's output)."""
    import torchseg_b200
    from torchseg_b200 import ops
    import ocrnet_oracle as tr
    sd = {prefix + "." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for kk, vv in sd.items():
        if vv.is_floating_point() and "running" not in kk:
            vv.requires_grad_(True)
    x32, p32 = x.clone().requires_grad_(True), proxy.clone().requires_grad_(True)
    y32 = fn(x32, p32, sd, prefix, stats={})
    (y32 * gy).sum().backward()
    ref32 = {kk: vv.grad.clone() for kk, vv in sd.items() if vv.grad is not None}
    for vv in sd.values():
        vv.grad = None
    xr, pr = x.clone().requires_grad_(True), proxy.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = fn(xr, pr, sd, prefix, stats={})
        (yr * gy).sum().backward()
    finally:
        tr.set_bf16_emulation(False)
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    pd = ops.to_nhwc(proxy.to(cuda)).requires_grad_(True)
    y = mod(xd, pd)
    y.backward(ops.to_nhwc(gy.to(cuda)))
    torch.cuda.synchronize()
    assert _close(y, yr.detach(), y32.detach(), 1e-2, 2e-3), (norm_err(y, yr), norm_err(yr, y32))
    assert _close(xd.grad, xr.grad, x32.grad, 2e-2, 2e-3), (norm_err(xd.grad, xr.grad), norm_err(xr.grad, x32.grad))
    assert _close(pd.grad, pr.grad, p32.grad, 2e-2, 2e-3), (norm_err(pd.grad, pr.grad), norm_err(pr.grad, p32.grad))
    for n, p in mod.named_parameters():
        emu = sd[prefix + "." + n].grad
        assert float(emu.norm()) > 0, n
        assert _close(p.grad, emu, ref32[prefix + "." + n], 2e-2, 1e-2), (n, norm_err(p.grad, emu))


def test_object_attention_block_teacher_forced(cuda):
    """B·K = 38: the 1x1 ConvBnRelu of f_object and f_down run on the 2 x 19 region proxies"""
    from torchseg_b200.seg_opr.seg_oprs import ObjectAttentionBlock
    import ocrnet_oracle as tr
    torch.manual_seed(0)
    mod = ObjectAttentionBlock(512, 256)
    g = torch.Generator().manual_seed(1)
    x = bf16_round(torch.relu(torch.randn(2, 512, 21, 19, generator=g)))
    proxy = bf16_round(torch.randn(2, 512, 19, 1, generator=g))
    gy = torch.randn(2, 512, 21, 19, generator=g)
    _teacher_forced(cuda, mod, tr.object_attention, "m", x, proxy, gy)


def test_spatial_ocr_module_teacher_forced(cuda):
    from torchseg_b200.seg_opr.seg_oprs import SpatialOCRModule
    import ocrnet_oracle as tr
    torch.manual_seed(2)
    mod = SpatialOCRModule(512, 256, 512, dropout=0.0)
    g = torch.Generator().manual_seed(3)
    x = bf16_round(torch.relu(torch.randn(2, 512, 17, 17, generator=g)))
    proxy = bf16_round(torch.randn(2, 512, 19, 1, generator=g))
    gy = torch.randn(2, 512, 17, 17, generator=g)
    _teacher_forced(cuda, mod, tr.spatial_ocr, "m", x, proxy, gy)


# ------------------------------------------------------------------------------------------------------- step level
def _build(cuda, N=2, H=129, W=129, seed=0, criterion=None, classes=19, ignore=255):
    import torchseg_b200
    from torchseg_b200.networks import OCRNet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(seed)
    crit = torch.nn.CrossEntropyLoss(ignore_index=ignore) if criterion is None else criterion
    model = OCRNet(classes, crit, norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.spatial_ocr_head.conv_bn_dropout[1].p = 0.0
    model.dsn_head[1].p = 0.0
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = torch.randint(0, classes, (N, H, W), generator=g)
    y[:, :5] = ignore
    return model, sd, x, y


_HEAD = ("head.weight", "head.bias", "dsn_head.2.weight", "dsn_head.2.bias")


def _step_vs_oracle(cuda, model, sd, x, y, loss_fn):
    """one training step against the fp32 oracle and its bf16-storage emulation. The randomly initialised OCR head is
    sensitive to bf16 storage itself: the region proxies are soft averages over many pixels that differ little, and
    f_object's and f_down's BatchNorm renormalise their differences. At 2 x 129² the fp32 oracle and its emulation
    differ by ~1.4 % in the loss and by cos 0.73-0.86 in the classifiers' gradients. So the step is held to what bf16
    storage allows: the loss within 1e-2 of the emulation's; each classifier gradient's direction no farther from the
    fp32 oracle's than the emulation's is, less 0.1 (or within cos 0.9 of the emulation's); and, as in
    net_checks.check_step_vs_oracle, every weight's gradient magnitude within ±33 % of either oracle's, all finite. A
    weight whose two oracles already disagree by more than 10 % in magnitude (the dsn head's 3x3 conv, f_down, f_up
    here: up to a factor 2) may instead lie anywhere in the span of the two, widened by 1.5x."""
    from oracle.torch_ref import set_bf16_emulation
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    ref = []
    for emulate in (False, True):
        set_bf16_emulation(emulate)
        try:
            loss_ref, _ = loss_fn(x, y, sd)
            loss_ref.backward()
        finally:
            set_bf16_emulation(False)
        ref.append((loss_ref.item(), {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}))
        for v in sd.values():
            v.grad = None
    (l32, g32), (lemu, gemu) = ref
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - lemu) < 1e-2 * abs(lemu), (loss.item(), lemu, l32)

    def cos(a, b):
        a, b = a.float().cpu().reshape(-1), b.float().cpu().reshape(-1)
        return float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
    P = dict(model.named_parameters())
    for n in _HEAD:
        c32, cemu, c_emu32 = cos(P[n].grad, g32[n]), cos(P[n].grad, gemu[n]), cos(gemu[n], g32[n])
        assert c32 > c_emu32 - 0.1 or cemu > 0.9, (n, c32, cemu, c_emu32)
    bad = []
    for n, p in P.items():
        assert bool(torch.isfinite(p.grad).all()), n
        if p.dim() >= 2:
            gn = float(p.grad.float().norm().cpu())
            r_emu, r_ref = (gn / float(o[n].norm().clamp_min(1e-30)) for o in (gemu, g32))
            e = r_ref / r_emu   # |emulation's| / |fp32 oracle's|
            spread = abs(e - 1) > 0.1 and min(1.0, e) / 1.5 < r_ref < max(1.0, e) * 1.5
            if not (0.75 < r_emu < 1.33 or 0.75 < r_ref < 1.33 or spread):
                bad.append((n, round(r_emu, 3), round(r_ref, 3)))
    assert not bad, "|grad| / |emulating oracle's|, / |fp32 oracle's|: %s" % bad[:10]


def test_ocrnet_step_matches_oracle(cuda):
    """2 x 129² (a ragged 17 x 17 map, K = 19 regions) against the fp32 oracle and its bf16-storage emulation"""
    import ocrnet_oracle as tr
    model, sd, x, y = _build(cuda)
    _step_vs_oracle(cuda, model, sd, x, y, tr.ocrnet_loss)


def test_ocrnet_150_class_ignore_minus_one_step_matches_oracle(cuda):
    """150 classes (Kp = 192, Nk = 150), ignore −1, through head_loss"""
    import ocrnet_oracle as tr
    model, sd, x, y = _build(cuda, classes=150, ignore=-1, seed=4)
    _step_vs_oracle(cuda, model, sd, x, y, lambda a, b, s: tr.ocrnet_loss(a, b, s, ignore_label=-1))


def _groups(model):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return groups


def test_ocrnet_train_steps_decrease_loss_and_reproduce(cuda):
    from torchseg_b200 import optim

    def make():
        model, _, x, y = _build(cuda, N=2, H=97, W=113, seed=3)
        return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_train_reproducible(make)


def test_ocrnet_graphed_step_matches_eager_and_runs_no_aten_gemm(cuda):
    from torchseg_b200 import optim
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d

    def make():
        crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=2 * 96 * 96 // 16)
        model, _, x, y = _build(cuda, N=2, H=96, W=96, seed=7, criterion=crit)
        return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_graphed_matches_eager(make, kernels=("attn_fwd_kernel", "attn_bwd_kv_kernel", "attn_bwd_q_kernel",
                                               "attn_delta_kernel", "ssm_partial_kernel", "ssm_apply_kernel",
                                               "ssm_bwd_partial_kernel", "ssm_bwd_apply_kernel"),
                                extra_aten=("aten::scaled_dot_product", "aten::_scaled_dot_product",
                                            "aten::_flash_attention", "aten::_efficient_attention", "aten::softmax",
                                            "aten::_softmax"),
                                extra_libs=("flash", "fmha"))


def test_ocrnet_full_size_step_runs(cuda):
    """the Cityscapes shape: 8 x 769², 19 classes, OHEM; one training step with a finite loss and finite, non-zero
    gradients in the object attention and the dsn classifier"""
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=8 * 769 * 769 // 16)
    model, _, _, _ = _build(cuda, N=1, H=64, W=64, seed=9, criterion=crit)
    g = torch.Generator(device=cuda).manual_seed(0)
    x = torch.randn(8, 3, 769, 769, device=cuda, generator=g)
    y = torch.randint(0, 19, (8, 769, 769), device=cuda, generator=g)
    loss = model(x, y)
    loss.backward()
    torch.cuda.synchronize()
    assert loss.item() == loss.item()
    blk = model.spatial_ocr_head.object_context_block
    params = [c.conv.weight for c in (*blk.f_pixel, *blk.f_object, blk.f_down, blk.f_up)]
    for p in params + [model.dsn_head[2].weight]:
        assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().max()) > 0


def test_ocrnet_eval_forward_matches_oracle_and_sliding_eval(cuda):
    from torchseg_b200.networks import OCRNet
    import ocrnet_oracle as tr
    check_eval_vs_oracle_and_sliding(cuda, lambda: OCRNet(19, None), tr.ocrnet_eval, 19)
