"""DANet on the H100: the fused attention kernels at (d_k, d_v) = (64, 512) against float64 autograd of the materialised
softmax(scale · q kᵀ) v, exact one-hot and uniform cases, channel slices, bounds, determinism and dq_accumulate; the
channel-attention and gamma-residual ops against float64; PAM, CAM and the head teacher-forced against the
bf16-emulating oracle; and the whole training and eval step against the fp32 oracle (tests/danet_oracle.py on the
blocks of oracle/torch_ref.py, pinned to the live reference composition by tests/test_cpu_danet.py)."""
import pytest
import torch

from util import norm_err, bf16_round
from net_checks import (check_step_vs_oracle, check_train_reproducible, check_graphed_matches_eager,
                        check_eval_vs_oracle_and_sliding)

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d
DK, DV = 64, 512
WIDE_KERNELS = ("attn_fwd_wide_kernel", "attn_bwd_dv_wide_kernel", "attn_bwd_ds_wide_kernel", "attn_delta_wide_kernel")


# ------------------------------------------------------------------------------------------------------- kernels
def _rows(B, N, cs, dev, fill=0.0):
    return torch.full((B, N, cs), fill, dtype=torch.bfloat16, device=dev)


def _fwd(q, k, v, o=None, lse=True, scale=1.0):
    from torchseg_b200._lib import call, ptr, stream
    B, N = q.shape[:2]
    o = _rows(B, N, DV, q.device) if o is None else o
    lse_t = torch.empty((B, N), dtype=torch.float32, device=q.device) if lse else None
    call("tsb_attention_fwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(lse_t), B, N, DK, DV, float(scale), stream())
    return o, lse_t


def _bwd(q, k, v, o, do, lse, dq=None, dk=None, dv=None, accumulate=False, scale=1.0):
    from torchseg_b200._lib import call, ptr, stream
    B, N = q.shape[:2]
    dev = q.device
    dq = _rows(B, N, DK, dev) if dq is None else dq
    dk = _rows(B, N, DK, dev) if dk is None else dk
    dv = _rows(B, N, DV, dev) if dv is None else dv
    delta = torch.empty((B, N), dtype=torch.float32, device=dev)
    call("tsb_attention_bwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(do), do.stride(1), ptr(lse), ptr(delta), ptr(dq), dq.stride(1), ptr(dk), dk.stride(1), ptr(dv),
         dv.stride(1), int(accumulate), B, N, DK, DV, float(scale), stream())
    return dq, dk, dv


def _ref64(q, k, v, do, scale=1.0):
    """float64 autograd of the materialised form on the same bf16 inputs: (o, lse, dq, dk, dv)"""
    q64 = q[..., :DK].double().requires_grad_(True)
    k64 = k[..., :DK].double().requires_grad_(True)
    v64 = v[..., :DV].double().requires_grad_(True)
    s = torch.matmul(q64, k64.transpose(1, 2)) * scale
    o = torch.matmul(torch.softmax(s, -1), v64)
    o.backward(do[..., :DV].double())
    return o.detach(), torch.logsumexp(s, -1).detach(), q64.grad, k64.grad, v64.grad


def _rand(B, N, d, dev, g, cs=None, std=1.0):
    t = _rows(B, N, d if cs is None else cs, dev, float("nan"))
    t[..., :d] = (torch.randn(B, N, d, device=dev, generator=g) * std).to(torch.bfloat16)
    return t


def _qkvdo(B, N, dev, g):
    """q, k at std 0.35 (scores of std ~1 at scale 1, DANet's unscaled product), v and dout at std 1"""
    return (_rand(B, N, DK, dev, g, std=0.35), _rand(B, N, DK, dev, g, std=0.35), _rand(B, N, DV, dev, g),
            _rand(B, N, DV, dev, g))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [1, 37, 64, 100, 1000, 9409])
def test_wide_attention_kernels_vs_float64(cuda, B, N):
    g = torch.Generator(device=cuda).manual_seed(N * 11 + B)
    q, k, v, do = _qkvdo(B, N, cuda, g)
    o, lse = _fwd(q, k, v)
    dq, dk, dv = _bwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    ro, rlse, rdq, rdk, rdv = _ref64(q, k, v, do)
    assert norm_err(o, ro) < 6e-3, norm_err(o, ro)
    assert float((lse.double() - rlse).abs().max()) < 2e-4 * max(1.0, float(rlse.abs().max()))
    if N == 1:
        # one key: P = 1, so o = v and dv = dout exactly, and dS = dout·v − dout·o is 0 up to the fp32 summation order
        assert torch.equal(o, v[..., :DV]) and torch.equal(dv, do[..., :DV])
        assert float(dq.float().abs().max()) < 1e-4 and float(dk.float().abs().max()) < 1e-4
        return
    for name, a, b in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        assert norm_err(a, b) < 1.5e-2, (name, norm_err(a, b))


@pytest.mark.parametrize("N", [37, 64])
def test_wide_attention_one_hot_exact(cuda, N):
    """q_i = 12·e_i, k_perm(i) = 12·e_i at scale 1: the score gap 144 makes every other weight underflow to 0 in fp32, so
    o = v[perm], dv = dout[perm⁻¹] and dq = dk = 0 exactly (v, dout small integers: every dot product is exact)"""
    B = 2
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(N)).to(cuda)
    eye = torch.eye(DK, device=cuda)[:N] * 12
    q = _rows(B, N, DK, cuda)
    k = _rows(B, N, DK, cuda)
    q[:] = eye.to(torch.bfloat16)
    k[:, perm] = eye.to(torch.bfloat16)
    g = torch.Generator(device=cuda).manual_seed(3)
    v = torch.randint(-4, 5, (B, N, DV), device=cuda, generator=g).to(torch.bfloat16)
    do = torch.randint(-4, 5, (B, N, DV), device=cuda, generator=g).to(torch.bfloat16)
    o, lse = _fwd(q, k, v)
    dq, dk, dv = _bwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    assert torch.equal(o, v[:, perm])
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(N, device=cuda)
    assert torch.equal(dv, do[:, inv])
    assert int(dq.float().abs().max()) == 0 and int(dk.float().abs().max()) == 0


@pytest.mark.parametrize("N", [64, 128, 4096])
def test_wide_attention_uniform_exact(cuda, N):
    """k = 0: every weight is 1/N, and with small-integer v the output is the exact mean in both value slices"""
    B = 2
    g = torch.Generator(device=cuda).manual_seed(N)
    q = _rand(B, N, DK, cuda, g)
    k = _rows(B, N, DK, cuda)
    v = torch.randint(-8, 9, (B, N, DV), device=cuda, generator=g).to(torch.bfloat16)
    o, _ = _fwd(q, k, v)
    torch.cuda.synchronize()
    ref = (v.double().sum(1, keepdim=True) / N).expand(B, N, DV).float().to(torch.bfloat16)
    assert torch.equal(o, ref)


def test_wide_attention_channel_slices_and_bounds(cuda):
    """inputs as channel slices of wider buffers whose other channels are NaN give the dense results bit for bit; the
    outputs' other channels and the rows past B·N keep their sentinel"""
    B, N = 2, 333
    g = torch.Generator(device=cuda).manual_seed(4)
    dense = list(_qkvdo(B, N, cuda, g))
    o0, lse0 = _fwd(*dense[:3])
    grads0 = _bwd(*dense[:3], o0, dense[3], lse0)
    wide = []
    for t, cs in zip(dense, (72, 128, 520, 576)):
        w = _rows(B, N, cs, cuda, float("nan"))
        w[..., :t.shape[-1]] = t
        wide.append(w)
    sentinel = -3.5

    def out_buf(cs):
        buf = torch.full((B * N + 64, cs), sentinel, dtype=torch.bfloat16, device=cuda)
        return buf, buf[:B * N].view(B, N, cs)

    ob, o = out_buf(544)
    o, lse = _fwd(*wide[:3], o=o)
    bufs = [out_buf(cs) for cs in (80, 136, 528)]
    _bwd(*wide[:3], o, wide[3], lse, dq=bufs[0][1], dk=bufs[1][1], dv=bufs[2][1])
    torch.cuda.synchronize()
    assert torch.equal(o[..., :DV], o0) and torch.equal(lse, lse0)
    for (buf, view), ref in zip([(ob, o)] + bufs, (o0,) + tuple(grads0)):
        d = ref.shape[-1]
        assert torch.equal(view[..., :d], ref)
        assert bool((buf[B * N:] == sentinel).all()) and bool((buf[:, d:] == sentinel).all())


def test_wide_attention_deterministic_and_batch_independent(cuda):
    N = 1500
    g = torch.Generator(device=cuda).manual_seed(6)
    q, k, v, do = _qkvdo(3, N, cuda, g)
    runs = []
    for _ in range(3):
        o, lse = _fwd(q, k, v)
        runs.append((o, lse) + _bwd(q, k, v, o, do, lse))
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)
    for b in range(3):
        sl = [t[b:b + 1].contiguous() for t in (q, k, v, do)]
        o1, lse1 = _fwd(*sl[:3])
        one = (o1, lse1) + _bwd(*sl[:3], o1, sl[3], lse1)
        for a, c in zip(runs[0], one):
            assert torch.equal(a[b:b + 1], c)


def test_wide_attention_dq_accumulate(cuda):
    """dq_accumulate adds dQ onto dq (onto zeros: the plain result bit for bit), and with dq == dk the one buffer holds
    dQ + dK, since dK is finished before dQ is added"""
    B, N = 2, 500
    g = torch.Generator(device=cuda).manual_seed(9)
    q, k, v, do = _qkvdo(B, N, cuda, g)
    o, lse = _fwd(q, k, v)
    dq0, dk0, dv0 = _bwd(q, k, v, o, do, lse)
    dq1, _, _ = _bwd(q, k, v, o, do, lse, dq=_rows(B, N, DK, cuda), accumulate=True)
    both = _rows(B, N, DK, cuda)
    _, _, dv2 = _bwd(q, k, v, o, do, lse, dq=both, dk=both, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(dq1, dq0) and torch.equal(dv2, dv0)
    _, _, rdq, rdk, _ = _ref64(q, k, v, do)
    assert norm_err(both, rdq + rdk) < 1.5e-2, norm_err(both, rdq + rdk)


def test_attention_fn_wide_eval_skips_lse_and_matches_training_forward(cuda):
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(8)
    q = ops.to_nhwc(torch.randn(2, DK, 13, 11, device=cuda, generator=g) * 0.35)
    k = ops.to_nhwc(torch.randn(2, DK, 13, 11, device=cuda, generator=g) * 0.35)
    v = ops.to_nhwc(torch.randn(2, DV, 13, 11, device=cuda, generator=g))
    with torch.no_grad():
        o_eval = ops.AttentionFn.apply(q, k, v, 1.0)
    qq, kk, vv = (t.detach().requires_grad_(True) for t in (q, k, v))
    o_train = ops.AttentionFn.apply(qq, kk, vv, 1.0)
    assert torch.equal(o_eval, o_train.detach()) and tuple(o_train.shape) == (2, DV, 13, 11)
    o_train.float().sum().backward()
    for t in (qq, kk, vv):
        assert t.grad is not None and bool(torch.isfinite(t.grad.float()).all())


# ----------------------------------------------------------------------------------- channel attention, gamma residual
def _cam_ref64(x, gy):
    """float64 CAM product A X (without the residual) and its input gradient for the upstream gy, on the bf16 x"""
    B, C, h, w = x.shape
    X = x.double().reshape(B, C, -1).requires_grad_(True)
    E = torch.bmm(X, X.transpose(1, 2))
    A = torch.softmax(E.max(-1, keepdim=True)[0] - E, -1)
    out = torch.bmm(A, X)
    out.backward(gy.double().reshape(B, C, -1))
    return out.detach().reshape(B, C, h, w), X.grad.reshape(B, C, h, w)


@pytest.mark.parametrize("B,h,w", [(1, 7, 9), (3, 17, 17), (2, 97, 97)])
def test_channel_attention_fn_vs_float64(cuda, B, h, w):
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(B * 100 + h)
    x = bf16_round(torch.randn(B, 512, h, w, generator=g) * (0.6 / (h * w) ** 0.5))
    gy = torch.randn(B, 512, h, w, generator=g)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    out = ops.ChannelAttentionFn.apply(xd)
    out.backward(ops.to_nhwc(gy.to(cuda)))
    torch.cuda.synchronize()
    ro, rdx = _cam_ref64(x, bf16_round(gy))
    assert norm_err(out, ro) < 1e-2, norm_err(out, ro)
    assert norm_err(xd.grad, rdx) < 2e-2, norm_err(xd.grad, rdx)


def test_chan_attn_softmax_kernels_vs_float64_and_symmetric(cuda):
    """A = softmax(rowmax − E) within bf16 rounding of float64; G = −(dẼ + dẼᵀ) exactly symmetric and within bf16
    rounding of float64"""
    from torchseg_b200._lib import call, ptr, stream
    B, C = 3, 512
    g = torch.Generator(device=cuda).manual_seed(12)
    E = torch.randn(B, C, C, device=cuda, generator=g) * 2
    dA = torch.randn(B, C, C, device=cuda, generator=g)
    A = torch.empty(B, C, C, dtype=torch.bfloat16, device=cuda)
    G = torch.empty_like(A)
    rowdot = torch.empty(B, C, device=cuda)
    call("tsb_chan_attn_softmax_fwd", ptr(E), ptr(A), B, C, stream())
    call("tsb_chan_attn_softmax_bwd", ptr(A), ptr(dA), ptr(rowdot), ptr(G), B, C, stream())
    torch.cuda.synchronize()
    E64 = E.double()
    rA = torch.softmax(E64.max(-1, keepdim=True)[0] - E64, -1)
    assert float((A.double() - rA).abs().max()) <= 2 ** -8 * float(rA.abs().max())
    A64 = A.double()
    dt = A64 * (dA.double() - (A64 * dA.double()).sum(-1, keepdim=True))
    rG = -(dt + dt.transpose(1, 2))
    assert torch.equal(G, G.transpose(1, 2))
    assert norm_err(G, rG) < 4e-3, norm_err(G, rG)


def test_gamma_residual_fn_vs_float64_and_reproducible_dgamma(cuda):
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(14)
    x, o, gy = (bf16_round(torch.randn(2, 512, 33, 29, generator=g)) for _ in range(3))
    runs = []
    for _ in range(3):
        gamma = torch.nn.Parameter(torch.full((1,), 0.375, device=cuda))
        xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
        od = ops.to_nhwc(o.to(cuda)).requires_grad_(True)
        y = ops.GammaResidualFn.apply(xd, od, gamma)
        y.backward(ops.to_nhwc(gy.to(cuda)))
        torch.cuda.synchronize()
        runs.append((y.detach(), xd.grad, od.grad, gamma.grad.clone()))
    y, dx, do, dgamma = runs[0]
    ref = 0.375 * o.double() + x.double()
    assert norm_err(y, ref) < 4e-3 and float((y.double().cpu() - ref).abs().max()) <= 2 ** -8 * float(ref.abs().max())
    assert torch.equal(dx.float().cpu(), gy)
    assert torch.equal(do.float().cpu(), bf16_round(0.375 * gy))
    rg = float((gy.double() * o.double()).sum())
    assert abs(float(dgamma) - rg) <= 1e-4 * float((gy.double() * o.double()).abs().sum())
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------- module level
def _teacher_forced(cuda, mod, fn, prefix, x, gys, zero_grad=(), tol_out=1e-2):
    """module vs the bf16-emulating oracle: outputs, input gradient and parameter gradients (norm), the gradients within
    2e-2 or within 1.5x the distance between the fp32 oracle and its emulation (+1e-2). The module's output (a tensor or
    a tuple) is dotted with gys. Parameters in `zero_grad` have an exact gradient of 0, so every implementation returns
    rounding noise there: they are only checked to be finite."""
    import torchseg_b200
    from torchseg_b200 import ops
    import danet_oracle as tr
    sd = {prefix + "." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for kk, vv in sd.items():
        if vv.is_floating_point() and "running" not in kk:
            vv.requires_grad_(True)

    def as_tuple(y):
        return y if isinstance(y, tuple) else (y,)

    def run_oracle(xr):
        ys = as_tuple(fn(xr, sd, prefix))
        sum((y * gy).sum() for y, gy in zip(ys, gys)).backward()
        return ys

    x32 = x.clone().requires_grad_(True)
    run_oracle(x32)
    ref32 = {kk: vv.grad.clone() for kk, vv in sd.items() if vv.grad is not None}
    for vv in sd.values():
        vv.grad = None
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yrs = run_oracle(xr)
    finally:
        tr.set_bf16_emulation(False)
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    ys = as_tuple(mod(xd))
    torch.autograd.backward(ys, [gy.to(cuda) if y.dtype == torch.float32 else ops.to_nhwc(gy.to(cuda))
                                 for y, gy in zip(ys, gys)])
    torch.cuda.synchronize()
    for y, yr in zip(ys, yrs):
        assert norm_err(y, yr) < tol_out, norm_err(y, yr)
    e = norm_err(xd.grad, xr.grad)
    assert e < 2e-2 or norm_err(xd.grad, x32.grad) <= 1.5 * norm_err(xr.grad, x32.grad) + 1e-2, e
    for n, p in mod.named_parameters():
        emu = sd[prefix + "." + n].grad
        if n in zero_grad:
            assert bool(torch.isfinite(p.grad).all()), n
            continue
        assert float(emu.norm()) > 0, n
        e = norm_err(p.grad, emu)
        assert e < 2e-2 or norm_err(p.grad, ref32[prefix + "." + n]) <= 1.5 * norm_err(emu, ref32[prefix + "." + n]) + 1e-2, (n, e)


def _set_gamma(mod, value):
    with torch.no_grad():
        mod.gamma.fill_(value)


def test_pam_module_teacher_forced(cuda):
    from torchseg_b200.seg_opr.seg_oprs import PAM_Module
    import danet_oracle as tr
    torch.manual_seed(0)
    mod = PAM_Module(512)
    _set_gamma(mod, 0.5)
    with torch.no_grad():   # q, k of std ~0.35 as the head's BatchNorm'd input gives them: unsaturated attention
        mod.query_conv.weight.mul_(0.5)
        mod.key_conv.weight.mul_(0.5)
    g = torch.Generator().manual_seed(1)
    x = bf16_round(torch.relu(torch.randn(2, 512, 21, 19, generator=g)))
    gy = torch.randn(2, 512, 21, 19, generator=g)
    # a bias on every key shifts each query's scores by one constant, which the soft-max removes: its exact gradient is 0
    _teacher_forced(cuda, mod, tr.pam, "m", x, (gy,), zero_grad=("key_conv.bias",))


def test_cam_module_teacher_forced(cuda):
    from torchseg_b200.seg_opr.seg_oprs import CAM_Module
    import danet_oracle as tr
    mod = CAM_Module(512)
    _set_gamma(mod, 0.25)
    g = torch.Generator().manual_seed(3)
    x = bf16_round(torch.relu(torch.randn(2, 512, 17, 15, generator=g)) * 0.05)
    gy = torch.randn(2, 512, 17, 15, generator=g)
    _teacher_forced(cuda, mod, tr.cam, "m", x, (gy,))


def test_danet_head_teacher_forced(cuda):
    from torchseg_b200.networks import DANetHead
    import danet_oracle as tr
    torch.manual_seed(4)
    mod = DANetHead(2048, 19)
    for name in ("conv6", "conv7", "conv8"):
        getattr(mod, name)[0].p = 0.0
    _set_gamma(mod.sa, 0.5)
    _set_gamma(mod.sc, 0.25)
    g = torch.Generator().manual_seed(5)
    x = bf16_round(torch.relu(torch.randn(2, 2048, 13, 17, generator=g)))
    gys = tuple(torch.randn(2, 19, 13, 17, generator=g) for _ in range(3))

    def head(xx, sd, prefix):
        return tr.danet_head(xx, sd, prefix, stats={})

    _teacher_forced(cuda, mod, head, "head", x, gys, zero_grad=("sa.key_conv.bias",))


# ------------------------------------------------------------------------------------------------------- step level
def _build(cuda, N=2, H=129, W=129, seed=0, criterion=None):
    import torchseg_b200
    from torchseg_b200.networks import DANet
    from torchseg_b200.utils.init_func import init_weight
    import danet_oracle as tr
    torch.manual_seed(seed)
    crit = torch.nn.CrossEntropyLoss(ignore_index=255) if criterion is None else criterion
    model = DANet(19, crit, norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    for name in ("conv6", "conv7", "conv8"):
        getattr(model.head, name)[0].p = 0.0
    params = dict(model.named_parameters())
    with torch.no_grad():   # DANet zero-initialises both gammas; non-zero, the attention backward is exercised
        for k, v in tr.GAMMAS.items():
            params[k].fill_(v)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = torch.randint(0, 19, (N, H, W), generator=g)
    y[:, :5] = 255
    return model, sd, x, y


def test_danet_step_matches_oracle(cuda):
    """2 x 129² (a ragged 17 x 17 attention map): loss within 1e-2 of the fp32 oracle, classifier gradient directions
    (cos > 0.9), per-weight gradient magnitudes within ±33 % of the fp32 oracle's or of its bf16-storage emulation's"""
    import danet_oracle as tr
    model, sd, x, y = _build(cuda)
    P = check_step_vs_oracle(cuda, model, sd, x, y, tr.danet_loss,
                             ("head.conv8.1.weight", "head.conv8.1.bias", "head.conv6.1.weight", "head.conv7.1.weight"))
    for n in ("head.sa.gamma", "head.sc.gamma"):
        assert float(P[n].grad.abs().max()) > 0, n


def _groups(model, lr=1e-2):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.backbone, BN, lr)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 10 * lr)
    return groups


def test_danet_train_steps_decrease_loss_and_reproduce(cuda):
    """five SGD steps at lr 2e-4 (business layers 2e-3): the loss falls and two seeded runs agree bit for bit. At the
    OCNet test's 1e-2 / 1e-1 this randomly initialised head, with its three summed losses, climbs within five steps"""
    from torchseg_b200 import optim

    def make():
        model, _, x, y = _build(cuda, N=2, H=97, W=113, seed=3)
        return model, optim.SGD(_groups(model, 2e-4), lr=2e-4, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_train_reproducible(make)


def test_danet_graphed_step_matches_eager_and_runs_no_aten_gemm(cuda):
    from torchseg_b200 import optim
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d

    def make():
        crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=2 * 96 * 96 // 16)
        model, _, x, y = _build(cuda, N=2, H=96, W=96, seed=7, criterion=crit)
        return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_graphed_matches_eager(make, kernels=WIDE_KERNELS + ("cam_softmax_fwd_kernel", "cam_softmax_bwd_kernel",
                                                              "gamma_residual_fwd_kernel", "gamma_residual_bwd_kernel"),
                                extra_aten=("aten::scaled_dot_product", "aten::_scaled_dot_product",
                                            "aten::_flash_attention", "aten::_efficient_attention", "aten::softmax",
                                            "aten::_softmax"),
                                extra_libs=("flash", "fmha"))


def test_danet_full_size_step_runs(cuda):
    """the Cityscapes shape: 8 x 769², 19 classes, OHEM; one training step with a finite loss and gradients"""
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
    head = model.head
    for p in (head.sa.query_conv.weight, head.sa.key_conv.weight, head.sa.value_conv.weight, head.sa.gamma,
              head.sc.gamma, head.conv5c.conv.weight):
        assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().max()) > 0


def test_danet_eval_forward_matches_oracle_and_sliding_eval(cuda):
    from torchseg_b200.networks import DANet
    import danet_oracle as tr

    def make():
        model = DANet(19, None)
        params = dict(model.named_parameters())
        with torch.no_grad():
            for k, v in tr.GAMMAS.items():
                params[k].fill_(v)
        return model

    check_eval_vs_oracle_and_sliding(cuda, make, tr.danet_eval, 19)
