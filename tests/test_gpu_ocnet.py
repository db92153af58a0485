"""OCNet on the H100: the fused attention kernels (tsb_attention_{fwd,bwd}) against float64 autograd of the
materialised softmax(scale · q kᵀ) v, exact one-hot and uniform cases, channel slices, bounds and determinism; the
attention block and Base-OC module teacher-forced against the bf16-emulating oracle; and the whole training and eval
step against the fp32 oracle (tests/ocnet_oracle.py on the blocks of oracle/torch_ref.py, pinned to the live reference
composition by tests/test_cpu_ocnet.py)."""
import pytest
import torch

from util import norm_err, bf16_round

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d
D = 256
SCALE = D ** -0.5


# ------------------------------------------------------------------------------------------------------- kernels
def _rows(B, N, cs, dev, fill=0.0):
    return torch.full((B, N, cs), fill, dtype=torch.bfloat16, device=dev)


def _fwd(q, k, v, o=None, lse=True, scale=SCALE):
    from torchseg_b200._lib import call, ptr, stream
    B, N = q.shape[:2]
    o = _rows(B, N, D, q.device) if o is None else o
    lse_t = torch.empty((B, N), dtype=torch.float32, device=q.device) if lse else None
    call("tsb_attention_fwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(lse_t), B, N, D, D, float(scale), stream())
    return o, lse_t


def _bwd(q, k, v, o, do, lse, dq=None, dk=None, dv=None, accumulate=False, scale=SCALE):
    from torchseg_b200._lib import call, ptr, stream
    B, N = q.shape[:2]
    dev = q.device
    dq = _rows(B, N, D, dev) if dq is None else dq
    dk = _rows(B, N, D, dev) if dk is None else dk
    dv = _rows(B, N, D, dev) if dv is None else dv
    delta = torch.empty((B, N), dtype=torch.float32, device=dev)
    call("tsb_attention_bwd", ptr(q), q.stride(1), ptr(k), k.stride(1), ptr(v), v.stride(1), ptr(o), o.stride(1),
         ptr(do), do.stride(1), ptr(lse), ptr(delta), ptr(dq), dq.stride(1), ptr(dk), dk.stride(1), ptr(dv),
         dv.stride(1), int(accumulate), B, N, D, D, float(scale), stream())
    return dq, dk, dv


def _ref64(q, k, v, do, shared=False, rows=None):
    """float64 autograd of the materialised form on the same bf16 inputs: (o, lse, dq, dk, dv); shared: k is q and dq is
    the gradient of softmax(q qᵀ) v with respect to q. rows: only these query rows (forward and dq restricted to them)"""
    q64 = q[..., :D].double().requires_grad_(True)
    k64 = q64 if shared else k[..., :D].double().requires_grad_(True)
    v64 = v[..., :D].double().requires_grad_(True)
    qs = q64 if rows is None else q64[:, rows]
    s = torch.matmul(qs, k64.transpose(1, 2)) * SCALE
    o = torch.matmul(torch.softmax(s, -1), v64)
    lse = torch.logsumexp(s, -1)
    g = do[..., :D].double() if rows is None else do[:, rows, :D].double()
    o.backward(g)
    return o.detach(), lse.detach(), q64.grad, (None if shared else k64.grad), v64.grad


def _rand(B, N, dev, g, cs=D):
    t = _rows(B, N, cs, dev, float("nan"))
    t[..., :D] = torch.randn(B, N, D, device=dev, generator=g).to(torch.bfloat16)
    return t


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [1, 37, 64, 100, 1000, 9409])
def test_attention_kernels_vs_float64(cuda, B, N):
    g = torch.Generator(device=cuda).manual_seed(N * 7 + B)
    q, k, v, do = (_rand(B, N, cuda, g) for _ in range(4))
    o, lse = _fwd(q, k, v)
    dq, dk, dv = _bwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    ro, rlse, rdq, rdk, rdv = _ref64(q, k, v, do)
    assert norm_err(o, ro) < 6e-3, norm_err(o, ro)
    assert float((lse.double() - rlse).abs().max()) < 2e-4 * max(1.0, float(rlse.abs().max()))
    if N == 1:
        # one key: P = 1, so o = v and dv = dout exactly, and dS = dout·v − dout·o is 0 up to the fp32 summation order
        assert torch.equal(o, v[..., :D]) and torch.equal(dv, do[..., :D])
        assert float(dq.float().abs().max()) < 1e-4 and float(dk.float().abs().max()) < 1e-4
        return
    for name, a, b in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        assert norm_err(a, b) < 1.5e-2, (name, norm_err(a, b))


@pytest.mark.parametrize("N", [37, 1000])
def test_attention_shared_query_key_gradient(cuda, N):
    """q = k in one buffer and dq == dk with dq_accumulate: the gradient of softmax(q qᵀ) v with respect to q. q is
    scaled down so that the self-score q_i·q_i does not saturate the soft-max (saturated, the exact gradient is smaller
    than the bf16 rounding of o that δ sees, in any implementation)"""
    B = 2
    g = torch.Generator(device=cuda).manual_seed(N)
    q, v, do = (_rand(B, N, cuda, g) for _ in range(3))
    q[..., :D] = (q[..., :D].float() * 0.25).to(torch.bfloat16)
    o, lse = _fwd(q, q, v)
    dqk = _rows(B, N, D, cuda)
    _, _, dv = _bwd(q, q, v, o, do, lse, dq=dqk, dk=dqk, accumulate=True)
    torch.cuda.synchronize()
    ro, _, rdq, _, rdv = _ref64(q, None, v, do, shared=True)
    assert norm_err(o, ro) < 6e-3
    assert norm_err(dqk, rdq) < 1.5e-2, norm_err(dqk, rdq)
    assert norm_err(dv, rdv) < 1.5e-2


def test_attention_32768_sampled_rows(cuda):
    """the whole-image eval size (128 x 256 map): forward, lse and dq on 64 sampled rows"""
    B, N = 1, 32768
    g = torch.Generator(device=cuda).manual_seed(1)
    q, k, v, do = (_rand(B, N, cuda, g) for _ in range(4))
    o, lse = _fwd(q, k, v)
    dq, dk, dv = _bwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    rows = torch.randperm(N, generator=torch.Generator().manual_seed(2))[:64].to(cuda)
    ro, rlse, rdq, _, _ = _ref64(q, k, v, do, rows=rows)
    assert norm_err(o[:, rows], ro) < 6e-3
    assert float((lse[:, rows].double() - rlse).abs().max()) < 2e-4 * max(1.0, float(rlse.abs().max()))
    assert norm_err(dq[:, rows], rdq[:, rows]) < 1.5e-2
    assert bool(torch.isfinite(dk.float()).all()) and bool(torch.isfinite(dv.float()).all())


@pytest.mark.parametrize("N", [37, 100, 200])
def test_attention_one_hot_exact(cuda, N):
    """q_i = 48·e_i, k_perm(i) = 48·e_i: the score gap 48²/16 = 144 makes every other weight underflow to 0 in fp32, so
    o = v[perm], dv = dout[perm⁻¹] and dq = dk = 0 exactly (v, dout small integers: every dot product is exact)"""
    B = 2
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(N)).to(cuda)
    eye = torch.eye(D, device=cuda)[:N] * 48
    q = _rows(B, N, D, cuda)
    k = _rows(B, N, D, cuda)
    q[:] = eye.to(torch.bfloat16)
    k[:, perm] = eye.to(torch.bfloat16)
    g = torch.Generator(device=cuda).manual_seed(3)
    v = torch.randint(-4, 5, (B, N, D), device=cuda, generator=g).to(torch.bfloat16)
    do = torch.randint(-4, 5, (B, N, D), device=cuda, generator=g).to(torch.bfloat16)
    o, lse = _fwd(q, k, v)
    dq, dk, dv = _bwd(q, k, v, o, do, lse)
    torch.cuda.synchronize()
    assert torch.equal(o, v[:, perm])
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(N, device=cuda)
    assert torch.equal(dv, do[:, inv])
    assert int(dq.float().abs().max()) == 0 and int(dk.float().abs().max()) == 0


@pytest.mark.parametrize("N", [64, 128, 4096])
def test_attention_uniform_exact(cuda, N):
    """k = 0: every weight is 1/N, and with small-integer v the output is the exact mean"""
    B = 2
    g = torch.Generator(device=cuda).manual_seed(N)
    q = _rand(B, N, cuda, g)
    k = _rows(B, N, D, cuda)
    v = torch.randint(-8, 9, (B, N, D), device=cuda, generator=g).to(torch.bfloat16)
    o, _ = _fwd(q, k, v)
    torch.cuda.synchronize()
    ref = (v.double().sum(1, keepdim=True) / N).expand(B, N, D).float().to(torch.bfloat16)
    assert torch.equal(o, ref)


def test_attention_channel_slices_and_bounds(cuda):
    """inputs as channel slices of wider buffers whose other channels are NaN give the dense results bit for bit; the
    outputs' other channels and the rows past B·N keep their sentinel"""
    B, N = 2, 333
    g = torch.Generator(device=cuda).manual_seed(4)
    dense = [_rand(B, N, cuda, g) for _ in range(4)]
    o0, lse0 = _fwd(*dense[:3])
    grads0 = _bwd(*dense[:3], o0, dense[3], lse0)
    wide = []
    for t, cs in zip(dense, (264, 512, 320, 272)):
        w = _rows(B, N, cs, cuda, float("nan"))
        w[..., :D] = t
        wide.append(w)
    sentinel = -3.5

    def out_buf(cs):
        buf = torch.full((B * N + 64, cs), sentinel, dtype=torch.bfloat16, device=cuda)
        return buf, buf[:B * N].view(B, N, cs)

    ob, o = out_buf(288)
    o, lse = _fwd(*wide[:3], o=o)
    bufs = [out_buf(cs) for cs in (264, 296, 512)]
    _bwd(*wide[:3], o, wide[3], lse, dq=bufs[0][1], dk=bufs[1][1], dv=bufs[2][1])
    torch.cuda.synchronize()
    assert torch.equal(o[..., :D], o0) and torch.equal(lse, lse0)
    for (buf, view), ref in zip([(ob, o)] + bufs, (o0,) + tuple(grads0)):
        assert torch.equal(view[..., :D], ref)
        assert bool((buf[B * N:] == sentinel).all()) and bool((buf[:, D:] == sentinel).all())


def test_attention_deterministic_and_batch_independent(cuda):
    N = 1500
    g = torch.Generator(device=cuda).manual_seed(6)
    q, k, v, do = (_rand(3, N, cuda, g) for _ in range(4))
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


def test_attention_fn_eval_skips_lse_and_matches_training_forward(cuda):
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(8)
    k = ops.to_nhwc(torch.randn(2, D, 13, 11, device=cuda, generator=g))
    v = ops.to_nhwc(torch.randn(2, D, 13, 11, device=cuda, generator=g))
    with torch.no_grad():
        o_eval = ops.AttentionFn.apply(k, None, v, SCALE)
    kk = k.detach().requires_grad_(True)
    o_train = ops.AttentionFn.apply(kk, None, v, SCALE)
    assert torch.equal(o_eval, o_train.detach())
    o_train.float().sum().backward()
    assert kk.grad is not None and bool(torch.isfinite(kk.grad.float()).all())


# ----------------------------------------------------------------------------------------------------- module level
def _nonzero_w(block):
    import ocnet_oracle as tr
    w, b = tr.nonzero_w(block.W.out_channels, block.W.in_channels)
    with torch.no_grad():
        block.W.weight.copy_(w)
        block.W.bias.copy_(b)


def _teacher_forced(cuda, mod, fn, prefix, x, gy, zero_grad=()):
    """module vs the bf16-emulating oracle: output, input gradient and parameter gradients (norm), the latter within
    2e-2 or within 1.5x the distance between the fp32 oracle and its emulation (+1e-2). Parameters in `zero_grad` have an
    exact gradient of 0, so every implementation returns rounding noise there: they are only checked to be finite."""
    import torchseg_b200
    from torchseg_b200 import ops
    import ocnet_oracle as tr
    sd = {prefix + "." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for kk, vv in sd.items():
        if vv.is_floating_point() and "running" not in kk:
            vv.requires_grad_(True)
    xp = x.clone().requires_grad_(True)
    (fn(xp, sd, prefix, stats={}) * gy).sum().backward()
    ref32 = {kk: vv.grad.clone() for kk, vv in sd.items() if vv.grad is not None}
    for vv in sd.values():
        vv.grad = None
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = fn(xr, sd, prefix, stats={})
        (yr * gy).sum().backward()
    finally:
        tr.set_bf16_emulation(False)
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    y = mod(xd)
    y.backward(ops.to_nhwc(gy.to(cuda)))
    torch.cuda.synchronize()
    assert norm_err(y, yr) < 1e-2, norm_err(y, yr)
    assert norm_err(xd.grad, xr.grad) < 2e-2, norm_err(xd.grad, xr.grad)
    for n, p in mod.named_parameters():
        emu = sd[prefix + "." + n].grad
        if n in zero_grad:
            assert bool(torch.isfinite(p.grad).all()), n
            continue
        assert float(emu.norm()) > 0, n
        e = norm_err(p.grad, emu)
        assert e < 2e-2 or norm_err(p.grad, ref32[prefix + "." + n]) <= 1.5 * norm_err(emu, ref32[prefix + "." + n]) + 1e-2, (n, e)


def test_self_attention_block_teacher_forced(cuda):
    from torchseg_b200.seg_opr.seg_oprs import SelfAttentionBlock
    import ocnet_oracle as tr
    torch.manual_seed(0)
    mod = SelfAttentionBlock(512, 256, 256, 512)
    _nonzero_w(mod)
    g = torch.Generator().manual_seed(1)
    x = bf16_round(torch.relu(torch.randn(2, 512, 21, 19, generator=g)))
    gy = torch.randn(2, 512, 21, 19, generator=g)
    _teacher_forced(cuda, mod, tr.self_attention, "m", x, gy)


def test_base_oc_module_teacher_forced(cuda):
    from torchseg_b200.seg_opr.seg_oprs import BaseOCModule
    import ocnet_oracle as tr
    torch.manual_seed(2)
    mod = BaseOCModule(512, 512, 256, 256, dropout=0.0)
    _nonzero_w(mod.stages[0])
    g = torch.Generator().manual_seed(3)
    x = bf16_round(torch.relu(torch.randn(2, 512, 17, 17, generator=g)))
    gy = torch.randn(2, 512, 17, 17, generator=g)
    # W's bias shifts channels of the concatenation that conv_bn_dropout's 1x1 conv mixes into per-channel shifts, which
    # its BatchNorm removes: the exact gradient is 0 (the attention-block test checks it where it is not)
    _teacher_forced(cuda, mod, tr.base_oc, "m", x, gy, zero_grad=("stages.0.W.bias",))


# ------------------------------------------------------------------------------------------------------- step level
def _build(cuda, N=2, H=129, W=129, seed=0, criterion=None):
    import torchseg_b200
    from torchseg_b200.networks import OCNet
    from torchseg_b200.utils.init_func import init_weight
    import ocnet_oracle as tr
    torch.manual_seed(seed)
    crit = torch.nn.CrossEntropyLoss(ignore_index=255) if criterion is None else criterion
    model = OCNet(19, crit, norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.context[1].conv_bn_dropout[1].p = 0.0
    model.aux_layer[1].p = 0.0
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = torch.randint(0, 19, (N, H, W), generator=g)
    y[:, :5] = 255
    return model, sd, x, y


def test_ocnet_step_matches_oracle(cuda):
    """2 x 129² (a ragged 17 x 17 attention map): loss within 1e-2 of the fp32 oracle, classifier gradient directions
    (cos > 0.9), per-weight gradient magnitudes within ±33 % of the fp32 oracle's or of its bf16-storage emulation's.
    init_weight re-initialises W like every business-layer conv, so the attention backward is exercised."""
    import ocnet_oracle as tr
    model, sd, x, y = _build(cuda)
    assert float(model.context[1].stages[0].W.weight.abs().max()) > 0
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    loss_ref, _ = tr.ocnet_loss(x, y, sd)
    loss_ref.backward()
    ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    tr.set_bf16_emulation(True)
    try:
        loss_emu, _ = tr.ocnet_loss(x, y, sd)
        loss_emu.backward()
    finally:
        tr.set_bf16_emulation(False)
    emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    P = dict(model.named_parameters())
    for n in ("cls.weight", "cls.bias", "aux_layer.2.weight", "aux_layer.2.bias"):
        a, b = P[n].grad.float().cpu().reshape(-1), ref[n].reshape(-1)
        cos = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        assert cos > 0.9, (n, cos)
    bad = []
    for n, p in P.items():
        assert bool(torch.isfinite(p.grad).all()), n
        if p.dim() >= 2:
            gn = float(p.grad.float().norm().cpu())
            r_emu, r_ref = (gn / float(o[n].norm().clamp_min(1e-30)) for o in (emu, ref))
            if not (0.75 < r_emu < 1.33 or 0.75 < r_ref < 1.33):
                bad.append((n, round(r_emu, 3), round(r_ref, 3)))
    assert not bad, "|grad| / |emulating oracle's|, / |fp32 oracle's|: %s" % bad[:10]


def _groups(model):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return groups


def test_ocnet_train_steps_decrease_loss_and_reproduce(cuda):
    from torchseg_b200 import optim
    runs = []
    for _ in range(2):
        model, _, x, y = _build(cuda, N=2, H=97, W=113, seed=3)
        opt = optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4)
        xs, ys = x.to(cuda), y.to(cuda)
        losses = []
        for _ in range(5):
            opt.zero_grad()
            loss = model(xs, ys)
            loss.backward()
            opt.step()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        runs.append((losses, [p.detach().clone() for p in model.parameters()]))
        del model, opt
    (l0, p0), (l1, p1) = runs
    vals = [float(l) for l in l0]
    assert all(v == v for v in vals) and vals[-1] < vals[0], vals
    for a, b in zip(l0, l1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (vals, [float(l) for l in l1])
    for a, b in zip(p0, p1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_ocnet_graphed_step_matches_eager_and_runs_no_aten_gemm(cuda):
    from torch.profiler import ProfilerActivity, profile
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        def make():
            crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=2 * 96 * 96 // 16)
            model, _, x, y = _build(cuda, N=2, H=96, W=96, seed=7, criterion=crit)
            return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

        model, opt, x, y = make()
        eager = []
        for i in range(4):
            opt.zero_grad()
            if i == 3:
                with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                    loss = model(x, y)
                    loss.backward()
                    torch.cuda.synchronize()
            else:
                loss = model(x, y)
                loss.backward()
            opt.step()
            eager.append(loss.detach().clone())
        names = [e.name for e in prof.events()]
        aten = ("aten::conv", "aten::_conv", "aten::cudnn", "aten::mm", "aten::bmm", "aten::baddbmm", "aten::matmul",
                "aten::addmm", "aten::linear", "aten::scaled_dot_product", "aten::_scaled_dot_product",
                "aten::_flash_attention", "aten::_efficient_attention", "aten::softmax", "aten::_softmax")
        bad = [n for n in names if n.startswith(aten) or any(t in n.lower() for t in ("cudnn", "cublas", "cutlass", "xmma",
                                                                                      "gemv", "flash", "fmha"))]
        assert not bad, sorted(set(bad))[:10]
        for k in ("attn_fwd_kernel", "attn_bwd_kv_kernel", "attn_bwd_q_kernel", "attn_delta_kernel"):
            assert any(k in n for n in names), k
        model, opt, x, y = make()
        step = GraphedTrainStep(model, opt, [x, y], warmup=2)
        assert step.graph is not None, step.error
        graphed = [step(x, y).detach().clone() for _ in range(2)]
        torch.cuda.synchronize()
        for a, b in zip(eager[2:], graphed):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), ([float(e) for e in eager],
                                                                           [float(e) for e in graphed])
        step.release()
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())


def test_ocnet_full_size_step_runs(cuda):
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
    blk = model.context[1].stages[0]
    for p in (blk.f_key.conv.weight, blk.f_value.weight, blk.W.weight):
        assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().max()) > 0


def test_ocnet_eval_forward_matches_oracle_and_sliding_eval(cuda):
    import numpy as np
    import torchseg_b200
    from torchseg_b200.engine.evaluator import Evaluator
    from torchseg_b200.networks import OCNet
    from torchseg_b200.utils.init_func import init_weight
    import ocnet_oracle as tr
    torch.manual_seed(11)
    model = OCNet(19, None)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = torch.Generator().manual_seed(12)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) * 1.5 + 0.5)
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = torch.randn(2, 3, 96, 130, generator=g)
    tr.set_bf16_emulation(True)
    try:
        with torch.no_grad():
            ref = tr.ocnet_eval(x, sd)
    finally:
        tr.set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    with torch.no_grad():
        out = model(x.to(cuda))
    assert tuple(out.shape) == (2, 19, 96, 130) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97
    ev = Evaluator(dataset=None, class_num=19, image_mean=np.array([0.485, 0.456, 0.406]),
                   image_std=np.array([0.229, 0.224, 0.225]), network=None, multi_scales=[0.75, 1.0], is_flip=True,
                   devices=[0], crop_batch=2)
    ev.val_func = model
    img = np.random.default_rng(0).integers(0, 256, (150, 171, 3), dtype=np.uint8)
    host = ev.sliding_eval(img, 128, 2 / 3.0, cuda)
    dev = ev.sliding_eval_device(img, 128, 2 / 3.0, cuda)
    assert np.array_equal(dev.cpu().numpy(), host)
