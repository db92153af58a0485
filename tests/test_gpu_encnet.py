"""EncNet on the H100: the Encoding kernels (tsb_encoding_{fwd,bwd}) against float64 autograd of the direct form, the
channel mean and the SE-loss kernels, EncModule teacher-forced against the bf16-emulating oracle, and the whole training
and eval step against the fp32 oracle (tests/encnet_oracle.py on the blocks of oracle/torch_ref.py, pinned to the live
reference composition by tests/test_cpu_encnet.py)."""
import pytest
import torch
import torch.nn.functional as F

from util import norm_err, bf16_round

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d

# (B, h, w, K, D, channel stride of x, saturating scales): one pixel, odd maps, 3600 pixels (many CTAs per image and
# tiles per CTA), channel slices of wider buffers, every K instance
ENC_CASES = [(1, 1, 1, 8, 64, 64, False), (1, 61, 59, 32, 512, 512, False), (16, 60, 60, 8, 64, 72, False),
             (2, 60, 60, 32, 512, 520, False), (16, 61, 59, 32, 64, 64, False), (2, 37, 41, 24, 192, 200, False),
             (3, 23, 29, 16, 128, 128, False), (2, 60, 60, 32, 512, 512, True)]


def _ordered(t):
    i = t.view(torch.int16).int()
    return torch.where(i < 0, -(i & 0x7FFF), i)


def _within_bf16_ulp(got, ref64):
    """got (bf16) within one bf16 ulp of ref64 rounded to bf16 (adjacent bf16 values); results closer to 0 than 2^-10 of
    the largest are held to the ulp at that floor instead (the fp32 rounding of a cancelling sum of K terms). Returns the
    number of elements outside."""
    ref = ref64.double()
    floor = float(ref.abs().max()) * 2.0 ** -10
    ulp_floor = 2.0 ** (torch.floor(torch.log2(torch.tensor(max(floor, 1e-30)))).item() - 7)
    steps = (_ordered(got) - _ordered(ref.float().to(torch.bfloat16))).abs()
    small = (ref.abs() < floor) & ((got.double() - ref).abs() <= ulp_floor)
    return int(((steps > 1) & ~small).sum())


def _enc_ref(x64, c64, s64, dE64):
    """float64 autograd of the direct form: (a, d², E [B, K, D]) and the gradients of E·dE"""
    B, D = x64.shape[:2]
    X = x64.reshape(B, D, -1).transpose(1, 2)
    R = X.unsqueeze(2) - c64[None, None]
    d2 = R.pow(2).sum(3)
    A = F.softmax(s64[None, None] * d2, dim=2)
    E = (A.unsqueeze(3) * R).sum(1)
    E.backward(dE64)
    return A.detach(), d2.detach(), E.detach()


@pytest.mark.parametrize("case", ENC_CASES, ids=["B%dh%dw%dK%dD%dcs%d%s" % (c[:6] + ("_sat" if c[6] else "",))
                                                 for c in ENC_CASES])
def test_encoding_kernels_vs_float64(cuda, case):
    from torchseg_b200 import ops
    B, h, w, K, D, cs, sat = case
    N = h * w
    g = torch.Generator().manual_seed(B * 7 + N + K + D)
    x = bf16_round(torch.randn(B, D, h, w, generator=g) * 0.5)
    c = torch.randn(K, D, generator=g) * 0.5
    c[0] = x[0, :, 0, 0]                    # a pixel equal to a codeword: d² = 0
    s = -(torch.rand(K, generator=g) * (1.0 if sat else 4.0 / D)) - (1.0 if sat else 0.0)
    dE = bf16_round(torch.randn(B, K, D, generator=g))
    x64 = x.double().to(cuda).requires_grad_(True)
    c64 = c.double().to(cuda).requires_grad_(True)
    s64 = s.double().to(cuda).requires_grad_(True)
    A, d2r, Er = _enc_ref(x64, c64, s64, dE.double().to(cuda))
    xb = torch.zeros(B, h, w, cs, dtype=torch.bfloat16, device=cuda)
    xb[..., :D] = x.permute(0, 2, 3, 1).to(cuda, torch.bfloat16)
    xv = xb[..., :D].permute(0, 3, 1, 2)
    cd, sd = c.to(cuda).contiguous(), s.to(cuda).contiguous()
    dEd = dE.to(cuda, torch.bfloat16).permute(0, 2, 1).contiguous()    # [B·D rows][K]
    s_ = ops.stream()
    outs = []
    for _ in range(2):
        a = torch.empty(B * N, K, device=cuda)
        d2 = torch.empty(B * N, K, device=cuda)
        sa = torch.empty(B, K, device=cuda)
        E = torch.empty(B * D, K, dtype=torch.bfloat16, device=cuda)
        ops.call("tsb_encoding_fwd", xb.data_ptr(), cs, B, N, D, cd.data_ptr(), sd.data_ptr(), K, a.data_ptr(),
                 d2.data_ptr(), sa.data_ptr(), E.data_ptr(), *ops.det_ws(), s_)
        dx = torch.full((B, h, w, cs), 7.0, dtype=torch.bfloat16, device=cuda)
        dc = torch.zeros(K, D, device=cuda)
        ds = torch.zeros(K, device=cuda)
        ops.call("tsb_encoding_bwd", dEd.data_ptr(), xb.data_ptr(), cs, B, N, D, cd.data_ptr(), sd.data_ptr(), K,
                 a.data_ptr(), d2.data_ptr(), sa.data_ptr(), dx.data_ptr(), cs, dc.data_ptr(), ds.data_ptr(),
                 *ops.det_ws(), s_)
        outs.append((a, d2, sa, E, dx, dc, ds))
    torch.cuda.synchronize()
    for u, v in zip(*outs):
        assert torch.equal(u.view(torch.int16 if u.dtype == torch.bfloat16 else torch.int32),
                           v.view(torch.int16 if v.dtype == torch.bfloat16 else torch.int32)), "run to run"
    a, d2, sa, E, dx, dc, ds = outs[0]
    # a moves by a(1 − a)·ΔL <= ΔL / 4 under an error ΔL of the fp32 logit L = s_k·d²_ik: 1e-6 plus a few fp32 ulps of the
    # largest |L| (that term only matters where large |s| saturates the soft-max)
    L = float((s64[None, None] * d2r).abs().max())
    assert float((a.double() - A.reshape(B * N, K)).abs().max()) <= 1e-6 + L * 2.0 ** -21 / 4
    assert float(d2.view(B, N, K)[0, 0, 0]) == 0.0
    assert float((sa.double() - A.sum(1)).abs().max()) <= 1e-6 * N
    Eref = Er.permute(0, 2, 1).reshape(B * D, K)
    assert _within_bf16_ulp(E, Eref) == 0, _within_bf16_ulp(E, Eref)
    dxr = x64.grad.permute(0, 2, 3, 1)
    assert _within_bf16_ulp(dx[..., :D], dxr) == 0, _within_bf16_ulp(dx[..., :D], dxr)
    assert bool((dx[..., D:] == 7.0).all()), "channels past D were written"
    assert norm_err(dc, c64.grad) <= 1e-5, norm_err(dc, c64.grad)
    if sat:   # a saturated soft-max makes g (hence dscale) vanish: both sides are rounding noise
        assert float((ds.double() - s64.grad).abs().max()) <= 1e-5 * float(c64.grad.norm())
    else:
        assert norm_err(ds, s64.grad) <= 1e-5, norm_err(ds, s64.grad)


def test_encoding_fwd_without_saved_assignments(cuda):
    """inference (a, d² NULL): the same E and Σa bits as the training form"""
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = ops.to_nhwc(bf16_round(torch.randn(2, 64, 13, 17, generator=g)).to(cuda))
    c, s = (torch.randn(8, 64, generator=g) * 0.3).to(cuda), -torch.rand(8, generator=g).to(cuda) * 0.1
    E1 = ops.encoding_infer(x, c, s)
    E2 = ops.EncodingFn.apply(x, c, s)
    torch.cuda.synchronize()
    assert torch.equal(E1.view(torch.int16), E2.view(torch.int16)) and tuple(E1.shape) == (2, 8, 64, 1)


def test_chan_mean_exact(cuda):
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randint(-8, 9, (3, 32, 50, 1), generator=g).float()
    xd = ops.to_nhwc(x.to(cuda))
    y = ops.ChanMeanFn.apply(xd.requires_grad_(True))
    dy = torch.randint(-8, 9, (3, 50, 1, 1), generator=g).float()
    y.backward(dy.to(cuda, torch.bfloat16))
    torch.cuda.synchronize()
    assert torch.equal(y.float().cpu().reshape(3, 50), bf16_round(x.mean(1).reshape(3, 50)))
    assert torch.equal(xd.grad.float().cpu(), (dy.reshape(3, 1, 50, 1) / 32).expand(3, 32, 50, 1))


def _se_ref(z, label, C):
    pres = torch.stack([torch.histc(l.double(), bins=C, min=0, max=C - 1) > 0 for l in label]).double()
    z64 = z.double().requires_grad_(True)
    loss = torch.nn.BCELoss()(torch.sigmoid(z64), pres)
    loss.backward()
    return pres, loss.detach(), z64.grad


@pytest.mark.parametrize("B, C, hw", [(2, 150, (37, 41)), (16, 150, (60, 60)), (3, 19, (64, 64)), (1, 33, (5, 7))])
def test_se_loss_vs_float64(cuda, B, C, hw):
    """presence exact against torch.histc with labels −1, 255, C−1 and absent classes; loss and gradient within 1e-6 of
    float64 BCELoss(sigmoid(z)), with logits up to ±200 where the −100 log clamp decides"""
    from torchseg_b200 import ops
    g = torch.Generator().manual_seed(B * C)
    label = torch.randint(-1, C // 2, (B,) + hw, generator=g)
    label[:, 0, :3] = torch.tensor([255, C - 1, -1])
    label[0, 1, 0] = C + 3
    z = torch.randn(B, C, generator=g) * 4
    z.view(-1)[::7] = torch.linspace(-200, 200, z.view(-1)[::7].numel())
    pres, lref, gref = _se_ref(z, label, C)
    zs = (C + 31) // 32 * 32
    zd = torch.zeros(B, zs, device=cuda)
    zd[:, :C] = z.to(cuda)
    nw = (C + 31) // 32
    presence = torch.empty(B, nw, dtype=torch.int32, device=cuda)
    loss = torch.empty((), device=cuda)
    dz = torch.zeros(B, zs, device=cuda)
    ld = label.to(cuda)
    ops.call("tsb_se_loss_fwd_bwd", ld.data_ptr(), B, hw[0] * hw[1], zd.data_ptr(), zs, C, presence.data_ptr(),
             loss.data_ptr(), dz.data_ptr(), zs, ops.stream())
    torch.cuda.synchronize()
    bits = presence.cpu().view(torch.int32)
    got = torch.tensor([[(int(bits[b, c // 32]) >> (c % 32)) & 1 for c in range(C)] for b in range(B)]).double()
    assert torch.equal(got, pres)
    assert abs(float(loss) - float(lref)) <= 1e-6 * max(1.0, abs(float(lref)))
    assert float((dz[:, :C].double().cpu() - gref).abs().max()) <= 1e-6
    # the autograd wrapper, inside a captured graph (no host synchronisation)
    zn = torch.zeros(B, 1, 1, zs, device=cuda)
    zn[..., :C] = z.to(cuda).reshape(B, 1, 1, C)
    zin = zn[..., :C].permute(0, 3, 1, 2)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        ops.SELossFn.apply(zin, ld, C)           # warm-up outside the capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=st):
            out = ops.SELossFn.apply(zin, ld, C)
    graph.replay()
    torch.cuda.synchronize()
    assert float(out) == float(loss)


# ----------------------------------------------------------------------------------------------------- module level
def test_encmodule_teacher_forced(cuda):
    """train: y, SE logits, df and the running statistics within 1e-2 (norm) of the bf16-emulating oracle; every parameter
    gradient within 2e-2 of it, or within 1.5x the distance between the fp32 oracle and its bf16-storage emulation
    (+1e-2) of the fp32 oracle: dscale = Σ g d² cancels heavily and follows the bf16 rounding of dE, as the ASPP's
    gradients do (DESIGN §5). The oracle computes relu(f + f·γ), the module f·(1 + γ). Eval (no_grad): within 1e-2 of the
    oracle's eval"""
    import torchseg_b200
    from torchseg_b200 import ops
    from torchseg_b200.networks.encnet import EncModule
    import encnet_oracle as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(5)
    mod = EncModule(512, 150)
    with torch.no_grad():   # codewords and smoothing factors that leave the soft-max unsaturated, so dscale is not noise
        mod.encoding.codewords.copy_(torch.randn(32, 512, generator=g) * 0.5 + 0.5)
        mod.encoding.scale.copy_(-torch.rand(32, generator=g) * (4.0 / 512))
    sd = {"m." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    f = bf16_round(torch.relu(torch.randn(4, 512, 23, 19, generator=g)))
    gy = torch.randn(4, 512, 23, 19, generator=g)
    gse = torch.randn(4, 150, generator=g)
    fp = f.clone().requires_grad_(True)
    yp, sep = tr.enc_module(fp, sd, "m", stats={})
    (yp * gy).sum().add((sep * gse).sum()).backward()
    ref32 = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    fr = f.clone().requires_grad_(True)
    stats = {}
    tr.set_bf16_emulation(True)
    try:
        yr, ser = tr.enc_module(fr, sd, "m", stats=stats)
        (yr * gy).sum().add((ser * gse).sum()).backward()
    finally:
        tr.set_bf16_emulation(False)
    fd = ops.to_nhwc(f.to(cuda)).requires_grad_(True)
    y, se = mod(fd)
    torch.autograd.backward([y, se], [ops.to_nhwc(gy.to(cuda)), gse.reshape(4, 150, 1, 1).to(cuda)])
    torch.cuda.synchronize()
    assert norm_err(y, yr) < 1e-2, norm_err(y, yr)
    assert norm_err(se.reshape(4, 150), ser) < 1e-2, norm_err(se.reshape(4, 150), ser)
    # where f = 0 the oracle's relu(f + f·γ) passes no gradient and f·(1 + γ) does; in the network f is conv5's ReLU
    # output, whose backward zeroes exactly those positions, so the two agree wherever f > 0
    live = (f > 0).to(cuda)
    assert norm_err(fd.grad * live, fr.grad.to(cuda) * live) < 1e-2, norm_err(fd.grad * live, fr.grad.to(cuda) * live)
    for n, p in mod.named_parameters():
        emu = sd["m." + n].grad
        e = norm_err(p.grad, emu)
        assert e < 2e-2 or norm_err(p.grad, ref32["m." + n]) <= 1.5 * norm_err(emu, ref32["m." + n]) + 1e-2, (n, e)
    msd = mod.state_dict()
    for k, v in stats.items():
        e = float((msd[k[2:]].float().cpu() - v).abs().max()) / max(float(v.abs().max()), 1e-2)
        assert e < 1e-2, (k, e)
    mod.eval()
    with torch.no_grad():
        ye, _ = mod(fd.detach(), with_se=False)
        sde = {k: v.detach() for k, v in sd.items()}
        sde.update({"m." + k: v.detach().cpu() for k, v in mod.state_dict().items() if "running" in k})
        tr.set_bf16_emulation(True)
        try:
            yre, _ = tr.enc_module(f, sde, "m", training=False, momentum=0.0)
        finally:
            tr.set_bf16_emulation(False)
    assert norm_err(ye, yre) < 1e-2, norm_err(ye, yre)


# ------------------------------------------------------------------------------------------------------- step level
def _build(cuda, N=4, H=80, W=112, seed=0):
    import torchseg_b200
    from torchseg_b200.networks import EncNet
    from torchseg_b200.utils.init_func import init_weight
    import encnet_oracle as tr
    torch.manual_seed(seed)
    model = EncNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1), norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.head.conv6[0].p = 0.0
    model.aux_layer[1].p = 0.0
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    x, y, _ = tr.encnet_case(N=N, HW=H, seed=seed + 1)
    if W != H:
        g = torch.Generator().manual_seed(seed + 1)
        x = torch.randn(N, 3, H, W, generator=g)
        y = torch.randint(-1, 40, (N, H, W), generator=g)
    return model, sd, x, y


def test_encnet_step_matches_oracle(cuda):
    """the bar of the other untrained R101 lines (DESIGN §5): loss within 1e-2 of the fp32 oracle, classifier and SE
    gradient directions (cos > 0.9), per-weight gradient magnitudes (codewords included) within ±33 % of the fp32 oracle's
    or of its bf16-storage emulation's. The smoothing factors are left out: at initialisation d² ≈ ‖x‖² is in the
    hundreds, s_k·d² saturates the soft-max, and g (hence dscale) is rounding noise in every implementation; the kernel
    test above checks dscale where the soft-max is not saturated."""
    import encnet_oracle as tr
    model, sd, x, y = _build(cuda, N=4, H=72, W=88)
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    loss_ref, _ = tr.encnet_loss(x, y, sd)
    loss_ref.backward()
    ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    tr.set_bf16_emulation(True)
    try:
        loss_emu, _ = tr.encnet_loss(x, y, sd)
        loss_emu.backward()
    finally:
        tr.set_bf16_emulation(False)
    emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    P = dict(model.named_parameters())
    for n in ("head.conv6.1.weight", "head.conv6.1.bias", "head.encmodule.selayer.weight",
              "head.encmodule.selayer.bias"):
        a, b = P[n].grad.float().cpu().reshape(-1), ref[n].reshape(-1)
        cos = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        assert cos > 0.9, (n, cos)
    for n, p in P.items():
        assert bool(torch.isfinite(p.grad).all()), n
    assert float(P["head.encmodule.encoding.scale"].grad.abs().max()) > 0.0
    bad = []
    for n, p in P.items():
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


def test_encnet_train_steps_decrease_loss_and_reproduce(cuda):
    """five SGD steps lower the loss, and a second run from the same seed, with the first run's model freed, gives the
    same bits"""
    from torchseg_b200 import optim
    runs = []
    for _ in range(2):
        model, _, x, y = _build(cuda, seed=3)
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


def test_encnet_graphed_step_matches_eager_and_runs_no_aten_gemm(cuda):
    from torch.profiler import ProfilerActivity, profile
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        def make():
            model, _, x, y = _build(cuda, seed=7)
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
                "aten::addmm", "aten::linear")
        bad = [n for n in names if n.startswith(aten) or any(t in n.lower() for t in ("cudnn", "cublas", "cutlass", "xmma",
                                                                                      "gemv"))]
        assert not bad, sorted(set(bad))[:10]
        assert any("enc_fwd_kernel" in n for n in names) and any("enc_bwd_kernel" in n for n in names)
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


def test_encnet_full_size_step_runs(cuda):
    """the ADE shape: 16 x 480², 150 classes, one training step with a finite loss and gradients"""
    model, _, _, _ = _build(cuda, N=1, H=64, W=64, seed=9)
    g = torch.Generator(device=cuda).manual_seed(0)
    x = torch.randn(16, 3, 480, 480, device=cuda, generator=g)
    y = torch.randint(-1, 150, (16, 480, 480), device=cuda, generator=g)
    loss = model(x, y)
    loss.backward()
    torch.cuda.synchronize()
    assert loss.item() == loss.item()
    enc = model.head.encmodule.encoding
    assert bool(torch.isfinite(enc.codewords.grad).all()) and bool(torch.isfinite(enc.scale.grad).all())


def test_encnet_eval_forward_matches_oracle_and_sliding_eval(cuda):
    import numpy as np
    import torchseg_b200
    from torchseg_b200.engine.evaluator import Evaluator
    from torchseg_b200.networks import EncNet
    from torchseg_b200.utils.init_func import init_weight
    import encnet_oracle as tr
    torch.manual_seed(11)
    model = EncNet(150, None)
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
            ref = tr.encnet_eval(x, sd)
    finally:
        tr.set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    with torch.no_grad():
        out = model(x.to(cuda))
    assert tuple(out.shape) == (2, 150, 96, 130) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97
    ev = Evaluator(dataset=None, class_num=150, image_mean=np.array([0.485, 0.456, 0.406]),
                   image_std=np.array([0.229, 0.224, 0.225]), network=None, multi_scales=[0.75, 1.0], is_flip=True,
                   devices=[0], crop_batch=2)
    ev.val_func = model
    img = np.random.default_rng(0).integers(0, 256, (150, 171, 3), dtype=np.uint8)
    host = ev.sliding_eval(img, 128, 2 / 3.0, cuda)
    dev = ev.sliding_eval_device(img, 128, 2 / 3.0, cuda)
    assert np.array_equal(dev.cpu().numpy(), host)
