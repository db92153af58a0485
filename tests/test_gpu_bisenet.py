"""End-to-end parity of the libtsb BiSeNet-R18 training step against the oracle (oracle/torch_ref.py, pinned to
the live reference).

Two layers of evidence, because a randomly initialised batch-stat BN network amplifies bf16-level noise by
~4x per layer (tools/diag_chain.py, DESIGN.md §parity):
  1. TEACHER-FORCED blocks: every module type of the network gets the oracle's (bf16-exact) inputs and upstream
     gradients; outputs, input gradients and parameter gradients must match the bf16-storage-emulating oracle
     within the 1e-2 bf16 tolerance (observed ~1e-4..1e-3).
  2. WHOLE STEP: the loss matches the fp32 oracle within 1e-2, every parameter gradient stays well aligned
     (cosine) with the oracle's, BN running statistics follow the reference update, the loss decreases under
     the fused SGD.
"""
import pytest
import torch
import torch.nn.functional as F

from util import rel_err, norm_err, make_labels, bf16_round

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d


def _sd_of(mod, prefix="m."):
    sd = {prefix + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    return sd


def _prep(mod, cuda):
    import torchseg_b200
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    return mod


def _check(mod, sd, outs_dev, outs_ref, ins_dev, ins_ref, tol=1e-2):
    for i, (a, b) in enumerate(zip(outs_dev, outs_ref)):
        assert norm_err(a, b) < tol, "output %d: %g" % (i, norm_err(a, b))
    for i, (a, b) in enumerate(zip(ins_dev, ins_ref)):
        if b.grad is not None:
            assert norm_err(a.grad, b.grad) < tol, "input grad %d: %g" % (i, norm_err(a.grad, b.grad))
    for n, p in mod.named_parameters():
        ref = sd["m." + n].grad
        e = norm_err(p.grad, ref)
        assert e < 2 * tol, "param grad %s: %g" % (n, e)


def _rand(shape, g, relu=False):
    t = torch.randn(*shape, generator=g)
    if relu:
        t = torch.relu(t)
    return bf16_round(t)


@pytest.mark.parametrize("cfg", [(64, 64, 3, 1, 1), (64, 128, 3, 2, 1), (64, 128, 1, 1, 0), (3, 64, 7, 2, 3)],
                         ids=["3x3s1", "3x3s2", "1x1", "stem7x7"])
def test_conv_bn_relu_teacher_forced(cuda, cfg):
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr.seg_oprs import ConvBnRelu
    from oracle import torch_ref as tr
    cin, cout, k, st, pd = cfg
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    mod = ConvBnRelu(cin, cout, k, st, pd)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    x = _rand((8, cin, 48, 64), g, relu=cin != 3)
    xr = x.clone().requires_grad_(cin != 3)
    tr.set_bf16_emulation(True)
    try:
        yr = tr.conv_bn_relu(xr, sd, "m", st, pd)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = (ops.to_nhwc(x.to(cuda)) if cin != 3 else x.to(cuda)).requires_grad_(cin != 3)
    yd = mod(xd)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    _check(mod, sd, [yd], [yr], [xd] if cin != 3 else [], [xr] if cin != 3 else [])


@pytest.mark.parametrize("down", [False, True])
def test_basic_block_teacher_forced(cuda, down):
    from torchseg_b200 import ops
    from torchseg_b200.base_model.resnet import BasicBlock
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(2)
    cin, cout, st = (64, 128, 2) if down else (64, 64, 1)
    ds = None
    if down:
        ds = torch.nn.Sequential(torch.nn.Conv2d(cin, cout, 1, st, bias=False), BN(cout))
    mod = BasicBlock(cin, cout, st, BN, 1e-5, 0.1, ds, True)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    x = _rand((8, cin, 32, 32), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = tr.basic_block(xr, sd, "m", st, down, 1e-5, 0.1, True)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = mod(xd)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    _check(mod, sd, [yd], [yr], [xd], [xr])


def test_arm_ffm_teacher_forced(cuda):
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr.seg_oprs import AttentionRefinement, FeatureFusion
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(3)
    arm = AttentionRefinement(256, 128, BN)
    sda = _sd_of(arm)
    _prep(arm, cuda)
    ffm = FeatureFusion(256, 256, 1, BN)
    sdf = _sd_of(ffm)
    _prep(ffm, cuda)
    x = _rand((16, 256, 16, 16), g, relu=True)
    last = _rand((16, 128, 16, 16), g, relu=True)
    x1 = _rand((16, 128, 24, 24), g, relu=True)
    x2 = _rand((16, 128, 24, 24), g, relu=True)
    xr, lr_, x1r, x2r = [t.clone().requires_grad_(True) for t in (x, last, x1, x2)]
    tr.set_bf16_emulation(True)
    try:
        ya = tr.q(tr.attention_refinement(xr, sda, "m", 1e-5, 0.1, True) + lr_)
        ga = _rand(tuple(ya.shape), g)
        ya.backward(ga)
        yf = tr.feature_fusion(x1r, x2r, sdf, "m", 1e-5, 0.1, True)
        gf = _rand(tuple(yf.shape), g)
        yf.backward(gf)
    finally:
        tr.set_bf16_emulation(False)
    xd, ld, x1d, x2d = [ops.to_nhwc(t.to(cuda)).requires_grad_(True) for t in (x, last, x1, x2)]
    yad = arm(xd, add=ld)
    yad.backward(ops.to_nhwc(ga.to(cuda)))
    _check(arm, sda, [yad], [ya], [xd, ld], [xr, lr_], tol=2e-2)
    yfd = ffm(x1d, x2d)
    yfd.backward(ops.to_nhwc(gf.to(cuda)))
    _check(ffm, sdf, [yfd], [yf], [x1d, x2d], [x1r, x2r], tol=2e-2)


def test_head_loss_teacher_forced(cuda):
    """3x3 CBR → 1x1 classifier (+bias) → bilinear x8 → OHEM CE, fused on the device side"""
    from torchseg_b200 import ops
    from torchseg_b200.networks.bisenet import BiSeNetHead
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(4)
    N, h, w, s = 4, 16, 16, 8
    head = BiSeNetHead(128, 19, s, True, BN)
    sd = _sd_of(head)
    _prep(head, cuda)
    labels = make_labels(N, h * s, w * s, 19, 255, g)
    mk = N * h * s * w * s // 16
    crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=mk)
    x = _rand((N, 128, h, w), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        lo = tr.bisenet_head_logits(xr, sd, "m", 1e-5, 0.1, True)
        loss_r = tr.ohem_ce(F.interpolate(lo, scale_factor=s, mode="bilinear", align_corners=True), labels, 255, 0.7, mk)
        loss_r.backward()
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    lod = head.lowres_logits(xd)
    loss_d = crit.forward_lowres(lod, labels.to(cuda), 19)
    loss_d.backward()
    assert abs(loss_d.item() - loss_r.item()) < 2e-3 * abs(loss_r.item())
    _check(head, sd, [lod], [lo], [xd], [xr], tol=2e-2)
    # the reference-boundary form (materialised NCHW fp32 logits through BiSeNetHead.forward + criterion)
    for p in head.parameters():
        p.grad = None
    xd2 = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    loss_m = crit(head(xd2), labels.to(cuda))
    loss_m.backward()
    assert abs(loss_m.item() - loss_r.item()) < 2e-3 * abs(loss_r.item())
    assert norm_err(xd2.grad, xr.grad) < 2e-2


def _build(cuda, N=8, HW=128, seed=0):
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(seed)
    H = W = HW
    crit = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=N * H * W // 16, use_weight=False)
    model = BiSeNet(19, True, crit, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = make_labels(N, H, W, 19, 255, g)
    return model, sd, x, y, N * H * W // 16


def test_bisenet_step_matches_oracle(cuda):
    from oracle import torch_ref
    model, sd, x, y, min_kept = _build(cuda)
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    stats = {}
    loss_ref, _ = torch_ref.bisenet_r18_loss(x, y, sd, min_kept, stats=stats)   # plain fp32 reference
    loss_ref.backward()
    grads_ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    # the same oracle with bf16 STORAGE emulated: |fp32 − emulation| is what the storage policy alone does to each gradient
    torch_ref.set_bf16_emulation(True)
    try:
        loss_emu, _ = torch_ref.bisenet_r18_loss(x, y, sd, min_kept)
        loss_emu.backward()
    finally:
        torch_ref.set_bf16_emulation(False)
    grads_emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    bad, outside = [], []
    for n, p in model.named_parameters():
        a, b, c = p.grad.float().cpu(), grads_ref[n], grads_emu[n]
        af, bf = a.reshape(-1), b.reshape(-1)
        cos = float(torch.dot(af, bf) / (af.norm() * bf.norm()).clamp_min(1e-30))
        ratio = float(af.norm() / bf.norm().clamp_min(1e-30))
        if cos < 0.8 or not (0.7 < ratio < 1.4):
            bad.append((n, round(cos, 3), round(ratio, 3)))
        # every conv / classifier weight: as close to the fp32 oracle as the bf16-storage emulation is (x1.5 + 2e-2)
        if p.dim() == 4:
            e, spread = norm_err(a, b), norm_err(c, b)
            if e > 1.5 * spread + 2e-2:
                outside.append((n, round(e, 4), round(spread, 4)))
    assert not bad, "gradient direction / magnitude off: %s" % bad[:10]
    assert not outside, "gradient farther from the fp32 oracle than 1.5 x the bf16-storage spread + 2e-2: %s" % outside[:10]
    msd = model.state_dict()
    for k, v in stats.items():   # running stats: momentum 0.1, unbiased variance (SURVEY App. A3)
        assert rel_err(msd[k], v) < 3e-2, k


def test_bisenet_train_steps_decrease_loss(cuda):
    """optimiser steps with the fused flat SGD: loss decreases, parameters stay finite"""
    from torchseg_b200 import optim
    from torchseg_b200.utils.init_func import group_weight
    model, sd, x, y, _ = _build(cuda, N=4, HW=128, seed=3)
    groups = group_weight([], model.context_path, BN, 1e-2)
    for m in (model.spatial_path, model.global_context, model.arms, model.refines, model.heads, model.ffm):
        groups = group_weight(groups, m, BN, 1e-1)
    opt = optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)
    xs, ys = x.to(cuda), y.to(cuda)
    losses = []
    for it in range(5):
        opt.zero_grad()
        loss = model(xs, ys)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(l == l for l in losses)
    assert losses[-1] < losses[0], losses
    for p in model.parameters():
        assert torch.isfinite(p).all()


def test_bottleneck_dilated_teacher_forced(cuda):
    """Bottleneck (1x1 → dilated 3x3 → 1x1 + residual) as rewritten by PSPNet._nostride_dilate (dilation 2)"""
    from torchseg_b200 import ops
    from torchseg_b200.base_model.resnet import Bottleneck
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(6)
    mod = Bottleneck(256, 64, 1, BN, 1e-5, 0.1, None, True)
    mod.conv2.dilation, mod.conv2.padding = (2, 2), (2, 2)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    x = _rand((8, 256, 24, 24), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = tr.bottleneck(xr, sd, "m", 1, 2, False, 1, 1e-5, 0.1, True)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = mod(xd)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    _check(mod, sd, [yd], [yr], [xd], [xr])


def test_pspnet_r101_step_matches_oracle(cuda):
    """PSPNet-R101_v1c dilated-8, 150 classes (BASELINE configs[2] family at a small spatial size): deep stem via
    the 3x3/2 space-to-depth kernel, dilated bottlenecks, pyramid pooling (S = 1,2,3,6), concat, materialised
    x8 logits + cross-entropy(ignore -1). Loss vs the fp32 oracle, gradients aligned."""
    import torchseg_b200
    from torchseg_b200.networks import PSPNet
    from oracle import torch_ref
    torch.manual_seed(2)
    N, HW = 8, 96
    m = PSPNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout2d):
            mod.p = 0.0
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(-1, 150, (N, HW, HW), generator=g)
    loss_ref, _ = torch_ref.pspnet_loss(x, y, sd)
    loss_ref.backward()
    m.to(cuda)
    torchseg_b200.prepare_model(m)
    m.train()
    loss = m(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    # An untrained 100-layer batch-stat-BN network has exploding, chaotic gradients (|g| grows 1e-1 → 4e+1 towards the
    # input; even the fp32 oracle and its own bf16-storage emulation decorrelate below layer4, tools/diag_psp.py), so
    # direction is only checked where it is well conditioned (the two classifiers); everywhere else the gradient
    # MAGNITUDE must track the oracle, which catches missing / double-counted paths and wrong scales.
    P = dict(m.named_parameters())
    for n in ("psp_layer.conv6.2.weight", "aux_layer.2.weight"):
        a, b = P[n].grad.float().cpu().reshape(-1), sd[n].grad.reshape(-1)
        cos = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        assert cos > 0.9, (n, cos)
    checked = 0
    for n, p in P.items():
        if p.dim() == 4:
            ratio = float(p.grad.float().norm().cpu() / sd[n].grad.norm().clamp_min(1e-30))
            assert 0.8 < ratio < 1.25, (n, ratio)
            checked += 1
    assert checked >= 100


def test_flat_bf16_mirror_matches_per_tensor_pack(cuda):
    """after an optimiser step the bf16 mirror written by tsb_sgd_flat_pack / tsb_pack_wt_multi must be bit-identical to
    the per-tensor tsb_pack_weight operands (fprop/wgrad KRSC copy and the flipped-transposed dgrad copy)"""
    from torchseg_b200 import optim, ops
    from torchseg_b200.utils.init_func import group_weight
    model, sd, x, y, _ = _build(cuda, N=2, HW=64, seed=5)
    groups = group_weight([], model, BN, 1e-2)
    opt = optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)
    opt.zero_grad()
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    opt.step()
    checked = 0
    for n, p in model.named_parameters():
        if p.dim() != 4 or p.shape[1] % 8 != 0 or p.shape[0] % 8 != 0:
            continue
        fp, idx = p._tsb_pack
        hit = fp.lookup(p, idx, True)
        assert hit is not None, n
        wb, wt = hit
        K, C, R, S = p.shape
        ref_b = p.detach().permute(0, 2, 3, 1).to(torch.bfloat16)
        ref_t = ref_b.flip(1, 2).permute(3, 1, 2, 0).contiguous()
        assert torch.equal(wb, ref_b), n
        assert torch.equal(wt, ref_t), n
        checked += 1
    assert checked >= 30
    # an in-place edit of a weight invalidates its mirror entry (falls back to the per-tensor pack)
    p = model.ffm.conv_1x1.conv.weight
    with torch.no_grad():
        p.mul_(0.5)
    assert p._tsb_pack[0].lookup(p, p._tsb_pack[1], False) is None


def test_graphed_train_step_matches_eager(cuda):
    """GraphedTrainStep (whole step as one CUDA graph: zero_grad → forward → backward → fused SGD) follows the eager
    trajectory: same losses step by step (up to the non-deterministic summation order of the atomics), LR changes
    between replays are honoured (push_hyperparams → the device tensor the captured kernel reads)"""
    import os
    if os.environ.get("TSB_TEST_GRAPH", "1") == "0":
        pytest.skip("TSB_TEST_GRAPH=0")
    # (round 1 gated this test behind an environment variable: the capture failed "intermittently". Root cause, round 2:
    # a live autograd graph of an eager step — see engine/graph.py. Nothing of the kind is alive here: the eager trajectory
    # below keeps only loss.item().)
    torch.cuda.set_stream(torch.cuda.Stream())
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    from torchseg_b200.utils.init_func import group_weight

    def make():
        model, sd, x, y, _ = _build(cuda, N=4, HW=128, seed=7)
        groups = group_weight([], model, BN, 1e-2)
        g2 = torch.Generator().manual_seed(99)
        x2 = torch.randn(x.shape, generator=g2)
        y2 = make_labels(4, 128, 128, 19, 255, g2)
        data = [(x.to(cuda), y.to(cuda)), (x2.to(cuda), y2.to(cuda))]     # two different batches, alternating
        return model, optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4), data

    lrs = [1e-2, 1e-2, 8e-3, 6e-3, 0.0, 0.0]
    batch_of = lambda k: 0 if k < 2 else (k & 1)     # steps 0, 1 = the constructor's warm-up on its static inputs
    # eager reference trajectory
    model, opt, data = make()
    eager = []
    for k, lr in enumerate(lrs):
        for g in opt.param_groups:
            g["lr"] = lr
        opt.zero_grad()
        loss = model(*data[batch_of(k)])
        loss.backward()
        opt.step()
        eager.append(loss.item())
    # graphed: the constructor runs trajectory steps 0 and 1 eagerly on a SIDE stream (PyTorch's capture requirement),
    # then captures; every later step is a replay fed with fresh data
    model, opt, data = make()
    for g in opt.param_groups:
        g["lr"] = lrs[0]
    step = GraphedTrainStep(model, opt, list(data[0]), warmup=2)
    if step.graph is None:   # experimental feature (engine/graph.py)
        pytest.skip("CUDA graph capture unavailable: %s" % (step.error or "")[:200])
    assert step.launches_per_step > 100
    graphed = []
    frozen = None
    for k in range(2, len(lrs)):
        for g in opt.param_groups:
            g["lr"] = lrs[k]
        if lrs[k] == 0.0 and frozen is None:
            torch.cuda.synchronize()
            frozen = opt.flat_param.clone()
        graphed.append(step(*data[batch_of(k)]).item())    # fresh data copied into the static inputs every step
    # lr = 0 pushed for the last two replays (device tensor read by the captured SGD kernel): nothing may move
    assert torch.equal(opt.flat_param, frozen), "the staged learning rate did not reach the captured SGD kernel"
    for k, (a, b) in enumerate(zip(eager[2:], graphed)):
        assert abs(a - b) < 2e-2 * abs(a), (k, eager, graphed)
    # (a replay that kept a stale packed image cannot be told apart here: with untrained weights two batches give losses
    #  within the run-to-run spread of the atomics; the cache-key logic is unit-tested in tests/test_cpu_host.py)
    # (p -= lr * momentum_buffer: with lr = 0 nothing moves; a stale capture-time lr of 1e-2 would change the loss)
    # (steps 4 and 5 use different batches, so compare each with its eager twin instead of with each other)
    assert abs(graphed[-1] - eager[-1]) < 2e-2 * abs(eager[-1]) and abs(graphed[-2] - eager[-2]) < 2e-2 * abs(eager[-2])
    # and an eager step right after the replays must see the CURRENT weights (no stale bf16 packs): with lr = 0 the
    # parameters are frozen, so it reproduces the last loss on the same batch
    for g in opt.param_groups:
        g["lr"] = 0.0
    opt.zero_grad()
    l_after = model(*data[batch_of(len(lrs) - 1)])
    l_after.backward()
    opt.step()
    assert abs(l_after.item() - graphed[-1]) < 5e-3 * abs(graphed[-1]), (l_after.item(), graphed[-1])
    for p in model.parameters():
        assert torch.isfinite(p).all()
    step.release()
    # restore_after_warmup: constructing the object leaves parameters, momentum and BN statistics untouched, and the
    # first replay then computes the same loss as an eager step from that state
    model, opt, data = make()
    before = (opt.flat_param.clone(), opt.flat_mom.clone(), [b.clone() for b in model.buffers()])
    for g in opt.param_groups:
        g["lr"] = 0.0
    step2 = GraphedTrainStep(model, opt, list(data[0]), warmup=2, restore_after_warmup=True)
    assert step2.graph is not None, step2.error
    assert torch.equal(opt.flat_param, before[0]) and torch.equal(opt.flat_mom, before[1])
    assert all(torch.equal(a, b) for a, b in zip(model.buffers(), before[2]))
    l_graph = step2(*data[0]).item()
    assert abs(l_graph - eager[0]) < 5e-3 * abs(eager[0]), (l_graph, eager[0])
    step2.release()
    torch.cuda.set_stream(torch.cuda.default_stream())


def test_bisenet_eval_forward_matches_oracle(cuda):
    """inference branch of BiSeNet.forward (network.py:110-111): eval-mode BN from the running statistics (scale / shift
    through tsb_bn_finalize with count 1), main head only, x8 bilinear, log_softmax — vs the oracle in eval mode"""
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    from oracle import torch_ref as tr
    torch.manual_seed(11)
    model = BiSeNet(19, False, None, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = torch.Generator().manual_seed(12)
    with torch.no_grad():   # non-trivial running statistics and affine parameters
        for m in model.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) * 1.5 + 0.5)
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = torch.randn(2, 3, 128, 160, generator=g)
    tr.set_bf16_emulation(True)
    try:
        with torch.no_grad():
            lo, _ = tr.bisenet_r18_forward(x, sd, training=False)
            ref = F.log_softmax(F.interpolate(lo[2], scale_factor=8, mode="bilinear", align_corners=True), dim=1)
    finally:
        tr.set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    rm_before = model.context_path.bn1.running_mean.clone()
    with torch.no_grad():
        out = model(x.to(cuda))
    assert tuple(out.shape) == (2, 19, 128, 160) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97
    assert torch.equal(model.context_path.bn1.running_mean, rm_before), "eval must not touch the running statistics"


def test_bisenet_eval_bn_folding_matches_unfolded(cuda):
    """evaluator forward with the BatchNorm folded into the conv operands (bias + shortcut + ReLU in the conv epilogue,
    tsb_conv2d_fprop_fused / tsb_conv_stem_fprop_fused) against the un-folded eval path (raw conv → tsb_bn_apply): same
    log-probabilities up to the bf16 rounding of the folded weights, far fewer kernel launches, no BN pass"""
    import torchseg_b200
    from torchseg_b200 import _lib
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.seg_opr import seg_oprs
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(13)
    model = BiSeNet(19, False, None, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = torch.Generator().manual_seed(14)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) * 1.5 + 0.5)
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    x = torch.randn(2, 3, 256, 320, generator=g).to(cuda)
    outs, launches = {}, {}
    try:
        for fold in (False, True):
            seg_oprs.EVAL_FOLD_BN = fold
            with torch.no_grad():
                model(x)                                  # warm (packs, fold cache)
                n0 = _lib.launch_count()
                outs[fold] = model(x)
                launches[fold] = _lib.launch_count() - n0
    finally:
        seg_oprs.EVAL_FOLD_BN = True
    assert norm_err(outs[True], outs[False]) < 1e-2, norm_err(outs[True], outs[False])
    # (untrained weights: many pixels have near-tied classes, so the arg-max is only required to agree on > 97 %)
    assert (outs[True].argmax(1) == outs[False].argmax(1)).float().mean() > 0.97
    assert launches[True] <= launches[False] - 40, launches     # ~30 BN layers: finalize + apply launches are gone
    # parameters change → the folded operands follow (version / optimiser-step keyed cache)
    with torch.no_grad():
        model.ffm.conv_1x1.bn.weight.mul_(1.5)
        changed = model(x)
    assert norm_err(changed, outs[True]) > 1e-3


def test_pspnet_odd_input_size_matches_oracle(cuda):
    """BASELINE configs[2] asks for 713 x 713 (not a multiple of 8): the heads up-sample to the INPUT size (`size=`
    semantics, identical numbers to scale_factor=8 where that is defined), the stem pads the odd image. Small odd size
    here (105 → 53 → 27 → 14 feature map), loss against the oracle patched the same way (oracle/torch_ref._up8)."""
    import torchseg_b200
    from torchseg_b200.networks import PSPNet
    from oracle import torch_ref
    torch.manual_seed(4)
    N, HW = 4, 105
    m = PSPNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout2d):
            mod.p = 0.0
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(-1, 150, (N, HW, HW), generator=g)
    loss_ref, (psp_ref, _) = torch_ref.pspnet_loss(x, y, sd)
    assert tuple(psp_ref.shape[2:]) == (HW, HW)
    m.to(cuda)
    torchseg_b200.prepare_model(m)
    m.train()
    loss = m(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
    m.eval()
    with torch.no_grad():
        out = m(x.to(cuda))
    assert tuple(out.shape) == (N, 150, HW, HW)
