"""Checks shared by the step-level GPU tests of the ResNet-101 network lines (DeepLabV3+, EncNet, OCNet, DenseASPP), and
the eval-mode BatchNorm randomisation of the eval tests. What differs from line to line (constructor, oracle functions,
class count, classifier names, parameter filter, required kernels) comes in as arguments."""
import torch

from util import norm_err

BN = torch.nn.BatchNorm2d
# ATen ops and library kernel names (lower-cased substrings) of a GEMM or convolution libtsb should have run instead
ATEN_GEMM = ("aten::conv", "aten::_conv", "aten::cudnn", "aten::mm", "aten::bmm", "aten::baddbmm", "aten::matmul",
             "aten::addmm", "aten::linear")
LIB_GEMM = ("cudnn", "cublas", "cutlass", "xmma", "gemv")


def randomize_bn(model, seed):
    """non-trivial running statistics and affine parameters for the eval tests, drawn BN module by BN module; returns
    the generator, from which the caller draws its input next"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) * 1.5 + 0.5)
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    return g


def check_step_vs_oracle(cuda, model, sd, x, y, oracle_loss, classifier, keep=lambda p: p.dim() >= 2, finite=True):
    """one training step of `model` (prepared, train mode) against oracle_loss(x, y, sd) run in fp32 and with
    bf16-storage emulation: loss within 1e-2 of the fp32 oracle, gradient direction of the `classifier` parameters
    (cos > 0.9), and for every parameter p with keep(p) a gradient magnitude within ±33 % of the fp32 oracle's or of the
    emulation's. `finite`: every parameter gradient is finite too. Returns the model's named parameters for
    line-specific asserts."""
    from oracle.torch_ref import set_bf16_emulation
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    loss_ref, _ = oracle_loss(x, y, sd)
    loss_ref.backward()
    ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    set_bf16_emulation(True)
    try:
        loss_emu, _ = oracle_loss(x, y, sd)
        loss_emu.backward()
    finally:
        set_bf16_emulation(False)
    emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    P = dict(model.named_parameters())
    for n in classifier:
        a, b = P[n].grad.float().cpu().reshape(-1), ref[n].reshape(-1)
        cos = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        assert cos > 0.9, (n, cos)
    bad = []
    for n, p in P.items():
        if finite:
            assert bool(torch.isfinite(p.grad).all()), n
        if keep(p):
            gn = float(p.grad.float().norm().cpu())
            r_emu, r_ref = (gn / float(o[n].norm().clamp_min(1e-30)) for o in (emu, ref))
            if not (0.75 < r_emu < 1.33 or 0.75 < r_ref < 1.33):
                bad.append((n, round(r_emu, 3), round(r_ref, 3)))
    assert not bad, "|grad| / |emulating oracle's|, / |fp32 oracle's|: %s" % bad[:10]
    return P


def _train_step(model, opt, x, y):
    opt.zero_grad()
    loss = model(x, y)
    loss.backward()
    opt.step()
    return loss.detach().clone()


def check_train_reproducible(make, steps=5):
    """`steps` optimiser steps lower the loss, and a second run from make() (model, optimiser, x, y on the device), with
    the first run's model freed, gives the same loss and parameter bits"""
    runs = []
    for _ in range(2):
        model, opt, x, y = make()
        losses = [_train_step(model, opt, x, y) for _ in range(steps)]
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


def check_graphed_matches_eager(make, kernels=None, extra_aten=(), extra_libs=()):
    """four eager steps of make() (model, optimiser, x, y on the device), then a fresh make() captured by
    GraphedTrainStep (warm-up 2): its two replays equal eager steps 3 and 4 bit for bit. With `kernels`, the fourth
    eager step's forward and backward are profiled: no ATen / cuDNN / cuBLAS GEMM (nor an op of `extra_aten`, a kernel
    name containing one of `extra_libs`) runs, and a kernel whose name contains each of `kernels` does"""
    from torch.profiler import ProfilerActivity, profile
    from torchseg_b200.engine.graph import GraphedTrainStep
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        model, opt, x, y = make()
        eager = []
        for i in range(4):
            if kernels is not None and i == 3:
                opt.zero_grad()
                with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                    loss = model(x, y)
                    loss.backward()
                    torch.cuda.synchronize()
                opt.step()
                eager.append(loss.detach().clone())
            else:
                eager.append(_train_step(model, opt, x, y))
        if kernels is not None:
            names = [e.name for e in prof.events()]
            aten, libs = ATEN_GEMM + tuple(extra_aten), LIB_GEMM + tuple(extra_libs)
            bad = [n for n in names if n.startswith(aten) or any(t in n.lower() for t in libs)]
            assert not bad, sorted(set(bad))[:10]
            for k in kernels:
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


def check_eval_vs_oracle_and_sliding(cuda, make_model, oracle_eval, classes):
    """eval forward of make_model() (business layers Kaiming-initialised, BatchNorm randomised) on 2 x 96 x 130 within
    2e-2 (norm) of the bf16-emulating oracle_eval(x, sd) with > 97 % arg-max agreement, and the device sliding-window
    evaluation equal to the host one"""
    import numpy as np
    import torchseg_b200
    from torchseg_b200.engine.evaluator import Evaluator
    from torchseg_b200.utils.init_func import init_weight
    from oracle.torch_ref import set_bf16_emulation
    torch.manual_seed(11)
    model = make_model()
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = randomize_bn(model, 12)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = torch.randn(2, 3, 96, 130, generator=g)
    set_bf16_emulation(True)
    try:
        with torch.no_grad():
            ref = oracle_eval(x, sd)
    finally:
        set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    with torch.no_grad():
        out = model(x.to(cuda))
    assert tuple(out.shape) == (2, classes, 96, 130) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97
    ev = Evaluator(dataset=None, class_num=classes, image_mean=np.array([0.485, 0.456, 0.406]),
                   image_std=np.array([0.229, 0.224, 0.225]), network=None, multi_scales=[0.75, 1.0], is_flip=True,
                   devices=[0], crop_batch=2)
    ev.val_func = model
    img = np.random.default_rng(0).integers(0, 256, (150, 171, 3), dtype=np.uint8)
    host = ev.sliding_eval(img, 128, 2 / 3.0, cuda)
    dev = ev.sliding_eval_device(img, 128, 2 / 3.0, cuda)
    assert np.array_equal(dev.cpu().numpy(), host)
