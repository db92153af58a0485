"""BiSeNet-X39 on the H100: the depthwise 3x3 kernels (tsb_dwconv_*) bit for bit against a float64 reference, the
Xception modules teacher-forced against the bf16-emulating oracle, and the whole training step against the fp32
oracle (tests/x39_oracle.py on the blocks of oracle/torch_ref.py, pinned to the live reference by
tests/test_cpu_x39.py)."""
import pytest
import torch
import torch.nn.functional as F

from util import rel_err, norm_err, make_labels, bf16_round
from net_checks import randomize_bn

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d

# every depthwise conv of the X39 step at 1024^2 as (C, input H = W, stride), at batch 2
X39_DW_SHAPES = [(8, 256, 2), (16, 128, 1), (64, 128, 1), (64, 128, 2), (32, 64, 1), (128, 64, 1), (128, 64, 2),
                 (64, 32, 1), (256, 32, 1)]
# (N, C, H, W, stride, channel stride of x / y): odd sizes, channel slices of wider buffers, a batch of 1
EXTRA_DW_SHAPES = [(2, 24, 33, 47, 2, 24), (2, 24, 33, 47, 1, 24), (2, 16, 40, 24, 1, 64), (2, 16, 41, 23, 2, 64),
                   (1, 64, 17, 9, 2, 64), (1, 8, 5, 7, 1, 8)]


def _cases():
    out = [(2, C, H, H, s, C) for C, H, s in X39_DW_SHAPES] + EXTRA_DW_SHAPES
    return out, ["N%dC%dH%dW%ds%dcs%d" % c for c in out]


def _small_int(shape, g, lo=-2, hi=3):
    return torch.randint(lo, hi, shape, generator=g).to(torch.float32)


def _nhwc(t, cs, cuda, fill=0.0):
    """bf16 NHWC buffer of channel stride cs holding t ([N,C,H,W]) in its first C channels; the rest = fill"""
    N, C, H, W = t.shape
    buf = torch.full((N, H, W, cs), fill, dtype=torch.bfloat16, device=cuda)
    buf[..., :C] = t.permute(0, 2, 3, 1).to(cuda, torch.bfloat16)
    return buf


@pytest.mark.parametrize("case", _cases()[0], ids=_cases()[1])
def test_dwconv_kernels_exact(cuda, case):
    """small-integer operands: every fp32 partial sum is exact, so fprop, dgrad (plain and accumulating) and wgrad must
    equal the float64 grouped convolution bit for bit; channels outside the slice are never touched"""
    from torchseg_b200 import ops
    N, C, H, W, st, cs = case
    P, Q = (H - 1) // st + 1, (W - 1) // st + 1
    g = torch.Generator().manual_seed(C * 1000 + H + st)
    x, w, dy = _small_int((N, C, H, W), g), _small_int((C, 1, 3, 3), g), _small_int((N, C, P, Q), g)
    old = _small_int((N, C, H, W), g)
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, None, st, 1, 1, C)
    y64.backward(dy.double())
    xb, dyb = _nhwc(x, cs, cuda), _nhwc(dy, cs, cuda)
    wd = w.to(cuda).reshape(C, 9).contiguous()
    s = ops.stream()
    y = _nhwc(torch.zeros(N, C, P, Q), cs, cuda, fill=7.0)
    ops.call("tsb_dwconv_fprop", xb.data_ptr(), cs, wd.data_ptr(), y.data_ptr(), cs, N, H, W, C, st, s)
    dx = _nhwc(torch.zeros(N, C, H, W), cs, cuda, fill=7.0)
    ops.call("tsb_dwconv_dgrad", dyb.data_ptr(), cs, wd.data_ptr(), dx.data_ptr(), cs, N, H, W, C, st, 0, s)
    dxa = _nhwc(old, cs, cuda, fill=7.0)
    ops.call("tsb_dwconv_dgrad", dyb.data_ptr(), cs, wd.data_ptr(), dxa.data_ptr(), cs, N, H, W, C, st, 1, s)
    dws = []
    for _ in range(2):
        dw = torch.zeros(C, 9, dtype=torch.float32, device=cuda)
        ops.call("tsb_dwconv_wgrad", xb.data_ptr(), cs, dyb.data_ptr(), cs, dw.data_ptr(), N, H, W, C, st,
                 *ops.det_ws(), s)
        dws.append(dw)
    torch.cuda.synchronize()
    nchw = lambda b: b[..., :C].permute(0, 3, 1, 2).double().cpu()
    assert torch.equal(nchw(y), y64.detach()), "fprop"
    assert torch.equal(nchw(dx), x64.grad), "dgrad"
    assert torch.equal(nchw(dxa), x64.grad + old.double()), "dgrad accumulate"
    assert torch.equal(dws[0].double().cpu().reshape(C, 1, 3, 3), w64.grad), "wgrad"
    assert torch.equal(dws[0].view(torch.int32), dws[1].view(torch.int32)), "wgrad is not reproducible"
    if cs > C:
        for b in (y, dx, dxa):
            assert bool((b[..., C:].float() == 7.0).all()), "wrote outside the channel slice"


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


def _rand(shape, g, relu=False):
    t = torch.randn(*shape, generator=g)
    return bf16_round(torch.relu(t) if relu else t)


def _padded_input(x, cuda):
    """x as the 64-padded activation a padded pointwise conv leaves behind (pad channels exact zeros)"""
    from torchseg_b200 import ops
    N, C, H, W = x.shape
    Cp = (C + 63) // 64 * 64
    buf = ops.nhwc_zeros(N, Cp, H, W, device=cuda)
    with torch.no_grad():
        buf[:, :C].copy_(x.to(cuda))
    return buf.requires_grad_(True)


def _check_params(mod, sd, tol=1e-2):
    for n, p in mod.named_parameters():
        e = norm_err(p.grad, sd["m." + n].grad)
        assert e < 2 * tol, "param grad %s: %g" % (n, e)


@pytest.mark.parametrize("cfg", [(8, 64, 2, False), (16, 16, 1, True), (64, 32, 2, True), (32, 128, 1, False)],
                         ids=["8to64s2", "16to16s1relu", "64to32s2relu", "32to128s1"])
def test_separable_conv_teacher_forced(cuda, cfg):
    from torchseg_b200 import ops
    from torchseg_b200.base_model.xception import SeparableConvBnRelu
    import x39_oracle as tr
    cin, cout, st, relu = cfg
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(3)
    mod = SeparableConvBnRelu(cin, cout, 3, st, 1, has_relu=relu)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    x = _rand((8, cin, 40, 48), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = tr.separable_conv_bn_relu(xr, sd, "m", st, relu)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = _padded_input(x, cuda)
    yd = mod(xd)
    Kp = (cout + 63) // 64 * 64
    assert yd.shape[1] == Kp
    gyd = ops.nhwc_zeros(yd.shape[0], Kp, yd.shape[2], yd.shape[3], device=cuda)
    with torch.no_grad():
        gyd[:, :cout].copy_(gy.to(cuda))
    yd.backward(gyd)
    assert norm_err(yd[:, :cout], yr) < 1e-2, norm_err(yd[:, :cout], yr)
    assert norm_err(xd.grad[:, :cin], xr.grad) < 1e-2, norm_err(xd.grad[:, :cin], xr.grad)
    assert bool((yd[:, cout:] == 0).all()), "forward pad channels are not zero"
    assert bool((xd.grad[:, cin:] == 0).all()), "backward pad channels are not zero"
    _check_params(mod, sd)


@pytest.mark.parametrize("proj", [True, False], ids=["proj_s2", "identity"])
def test_xception_block_teacher_forced(cuda, proj):
    from torchseg_b200 import ops
    from torchseg_b200.base_model.xception import Block
    import x39_oracle as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(4)
    cin, mid, st = (64, 32, 2) if proj else (128, 32, 1)
    mod = Block(cin, mid, proj, st, norm_layer=BN)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    x = _rand((8, cin, 32, 32), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        yr = tr.xception_block(xr, sd, "m", st, proj)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = mod(xd)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    assert norm_err(yd, yr) < 1e-2, norm_err(yd, yr)
    assert norm_err(xd.grad, xr.grad) < 1e-2, norm_err(xd.grad, xr.grad)
    _check_params(mod, sd)


def _build(cuda, N=8, HW=128, seed=0):
    import torchseg_b200
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(seed)
    H = W = HW
    ohem = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=N * H * W // 16, use_weight=False)
    model = BiSeNet(19, True, torch.nn.CrossEntropyLoss(ignore_index=255), ohem, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = make_labels(N, H, W, 19, 255, g)
    return model, sd, x, y, N * H * W // 16


def test_bisenet_x39_step_matches_oracle(cuda):
    import x39_oracle as torch_ref
    model, sd, x, y, min_kept = _build(cuda)
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    stats = {}
    loss_ref, _ = torch_ref.bisenet_x39_loss(x, y, sd, min_kept, stats=stats)
    loss_ref.backward()
    grads_ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    torch_ref.set_bf16_emulation(True)
    try:
        stats_emu = {}
        loss_emu, _ = torch_ref.bisenet_x39_loss(x, y, sd, min_kept, stats=stats_emu)
        loss_emu.backward()
    finally:
        torch_ref.set_bf16_emulation(False)
    grads_emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    # X39 chains ~60 batch-statistics BN layers: at initialisation bf16 STORAGE alone (the emulating oracle) already
    # turns many fp32 gradients to cosines of 0.4-0.7 (measured on the CPU). The direction / magnitude bar of the R18
    # test therefore applies where the emulation resolves the fp32 gradient (cosine >= 0.95); every gradient keeps its
    # magnitude within 2x, and every conv weight gradient stays within the bf16-storage spread bar.
    bad, outside, resolved = [], [], 0
    for n, p in model.named_parameters():
        a, b, c = p.grad.float().cpu(), grads_ref[n], grads_emu[n]
        af, bf, cf = a.reshape(-1), b.reshape(-1), c.reshape(-1)
        cos = float(torch.dot(af, bf) / (af.norm() * bf.norm()).clamp_min(1e-30))
        cos_emu = float(torch.dot(cf, bf) / (cf.norm() * bf.norm()).clamp_min(1e-30))
        ratio = float(af.norm() / bf.norm().clamp_min(1e-30))
        if cos_emu >= 0.95:
            resolved += 1
            if cos < 0.8 or not (0.7 < ratio < 1.4):
                bad.append((n, round(cos, 3), round(ratio, 3)))
        elif not (0.5 < ratio < 2.0):
            bad.append((n, round(cos, 3), round(ratio, 3)))
        if p.dim() == 4:
            e, spread = norm_err(a, b), norm_err(c, b)
            if e > 1.5 * spread + 2e-2:
                outside.append((n, round(e, 4), round(spread, 4)))
    assert not bad, "gradient direction / magnitude off: %s" % bad[:10]
    assert not outside, "gradient farther from the fp32 oracle than 1.5 x the bf16-storage spread + 2e-2: %s" % outside[:10]
    assert resolved >= 5, resolved   # the classifiers and the last layers
    msd = model.state_dict()
    for k, v in stats.items():   # running statistics: within the bf16-storage spread of the same update (+3e-2)
        assert rel_err(msd[k], v) < 1.5 * rel_err(stats_emu[k], v) + 3e-2, (k, rel_err(msd[k], v), rel_err(stats_emu[k], v))


def _groups(model):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.context_path, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return groups


def test_bisenet_x39_train_steps_decrease_loss(cuda):
    from torchseg_b200 import optim
    model, _, x, y, _ = _build(cuda, N=4, HW=128, seed=3)
    opt = optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4)
    xs, ys = x.to(cuda), y.to(cuda)
    losses = []
    for _ in range(5):
        opt.zero_grad()
        loss = model(xs, ys)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(l == l for l in losses)
    assert losses[-1] < losses[0], losses
    for p in model.parameters():
        assert torch.isfinite(p).all()


def test_bisenet_x39_step_is_bit_reproducible(cuda):
    """two identical models and batches: identical loss bits and identical gradient bits"""
    runs = []
    for _ in range(2):
        model, _, x, y, _ = _build(cuda, N=4, HW=128, seed=5)
        loss = model(x.to(cuda), y.to(cuda))
        loss.backward()
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), [p.grad.detach().clone() for p in model.parameters()]))
    (l0, g0), (l1, g1) = runs
    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32)), (l0.item(), l1.item())
    for a, b in zip(g0, g1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_bisenet_x39_graphed_step_matches_eager(cuda):
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        def make():
            model, _, x, y, _ = _build(cuda, N=4, HW=128, seed=7)
            return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

        model, opt, x, y = make()
        eager = []
        for _ in range(4):
            opt.zero_grad()
            loss = model(x, y)
            loss.backward()
            opt.step()
            eager.append(loss.item())
        model, opt, x, y = make()
        step = GraphedTrainStep(model, opt, [x, y], warmup=2)
        assert step.graph is not None, step.error
        graphed = [step(x, y).item() for _ in range(2)]
        for a, b in zip(eager[2:], graphed):
            assert abs(a - b) < 5e-3 * abs(a), (eager, graphed)
        step.release()
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())


def test_bisenet_x39_eval_forward_matches_oracle(cuda):
    import torchseg_b200
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    from torchseg_b200.utils.init_func import init_weight
    import x39_oracle as tr
    torch.manual_seed(11)
    model = BiSeNet(19, False, None, None, None, BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = randomize_bn(model, 12)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = torch.randn(2, 3, 128, 160, generator=g)
    tr.set_bf16_emulation(True)
    try:
        with torch.no_grad():
            ref = tr.bisenet_x39_eval(x, sd)
    finally:
        tr.set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    with torch.no_grad():
        out = model(x.to(cuda))
    assert tuple(out.shape) == (2, 19, 128, 160) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97
