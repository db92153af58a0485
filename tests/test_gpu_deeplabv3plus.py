"""DeepLabV3+ on the H100: the dilated depthwise 3x3 kernels (tsb_dwconv2d_*) bit for bit against a float64 reference,
SeparableConvBnRelu / ASPP / decoder teacher-forced against the bf16-emulating oracle, and the whole training step against
the fp32 oracle (tests/deeplabv3plus_oracle.py on the blocks of oracle/torch_ref.py, pinned to the live reference
composition by tests/test_cpu_deeplabv3plus.py)."""
import pytest
import torch
import torch.nn.functional as F

from util import norm_err, make_labels, bf16_round
from net_checks import (check_step_vs_oracle, check_train_reproducible, check_graphed_matches_eager,
                        check_eval_vs_oracle_and_sliding)

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d

# (N, C, H, W, stride, dilation, channel stride of x / y): odd sizes, maps smaller than the dilation (only the centre tap
# lands inside), the 304 / 2048 channels of the decoder and the ASPP as channel slices of wider buffers
DW2D_CASES = [(2, 8, 9, 11, 1, 1, 16), (2, 8, 9, 11, 2, 1, 16), (2, 304, 17, 13, 1, 1, 320), (2, 304, 17, 13, 2, 1, 320),
              (2, 16, 21, 19, 1, 2, 24), (1, 8, 5, 7, 1, 6, 8), (2, 304, 25, 23, 1, 6, 320), (2, 2048, 8, 6, 1, 6, 2056),
              (2, 2048, 9, 11, 1, 12, 2056), (2, 2048, 7, 5, 1, 18, 2056), (1, 8, 13, 40, 1, 12, 16),
              (2, 24, 37, 41, 1, 18, 32), (4, 64, 64, 64, 1, 12, 64)]


def _small_int(shape, g, lo=-2, hi=3):
    return torch.randint(lo, hi, shape, generator=g).to(torch.float32)


def _nhwc(t, cs, cuda, fill=0.0):
    """bf16 NHWC buffer of channel stride cs holding t ([N,C,H,W]) in its first C channels; the rest = fill"""
    N, C, H, W = t.shape
    buf = torch.full((N, H, W, cs), fill, dtype=torch.bfloat16, device=cuda)
    buf[..., :C] = t.permute(0, 2, 3, 1).to(cuda, torch.bfloat16)
    return buf


@pytest.mark.parametrize("case", DW2D_CASES, ids=["N%dC%dH%dW%ds%dd%dcs%d" % c for c in DW2D_CASES])
def test_dwconv2d_kernels_exact(cuda, case):
    """small-integer operands: every fp32 partial sum is exact, so fprop, dgrad (plain and accumulating) and wgrad (over
    several CTAs) must equal the float64 grouped convolution bit for bit; channels outside the slice are never touched;
    at dilation 1 the tsb_dwconv_* entry points give the same bits"""
    from torchseg_b200 import ops
    N, C, H, W, st, d, cs = case
    P, Q = (H - 1) // st + 1, (W - 1) // st + 1
    g = torch.Generator().manual_seed(C * 1000 + H + st + 7 * d)
    x, w, dy = _small_int((N, C, H, W), g), _small_int((C, 1, 3, 3), g), _small_int((N, C, P, Q), g)
    old = _small_int((N, C, H, W), g)
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, None, st, d, d, C)
    assert tuple(y64.shape[2:]) == (P, Q)
    y64.backward(dy.double())
    xb, dyb = _nhwc(x, cs, cuda), _nhwc(dy, cs, cuda)
    wd = w.to(cuda).reshape(C, 9).contiguous()
    s = ops.stream()
    y = _nhwc(torch.zeros(N, C, P, Q), cs, cuda, fill=7.0)
    ops.call("tsb_dwconv2d_fprop", xb.data_ptr(), cs, wd.data_ptr(), y.data_ptr(), cs, N, H, W, C, st, d, s)
    dx = _nhwc(torch.zeros(N, C, H, W), cs, cuda, fill=7.0)
    ops.call("tsb_dwconv2d_dgrad", dyb.data_ptr(), cs, wd.data_ptr(), dx.data_ptr(), cs, N, H, W, C, st, d, 0, s)
    dxa = _nhwc(old, cs, cuda, fill=7.0)
    ops.call("tsb_dwconv2d_dgrad", dyb.data_ptr(), cs, wd.data_ptr(), dxa.data_ptr(), cs, N, H, W, C, st, d, 1, s)
    dws = []
    for _ in range(2):
        dw = torch.zeros(C, 9, dtype=torch.float32, device=cuda)
        ops.call("tsb_dwconv2d_wgrad", xb.data_ptr(), cs, dyb.data_ptr(), cs, dw.data_ptr(), N, H, W, C, st, d,
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
    if d == 1:
        y1 = _nhwc(torch.zeros(N, C, P, Q), cs, cuda, fill=7.0)
        ops.call("tsb_dwconv_fprop", xb.data_ptr(), cs, wd.data_ptr(), y1.data_ptr(), cs, N, H, W, C, st, s)
        dx1 = _nhwc(old, cs, cuda, fill=7.0)
        ops.call("tsb_dwconv_dgrad", dyb.data_ptr(), cs, wd.data_ptr(), dx1.data_ptr(), cs, N, H, W, C, st, 1, s)
        dw1 = torch.zeros(C, 9, dtype=torch.float32, device=cuda)
        ops.call("tsb_dwconv_wgrad", xb.data_ptr(), cs, dyb.data_ptr(), cs, dw1.data_ptr(), N, H, W, C, st,
                 *ops.det_ws(), s)
        torch.cuda.synchronize()
        assert torch.equal(y1.view(torch.int16), y.view(torch.int16))
        assert torch.equal(dx1.view(torch.int16), dxa.view(torch.int16))
        assert torch.equal(dw1.view(torch.int32), dws[0].view(torch.int32))


def test_dwconv2d_wgrad_runs_several_ctas(cuda):
    """the wgrad grid of the exactness cases above: more than one CTA slot is summed by tsb_det_reduce"""
    from torchseg_b200 import ops
    N, C, H, W, st, d, cs = DW2D_CASES[-1]
    x = torch.zeros(N, H, W, cs, dtype=torch.bfloat16, device=cuda)
    dw = torch.zeros(C, 9, dtype=torch.float32, device=cuda)
    ws, _ = ops.det_ws()
    with pytest.raises(RuntimeError, match="workspace needs"):   # one CTA's slot is not enough: the grid is wider
        ops.call("tsb_dwconv2d_wgrad", x.data_ptr(), cs, x.data_ptr(), cs, dw.data_ptr(), N, H, W, C, st, d, ws, C * 9,
                 ops.stream())


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


def _check_param_grads(named, ref, tol=1e-2):
    """every parameter gradient within 2·tol (norm) of the oracle's. The β of the BN between the depthwise and the
    pointwise conv is the exception: its gradient Σ dz is exactly 0 in exact arithmetic (a per-channel shift of the
    pointwise conv's input is removed by the pointwise BN's batch mean), so both sides hold rounding noise; its error is
    measured against the norm of the same BN's dγ instead."""
    for n, p in named:
        pre = n[:-len("bn.bias")]
        if n.endswith("bn.bias") and pre + "conv1.weight" in ref:   # SeparableConvBnRelu.bn
            e = float((p.grad.float().cpu() - ref[n]).norm() / ref[pre + "bn.weight"].norm())
        else:
            e = norm_err(p.grad, ref[n])
        assert e < 2 * tol, "param grad %s: %g" % (n, e)


def _check_params(mod, sd, tol=1e-2):
    _check_param_grads(mod.named_parameters(), {k[2:]: v.grad for k, v in sd.items() if v.grad is not None}, tol)


def _check_running(mod, stats, tol=1e-2):
    """running statistics within tol of the oracle's, relative to their largest entry or 1e-2, whichever is larger: the
    pointwise BN's batch mean is ~0 (its input is a conv of a batch-normalised map), so its entries are rounding noise"""
    msd = mod.state_dict()
    for k, v in stats.items():
        e = float((msd[k[2:]].float().cpu() - v).abs().max()) / max(float(v.abs().max()), 1e-2)
        assert e < tol, (k, e)


@pytest.mark.parametrize("cfg", [(304, 256, 1, True, 320), (256, 256, 1, True, 256), (2048, 256, 6, True, 2048),
                                 (64, 32, 12, False, 64), (16, 64, 18, True, 64)],
                         ids=["304to256d1_cs320", "256to256d1", "2048to256d6", "64to32d12", "16to64d18_map_smaller"])
def test_separable_conv_bn_relu_teacher_forced(cuda, cfg):
    """train: y, dx, dW, dγ, dβ and the running statistics within 1e-2 of the bf16-emulating oracle; the input's pad
    channels get exact-zero gradients and the 64-padded output's pad channels stay zero; eval against the oracle too"""
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr.seg_oprs import SeparableConvBnRelu
    import deeplabv3plus_oracle as tr
    cin, cout, d, relu, cs = cfg
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(3)
    mod = SeparableConvBnRelu(cin, cout, 3, 1, d, d, has_relu=relu)
    sd = _sd_of(mod)
    _prep(mod, cuda)
    HW = (13, 11) if d == 18 else (24, 20)
    x = _rand((4, cin) + HW, g, relu=True)
    xr = x.clone().requires_grad_(True)
    stats = {}
    tr.set_bf16_emulation(True)
    try:
        yr = tr.separable_conv_bn_relu(xr, sd, "m", d, relu, stats=stats)
        gy = _rand(tuple(yr.shape), g)
        yr.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.nhwc_zeros(4, cs, HW[0], HW[1], device=cuda)
    with torch.no_grad():
        xd[:, :cin].copy_(x.to(cuda))
    xd.requires_grad_(True)
    yd = mod(xd)
    Kp = yd.shape[1]
    gyd = ops.nhwc_zeros(yd.shape[0], Kp, yd.shape[2], yd.shape[3], device=cuda)
    with torch.no_grad():
        gyd[:, :cout].copy_(gy.to(cuda))
    yd.backward(gyd)
    torch.cuda.synchronize()
    assert norm_err(yd[:, :cout], yr) < 1e-2, norm_err(yd[:, :cout], yr)
    assert norm_err(xd.grad[:, :cin], xr.grad) < 1e-2, norm_err(xd.grad[:, :cin], xr.grad)
    assert bool((yd[:, cout:] == 0).all()), "forward pad channels are not zero"
    assert bool((xd.grad[:, cin:] == 0).all()), "backward pad channels are not zero"
    _check_params(mod, sd)
    _check_running(mod, stats)
    # eval: the depthwise BN on its running statistics, the pointwise CBR folded
    mod.eval()
    with torch.no_grad():
        ye = mod(xd.detach())
        tr.set_bf16_emulation(True)
        try:
            sde = {k: v.detach() for k, v in sd.items()}
            sde.update({"m." + k: v.detach().cpu() for k, v in mod.state_dict().items() if "running" in k})
            yre = tr.separable_conv_bn_relu(x, sde, "m", d, relu, training=False, momentum=0.0)
        finally:
            tr.set_bf16_emulation(False)
    assert norm_err(ye[:, :cout], yre) < 1e-2, norm_err(ye[:, :cout], yre)


def test_aspp_and_decoder_teacher_forced(cuda):
    """the ASPP (rates larger than the 1/16 map) and the decoder (ragged 48 / 304 channels), train and eval. The
    image-pooling branch normalises over the batch of 4 pooled vectors, which makes the ASPP's gradients sensitive to
    bf16 storage: every output and gradient must lie within 1.5x the distance between the fp32 oracle and its
    bf16-storage emulation (+1e-2) of the fp32 oracle, as DESIGN §5 asks of the X39 step."""
    from torchseg_b200 import ops
    from torchseg_b200.networks.deeplabv3plus import ASPP, Decoder
    import deeplabv3plus_oracle as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(5)

    class Head(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.aspp = ASPP(2048, 256, (6, 12, 18))
            self.decoder = Decoder(19)
            self.aspp.dropout.p = 0.0

        def forward(self, x, low):
            return self.decoder(self.aspp(x), low)

    mod = Head()
    sd = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    _prep(mod, cuda)
    x, low = _rand((4, 2048, 9, 7), g, relu=True), _rand((4, 256, 33, 27), g, relu=True)
    glo = torch.randn(4, 19, 33, 27, generator=g)
    runs = {}
    for emulate in (False, True):
        xr, lowr = x.clone().requires_grad_(True), low.clone().requires_grad_(True)
        tr.set_bf16_emulation(emulate)
        try:
            lr = tr.decoder(tr.aspp(xr, sd, "aspp"), lowr, sd, "decoder")
            lr.backward(glo)
        finally:
            tr.set_bf16_emulation(False)
        runs[emulate] = dict(y=lr.detach(), dx=xr.grad, dlow=lowr.grad,
                             **{k: v.grad.clone() for k, v in sd.items() if v.grad is not None})
        for v in sd.values():
            v.grad = None
    xd, lowd = ops.to_nhwc(x.to(cuda)).requires_grad_(True), ops.to_nhwc(low.to(cuda)).requires_grad_(True)
    lo = mod(xd, lowd)
    lo.backward(glo.to(cuda))
    torch.cuda.synchronize()
    ours = dict(y=lo[:, :19], dx=xd.grad, dlow=lowd.grad, **{n: p.grad for n, p in mod.named_parameters()})
    ref, emu = runs[False], runs[True]
    outside = []
    for k, v in ours.items():
        e, spread = norm_err(v, ref[k]), norm_err(emu[k], ref[k])
        if e > 1.5 * spread + 1e-2:
            outside.append((k, round(e, 4), round(spread, 4)))
    assert not outside, outside[:10]
    mod.eval()
    with torch.no_grad():
        le = mod(xd.detach(), lowd.detach())
        sde = {k: v.detach().cpu() for k, v in mod.state_dict().items()}
        tr.set_bf16_emulation(True)
        try:
            lre = tr.decoder(tr.aspp(x, sde, "aspp", training=False), low, sde, "decoder", training=False)
        finally:
            tr.set_bf16_emulation(False)
    assert norm_err(le[:, :19], lre) < 1e-2, norm_err(le[:, :19], lre)


def _build(cuda, N=4, H=80, W=112, seed=0, ohem=True):
    import torchseg_b200
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(seed)
    crit = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=N * H * W // 16, use_weight=False)
    model = DeepLabV3Plus(19, crit, norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    model.aspp.dropout.p = 0.0
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = make_labels(N, H, W, 19, 255, g)
    return model, sd, x, y, N * H * W // 16


def test_deeplabv3plus_step_matches_oracle(cuda):
    """a non-square crop that is not a multiple of 16, with the bar of the other untrained R101 lines (DESIGN §5): loss
    within 1e-2 of the fp32 oracle, classifier-gradient direction (cos > 0.9), per-parameter gradient magnitudes within
    ±33 % of the fp32 oracle's or of its bf16-storage emulation's (`set_bf16_emulation`): below the ASPP the
    batch-statistics BN layers of the untrained network amplify bf16 rounding into the gradient's size, which the
    emulation reproduces and the fp32 oracle does not; in the ASPP it is the other way round."""
    import deeplabv3plus_oracle as tr
    model, sd, x, y, min_kept = _build(cuda, N=4, H=90, W=118)
    check_step_vs_oracle(cuda, model, sd, x, y, lambda x, y, sd: tr.deeplabv3plus_loss(x, y, sd, min_kept),
                         ("decoder.classifier.weight", "decoder.classifier.bias"), keep=lambda p: p.dim() == 4,
                         finite=False)


def _groups(model):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return groups


def _make(cuda, seed):
    from torchseg_b200 import optim
    model, _, x, y, _ = _build(cuda, seed=seed)
    return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)


def test_deeplabv3plus_train_steps_decrease_loss_and_reproduce(cuda):
    check_train_reproducible(lambda: _make(cuda, 3))


def test_deeplabv3plus_graphed_step_matches_eager(cuda):
    check_graphed_matches_eager(lambda: _make(cuda, 7))


def test_deeplabv3plus_eval_forward_matches_oracle_and_sliding_eval(cuda):
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    import deeplabv3plus_oracle as tr
    check_eval_vs_oracle_and_sliding(cuda, lambda: DeepLabV3Plus(19, None), tr.deeplabv3plus_eval, 19)
