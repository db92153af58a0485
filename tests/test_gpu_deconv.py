"""Transposed convolution (DeConvBnRelu, seg_oprs.py:49-73) on the wgmma kernels.

Bit-exact part: small-integer operands (every product and partial sum an exact fp32 number) against float64 autograd
of F.conv_transpose2d, dense and as channel slices of NaN-padded buffers written into sentinel-filled outputs, in the
style of test_gpu_conv_exact.py. The forward is tsb_conv_transpose2d_fprop (dgrad-form parity-class launches with the
fprop epilogue); dx and dW are the adjoint conv's fprop and wgrad. Module part: DeConvBnRelu against the stock
nn.ConvTranspose2d + BatchNorm2d + ReLU in fp32, and a small encoder-decoder trained with the fused SGD, eagerly and
as a captured CUDA graph."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from util import norm_err, rel_err

pytestmark = pytest.mark.gpu

# (N, Ci, Co, H, W, k, stride, pad, out_pad, dil) of ConvTranspose2d(Ci, Co, k, stride, pad, out_pad, dil) on H x W
CASES = [
    (2, 64, 64, 9, 7, 1, 1, 0, 0, 1),      # 1x1 stride 1: the flat GEMM
    (2, 64, 64, 9, 7, 1, 2, 0, 0, 1),      # 1x1 stride 2: three parity classes no tap reaches
    (2, 64, 128, 9, 7, 1, 2, 0, 1, 1),     # ... with output_padding 1 (odd rows / columns are tap-less)
    (2, 64, 128, 8, 8, 2, 2, 0, 0, 1),     # 2x2/2 up-conv: one tap per class, BN = 128 tile
    (2, 128, 64, 9, 7, 3, 1, 1, 0, 1),     # 3x3 stride 1
    (2, 128, 64, 9, 7, 3, 2, 1, 1, 1),     # 3x3/2 output_padding 1: classes of 1, 2 and 4 taps
    (2, 64, 192, 7, 5, 4, 2, 1, 0, 1),     # 4x4/2 (FCN upscore), Co = 192: two N tiles, the second half empty
    (2, 192, 64, 5, 9, 3, 2, 0, 0, 2),     # dilation 2, pad 0, stride 2
    (1, 64, 64, 6, 5, 4, 1, 1, 0, 1),      # 4x4 stride 1: 16 taps
    (2, 64, 64, 5, 5, 3, 1, 2, 0, 2),      # dilated stride 1
    (2, 64, 64, 11, 13, 2, 2, 0, 1, 1),    # odd sizes with output_padding
    (1, 64, 64, 4, 100, 3, 1, 1, 0, 1),    # long rows: row tiles with grouped taps
    (1, 128, 64, 3, 120, 4, 2, 1, 0, 1),   # stride-2 classes of 120 columns: row tiles per class
]
MODES = ["bf16", "bias_relu_bf16", "bias_f32", "stats", "bias_relu_stats"]
_SENT16, _SENT32 = 0x7FA5, 0x7FA5A5A5
_OFF = 8


def _ints(shape, lo, hi, g, dev):
    return torch.randint(lo, hi + 1, shape, device=dev, generator=g).double()


def _slice_in(t, off, cs, fill=float("nan")):
    N, C, H, W = t.shape
    buf = torch.full((N, H, W, cs), fill, dtype=torch.bfloat16, device=t.device)
    buf[..., off:off + C] = t.permute(0, 2, 3, 1).to(torch.bfloat16)
    return buf, buf[..., off:off + C].permute(0, 3, 1, 2)


def _dense(t):
    from torchseg_b200 import ops
    return ops.to_nhwc(t.float())


def _sentinel(N, H, W, cs, dtype, dev):
    bits, sent = (torch.int32, _SENT32) if dtype == torch.float32 else (torch.int16, _SENT16)
    return torch.full((N, H, W, cs), sent, dtype=bits, device=dev).view(dtype)


def _untouched(buf, lo, hi):
    bits, sent = (torch.int32, _SENT32) if buf.dtype == torch.float32 else (torch.int16, _SENT16)
    b = buf.view(bits)
    return bool((b[..., :lo] == sent).all()) and bool((b[..., hi:] == sent).all())


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _pack(ops, w):
    """deconv weight [Ci][Co][k][k] → (wb [Ci][k][k][Co], wt [Co][k][k][Ci] flipped): the adjoint conv's two packs"""
    Ci, Co, R, _ = w.shape
    wk = w.float().permute(0, 2, 3, 1).contiguous()
    wb = torch.empty((Ci, R, R, Co), dtype=torch.bfloat16, device=w.device)
    wt = torch.empty((Co, R, R, Ci), dtype=torch.bfloat16, device=w.device)
    ops.call("tsb_pack_weight", ops.ptr(wk), Ci, R, R, Co, ops.ptr(wb), ops.ptr(wt), ops.stream())
    return wb, wt


def _out_size(case):
    N, Ci, Co, H, W, k, s, p, op, d = case
    return (H - 1) * s - 2 * p + d * (k - 1) + op + 1, (W - 1) * s - 2 * p + d * (k - 1) + op + 1


def _ids(c):
    return "N%d_Ci%d_Co%d_%dx%d_k%d_s%d_p%d_op%d_d%d" % c


@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_deconv_forward_exact(cuda, case, mode, layout):
    """y = relu?(conv_transpose(x, W) + bias) bit for bit; with statistics, Σ and Σ² of the rounded bf16 outputs (every
    output position, including those no tap reaches) bit for bit as well"""
    from torchseg_b200 import ops
    N, Ci, Co, H, W, k, s, p, op, d = case
    Ho, Wo = _out_size(case)
    stats = "stats" in mode
    has_bias, relu, f32 = "bias" in mode, "relu" in mode, "f32" in mode
    g = torch.Generator(device="cuda").manual_seed(31)
    if stats:   # integer outputs: every partial sum of Σ and Σ² is an exact fp32 integer below 2^24 (checked below)
        x, w = _ints((N, Ci, H, W), -1, 1, g, cuda), _ints((Ci, Co, k, k), -1, 1, g, cuda)
        b = _ints((Co,), -3, 3, g, cuda)
    else:       # |x| <= 2, W and bias in quarters of [-2, 2]: Ci·k² products of <= 4 on a 0.25 grid stay exact
        assert Ci * k * k * 4 / 0.25 < 2 ** 24
        x, w = _ints((N, Ci, H, W), -2, 2, g, cuda), _ints((Ci, Co, k, k), -8, 8, g, cuda) / 4
        b = _ints((Co,), -8, 8, g, cuda) / 4
    ref = F.conv_transpose2d(x, w, b if has_bias else None, s, p, op, 1, d)
    assert tuple(ref.shape[2:]) == (Ho, Wo)
    if relu:
        ref = ref.clamp_min(0)
    _, wt = _pack(ops, w)
    bias = b.float() if has_bias else None
    odt = torch.float32 if f32 else torch.bfloat16
    st = torch.zeros((2, Co), dtype=torch.float32, device=cuda) if stats else None
    if layout == "sliced":
        _, xd = _slice_in(x, _OFF, Ci + 24)
        ybuf = _sentinel(N, Ho, Wo, Co + 16, odt, cuda)
        yv = ybuf[..., _OFF:_OFF + Co].permute(0, 3, 1, 2)
        ops.conv_transpose_fprop(xd, wt, Co, k, s, p, d, op, bias=bias, relu=relu, out=yv, stats=st)
        assert _untouched(ybuf, _OFF, _OFF + Co), "a write outside the output slice"
    else:
        yv = ops.conv_transpose_fprop(_dense(x), wt, Co, k, s, p, d, op, bias=bias, relu=relu, out_dtype=odt, stats=st)
    want = ref.float() if f32 else ref.to(torch.bfloat16)
    assert torch.equal(yv.contiguous(), want.contiguous()), "forward differs"
    if stats:
        r = ref.to(torch.bfloat16).double()
        assert float(r.abs().sum(dim=(0, 2, 3)).max()) < 2 ** 24 and float((r * r).sum(dim=(0, 2, 3)).max()) < 2 ** 24
        assert torch.equal(st[0], r.sum(dim=(0, 2, 3)).float()), "Σ differs"
        assert torch.equal(st[1], (r * r).sum(dim=(0, 2, 3)).float()), "Σ² differs"


@pytest.mark.parametrize("layout", ["dense", "sliced"])
@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_deconv_backward_exact(cuda, case, layout):
    """dx = the adjoint conv's fprop of dy (fp32 output), dW = its wgrad with x and dy exchanged, into a KRSC buffer:
    both bit for bit against float64 autograd"""
    from torchseg_b200 import ops
    N, Ci, Co, H, W, k, s, p, op, d = case
    Ho, Wo = _out_size(case)
    g = torch.Generator(device="cuda").manual_seed(37)
    assert Co * k * k * 4 / 0.25 < 2 ** 24 and N * H * W * 4 < 2 ** 24
    x = _ints((N, Ci, H, W), -2, 2, g, cuda)
    w = _ints((Ci, Co, k, k), -8, 8, g, cuda) / 4
    gy = _ints((N, Co, Ho, Wo), -2, 2, g, cuda)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    F.conv_transpose2d(xr, wr, None, s, p, op, 1, d).backward(gy)
    wb, _ = _pack(ops, w)
    if layout == "sliced":
        _, xd = _slice_in(x, _OFF, Ci + 24)
        _, gyd = _slice_in(gy, _OFF, Co + 16)
        dxbuf = _sentinel(N, H, W, Ci + 16, torch.float32, cuda)
        ops.conv_fprop(gyd, wb, Ci, k, s, p, d, out=dxbuf[..., _OFF:_OFF + Ci].permute(0, 3, 1, 2))
        assert _untouched(dxbuf, _OFF, _OFF + Ci)
        dx = dxbuf[..., _OFF:_OFF + Ci]
    else:
        xd, gyd = _dense(x), _dense(gy)
        dx = ops.conv_fprop(gyd, wb, Ci, k, s, p, d, out_dtype=torch.float32).permute(0, 2, 3, 1)
    assert torch.equal(dx.contiguous(), xr.grad.permute(0, 2, 3, 1).float().contiguous()), "dx differs"
    dw = torch.zeros((Ci, k, k, Co), dtype=torch.float32, device=cuda)
    ops.conv_wgrad(gyd, xd, Ci, k, s, p, d, dw)
    assert torch.equal(dw, wr.grad.permute(0, 2, 3, 1).float()), "dW differs"


def test_deconv_stats_and_wgrad_repeat_bitwise(cuda):
    """random operands, many CTAs and all four parity classes: the statistics and dW repeat bit for bit"""
    from torchseg_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(41)
    N, Ci, Co, H, W, k, s, p, op = 16, 128, 64, 32, 32, 4, 2, 1, 0
    x = ops.to_nhwc(torch.randn((N, Ci, H, W), device=cuda, generator=g))
    gy = ops.to_nhwc(torch.randn((N, Co, 2 * H, 2 * W), device=cuda, generator=g))
    w = torch.randn((Ci, Co, k, k), device=cuda, generator=g) * 0.05
    _, wt = _pack(ops, w)
    outs = []
    for _ in range(2):
        st = torch.zeros((2, Co), dtype=torch.float32, device=cuda)
        ops.conv_transpose_fprop(x, wt, Co, k, s, p, 1, op, stats=st)
        dw = torch.zeros((Ci, k, k, Co), dtype=torch.float32, device=cuda)
        ops.conv_wgrad(gy, x, Ci, k, s, p, 1, dw)
        outs.append((st, dw))
    assert _same_bits(outs[0][0], outs[1][0]) and _same_bits(outs[0][1], outs[1][1])
    assert bool(torch.isfinite(outs[0][0]).all()) and float(outs[0][1].abs().sum()) > 0


def test_deconv_runs_no_library_convolution(cuda):
    """forward + backward of DeConvBnRelu launch only libtsb kernels: the wgmma conv kernels, no cuDNN / ATen conv"""
    import torchseg_b200
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    from torch.profiler import ProfilerActivity, profile
    m = torchseg_b200.prepare_model(DeConvBnRelu(128, 64, 4, 2, 1, 0).to(cuda))
    x = torch.randn(2, 128, 16, 16, device=cuda).to(torch.bfloat16).to(memory_format=torch.channels_last).requires_grad_(True)
    m(x).float().sum().backward()   # warm-up: packs, workspaces
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        y = m(x)
        y.backward(torch.ones_like(y))
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad = [n for n in names if any(t in n.lower() for t in ("cudnn", "convolution", "conv_transpose", "xmma", "implicit_gemm"))]
    assert not bad, bad
    assert any("igemm_v2_kernel" in n for n in names)
    assert any("wgrad" in n for n in names)


# ------------------------------------------------------------------------------------------------ module level
class _RefCBR(nn.Module):
    """stock-torch twin of ConvBnRelu / DeConvBnRelu with the same children and state_dict keys"""

    def __init__(self, conv, has_bn, has_relu):
        super().__init__()
        self.conv = conv
        if has_bn:
            self.bn = nn.BatchNorm2d(conv.out_channels)
        self.has_bn, self.has_relu = has_bn, has_relu

    def forward(self, x):
        x = self.conv(x)
        if self.has_bn:
            x = self.bn(x)
        return F.relu(x) if self.has_relu else x


def _ref_deconv(ci, co, k, s, p, op, d=1, has_bn=True, has_relu=True, bias=False):
    return _RefCBR(nn.ConvTranspose2d(ci, co, k, s, p, op, dilation=d, bias=bias), has_bn, has_relu)


def _randomize_bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.2)
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)


def _masked_backward(ref, xr, y, g, cuda):
    """ref forward on xr and backward of a random gradient into xr and ref's parameters, with ref's ReLU derivative taken
    where OUR output y is positive: an input that rounds to either side of zero in bf16 would otherwise flip the mask
    and move the gradient by O(1) at that position, which says nothing about the convolution. y.backward runs with the
    same gradient. Returns ref's output."""
    pre = ref.bn(ref.conv(xr)) if ref.has_bn else ref.conv(xr)
    assert tuple(y.shape) == tuple(pre.shape)
    gy = torch.randn(pre.shape, generator=g).to(cuda)
    y.float().backward(gy)
    if ref.has_relu:
        pre.backward(gy * (y.float() > 0).float())
        return F.relu(pre)
    pre.backward(gy)
    return pre


def _pair(cuda, ci, co, k, s, p, op, seed, **kw):
    import torchseg_b200
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    torch.manual_seed(seed)
    has_bn = kw.get("has_bn", True)
    ours = DeConvBnRelu(ci, co, k, s, p, op, has_bn=has_bn, has_bias=kw.get("bias", False),
                        has_relu=kw.get("has_relu", True))
    _randomize_bn(ours, seed)
    ref = _ref_deconv(ci, co, k, s, p, op, has_bn=has_bn, has_relu=kw.get("has_relu", True), bias=kw.get("bias", False))
    ref.load_state_dict(ours.state_dict())
    return torchseg_b200.prepare_model(ours.to(cuda)), ref.to(cuda)


@pytest.mark.parametrize("geo", [(64, 64, 4, 2, 1, 0), (128, 64, 3, 2, 1, 1), (64, 128, 2, 2, 0, 0), (19, 19, 4, 2, 1, 0)],
                         ids=["4x4s2", "3x3s2op1", "2x2s2", "ragged19"])
def test_deconv_module_train_matches_torch(cuda, geo):
    ci, co, k, s, p, op = geo
    ours, ref = _pair(cuda, ci, co, k, s, p, op, seed=5)
    ours.train()
    ref.train()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(4, ci, 17, 15, generator=g).to(cuda)
    xo = x.clone().requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    y = ours(xo)
    yr = _masked_backward(ref, xr, y, g, cuda)
    assert rel_err(y, yr) < 1e-2, rel_err(y, yr)
    assert norm_err(xo.grad, xr.grad) < 1e-2, norm_err(xo.grad, xr.grad)
    for name in ("conv.weight", "bn.weight", "bn.bias"):
        a, b = ours.get_parameter(name).grad, ref.get_parameter(name).grad
        assert norm_err(a, b) < 1e-2, (name, norm_err(a, b))
    assert norm_err(ours.bn.running_mean, ref.bn.running_mean) < 1e-2
    assert norm_err(ours.bn.running_var, ref.bn.running_var) < 1e-2


@pytest.mark.parametrize("geo", [(64, 64, 4, 2, 1, 0), (128, 64, 3, 2, 1, 1), (128, 128, 1, 2, 0, 1)],
                         ids=["4x4s2", "3x3s2op1", "1x1s2op1"])
def test_deconv_module_eval_folded_matches_torch(cuda, geo):
    ci, co, k, s, p, op = geo
    ours, ref = _pair(cuda, ci, co, k, s, p, op, seed=7)
    ours.eval()
    ref.eval()
    x = torch.randn(2, ci, 13, 16, generator=torch.Generator().manual_seed(8)).to(cuda)
    with torch.no_grad():
        y, yr = ours(x), ref(x)
    assert rel_err(y, yr) < 1e-2, rel_err(y, yr)


@pytest.mark.parametrize("geo", [(64, 64, 4, 2, 1, 0), (19, 19, 4, 2, 1, 0), (64, 128, 3, 1, 1, 0)],
                         ids=["4x4s2", "ragged19", "3x3s1"])
@pytest.mark.parametrize("relu", [False, True])
def test_deconv_module_bias_without_bn(cuda, geo, relu):
    ci, co, k, s, p, op = geo
    ours, ref = _pair(cuda, ci, co, k, s, p, op, seed=9, has_bn=False, bias=True, has_relu=relu)
    with torch.no_grad():
        ours.conv.bias.copy_(torch.randn(co) * 0.3)
        ref.conv.bias.copy_(ours.conv.bias)
    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, ci, 11, 12, generator=g).to(cuda)
    xo, xr = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    y = ours(xo)
    yr = _masked_backward(ref, xr, y, g, cuda)
    assert rel_err(y, yr) < 1e-2, rel_err(y, yr)
    assert norm_err(xo.grad, xr.grad) < 1e-2
    assert norm_err(ours.conv.weight.grad, ref.conv.weight.grad) < 1e-2
    assert norm_err(ours.conv.bias.grad, ref.conv.bias.grad) < 1e-2


# ------------------------------------------------------------------------------------------------ encoder-decoder
def _encdec(stock):
    """ConvBnRelu ↓2 → DeConvBnRelu 4x4/2 ↑2 → ConvBnRelu ↓2 → DeConvBnRelu 3x3/2 op 1 ↑2 → 1x1 19-class head"""
    if stock:
        C = lambda ci, co, k, s, p: _RefCBR(nn.Conv2d(ci, co, k, s, p, bias=False), True, True)  # noqa: E731
        D = _ref_deconv
        head = _RefCBR(nn.Conv2d(64, 19, 1, bias=True), False, False)
    else:
        from torchseg_b200.seg_opr.seg_oprs import ConvBnRelu, DeConvBnRelu
        C = lambda ci, co, k, s, p: ConvBnRelu(ci, co, k, s, p)  # noqa: E731
        D = DeConvBnRelu
        head = ConvBnRelu(64, 19, 1, 1, 0, has_bn=False, has_relu=False, has_bias=True)
    return nn.Sequential(C(64, 128, 3, 2, 1), D(128, 64, 4, 2, 1, 0), C(64, 128, 3, 2, 1), D(128, 64, 3, 2, 1, 1), head)


class _Net(nn.Module):
    def __init__(self, stock):
        super().__init__()
        self.body = _encdec(stock)

    def forward(self, x, y):
        # log-softmax, gather and mean: a loss whose forward and backward have a fixed summation order
        lp = self.body(x).float().log_softmax(1)
        return -lp.gather(1, y[:, None]).mean()


def _make_net(cuda, seed):
    import torchseg_b200
    torch.manual_seed(seed)
    net = _Net(False)
    _randomize_bn(net, seed)
    return torchseg_b200.prepare_model(net.to(cuda))


def _data(cuda, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(4, 64, 32, 32, generator=g).to(cuda), torch.randint(0, 19, (4, 32, 32), generator=g).to(cuda)


def test_encoder_decoder_matches_stock_torch_and_trains(cuda):
    from torchseg_b200 import optim
    net = _make_net(cuda, 12)
    ref = _Net(True).to(cuda)
    ref.load_state_dict(net.state_dict())     # identical keys: the stock twin takes our checkpoint as it is
    x, y = _data(cuda, 13)
    net.train()
    ref.train()
    loss = net(x, y)
    loss.backward()
    lr = ref(x, y)
    lr.backward()
    assert abs(loss.item() - lr.item()) < 1e-2 * abs(lr.item()), (loss.item(), lr.item())
    for (n, a), (_, b) in zip(net.named_parameters(), ref.named_parameters()):
        cos = F.cosine_similarity(a.grad.flatten().float(), b.grad.flatten().float(), dim=0).item()
        assert cos > 0.8, (n, cos)
    net.zero_grad(set_to_none=True)
    opt = optim.SGD(net.parameters(), lr=0.05, momentum=0.9)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = net(x, y)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0], losses


def test_encoder_decoder_graphed_step_matches_eager_bitwise(cuda):
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        def make():
            net = _make_net(cuda, 14)
            net.train()
            x, y = _data(cuda, 15)
            return net, optim.SGD(net.parameters(), lr=0.02, momentum=0.9, weight_decay=1e-4), x, y

        net, opt, x, y = make()
        eager = []
        for _ in range(4):
            opt.zero_grad()
            loss = net(x, y)
            loss.backward()
            opt.step()
            eager.append(loss.detach().clone())
        del loss
        net, opt, x, y = make()
        step = GraphedTrainStep(net, opt, [x, y], warmup=2)
        assert step.graph is not None, step.error
        graphed = [step(x, y).detach().clone() for _ in range(2)]
        for a, b in zip(eager[2:], graphed):
            assert _same_bits(a, b), ([e.item() for e in eager], [g.item() for g in graphed])
        step.release()
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())
