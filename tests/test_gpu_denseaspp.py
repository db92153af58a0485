"""DenseASPP on the H100: the pre-activation 1x1 kernels (tsb_conv1x1_bnrelu_{fprop,wgrad}) bit for bit against
tsb_bn_apply followed by the plain convolution, tsb_bn_bwd_apply_add against tsb_bn_bwd_apply and float64, the dilated
3x3 convolutions of the head against float64, the DenseASPP module teacher-forced against the bf16-emulating oracle,
its peak memory, and the whole training and eval step against the fp32 oracle (tests/denseaspp_oracle.py, pinned to the
live reference composition by tests/test_cpu_denseaspp.py)."""
import ctypes

import pytest
import torch

from util import norm_err, bf16_round
from net_checks import (check_step_vs_oracle, check_train_reproducible, check_graphed_matches_eager,
                        check_eval_vs_oracle_and_sliding)

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d


# ------------------------------------------------------------------------------------------------------- kernels
def _act(N, C, H, W, dev, g, cs=None, nan_pad=True):
    """bf16 NHWC [N,C,H,W] channel slice of a [.., cs] buffer whose channels past C hold NaN"""
    from torchseg_b200 import ops
    cs = C if cs is None else cs
    buf = torch.full((N, H, W, cs), float("nan") if nan_pad else 0.0, dtype=torch.bfloat16, device=dev)
    buf[..., :C] = torch.randn(N, H, W, C, generator=g, device=dev).to(torch.bfloat16)
    return buf[..., :C].permute(0, 3, 1, 2)


def _bn_apply_relu(x, sc, sh):
    from torchseg_b200 import ops
    N, C, H, W = x.shape
    y = ops.nhwc_empty(N, C, H, W, device=x.device)
    ops.call("tsb_bn_apply", ops.ptr(x), ops.cs_of(x), ops.ptr(sc), ops.ptr(sh), None, 0, 1, ops.ptr(y), C, N * H * W, C,
             ops.stream())
    return y


def _scale_shift(C, dev, g):
    sc = (torch.randn(C, generator=g, device=dev) * 0.8).contiguous()     # negative scales included
    sh = (torch.randn(C, generator=g, device=dev) * 0.5).contiguous()
    return sc, sh


@pytest.mark.parametrize("N,H,W", [(2, 97, 97), (1, 8, 16)])
@pytest.mark.parametrize("C", [64, 2176, 2560])
@pytest.mark.parametrize("K", [64, 512])
def test_conv1x1_bnrelu_fprop_bit_exact(cuda, N, H, W, C, K):
    """training form (statistics epilogue) and eval form (bias + ReLU) against tsb_bn_apply(relu) + tsb_conv2d_fprop /
    tsb_conv2d_fprop_fused: y, sum and sumsq bit for bit; the input a NaN-padded channel slice, the output a slice"""
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C + K + H)
    x = _act(N, C, H, W, cuda, g, cs=C + 64)
    sc, sh = _scale_shift(C, cuda, g)
    aux = torch.stack([sc, sh, sc, sh]).contiguous()
    w = (torch.randn(K, 1, 1, C, generator=g, device=cuda) * C ** -0.5).to(torch.bfloat16).contiguous()
    bias = torch.randn(K, generator=g, device=cuda).contiguous()
    xh = _bn_apply_relu(x, sc, sh)
    shp = ops.make_shape(N, H, W, C, K, 1, 1, 0, 1)
    for train in (True, False):
        outs = []
        for fused in (True, False):
            ybuf = torch.full((N, H, W, K + 32), 7.0, dtype=torch.bfloat16, device=cuda)
            y = ybuf[..., 16:16 + K].permute(0, 3, 1, 2)
            st = torch.zeros((2, K), dtype=torch.float32, device=cuda) if train else None
            s1, s2 = (None, None) if st is None else (st[0], st[1])
            if fused:
                ops.call("tsb_conv1x1_bnrelu_fprop", ctypes.byref(shp), ops.ptr(x), ops.cs_of(x), ops.ptr(aux[2]), ops.ptr(aux[3]),
                         ops.ptr(w), None if train else ops.ptr(bias), 0 if train else 1, ops.ptr(y), 1, K + 32,
                         ops.ptr(s1), ops.ptr(s2), *ops.det_ws(), ops.stream())
            elif train:
                ops.call("tsb_conv2d_fprop", ctypes.byref(shp), ops.ptr(xh), C, ops.ptr(w), None, ops.ptr(y), 1, K + 32, ops.ptr(s1),
                         ops.ptr(s2), *ops.det_ws(), ops.stream())
            else:
                ops.call("tsb_conv2d_fprop_fused", ctypes.byref(shp), ops.ptr(xh), C, ops.ptr(w), ops.ptr(bias), None, 0, 1, ops.ptr(y),
                         1, K + 32, ops.stream())
            outs.append((ybuf.clone(), None if st is None else st.clone()))
        (ya, sa), (yb, sb) = outs
        assert torch.equal(ya.view(torch.int16), yb.view(torch.int16)), train
        assert bool((ya[..., :16] == 7).all() and (ya[..., 16 + K:] == 7).all())
        if train:
            assert torch.equal(sa.view(torch.int32), sb.view(torch.int32))


@pytest.mark.parametrize("C,K,npix", [(64, 512, 2 * 97 * 97), (2176, 512, 2 * 97 * 97), (2560, 64, 1000),
                                      (2432, 512, 75272)])
@pytest.mark.parametrize("ws", [True, False])
def test_conv1x1_bnrelu_wgrad_bit_exact(cuda, C, K, npix, ws):
    """dw against tsb_bn_apply(relu) + tsb_conv2d_wgrad, with the multi-split workspace and with none (one split adding
    in place), into a non-zero dw"""
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C + K)
    x = _act(1, C, 1, npix, cuda, g, cs=C + 8)
    dy = _act(1, K, 1, npix, cuda, g)
    sc, sh = _scale_shift(C, cuda, g)
    xh = _bn_apply_relu(x, sc, sh)
    shp = ops.make_shape(1, 1, npix, C, K, 1, 1, 0, 1)
    w0 = torch.randn(K, 1, 1, C, generator=g, device=cuda)
    wsp = ops.det_ws() if ws else (None, 0)
    a, b = w0.clone(), w0.clone()
    ops.call("tsb_conv1x1_bnrelu_wgrad", ctypes.byref(shp), ops.ptr(x), C + 8, ops.ptr(sc), ops.ptr(sh), ops.ptr(dy), K, ops.ptr(a),
             *wsp, ops.stream())
    ops.call("tsb_conv2d_wgrad", ctypes.byref(shp), ops.ptr(xh), C, ops.ptr(dy), K, ops.ptr(b), *wsp, ops.stream())
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert float((a - w0).abs().max()) > 0


def _bwd_apply(name, dy, x, aux, gamma, red, count, dx, fold=None):
    from torchseg_b200 import ops
    N, C, H, W = x.shape
    ops.call(name, ops.ptr(dy), ops.cs_of(dy), None, 0, ops.ptr(x), ops.cs_of(x), ops.ptr(aux[0]), ops.ptr(aux[1]),
             ops.ptr(gamma), ops.ptr(red[0]), ops.ptr(red[1]), count, 1, ops.ptr(dx), ops.cs_of(dx), None, 0, N * H * W, C,
             None if fold is None else ops.ptr(fold[0]), None if fold is None else ops.ptr(fold[1]), ops.ptr(aux[2]),
             ops.ptr(aux[3]), ops.stream())


@pytest.mark.parametrize("C", [64, 2176])
def test_bn_bwd_apply_add(cuda, C):
    """onto a zero dx: tsb_bn_bwd_apply's result; onto a non-zero dx slice: within one bf16 ulp of float64
    dx + r, deterministic, the parameter-gradient folding as tsb_bn_bwd_apply's"""
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C)
    N, H, W = 2, 33, 31
    x, dy = _act(N, C, H, W, cuda, g, cs=C + 64), _act(N, C, H, W, cuda, g)
    gamma = torch.rand(C, generator=g, device=cuda) + 0.5
    mean, invstd = torch.randn(C, generator=g, device=cuda) * 0.1, torch.rand(C, generator=g, device=cuda) + 0.5
    sc, sh = gamma * invstd, torch.randn(C, generator=g, device=cuda) * 0.3
    aux = torch.stack([mean, invstd, sc, sh]).contiguous()
    red = torch.randn(2, C, generator=g, device=cuda) * 50
    count = float(N * H * W)
    zero = ops.nhwc_zeros(N, C, H, W, device=cuda)
    plain = ops.nhwc_empty(N, C, H, W, device=cuda)
    fa, fb = torch.zeros(2, C, device=cuda), torch.zeros(2, C, device=cuda)
    _bwd_apply("tsb_bn_bwd_apply_add", dy, x, aux, gamma, red, count, zero, fold=fa)
    _bwd_apply("tsb_bn_bwd_apply", dy, x, aux, gamma, red, count, plain, fold=fb)
    assert torch.equal(zero, plain) and torch.equal(fa, fb)
    base = _act(N, C, H, W, cuda, g, cs=C + 128)
    outs = []
    for _ in range(2):
        dbuf = torch.full((N, H, W, C + 16), float("nan"), dtype=torch.bfloat16, device=cuda)
        dbuf[..., 8:8 + C] = base.permute(0, 2, 3, 1)
        d = dbuf[..., 8:8 + C].permute(0, 3, 1, 2)
        _bwd_apply("tsb_bn_bwd_apply_add", dy, x, aux, gamma, red, count, d)
        outs.append(dbuf.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    assert bool(outs[0][..., :8].isnan().all() and outs[0][..., 8 + C:].isnan().all())
    got = outs[0][..., 8:8 + C].double()
    # float64 r: A·dz + B·x + C with the mask recomputed from scale / shift
    xd, gd = x.permute(0, 2, 3, 1).double(), dy.permute(0, 2, 3, 1).double()
    m, i_s, ga = mean.double(), invstd.double(), gamma.double()
    gd = torch.where(torch.addcmul(sh.double(), xd, sc.double()) > 0, gd, torch.zeros_like(gd))
    A = ga * i_s
    B = -A * i_s * red[1].double() / count
    Cc = -A * red[0].double() / count - B * m
    ref = base.permute(0, 2, 3, 1).double() + A * gd + B * xd + Cc
    ulp = torch.maximum(ref.abs(), torch.full_like(ref, 1e-30)).log2().floor().exp2() * 2.0 ** -7
    assert bool(((got - ref).abs() <= ulp * 1.0001 + 1e-6).all()), float(((got - ref).abs() / ulp).max())


@pytest.mark.parametrize("HW", [97, 17])
@pytest.mark.parametrize("d", [3, 6, 12, 18, 24])
def test_dilated_3x3_convs_vs_float64(cuda, HW, d):
    """the head's 3x3 convs, 512 → 128 at dilation d: fprop (+bias), dgrad and wgrad against float64 on the same bf16
    operands. At 17 x 17, d >= 18 puts every off-centre tap wholly outside the map."""
    import torch.nn.functional as F
    from torchseg_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(d * 100 + HW)
    N, C, K = 2, 512, 128
    x = ops.to_nhwc(torch.randn(N, C, HW, HW, generator=g, device=cuda))
    w = torch.randn(K, C, 3, 3, generator=g, device=cuda) * (9 * C) ** -0.5
    wk = w.permute(0, 2, 3, 1).contiguous()
    wb = wk.to(torch.bfloat16)
    wt = torch.empty((C, 3, 3, K), dtype=torch.bfloat16, device=cuda)
    ops.call("tsb_pack_weight", ops.ptr(wk), K, 3, 3, C, None, ops.ptr(wt), ops.stream())
    bias = torch.randn(K, generator=g, device=cuda)
    dy = ops.to_nhwc(torch.randn(N, K, HW, HW, generator=g, device=cuda))
    y = ops.conv_fprop(x, wb, K, 3, 1, d, d, bias=bias)
    dx = ops.conv_dgrad(dy, wt, x.shape, K, 3, 1, d, d)
    dw = torch.zeros(K, 3, 3, C, device=cuda)
    ops.conv_wgrad(x, dy, K, 3, 1, d, d, dw)
    x64 = x.double().requires_grad_(True)
    w64 = wb.permute(0, 3, 1, 2).double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, bias.double(), 1, d, d)
    y64.backward(dy.double())
    assert norm_err(y, y64) < 5e-3, norm_err(y, y64)
    assert norm_err(dx, x64.grad) < 5e-3, norm_err(dx, x64.grad)
    assert norm_err(dw.permute(0, 3, 1, 2), w64.grad) < 1e-4, norm_err(dw.permute(0, 3, 1, 2), w64.grad)
    if HW == 17 and d >= 18:   # only the centre tap sees the map
        cen = F.conv2d(x.double(), w64.detach()[:, :, 1:2, 1:2], bias.double())
        assert norm_err(y, cen) < 5e-3


# ------------------------------------------------------------------------------------------------------- module
def _module(cuda, Cin=256, mid=128, out=64, rates=(3, 6, 12, 18, 24), seed=0):
    from torchseg_b200.seg_opr.seg_oprs import DenseASPPModule
    torch.manual_seed(seed)
    mod = DenseASPPModule(Cin, mid, out, rates, dropout=0.0)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, BN):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.2)
    return mod


def test_dense_aspp_module_teacher_forced(cuda):
    """DenseASPPModule (training) against the bf16-emulating oracle: output, input gradient, the running statistics
    after the forward, and every parameter gradient within 2e-2 of the emulation's or within 1.5x the distance between
    the fp32 oracle and its emulation (+1e-2): the later blocks' pre_bn sit at the end of a long bf16 chain"""
    import torchseg_b200
    from torchseg_b200 import ops
    import denseaspp_oracle as tr
    mod = _module(cuda)
    g = torch.Generator().manual_seed(3)
    x = bf16_round(torch.relu(torch.randn(2, 256, 23, 19, generator=g)))
    gy = torch.randn(2, 256 + 5 * 64, 23, 19, generator=g)
    sd = {"m." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    for kk, vv in sd.items():
        if vv.is_floating_point() and "running" not in kk:
            vv.requires_grad_(True)
    xp = x.clone().requires_grad_(True)
    (tr.dense_aspp(xp, sd, "m", stats={}) * gy).sum().backward()
    ref32 = {kk: vv.grad.clone() for kk, vv in sd.items() if vv.grad is not None}
    for vv in sd.values():
        vv.grad = None
    xr = x.clone().requires_grad_(True)
    stats = {}
    tr.set_bf16_emulation(True)
    try:
        yr = tr.dense_aspp(xr, sd, "m", stats=stats)
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
        emu = sd["m." + n].grad
        assert float(emu.norm()) > 0, n
        e = norm_err(p.grad, emu)
        assert e < 2e-2 or norm_err(p.grad, ref32["m." + n]) <= 1.5 * norm_err(emu, ref32["m." + n]) + 1e-2, (n, e)
    for n, b in mod.named_buffers():
        if "running" in n:
            assert norm_err(b, stats["m." + n]) < 1e-2, n


def test_dense_aspp_module_eval_matches_oracle(cuda):
    import torchseg_b200
    from torchseg_b200 import ops
    import denseaspp_oracle as tr
    mod = _module(cuda, seed=4)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, BN):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    sd = {"m." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    x = bf16_round(torch.relu(torch.randn(2, 256, 19, 21, generator=g)))
    tr.set_bf16_emulation(True)
    try:
        ref = tr.dense_aspp(x, sd, "m", training=False)
    finally:
        tr.set_bf16_emulation(False)
    mod.to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.eval()
    with torch.no_grad():
        y = mod(ops.to_nhwc(x.to(cuda)))
    assert norm_err(y, ref) < 1e-2, norm_err(y, ref)


def test_dense_aspp_forward_peak_memory(cuda):
    """the training forward of the full-width head at 8 x 97² (the 769² crop at output stride 8) allocates no more than
    the concatenation, each block's 512-channel BatchNorm tensors (raw and output), the largest 1x1 conv's
    statistics-free transients and 64 MB of slack: far below the 1.43 GB of normalised copies of the suffixes"""
    import torchseg_b200
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr.seg_oprs import DenseASPPModule
    mod = DenseASPPModule().to(cuda)
    torchseg_b200.prepare_model(mod)
    mod.train()
    N, H, W = 8, 97, 97
    x = ops.to_nhwc(torch.relu(torch.randn(N, 2048, H, W, device=cuda)))
    mod(x)   # packs, workspaces, zero arena
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    y = mod(x)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    px = N * H * W
    bound = px * 2688 * 2 + 5 * 2 * px * 512 * 2 + (64 << 20)
    assert grown <= bound, (grown, bound)
    assert grown < px * 9472 * 2, grown
    del y


# ------------------------------------------------------------------------------------------------------- step level
def _build(cuda, N=2, H=129, W=129, seed=0, criterion=None):
    import torchseg_b200
    from torchseg_b200.networks import DenseASPP
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(seed)
    crit = torch.nn.CrossEntropyLoss(ignore_index=255) if criterion is None else criterion
    model = DenseASPP(19, crit, norm_layer=BN)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    for blk in model.aspp.blocks:
        blk.dropout = 0.0
    model.dropout.p = 0.0
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = torch.randint(0, 19, (N, H, W), generator=g)
    y[:, :5] = 255
    return model, sd, x, y


def test_denseaspp_step_matches_oracle(cuda):
    """2 x 129² (a ragged 17 x 17 map): loss within 1e-2 of the fp32 oracle, classifier gradient direction (cos > 0.9),
    per-weight gradient magnitudes within ±33 % of the fp32 oracle's or of its bf16-storage emulation's"""
    import denseaspp_oracle as tr
    model, sd, x, y = _build(cuda)
    check_step_vs_oracle(cuda, model, sd, x, y, tr.denseaspp_loss, ("cls.weight", "cls.bias"))


def _groups(model, lr=1e-2):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.backbone, BN, lr)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 10 * lr)
    return groups


def test_denseaspp_train_steps_decrease_loss_and_reproduce(cuda):
    """five SGD steps at lr 2e-4 (business layers 2e-3): the loss falls and two seeded runs agree bit for bit. At the
    OCNet test's 1e-2 / 1e-1 this randomly initialised head diverges, in the fp32 oracle as here."""
    from torchseg_b200 import optim

    def make():
        model, _, x, y = _build(cuda, N=2, H=97, W=113, seed=3)
        for blk in model.aspp.blocks:
            blk.dropout = 0.1       # the dropout masks come from the seeded RNG too
        torch.manual_seed(17)
        return model, optim.SGD(_groups(model, 2e-4), lr=2e-4, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_train_reproducible(make)


def test_denseaspp_graphed_step_matches_eager_and_runs_no_aten_gemm(cuda):
    from torchseg_b200 import optim
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d

    def make():
        crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=2 * 96 * 96 // 16)
        model, _, x, y = _build(cuda, N=2, H=96, W=96, seed=7, criterion=crit)
        return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

    check_graphed_matches_eager(make, kernels=("igemm_v2_bnrelu_kernel", "wgrad_mnmajor_bnrelu_kernel",
                                               "bn_bwd_apply_add_kernel"))


def test_denseaspp_full_size_step_runs(cuda):
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
    for blk in model.aspp.blocks:
        for p in (blk.reduce.conv.weight, blk.conv.weight):
            assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().max()) > 0


def test_denseaspp_eval_forward_matches_oracle_and_sliding_eval(cuda):
    from torchseg_b200.networks import DenseASPP
    import denseaspp_oracle as tr
    check_eval_vs_oracle_and_sliding(cuda, lambda: DenseASPP(19, None), tr.denseaspp_eval, 19)
