"""GPU parity tests of the HBM-bound libtsb kernels against plain PyTorch fp32 references and the C oracle.
Tolerances: fp32 paths 1e-3 relative (north_star), bf16 paths 1e-2; OHEM selected indices bit-exact."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import rel_err, bf16_round, make_labels

pytestmark = pytest.mark.gpu


def _ops():
    from torchseg_b200 import ops
    return ops


# ----------------------------------------------------------------------------------------------- OHEM
def _ohem_case(regime, N=2, C=19, H=64, W=96, seed=0):
    g = torch.Generator().manual_seed(seed)
    labels = make_labels(N, H, W, C, 255, g)
    logits = torch.randn(N, C, H, W, generator=g)
    min_kept = N * H * W // 16
    if regime == "B":    # few hard pixels: threshold becomes the k-th smallest p (> 0.7)
        onehot = F.one_hot(labels.clamp(max=C - 1), C).permute(0, 3, 1, 2).float()
        logits = 8 * onehot + logits
    elif regime == "C":  # min_kept > num_valid → no OHEM
        min_kept = N * H * W
    elif regime == "D":  # min_kept = 0 → no filtering
        min_kept = 0
    elif regime == "E":  # everything ignored
        labels[:] = 255
    return logits, labels, min_kept


@pytest.mark.parametrize("regime", ["A", "B", "C", "D", "E"])
def test_ohem_materialised_bit_exact(cuda, regime):
    ops = _ops()
    from oracle import c_oracle
    logits, labels, min_kept = _ohem_case(regime)
    ref = c_oracle.ohem(logits.numpy(), labels.numpy(), 255, 0.7, min_kept, want_grad=True)
    pred = logits.to(cuda).requires_grad_(True)
    loss = ops.OhemCEFn.apply(pred, labels.to(cuda), 255, 0.7, min_kept, None)
    loss.backward(retain_graph=True)
    fn = loss.grad_fn
    _, _, p, state, _ = fn.saved_tensors
    st = ops.ohem_state_dict(state)
    p = p.cpu().numpy()
    assert np.array_equal(p.view(np.uint32), ref["p"].view(np.uint32)), "p_target bits differ from the oracle"
    assert st["active"] == ref["active"]
    if ref["active"]:
        assert np.float32(st["T"]).view(np.uint32) == np.float32(ref["T"]).view(np.uint32)
    lab = labels.numpy().reshape(-1)
    kept = (lab != 255) & ((not st["active"]) | (p <= np.float32(st["T"])))
    assert np.array_equal(kept, ref["kept"]), "kept index set differs from the oracle"
    assert st["kept"] == int(ref["kept"].sum())
    if regime == "E":
        assert np.isnan(loss.item()) and np.isnan(ref["loss"])
    else:
        assert abs(loss.item() - ref["loss"]) <= 1e-5 * abs(ref["loss"])
        assert rel_err(pred.grad, torch.from_numpy(ref["dlogits"])) < 1e-4


def test_ohem_matches_torch_reference_loss(cuda):
    ops = _ops()
    from oracle import torch_ref
    logits, labels, min_kept = _ohem_case("B", seed=3)
    ref = torch_ref.ohem_ce(logits.clone().requires_grad_(True), labels, 255, 0.7, min_kept)
    out = ops.OhemCEFn.apply(logits.to(cuda), labels.to(cuda), 255, 0.7, min_kept, None)
    assert abs(out.item() - ref.item()) < 1e-4 * abs(ref.item())


def test_ohem_class_weight_and_bf16(cuda):
    ops = _ops()
    from oracle import c_oracle
    logits, labels, min_kept = _ohem_case("A", seed=5)
    w = torch.linspace(0.5, 2.0, 19)
    lb = bf16_round(logits)
    ref = c_oracle.ohem(lb.numpy(), labels.numpy(), 255, 0.7, min_kept, class_weight=w.numpy())
    out = ops.OhemCEFn.apply(lb.to(cuda).to(torch.bfloat16), labels.to(cuda), 255, 0.7, min_kept, w.to(cuda))
    assert abs(out.item() - ref["loss"]) < 1e-5 * abs(ref["loss"])


@pytest.mark.parametrize("regime", ["A", "B"])
def test_ohem_fused_upsample(cuda, regime):
    """low-res fp32 NHWC logits → on-the-fly bilinear x8 → OHEM; p / kept bit-exact vs oracle, grad vs autograd"""
    ops = _ops()
    from oracle import c_oracle, torch_ref
    N, C, h, w, s = 2, 19, 16, 24, 8
    H, W = h * s, w * s
    g = torch.Generator().manual_seed(11)
    labels = make_labels(N, H, W, C, 255, g)
    lo = torch.randn(N, h, w, 32, generator=g)
    if regime == "B":
        lab_lo = labels[:, ::s, ::s].clamp(max=C - 1)
        lo[..., :C] += 8 * F.one_hot(lab_lo, C).float()
    min_kept = N * H * W // 16
    up = c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), C, H, W)
    ref = c_oracle.ohem(up, labels.numpy(), 255, 0.7, min_kept)
    lo_dev = lo.to(cuda).permute(0, 3, 1, 2)[:, :C].requires_grad_(True)  # logical [N,19,h,w], cs = 32
    loss = ops.OhemUpCEFn.apply(lo_dev, labels.to(cuda), H, W, C, 255, 0.7, min_kept, None)
    loss.backward(retain_graph=True)
    _, _, p, state, _ = loss.grad_fn.saved_tensors
    st = ops.ohem_state_dict(state)
    p = p.cpu().numpy()
    assert np.array_equal(p.view(np.uint32), ref["p"].view(np.uint32))
    lab = labels.numpy().reshape(-1)
    kept = (lab != 255) & ((not st["active"]) | (p <= np.float32(st["T"])))
    assert np.array_equal(kept, ref["kept"])
    assert abs(loss.item() - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    # gradient wrt the low-res logits vs autograd through F.interpolate + the torch restatement
    lo_t = lo[..., :C].permute(0, 3, 1, 2).clone().requires_grad_(True)
    l2 = torch_ref.ohem_ce(F.interpolate(lo_t, scale_factor=s, mode="bilinear", align_corners=True), labels, 255, 0.7,
                           min_kept)
    l2.backward()
    assert rel_err(lo_dev.grad, lo_t.grad) < 1e-3


def test_ohem_full_size_properties(cuda):
    """BASELINE size [16,19,1024,1024] fused form: size-independent properties (kept count ≥ min(k, valid),
    threshold monotonicity, loss finite, gradient sums to ~0 over classes)"""
    ops = _ops()
    N, C, h, w, s = 16, 19, 128, 128, 8
    H, W = h * s, w * s
    g = torch.Generator(device="cuda").manual_seed(1)
    lo = torch.randn(N, h, w, 32, device=cuda, generator=g) * 3
    labels = torch.randint(0, C, (N, H, W), device=cuda, generator=g)
    labels[:, :100] = 255
    min_kept = N * H * W // 16
    lo_v = lo.permute(0, 3, 1, 2)[:, :C].requires_grad_(True)
    loss = ops.OhemUpCEFn.apply(lo_v, labels, H, W, C, 255, 0.7, min_kept, None)
    loss.backward(retain_graph=True)
    _, _, p, state, _ = loss.grad_fn.saved_tensors
    st = ops.ohem_state_dict(state)
    assert st["num_valid"] == int((labels != 255).sum())
    assert st["active"] and np.float32(st["T"]) >= np.float32(0.7)
    kept = int(((labels.reshape(-1) != 255) & (p <= st["T"])).sum())
    assert kept == st["kept"]
    n_le = int((p <= st["T"]).sum())
    assert n_le >= min(min_kept, N * H * W)
    assert np.isfinite(loss.item())
    gsum = lo_v.grad.float().sum(dim=1).abs().max().item()
    assert gsum < 1e-4


# ----------------------------------------------------------------------------------------------- resize / pool
@pytest.mark.parametrize("shape", [(2, 128, 1, 1, 32, 32), (2, 128, 32, 32, 64, 64), (1, 64, 15, 20, 60, 60)])
def test_bilinear_fwd_bwd(cuda, shape):
    ops = _ops()
    N, C, Hi, Wi, Ho, Wo = shape
    g = torch.Generator().manual_seed(2)
    x = bf16_round(torch.randn(N, C, Hi, Wi, generator=g))
    xr = x.clone().requires_grad_(True)
    yr = F.interpolate(xr, size=(Ho, Wo), mode="bilinear", align_corners=True)
    gy = bf16_round(torch.randn(N, C, Ho, Wo, generator=g))
    yr.backward(gy)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = ops.BilinearFn.apply(xd, Ho, Wo)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    assert rel_err(yd, yr) < 1e-2
    assert rel_err(xd.grad, xr.grad) < 1e-2


def test_bilinear_logits_nchw(cuda):
    ops = _ops()
    from oracle import c_oracle
    g = torch.Generator().manual_seed(4)
    lo = torch.randn(2, 16, 16, 32, generator=g)
    ref = c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), 19, 128, 128)
    out = torch.empty(2, 19, 128, 128, device=cuda)
    ops.call("tsb_bilinear_fwd_nhwc_to_nchw", ops.ptr(lo.to(cuda)), ops.F32, 32, ops.ptr(out), 2, 19, 16, 16, 128, 128,
             ops.stream())
    assert np.array_equal(out.cpu().numpy().view(np.uint32), ref.view(np.uint32))  # pinned op order → bit exact
    aten = F.interpolate(lo[..., :19].permute(0, 3, 1, 2), scale_factor=8, mode="bilinear", align_corners=True)
    assert rel_err(out, aten) < 1e-5


@pytest.mark.parametrize("S,HW", [(1, (32, 32)), (1, (7, 9)), (2, (60, 60)), (3, (60, 60)), (6, (60, 60)), (3, (10, 14))])
def test_adaptive_avgpool(cuda, S, HW):
    ops = _ops()
    H, W = HW
    g = torch.Generator().manual_seed(5)
    x = bf16_round(torch.randn(2, 64, H, W, generator=g))
    xr = x.clone().requires_grad_(True)
    yr = F.adaptive_avg_pool2d(xr, S)
    gy = bf16_round(torch.randn(2, 64, S, S, generator=g))
    yr.backward(gy)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = ops.AdaptiveAvgPoolFn.apply(xd, S)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    assert rel_err(yd, yr) < 1e-2
    assert rel_err(xd.grad, xr.grad) < 1e-2


@pytest.mark.parametrize("HW", [(64, 64), (33, 47)])
def test_maxpool(cuda, HW):
    ops = _ops()
    H, W = HW
    g = torch.Generator().manual_seed(6)
    x = bf16_round(torch.randn(2, 64, H, W, generator=g))
    x[0, :, 4:8, 4:8] = 1.5  # ties: the first maximum in scan order must win
    xr = x.clone().requires_grad_(True)
    yr = F.max_pool2d(xr, 3, 2, 1)
    gy = bf16_round(torch.randn_like(yr))
    yr.backward(gy)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    yd = ops.MaxPool3x3S2Fn.apply(xd)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    assert rel_err(yd, yr) == 0.0
    assert rel_err(xd.grad, xr.grad) < 1e-2


# ----------------------------------------------------------------------------------------------- BN / attention
@pytest.mark.parametrize("relu,res", [(True, False), (True, True), (False, False)])
def test_bn_kernels(cuda, relu, res):
    ops = _ops()
    N, C, H, W = 4, 64, 24, 20
    g = torch.Generator().manual_seed(7)
    x = bf16_round(torch.randn(N, C, H, W, generator=g) * 2 + 0.5)
    r = bf16_round(torch.randn(N, C, H, W, generator=g))
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g)
    gy = bf16_round(torch.randn(N, C, H, W, generator=g))
    # reference
    xr = x.clone().requires_grad_(True); rr = r.clone().requires_grad_(True)
    gr = gamma.clone().requires_grad_(True); br = beta.clone().requires_grad_(True)
    rm, rv = torch.zeros(C), torch.ones(C)
    yr = F.batch_norm(xr, rm, rv, gr, br, True, 0.1, 1e-5)
    if res: yr = yr + rr
    if relu: yr = F.relu(yr)
    yr.backward(gy)
    # device
    xd = ops.to_nhwc(x.to(cuda)); rd = ops.to_nhwc(r.to(cuda)); gyd = ops.to_nhwc(gy.to(cuda))
    gam, bet = gamma.to(cuda), beta.to(cuda)
    stats = torch.zeros(2, C, device=cuda)
    npix = N * H * W
    ops.call("tsb_bn_stats", ops.ptr(xd), C, npix, C, ops.ptr(stats[0]), ops.ptr(stats[1]), *ops.det_ws(), ops.stream())
    aux = torch.empty(4, C, device=cuda)
    rmd, rvd = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    ops.call("tsb_bn_finalize", ops.ptr(stats[0]), ops.ptr(stats[1]), float(npix), C, ops.ptr(gam), ops.ptr(bet), 1e-5,
             0.1, ops.ptr(aux[0]), ops.ptr(aux[1]), ops.ptr(aux[2]), ops.ptr(aux[3]), ops.ptr(rmd), ops.ptr(rvd), ops.stream())
    yd = ops.nhwc_empty(N, C, H, W)
    ops.call("tsb_bn_apply", ops.ptr(xd), C, ops.ptr(aux[2]), ops.ptr(aux[3]), ops.ptr(rd) if res else None, C, int(relu),
             ops.ptr(yd), C, npix, C, ops.stream())
    assert rel_err(yd, yr) < 1e-2
    assert rel_err(rmd, rm) < 1e-3 and rel_err(rvd, rv) < 1e-3
    red = torch.zeros(2, C, device=cuda)
    # residual layers read the mask from y; the others recompute it from x*scale+shift (y = NULL)
    ymask = ops.ptr(yd) if (relu and res) else None
    ops.call("tsb_bn_bwd_reduce", ops.ptr(gyd), C, ymask, C, ops.ptr(xd), C, ops.ptr(aux[0]), ops.ptr(aux[1]),
             int(relu), npix, C, ops.ptr(red[0]), ops.ptr(red[1]), ops.ptr(aux[2]), ops.ptr(aux[3]), *ops.det_ws(), ops.stream())
    dx = ops.nhwc_empty(N, C, H, W); dres = ops.nhwc_empty(N, C, H, W)
    ops.call("tsb_bn_bwd_apply", ops.ptr(gyd), C, ymask, C, ops.ptr(xd), C, ops.ptr(aux[0]), ops.ptr(aux[1]),
             ops.ptr(gam), ops.ptr(red[0]), ops.ptr(red[1]), float(npix), int(relu), ops.ptr(dx), C,
             ops.ptr(dres) if res else None, C, npix, C, None, None, ops.ptr(aux[2]), ops.ptr(aux[3]), ops.stream())
    assert rel_err(dx, xr.grad) < 2e-2
    assert rel_err(red[1], gr.grad) < 1e-2 and rel_err(red[0], br.grad) < 1e-2
    if res:
        assert rel_err(dres, rr.grad) < 1e-2


@pytest.mark.parametrize("base,add", [(0.0, True), (1.0, False)])
def test_chan_scale(cuda, base, add):
    ops = _ops()
    N, C, H, W = 3, 128, 16, 12
    g = torch.Generator().manual_seed(8)
    x = bf16_round(torch.randn(N, C, H, W, generator=g)); a = bf16_round(torch.randn(N, C, 1, 1, generator=g))
    ad = bf16_round(torch.randn(N, C, H, W, generator=g)); gy = bf16_round(torch.randn(N, C, H, W, generator=g))
    xr = x.clone().requires_grad_(True); ar = a.clone().requires_grad_(True); adr = ad.clone().requires_grad_(True)
    yr = xr * (base + torch.sigmoid(ar)) + (adr if add else 0)
    yr.backward(gy)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True); a_d = ops.to_nhwc(a.to(cuda)).requires_grad_(True)
    add_d = ops.to_nhwc(ad.to(cuda)).requires_grad_(True) if add else None
    yd = ops.ChanScaleFn.apply(xd, a_d, add_d, base)
    yd.backward(ops.to_nhwc(gy.to(cuda)))
    assert rel_err(yd, yr) < 1e-2
    assert rel_err(xd.grad, xr.grad) < 1e-2
    assert rel_err(a_d.grad, ar.grad) < 2e-2
    if add:
        assert rel_err(add_d.grad, adr.grad) < 1e-2


def test_sgd_flat_matches_torch(cuda):
    from torchseg_b200 import optim
    g = torch.Generator().manual_seed(9)
    shapes = [(64, 3, 7, 7), (64,), (128, 64, 3, 3), (19,), (5, 3)]
    ref_p = [torch.randn(s, generator=g).requires_grad_(True) for s in shapes]
    dev_p = [torch.nn.Parameter(p.detach().clone().to(cuda)) for p in ref_p]
    groups = lambda ps: [dict(params=ps[:2], lr=0.01), dict(params=ps[2:4], lr=0.1, weight_decay=0.0), dict(params=ps[4:], lr=0.05)]
    o_ref = torch.optim.SGD(groups(ref_p), lr=0.01, momentum=0.9, weight_decay=5e-4)
    o_dev = optim.SGD(groups(dev_p), lr=0.01, momentum=0.9, weight_decay=5e-4)
    for it in range(3):
        o_ref.zero_grad(); o_dev.zero_grad()
        for pr, pd in zip(ref_p, dev_p):
            gr = torch.randn(pr.shape, generator=g)
            pr.grad = gr.clone()
            pd.grad.copy_(gr.to(cuda))
        for gi in range(3):
            o_ref.param_groups[gi]["lr"] *= 0.9; o_dev.param_groups[gi]["lr"] *= 0.9
        o_ref.step(); o_dev.step()
    for pr, pd in zip(ref_p, dev_p):
        assert rel_err(pd, pr) < 1e-5


def test_focal_loss(cuda):
    from torchseg_b200.seg_opr.loss_opr import SigmoidFocalLoss
    from oracle import torch_ref
    g = torch.Generator().manual_seed(10)
    pred = torch.randn(2, 1, 32, 40, generator=g)
    tgt = torch.randint(0, 2, (2, 32, 40), generator=g); tgt[:, :3] = 255
    pr = pred.clone().requires_grad_(True)
    lr = torch_ref.sigmoid_focal(pr, tgt, 255)
    lr.backward()
    pd = pred.to(cuda).requires_grad_(True)
    ld = SigmoidFocalLoss(255)(pd, tgt.to(cuda))
    ld.backward()
    assert abs(ld.item() - lr.item()) < 1e-4 * abs(lr.item())
    assert rel_err(pd.grad, pr.grad) < 1e-3


def test_cuda_prefetcher_delivers_batches_in_order(cuda):
    """CudaPrefetcher (double-buffered H2D on a side stream, train.py:119-124): every batch arrives intact and in order
    even when the consumer launches work that is still running while the next copy is issued"""
    from torchseg_b200.utils.prefetch import CudaPrefetcher
    g = torch.Generator().manual_seed(31)
    host = [{"data": torch.randn(4, 3, 64, 96, generator=g).pin_memory(),
             "label": torch.randint(0, 19, (4, 64, 96), generator=g).pin_memory(), "fn": "img%d" % i} for i in range(7)]
    loader = CudaPrefetcher(iter(host), cuda)
    seen = 0
    big = torch.randn(4096, 4096, device=cuda)
    for i, mb in enumerate(loader):
        acc = big @ big                      # keep the compute stream busy while the next batch is copied
        s = mb["data"].double().sum() + mb["label"].double().sum()
        ref = host[i]["data"].double().sum() + host[i]["label"].double().sum()
        assert mb["fn"] == "img%d" % i
        assert abs(float(s) - float(ref)) < 1e-6 * max(1.0, abs(float(ref)))
        assert torch.equal(mb["label"].cpu(), host[i]["label"])
        seen += 1
        del acc
    assert seen == 7


@pytest.mark.parametrize("cfg", [(19, 16, False), (21, 8, True), (20, 8, False), (19, 4, True), (19, (89, 301), False),
                                 (20, (89, 301), False)],
                         ids=["c19_x16", "c21_x8_weighted", "c20_generic", "c19_x4_weighted", "c19_89x301",
                              "c20_generic_89x301"])
def test_ohem_fused_upsample_variants(cuda, cfg):
    """exact-class-count band kernels (C = 19 / 21) and the generic fallback (C = 20), scales x4 / x8 / x16 and a
    non-integer one (12 x 40 -> 89 x 301: uneven column segments), class weights: p bits and kept set vs the C oracle,
    gradient vs autograd through F.interpolate + the torch restatement"""
    ops = _ops()
    from oracle import c_oracle, torch_ref
    C, size, weighted = cfg
    N, h, w = 2, 12, 40
    H, W = (h * size, w * size) if isinstance(size, int) else size
    g = torch.Generator().manual_seed(100 + C + H // h)
    labels = make_labels(N, H, W, C, 255, g)
    lo = torch.randn(N, h, w, 32, generator=g) * 2
    lab_lo = labels[:, torch.arange(h) * H // h][:, :, torch.arange(w) * W // w].clamp(max=C - 1)
    lo[..., :C] += 3 * F.one_hot(lab_lo, C).float()
    cwt = (torch.rand(C, generator=g) + 0.5) if weighted else None
    min_kept = N * H * W // 16
    up = c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), C, H, W)
    ref = c_oracle.ohem(up, labels.numpy(), 255, 0.7, min_kept, class_weight=None if cwt is None else cwt.numpy())
    lo_dev = lo.to(cuda).permute(0, 3, 1, 2)[:, :C].requires_grad_(True)
    loss = ops.OhemUpCEFn.apply(lo_dev, labels.to(cuda), H, W, C, 255, 0.7, min_kept, None if cwt is None else cwt.to(cuda))
    loss.backward(retain_graph=True)
    _, _, p, state, _ = loss.grad_fn.saved_tensors
    st = ops.ohem_state_dict(state)
    p = p.cpu().numpy()
    assert np.array_equal(p.view(np.uint32), ref["p"].view(np.uint32))
    kept = (labels.numpy().reshape(-1) != 255) & ((not st["active"]) | (p <= np.float32(st["T"])))
    assert np.array_equal(kept, ref["kept"])
    assert abs(loss.item() - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    lo_t = lo[..., :C].permute(0, 3, 1, 2).clone().requires_grad_(True)
    l2 = torch_ref.ohem_ce(F.interpolate(lo_t, size=(H, W), mode="bilinear", align_corners=True), labels, 255, 0.7,
                           min_kept, weight=cwt)
    l2.backward()
    assert rel_err(lo_dev.grad, lo_t.grad) < 1e-3


def test_ohem_exact_kernels_match_generic_at_full_size(cuda):
    """BASELINE size (16 x 19 x 1024 x 1024, x8): the exact-class-count kernels (C = 19) against the generic band
    kernels, reached with C = 20 on the same input: the extra class has low-res logit -1e4 and no label, so its exp
    flushes to exactly 0 and leaves every class-order sum unchanged (test_cpu_oracle.py checks this premise on the C
    oracle). Identical p bits / threshold / kept set / loss, the 19 real classes' gradients equal to fp32 summation
    order, and the extra class's gradient exactly 0."""
    ops = _ops()
    N, C, h, w, s = 16, 19, 128, 128, 8
    H, W = h * s, w * s
    g = torch.Generator(device="cuda").manual_seed(5)
    lo = torch.randn(N, h, w, 32, device=cuda, generator=g) * 3
    labels = torch.randint(0, C, (N, H, W), device=cuda, generator=g)
    labels[:, :100] = 255
    lo[..., C] = -1e4
    min_kept = N * H * W // 16
    res = []
    for c in (C, C + 1):
        lo_v = lo.permute(0, 3, 1, 2)[:, :c].detach().requires_grad_(True)
        loss = ops.OhemUpCEFn.apply(lo_v, labels, H, W, c, 255, 0.7, min_kept, None)
        loss.backward(retain_graph=True)
        _, _, p, state, _ = loss.grad_fn.saved_tensors
        res.append((p.clone(), ops.ohem_state_dict(state), loss.item(), lo_v.grad.clone()))
    (p1, s1, l1, g1), (p0, s0, l0, g0) = res
    assert torch.equal(p1.view(torch.int32), p0.view(torch.int32))
    assert s1["T"] == s0["T"] and s1["kept"] == s0["kept"] and s1["active"] == s0["active"]
    assert abs(l1 - l0) <= 1e-6 * abs(l0)
    assert rel_err(g1, g0[:, :C]) < 1e-4
    assert torch.count_nonzero(g0[:, C]) == 0


@pytest.mark.parametrize("cfg", [(150, 12, 20, 96, 160, -1), (150, 11, 13, 83, 99, -1), (21, 9, 9, 72, 72, 255), (37, 6, 70, 48, 560, 255)],
                         ids=["ade150_x8", "ade150_odd_size", "c21_x8", "c37_wide"])
def test_ce_up_fused_matches_torch(cuda, cfg):
    """fused bilinear up-sampling + cross-entropy for many classes (tsb_ce_up_*, the PSPNet / PSANet head tail): loss and
    d loss / d low-res logits against F.interpolate(size=, align_corners=True) + F.cross_entropy in fp32 on the GPU;
    x8 and non-integer scale (the 713 / 473 crops), ignored pixels, strips wider than one CTA"""
    ops = _ops()
    C, h, w, H, W, ign = cfg
    N = 3
    g = torch.Generator().manual_seed(C + h + W)
    lo = torch.randn(N, C, h, w, generator=g) * 2
    labels = torch.randint(0, C, (N, H, W), generator=g)
    labels[:, : max(1, H // 10)] = ign
    labels[torch.rand(N, H, W, generator=g) < 0.05] = ign
    cs = (C + 31) // 32 * 32
    lo_d = ops.nhwc_zeros(N, C, h, w, dtype=torch.float32, device=cuda, cs=cs)
    lo_d.copy_(lo.to(cuda))
    lo_d.requires_grad_(True)
    loss = ops.CEUpFn.apply(lo_d, labels.to(cuda), H, W, C, ign)
    (loss * 1.7).backward()
    lo_t = lo.to(cuda).clone().requires_grad_(True)
    ref = F.cross_entropy(F.interpolate(lo_t, size=(H, W), mode="bilinear", align_corners=True), labels.to(cuda), ignore_index=ign)
    (ref * 1.7).backward()
    assert abs(loss.item() - ref.item()) < 2e-5 * abs(ref.item()), (loss.item(), ref.item())
    assert rel_err(lo_d.grad, lo_t.grad) < 2e-4, rel_err(lo_d.grad, lo_t.grad)
    # channels beyond C in the padded NHWC gradient buffer stay untouched
    assert tuple(lo_d.grad.shape) == (N, C, h, w)


def test_ce_up_all_ignored_is_nan_like_torch(cuda):
    ops = _ops()
    lo = ops.nhwc_zeros(1, 150, 4, 4, dtype=torch.float32, device=cuda, cs=160)
    labels = torch.full((1, 32, 32), -1, dtype=torch.int64, device=cuda)
    loss = ops.CEUpFn.apply(lo, labels, 32, 32, 150, -1)
    assert loss.item() != loss.item()        # NaN: mean over zero valid pixels, like nn.CrossEntropyLoss
