"""BiSeNet lines R18.speed, X39.speed and R101 on the H100.

* The loss at label resolution: `forward_lowres` at up-scale factor 1 (the .speed main and aux1 heads) routes to the
  strided materialised OHEM pair reading the classifier's NHWC buffer in place; at factor 2 (the .speed aux0 head,
  W < 256 columns) it stays on the band kernels. p bits, threshold and kept set against the C oracle.
* Heads teacher-forced at both factors, and the whole step of each line against the oracle
  (tests/bisenet_lines_oracle.py, pinned to the live reference by tests/test_cpu_bisenet_lines.py), all at non-square
  shapes.
* Training behaviour (loss decrease, bit-reproducible steps, graph replay), eval mode (oracle, checkpoint load into the
  aux-head-free eval network, batch-1 graph replay) and one full-size step per line.
"""
import importlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import rel_err, norm_err, make_labels, bf16_round
from net_checks import randomize_bn

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d

# line → (module under torchseg_b200.networks, label down-sampling, takes ohem_criterion)
LINES = {
    "r18_speed": ("bisenet_speed", 8, True),
    "x39_speed": ("bisenet_x39_speed", 8, True),
    "r101": ("bisenet_r101", 1, False),
}
SPEED = ["r18_speed", "x39_speed"]
# small non-square training shape of each line (N, H, W)
SMALL = {"r18_speed": (4, 128, 256), "x39_speed": (4, 128, 256), "r101": (4, 128, 192)}


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _net(line, training, crit=None):
    mod, _, two_crit = LINES[line]
    cls = importlib.import_module("torchseg_b200.networks." + mod).BiSeNet
    if two_crit:
        return cls(19, training, torch.nn.CrossEntropyLoss(ignore_index=255) if training else None, crit, None, BN)
    return cls(19, training, crit, None, BN)


def _build(cuda, line, N, H, W, seed=0):
    import torchseg_b200
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import init_weight
    gt_down = LINES[line][1]
    min_kept = N * H * W // (16 * gt_down ** 2)      # train.py: batch·H·W // (16·gt_down_sampling²)
    torch.manual_seed(seed)
    crit = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    model = _net(line, True, crit)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 3, H, W, generator=g)
    y = make_labels(N, H // gt_down, W // gt_down, 19, 255, g)
    return model, sd, x, y, min_kept


def _groups(model):
    from torchseg_b200.utils.init_func import group_weight
    groups = group_weight([], model.context_path, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return groups


# ------------------------------------------------------------------------------------------ the loss at label resolution
@pytest.mark.parametrize("regime", ["A", "B"])
@pytest.mark.parametrize("scale", [1, 2])
def test_forward_lowres_matches_c_oracle(cuda, scale, regime):
    """p bits, threshold and kept set of forward_lowres equal the C oracle's on the up-scaled logits. Factor 1: the
    strided pair reads the fp32 NHWC buffer (channel stride 32) in place, and loss and gradient equal the materialised
    path on the same logits bit for bit. Factor 2: W = 192 is narrower than one 256-column band strip."""
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from oracle import c_oracle, torch_ref
    N, C = 2, 19
    h, w = (24, 40) if scale == 1 else (12, 96)
    H, W = h * scale, w * scale
    g = torch.Generator().manual_seed(100 * scale + ord(regime))
    lo = torch.randn(N, h, w, 32, generator=g)
    if regime == "B":
        # confident logits on 4x4-pixel label blocks (so that the up-scaled logits stay confident away from the block
        # edges) and min_kept = half the pixels: the k-th smallest p exceeds 0.7 and becomes the threshold
        blk = torch.randint(0, C, (N, h // 4 + 1, w // 4 + 1), generator=g)
        lab_lo = blk.repeat_interleave(4, 1).repeat_interleave(4, 2)[:, :h, :w]
        lo[..., :C] += 8 * F.one_hot(lab_lo, C).float()
        labels = lab_lo.repeat_interleave(scale, 1).repeat_interleave(scale, 2).contiguous()
        labels[:, : H // 10] = 255
        min_kept = N * H * W // 2
    else:
        labels = make_labels(N, H, W, C, 255, g)
        min_kept = N * H * W // 16
    up = lo[..., :C].permute(0, 3, 1, 2).contiguous().numpy() if scale == 1 else \
        c_oracle.bilinear_nhwc_to_nchw(lo.numpy(), C, H, W)
    ref = c_oracle.ohem(up, labels.numpy(), 255, 0.7, min_kept)
    crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=min_kept)
    lo_dev = lo.to(cuda).permute(0, 3, 1, 2)[:, :C].requires_grad_(True)   # logical [N,19,h,w], cs = 32
    lab_dev = labels.to(cuda)
    loss = crit.forward_lowres(lo_dev, lab_dev, C)
    loss.backward(retain_graph=True)
    saved = loss.grad_fn.saved_tensors
    p, state = saved[2], saved[3]
    if scale == 1:
        assert isinstance(loss.grad_fn, ops.OhemCEFn._backward_cls)
        assert saved[0].data_ptr() == lo_dev.data_ptr() and saved[0].stride() == lo_dev.stride()   # no copy
    else:
        assert isinstance(loss.grad_fn, ops.OhemUpCEFn._backward_cls)
    st = ops.ohem_state_dict(state)
    p = p.cpu().numpy()
    assert np.array_equal(p.view(np.uint32), ref["p"].view(np.uint32))
    assert st["active"] == ref["active"] and np.float32(st["T"]) == np.float32(ref["T"]), (st, ref["T"])
    if regime == "B":
        assert st["active"] and np.float32(st["T"]) > np.float32(0.7)
    lab = labels.numpy().reshape(-1)
    kept = (lab != 255) & ((not st["active"]) | (p <= np.float32(st["T"])))
    assert np.array_equal(kept, ref["kept"]) and st["kept"] == int(ref["kept"].sum())
    assert abs(loss.item() - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    if scale == 1:
        lo_m = lo_dev.detach().contiguous().requires_grad_(True)   # materialised NCHW copy of the same logits
        loss_m = ops.OhemCEFn.apply(lo_m, lab_dev, 255, 0.7, min_kept, None)
        loss_m.backward()
        assert torch.equal(_bits(loss), _bits(loss_m))
        assert torch.equal(_bits(lo_dev.grad), _bits(lo_m.grad))
    else:
        lo_t = lo[..., :C].permute(0, 3, 1, 2).clone().requires_grad_(True)
        l2 = torch_ref.ohem_ce(F.interpolate(lo_t, scale_factor=scale, mode="bilinear", align_corners=True), labels,
                               255, 0.7, min_kept)
        l2.backward()
        assert rel_err(lo_dev.grad, lo_t.grad) < 1e-3


@pytest.mark.parametrize("scale", [1, 2])
def test_head_loss_teacher_forced(cuda, scale):
    """3x3 CBR → 1x1 classifier → (x2) → OHEM at label resolution against the bf16-emulating oracle: the .speed aux0
    head (128 wide, x2) and main head (64 wide, x1), non-square"""
    from torchseg_b200 import ops
    from torchseg_b200.networks.bisenet import BiSeNetHead
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(5 + scale)
    N, h, w = 4, 16, 24
    cin, is_aux = (128, True) if scale == 2 else (256, False)
    head = BiSeNetHead(cin, 19, scale, is_aux, BN, aux_mid=128)
    sd = {"m." + k: v.detach().clone() for k, v in head.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    import torchseg_b200
    head.to(cuda)
    torchseg_b200.prepare_model(head)
    head.train()
    labels = make_labels(N, h * scale, w * scale, 19, 255, g)
    mk = N * h * w * scale * scale // 16
    crit = ProbOhemCrossEntropy2d(255, thresh=0.7, min_kept=mk)
    x = bf16_round(torch.relu(torch.randn(N, cin, h, w, generator=g)))
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        lo = tr.bisenet_head_logits(xr, sd, "m", 1e-5, 0.1, True)
        up = lo if scale == 1 else F.interpolate(lo, scale_factor=scale, mode="bilinear", align_corners=True)
        loss_r = tr.ohem_ce(up, labels, 255, 0.7, mk)
        loss_r.backward()
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    lod = head.lowres_logits(xd)
    loss_d = crit.forward_lowres(lod, labels.to(cuda), 19)
    loss_d.backward()
    assert abs(loss_d.item() - loss_r.item()) < 2e-3 * abs(loss_r.item()), (loss_d.item(), loss_r.item())
    assert norm_err(lod, lo) < 2e-2
    assert norm_err(xd.grad, xr.grad) < 2e-2, norm_err(xd.grad, xr.grad)
    for n, p in head.named_parameters():
        assert norm_err(p.grad, sd["m." + n].grad) < 4e-2, n


# ------------------------------------------------------------------------------------------------------- whole step
@pytest.mark.parametrize("line", list(LINES))
def test_step_matches_oracle(cuda, line):
    """the X39 two-tier bar (tests/test_gpu_xception.py): the R18 direction / magnitude bar wherever the bf16-storage
    emulation resolves the fp32 gradient (cosine >= 0.95); elsewhere the magnitude within 2x, or within 1.5x of the
    emulation's own magnitude ratio where bf16 storage alone moves it further (R101's ~100 batch-statistics BN layers
    decorrelate its whole context-path gradient at initialisation: cosines ~0 and magnitude ratios ~1.7 between the
    fp32 oracle and its bf16-storage emulation); conv weight gradients and BN running statistics within 1.5x the
    bf16-storage spread where the emulation keeps any correlation with the fp32 gradient"""
    import bisenet_lines_oracle as tr
    model, sd, x, y, min_kept = _build(cuda, line, *SMALL[line])
    for k in sd:
        if sd[k].is_floating_point() and "running" not in k:
            sd[k].requires_grad_(True)
    stats = {}
    loss_ref, _ = tr.bisenet_loss(line, x, y, sd, min_kept, stats=stats)
    loss_ref.backward()
    grads_ref = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    for v in sd.values():
        v.grad = None
    tr.set_bf16_emulation(True)
    try:
        stats_emu = {}
        loss_emu, _ = tr.bisenet_loss(line, x, y, sd, min_kept, stats=stats_emu)
        loss_emu.backward()
    finally:
        tr.set_bf16_emulation(False)
    grads_emu = {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}
    loss = model(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    bad, outside, resolved = [], [], 0
    for n, p in model.named_parameters():
        a, b, c = p.grad.float().cpu(), grads_ref[n], grads_emu[n]
        af, bf, cf = a.reshape(-1), b.reshape(-1), c.reshape(-1)
        cos = float(torch.dot(af, bf) / (af.norm() * bf.norm()).clamp_min(1e-30))
        cos_emu = float(torch.dot(cf, bf) / (cf.norm() * bf.norm()).clamp_min(1e-30))
        ratio = float(af.norm() / bf.norm().clamp_min(1e-30))
        ratio_emu = float(cf.norm() / bf.norm().clamp_min(1e-30))
        if cos_emu >= 0.95:
            resolved += 1
            if cos < 0.8 or not (0.7 < ratio < 1.4):
                bad.append((n, round(cos, 3), round(ratio, 3)))
        elif not (min(0.5, ratio_emu / 1.5) < ratio < max(2.0, 1.5 * ratio_emu)):
            bad.append((n, round(cos, 3), round(ratio, 3), round(ratio_emu, 3)))
        if p.dim() == 4:
            e, spread = norm_err(a, b), norm_err(c, b)
            # spread >= 1: the emulated gradient is uncorrelated with the fp32 one, and only the magnitude bar applies
            if spread < 1 and e > 1.5 * spread + 2e-2:
                outside.append((n, round(e, 4), round(spread, 4)))
    assert not bad, "gradient direction / magnitude off: %s" % bad[:10]
    assert not outside, "gradient farther from the fp32 oracle than 1.5 x the bf16-storage spread + 2e-2: %s" % outside[:10]
    assert resolved >= 5, resolved
    msd = model.state_dict()
    for k, v in stats.items():
        assert rel_err(msd[k], v) < 1.5 * rel_err(stats_emu[k], v) + 3e-2, (k, rel_err(msd[k], v), rel_err(stats_emu[k], v))


# ----------------------------------------------------------------------------------------------- training behaviour
@pytest.mark.parametrize("line", list(LINES))
def test_train_steps_decrease_loss(cuda, line):
    from torchseg_b200 import optim
    model, _, x, y, _ = _build(cuda, line, *SMALL[line], seed=3)
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


@pytest.mark.parametrize("line", list(LINES))
def test_step_is_bit_reproducible(cuda, line):
    """two identical models and batches: identical loss bits and identical gradient bits"""
    runs = []
    for _ in range(2):
        model, _, x, y, _ = _build(cuda, line, *SMALL[line], seed=5)
        loss = model(x.to(cuda), y.to(cuda))
        loss.backward()
        torch.cuda.synchronize()
        runs.append((loss.detach().clone(), [p.grad.detach().clone() for p in model.parameters()]))
    (l0, g0), (l1, g1) = runs
    assert torch.equal(_bits(l0), _bits(l1)), (l0.item(), l1.item())
    for a, b in zip(g0, g1):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("line", list(LINES))
def test_graphed_step_matches_eager(cuda, line):
    from torchseg_b200 import optim
    from torchseg_b200.engine.graph import GraphedTrainStep
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        def make():
            model, _, x, y, _ = _build(cuda, line, *SMALL[line], seed=7)
            return model, optim.SGD(_groups(model), lr=1e-2, momentum=0.9, weight_decay=5e-4), x.to(cuda), y.to(cuda)

        model, opt, x, y = make()
        eager = []
        for _ in range(4):
            opt.zero_grad()
            loss = model(x, y)
            loss.backward()
            opt.step()
            eager.append(loss.item())
        del loss
        model, opt, x, y = make()
        step = GraphedTrainStep(model, opt, [x, y], warmup=2)
        assert step.graph is not None, step.error
        graphed = [step(x, y).item() for _ in range(2)]
        assert graphed == eager[2:], (eager, graphed)   # bit for bit: the step is deterministic (DESIGN §5)
        step.release()
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())


# -------------------------------------------------------------------------------------------------------------- eval
@pytest.mark.parametrize("line", list(LINES))
def test_eval_forward_matches_oracle(cuda, line):
    """eval branch (network.py:113): BN on running statistics (folded), main head only, log_softmax — at 1/8 of the
    input for the .speed lines, x8 up-sampled for R101"""
    import torchseg_b200
    from torchseg_b200.utils.init_func import init_weight
    import bisenet_lines_oracle as tr
    torch.manual_seed(11)
    model = _net(line, False)
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    g = randomize_bn(model, 12)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    H, W = 128, 192
    x = torch.randn(2, 3, H, W, generator=g)
    tr.set_bf16_emulation(True)
    try:
        with torch.no_grad():
            ref = tr.bisenet_eval(line, x, sd)
    finally:
        tr.set_bf16_emulation(False)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    with torch.no_grad():
        out = model(x.to(cuda))
    d = LINES[line][1]
    assert tuple(out.shape) == (2, 19, H // d, W // d) and out.dtype == torch.float32
    assert norm_err(out, ref) < 2e-2, norm_err(out, ref)
    assert (out.argmax(1).cpu() == ref.argmax(1)).float().mean() > 0.97


@pytest.mark.parametrize("line", SPEED)
def test_training_checkpoint_loads_into_eval_network(cuda, line):
    """a training network's state_dict through utils.pyt_utils.load_model (non-strict: the aux heads are dropped) into
    the eval network gives the training network's own eval-mode output, bit for bit"""
    import torchseg_b200
    from torchseg_b200.utils.pyt_utils import load_model
    torch.manual_seed(21)
    train_net = _net(line, True)
    g = randomize_bn(train_net, 22)
    ckpt = {k: v.detach().clone() for k, v in train_net.state_dict().items()}
    eval_net = load_model(_net(line, False), ckpt)
    x = torch.randn(2, 3, 128, 256, generator=g).to(cuda)
    outs = []
    train_net.is_training = False   # the constructor flag selects the loss branch; .eval() alone keeps it
    for m in (train_net, eval_net):
        m.to(cuda)
        torchseg_b200.prepare_model(m)
        m.eval()
        with torch.no_grad():
            outs.append(m(x))
    assert tuple(outs[0].shape) == (2, 19, 16, 32)
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))


@pytest.mark.parametrize("line", SPEED)
def test_eval_batch1_graph_matches_eager(cuda, line):
    """a batch-1 768x1536 eval forward captured as one CUDA graph: a replay on a new frame equals the eager forward on
    that frame bit for bit"""
    import torchseg_b200
    torch.manual_seed(31)
    model = _net(line, False)
    g = randomize_bn(model, 32)
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.eval()
    frames = [torch.randn(1, 3, 768, 1536, generator=g).to(cuda) for _ in range(2)]
    torch.cuda.set_stream(torch.cuda.Stream())
    try:
        static_in = frames[0].clone()
        with torch.no_grad():
            for _ in range(2):
                model(static_in)          # packs and folded weights are made outside the capture
            eager = model(frames[1]).clone()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = model(static_in)
        static_in.copy_(frames[1])
        graph.replay()
        torch.cuda.synchronize()
        assert tuple(static_out.shape) == (1, 19, 96, 192)
        assert torch.equal(_bits(static_out), _bits(eager))
        del graph
    finally:
        torch.cuda.set_stream(torch.cuda.default_stream())


# --------------------------------------------------------------------------------------------------------- full size
def _twice(model, x, y):
    """two steps' forward + backward from the same state (no optimiser step): loss and gradient bits of each"""
    out = []
    for _ in range(2):
        for p in model.parameters():
            p.grad = None
        loss = model(x, y)
        loss.backward()
        torch.cuda.synchronize()
        out.append((loss.detach().clone(), [p.grad.detach().clone() for p in model.parameters()]))
        del loss
    return out


@pytest.mark.parametrize("line", list(LINES))
def test_full_size_step(cuda, line):
    """the reference training shape: .speed lines 16x768x1536 (labels 96x192), R101 16x1024². Finite loss and
    bit-identical repeated steps. R101 also against the fp32 oracle on cuDNN (forward only): at this size its ~100
    batch-statistics BN layers amplify rounding so far that bf16 storage alone (the emulating oracle) moves layer4 to a
    norm error of ~0.9 and the loss by 0.5-0.7 %. So the context-path stages must be as close to the fp32 oracle as
    the emulation is, and the loss within 1e-2 + 2x the emulation's loss spread (measured on an H100: 1.7e-2 from the
    fp32 oracle, whose bf16-storage emulation is 0.5e-2 from it; at 4x1024² and 16x512² both are ~0.2e-2)."""
    N, H, W = (16, 1024, 1024) if line == "r101" else (16, 768, 1536)
    model, sd, x, y, min_kept = _build(cuda, line, N, H, W, seed=12345)
    x, y = x.to(cuda), y.to(cuda)
    torch.cuda.reset_peak_memory_stats()
    (l0, g0), (l1, g1) = _twice(model, x, y)
    print("%s full size: loss %.6f, peak memory %.1f GiB" % (line, l0.item(), torch.cuda.max_memory_allocated() / 2 ** 30))
    assert np.isfinite(l0.item())
    assert torch.equal(_bits(l0), _bits(l1)), (l0.item(), l1.item())
    for a, b in zip(g0, g1):
        assert torch.equal(_bits(a), _bits(b))
    del g0, g1
    if line != "r101":
        return
    with torch.no_grad():
        ours = [b.float() for b in model.context_path(x)]
    del model
    torch.cuda.empty_cache()
    import bisenet_lines_oracle as tr
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    ref = {}
    try:
        sdc = {k: v.to(cuda) for k, v in sd.items()}
        for emu in (False, True):
            tr.set_bf16_emulation(emu)
            with torch.no_grad():
                blocks = [b.float() for b in tr.LINES[line][0](x, sdc, "context_path", 1e-5, 0.1, True)]
                loss_ref, _ = tr.bisenet_loss(line, x, y, sdc, min_kept)
            ref[emu] = (blocks, loss_ref.item())
    finally:
        tr.set_bf16_emulation(False)
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    (f32, loss_f32), (emu, loss_emu) = ref[False], ref[True]
    for i, (a, b, c) in enumerate(zip(ours, f32, emu)):
        e, spread = norm_err(a, b), norm_err(c, b)
        print("layer%d: norm error vs the fp32 oracle %.4f (bf16-storage oracle %.4f)" % (i + 1, e, spread))
        assert e < 1.1 * spread + 5e-3, (i + 1, e, spread)
    rel, rel_emu = abs(l0.item() - loss_f32) / abs(loss_f32), abs(loss_emu - loss_f32) / abs(loss_f32)
    print("r101 full size: loss %.6f, fp32 oracle %.6f (rel %.2e), bf16-storage oracle %.6f (rel %.2e)"
          % (l0.item(), loss_f32, rel, loss_emu, rel_emu))
    assert rel < 1e-2 + 2 * rel_emu, (l0.item(), loss_f32, loss_emu)
