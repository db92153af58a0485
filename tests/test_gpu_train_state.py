"""The cached training state against a cold rebuild, bit for bit.

Between the kernels and the training loop sit caches that decide which bytes the kernels read: the per-tensor bf16
packs (ops.pack_cache), the bf16 mirror of the flat parameters (optim.FlatPack, `wb` written by the SGD kernel, `wt`
filled lazily), the eval-mode folded weights (ops.fold_cache), the statistics arena (ops.zero_arena), the gradient
forks (ops.GradShare) and the captured whole step (engine.graph.GraphedTrainStep). A stale entry gives results that are
plausible and wrong, so every test here compares a model that has been through some sequence of steps, replays,
checkpoints or train/eval switches with its COLD TWIN: a fresh build of the same class that loads the model's and the
optimiser's state dicts and has never run a step, so that every operand it uses is packed from the fp32 masters. The
training step is deterministic (DESIGN §5), so the two must agree bit for bit: the loss, every gradient, and the
parameters, momentum and BN running statistics after the step; in eval, the output. Every test runs its sequence on two
cold builds side by side as well, and asserts that those agree: a warm-versus-cold difference then comes from state.

Networks: BiSeNet-R18 (the two-stem launch, the packed-image cache, GradShare forks, ARM / FFM, OHEM with C = 19),
DeepLabV3+ (ResNet-101 deep stem, BNFn and the depthwise direct gradients; the same object trains and evaluates) and
the DeConvBnRelu encoder-decoder of test_gpu_deconv.py (the transposed fold)."""
import copy

import pytest
import torch

from util import make_labels

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d
LR, MOM, WD = 1e-2, 0.9, 5e-4
NETS = ["bisenet", "deeplabv3plus", "deconv"]


# ------------------------------------------------------------------------------------------------------------ networks
def _ohem(N, H, W):
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    return ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=N * H * W // 16, use_weight=False)


def _kaiming(model):
    from torchseg_b200.utils.init_func import init_weight
    init_weight(model.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')


class _BiSeNet(object):
    N, H, W = 4, 128, 128

    def new(self):
        from torchseg_b200.networks import BiSeNet
        return BiSeNet(19, True, _ohem(self.N, self.H, self.W), None, BN)

    init = staticmethod(_kaiming)

    def groups(self, model):
        from torchseg_b200.utils.init_func import group_weight
        return group_weight([], model, BN, LR)

    def eval(self, model, x):
        model.is_training = False   # the network's eval branch (main head, log-softmax) on the training object
        try:
            return model(x)
        finally:
            model.is_training = True


class _DeepLab(object):
    N, H, W = 4, 80, 112

    def new(self):
        from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
        model = DeepLabV3Plus(19, _ohem(self.N, self.H, self.W), norm_layer=BN)
        model.aspp.dropout.p = 0.0
        return model

    init = staticmethod(_kaiming)

    def groups(self, model):
        from torchseg_b200.utils.init_func import group_weight
        groups = group_weight([], model.backbone, BN, LR)
        for m in model.business_layer:
            groups = group_weight(groups, m, BN, 10 * LR)
        return groups

    def eval(self, model, x):
        return model(x)             # label None: the eval branch


class _DeConv(object):
    N, H, W = 4, 32, 32

    def new(self):
        from test_gpu_deconv import _Net
        return _Net(False)

    def init(self, model):
        from test_gpu_deconv import _randomize_bn
        _randomize_bn(model, 12)

    def groups(self, model):
        return [dict(params=list(model.parameters()))]

    def eval(self, model, x):
        return model.body(x)


SPECS = {"bisenet": _BiSeNet(), "deeplabv3plus": _DeepLab(), "deconv": _DeConv()}


def _batches(spec, cuda, seed=1):
    """two different batches: a step that kept the previous batch's packed image would be caught"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(2):
        if isinstance(spec, _DeConv):
            x = torch.randn(spec.N, 64, spec.H, spec.W, generator=g)
            y = torch.randint(0, 19, (spec.N, spec.H, spec.W), generator=g)
        else:
            x = torch.randn(spec.N, 3, spec.H, spec.W, generator=g)
            y = make_labels(spec.N, spec.H, spec.W, 19, 255, g)
        out.append((x.to(cuda), y.to(cuda)))
    return out


def _optimizer(spec, model, torch_sgd=False):
    from torchseg_b200 import optim
    cls = torch.optim.SGD if torch_sgd else optim.SGD
    return cls(spec.groups(model), lr=LR, momentum=MOM, weight_decay=WD)


def _cold(spec, cuda, torch_sgd=False, seed=0):
    """a fresh build from the seed: two calls give the same model"""
    import torchseg_b200
    torch.manual_seed(seed)
    model = spec.new()
    spec.init(model)
    model = torchseg_b200.prepare_model(model.to(cuda))
    model.train()
    return model, _optimizer(spec, model, torch_sgd)


def _twin(spec, cuda, model, opt=None, state=None):
    """the cold twin of (model, opt): a fresh build that loads their state dicts (or `state` = the pair of them)"""
    import torchseg_b200
    msd, osd = state if state is not None else (model.state_dict(), opt.state_dict() if opt is not None else None)
    osd = copy.deepcopy(osd)   # torch.optim.SGD's state dict holds its live momentum buffers, not copies
    twin = spec.new()
    twin.load_state_dict(msd)
    twin = torchseg_b200.prepare_model(twin.to(cuda))
    twin.train(model.training if model is not None else True)
    if osd is None:
        return twin
    topt = _optimizer(spec, twin, torch_sgd=isinstance(opt, torch.optim.SGD))
    topt.load_state_dict(osd)
    return twin, topt


# ------------------------------------------------------------------------------------------------------- comparisons
def _bits(t):
    t = t.detach().contiguous()
    if not t.is_floating_point():
        return t
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(a, b, what):
    assert a.keys() == b.keys(), what
    bad = [k for k in a if a[k].shape != b[k].shape or not torch.equal(_bits(a[k]), _bits(b[k]))]
    assert not bad, "%s: %d of %d tensors differ bitwise: %s" % (what, len(bad), len(a), bad[:8])


def _momentum(opt):
    if isinstance(opt, torch.optim.SGD):
        ps = [p for g in opt.param_groups for p in g["params"]]
        return {"momentum.%d" % i: opt.state[p]["momentum_buffer"].clone() for i, p in enumerate(ps)
                if "momentum_buffer" in opt.state.get(p, {})}
    return {"momentum": opt.flat_mom.clone()}


def _after_step(model, opt):
    s = {"param." + n: p.detach().clone() for n, p in model.named_parameters()}
    s.update({"buffer." + n: b.detach().clone() for n, b in model.named_buffers()})
    s.update(_momentum(opt))
    return s


def _grads(model):
    return {"grad." + n: p.grad.detach().clone() for n, p in model.named_parameters()}


def _step(model, opt, batch, zero=None):
    """one eager training step: the loss, every gradient, then the state after the optimiser step"""
    (zero or opt.zero_grad)()
    loss = model(*batch)
    loss.backward()
    out = dict(loss=loss.detach().clone(), **_grads(model))
    del loss
    opt.step()
    out.update(_after_step(model, opt))
    return out


def _replay(step, model, opt, batch):
    loss = step(*batch)
    out = dict(loss=loss.detach().clone(), **_grads(model))   # .grad are the flat views the captured step writes
    out.update(_after_step(model, opt))
    return out


def _eval(spec, model, x):
    was = model.training
    model.eval()
    try:
        with torch.no_grad():
            return dict(out=spec.eval(model, x).clone())
    finally:
        model.train(was)


def _set_lr(opt, lr):
    for g in opt.param_groups:
        g["lr"] = lr


# ------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("flavour", ["fused", "torch_sgd"])
def test_eager_steps_match_cold_twin(cuda, net, flavour):
    """after each of steps 1..3 the next step matches a cold twin: the `wb` mirror written by the SGD kernel, the lazy
    `wt` of pack_wt_multi, pack invalidation, the arena reset and GradShare re-arming (fused); the optimizer-step
    post-hook that drops the per-tensor packs (torch.optim.SGD)"""
    spec = SPECS[net]
    torch_sgd = flavour == "torch_sgd"
    batches = _batches(spec, cuda)
    a, b = _cold(spec, cuda, torch_sgd), _cold(spec, cuda, torch_sgd)
    for k in range(4):
        twin = _twin(spec, cuda, *a) if k > 0 else None
        sa = _step(*a, batches[k % 2])
        _same(sa, _step(*b, batches[k % 2]), "step %d, cold build A vs B" % k)
        if twin is not None:
            _same(sa, _step(*twin, batches[k % 2]), "step %d after %d steps: warm vs cold twin" % (k, k))
        del twin, sa


@pytest.mark.parametrize("net", NETS)
def test_graph_replays_match_cold_twin(cuda, net):
    """the captured whole step: each replay (with a learning-rate change before it), an eager step between replays and
    the replay after it, and an eval after the replays (the fold cache must see the replayed parameter updates) against
    cold twins; two cold builds run the same sequence through their own graphs"""
    from torchseg_b200.engine.graph import GraphedTrainStep
    spec = SPECS[net]
    torch.cuda.set_stream(torch.cuda.Stream())
    steps = []
    try:
        batches = _batches(spec, cuda)
        pairs = [_cold(spec, cuda), _cold(spec, cuda)]
        for model, opt in pairs:
            steps.append(GraphedTrainStep(model, opt, list(batches[0]), warmup=2))
            assert steps[-1].graph is not None, steps[-1].error
        plan = [("replay", 1e-2, 1), ("replay", 8e-3, 0), ("eager", 6e-3, 1), ("replay", 4e-3, 0), ("replay", 2e-3, 1)]
        for i, (kind, lr, bi) in enumerate(plan):
            twin = _twin(spec, cuda, *pairs[0])    # takes the same step eagerly from the state before it
            _set_lr(twin[1], lr)
            tw = _step(*twin, batches[bi])
            del twin
            runs = []
            for (model, opt), step in zip(pairs, steps):
                _set_lr(opt, lr)
                if i == len(plan) - 1:   # an eval right before the last replay: its folds must not outlive the replay
                    _eval(spec, model, batches[1][0])
                runs.append(_replay(step, model, opt, batches[bi]) if kind == "replay" else _step(model, opt, batches[bi]))
            _same(runs[0], runs[1], "%s %d, cold build A vs B" % (kind, i))
            _same(runs[0], tw, "%s %d: warm vs the cold twin's eager step" % (kind, i))
            del runs, tw
        outs = [_eval(spec, model, batches[1][0]) for model, _ in pairs]
        _same(outs[0], outs[1], "eval after the replays, cold build A vs B")
        _same(outs[0], _eval(spec, _twin(spec, cuda, pairs[0][0]), batches[1][0]), "eval after the replays vs cold twin")
    finally:
        for s in steps:
            s.release()
        torch.cuda.set_stream(torch.cuda.default_stream())


def _edit_bn(model):
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, BN):
                m.weight.mul_(1.25)
                m.running_var.mul_(1.5)


@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("change", ["train_forward", "optimizer_step", "load_state_dict", "bn_edit"])
def test_eval_after_state_change_matches_cold_twin(cuda, net, change):
    """eval, then a change of state, then eval again on the same object, against the cold twin's eval. The train-mode
    forwards without an optimiser step (BN re-estimation) move only the running statistics, which tsb_bn_finalize writes
    through raw pointers; the folds involved are the plain, the stem (BiSeNet's two 7x7 stems, DeepLabV3+'s 3x3 deep
    stem) and the transposed one (the encoder-decoder)"""
    spec = SPECS[net]
    batches = _batches(spec, cuda)
    pairs = [_cold(spec, cuda), _cold(spec, cuda)]
    other = None
    if change == "load_state_dict":
        m2, o2 = _cold(spec, cuda, seed=5)
        _step(m2, o2, batches[1])
        other = {k: v.clone() for k, v in m2.state_dict().items()}
        del m2, o2
    outs = []
    for model, opt in pairs:
        _eval(spec, model, batches[0][0])          # builds the fold cache
        if change == "train_forward":
            with torch.no_grad():
                for x, y in batches:
                    model(x, y)
        elif change == "optimizer_step":
            _step(model, opt, batches[1])
        elif change == "load_state_dict":
            model.load_state_dict(other)
        else:
            _edit_bn(model)
        outs.append(_eval(spec, model, batches[0][0]))
    _same(outs[0], outs[1], "eval after %s, cold build A vs B" % change)
    _same(outs[0], _eval(spec, _twin(spec, cuda, pairs[0][0]), batches[0][0]), "eval after %s vs cold twin" % change)


@pytest.mark.parametrize("net", NETS)
def test_checkpoint_round_trip_mid_training(cuda, net):
    """a checkpoint taken after 2 steps, loaded (a) into a fresh model / optimiser pair and (b) back into the live pair
    (whose bf16 mirror and packs describe later weights by then): both continue exactly as the original did"""
    spec = SPECS[net]
    batches = _batches(spec, cuda)
    model, opt = _cold(spec, cuda)
    for k in range(2):
        _step(model, opt, batches[k % 2])
    ckpt = ({k: v.clone() for k, v in model.state_dict().items()}, opt.state_dict())
    ref = [_step(model, opt, batches[k % 2]) for k in range(2)]
    model.load_state_dict(ckpt[0])
    opt.load_state_dict(ckpt[1])
    for k in range(2):
        _same(ref[k], _step(model, opt, batches[k % 2]), "step %d after loading into the live pair" % k)
    fresh = _twin(spec, cuda, model, opt, state=ckpt)
    for k in range(2):
        _same(ref[k], _step(*fresh, batches[k % 2]), "step %d after loading into a fresh pair" % k)


@pytest.mark.parametrize("net", NETS)
def test_gradient_accumulation_and_zero_grad(cuda, net):
    """two forward / backward passes of the same batch without zero_grad accumulate exactly twice the gradient of one
    (training-mode BN uses the batch statistics, so both passes compute the same values and g + g is exact); and
    `model.zero_grad()` (set_to_none) between steps gives the same trajectory as the optimiser's zero_grad. A second
    backward through the same graph (retain_graph) adds the same gradient again: the block forks' GradShare must re-arm
    after its last contributor."""
    spec = SPECS[net]
    batches = _batches(spec, cuda)
    model, opt = _cold(spec, cuda)
    opt.zero_grad()
    losses, grads = [], []
    for _ in range(2):
        loss = model(*batches[0])
        loss.backward()
        losses.append(loss.detach().clone())
        grads.append(_grads(model))
        del loss
    _same(dict(loss=losses[0]), dict(loss=losses[1]), "the second pass's loss")
    _same({k: 2 * v for k, v in grads[0].items()}, grads[1], "two accumulated passes vs twice one pass")
    opt.zero_grad()
    loss = model(*batches[0])
    loss.backward(retain_graph=True)
    loss.backward()
    del loss
    _same({k: 2 * v for k, v in grads[0].items()}, _grads(model), "two backward passes through one graph")
    a, b = _cold(spec, cuda, seed=1), _cold(spec, cuda, seed=1)
    for k in range(3):
        _same(_step(*a, batches[k % 2]), _step(*b, batches[k % 2], zero=b[0].zero_grad),
              "step %d: opt.zero_grad() vs model.zero_grad()" % k)
