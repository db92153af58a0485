"""The many-class fused up-sampling loss (ce_up.cu) gives the same gradient bits on every run, and so does a PSPNet
training run rebuilt from the same seed. The backward's bands add into the low-resolution gradient one launch at a time
(row parity x strip phase), and the one-hot term is subtracted in the owning thread's own accumulator."""
import gc

import pytest
import torch

from util import norm_err

pytestmark = pytest.mark.gpu
BN = torch.nn.BatchNorm2d


# (N, C, h, w, H, W): the PSPNet / EncNet heads' x8, a non-integer up-scale, one low-res row, one low-res column (every
# strip writes the same column)
CASES = [(4, 150, 10, 14, 80, 112), (2, 150, 60, 60, 480, 480), (2, 40, 13, 9, 97, 70), (3, 150, 1, 17, 5, 130),
         (1, 5, 9, 1, 40, 300)]


@pytest.mark.parametrize("case", CASES, ids=["N%dC%dh%dw%dH%dW%d" % c for c in CASES])
def test_ce_up_bwd_bit_identical_across_runs(cuda, case):
    """eight backward passes over the same inputs, with freed NaN-filled buffers handed out in between, give the same
    bits, and they match the float64 gradient of F.interpolate + cross_entropy (labels from few classes, so many pixels
    of one strip share a target class)"""
    import torch.nn.functional as F
    from torchseg_b200 import ops
    N, C, h, w, H, W = case
    g = torch.Generator().manual_seed(C + h + W)
    lo = torch.randn(N, C, h, w, generator=g) * 3
    lab = torch.randint(-1, 4, (N, H, W), generator=g)
    lo64 = lo.double().to(cuda).requires_grad_(True)
    F.cross_entropy(F.interpolate(lo64, size=(H, W), mode="bilinear", align_corners=True), lab.to(cuda),
                    ignore_index=-1).backward()
    cs = (C + 31) // 32 * 32
    lod = ops.nhwc_zeros(N, C, h, w, dtype=torch.float32, device=cuda, cs=cs)
    lod.copy_(lo.to(cuda))
    labd = lab.to(cuda)
    outs = []
    for _ in range(8):
        junk = [torch.full((n,), float("nan"), device=cuda) for n in (N * h * w * cs, 4096, N * H * W)]
        del junk
        loss = ops.CEUpFn.apply(lod.requires_grad_(True), labd, H, W, C, -1)
        (d,) = torch.autograd.grad(loss, lod)
        outs.append(d.contiguous().clone())
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o.view(torch.int32), outs[0].view(torch.int32))
    assert norm_err(outs[0], lo64.grad) < 1e-5, norm_err(outs[0], lo64.grad)


def _pspnet(cuda):
    import torchseg_b200
    from torchseg_b200.networks import PSPNet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(3)
    model = PSPNet(150, torch.nn.CrossEntropyLoss(ignore_index=-1), norm_layer=BN)
    init_weight([model.psp_layer, model.aux_layer], torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in',
                nonlinearity='relu')
    model.psp_layer.conv6[1].p = 0.0
    model.aux_layer[1].p = 0.0
    model.to(cuda)
    torchseg_b200.prepare_model(model)
    model.train()
    return model


def test_pspnet_train_steps_reproduce_with_models_freed(cuda):
    """four PSPNet-R101 SGD steps (150 classes, ignore -1), run four times from the same seed with each model freed
    before the next is built: every loss and every parameter gradient is bit-identical"""
    from torchseg_b200 import optim
    g = torch.Generator().manual_seed(4)
    x = torch.randn(4, 3, 80, 112, generator=g).to(cuda)
    y = torch.randint(-1, 40, (4, 80, 112), generator=g).to(cuda)
    runs = []
    for _ in range(4):
        model = _pspnet(cuda)
        opt = optim.SGD([dict(params=list(model.parameters()), lr=1e-2)], lr=1e-2, momentum=0.9, weight_decay=5e-4)
        rec = []
        for _ in range(4):
            opt.zero_grad()
            loss = model(x, y)
            loss.backward()
            rec.append((loss.detach().clone(), [p.grad.detach().clone() for p in model.parameters()]))
            opt.step()
        torch.cuda.synchronize()
        runs.append(rec)
        del model, opt, rec
        gc.collect()
    for rec in runs[1:]:
        for (l0, g0), (l1, g1) in zip(runs[0], rec):
            assert torch.equal(l0.view(torch.int32), l1.view(torch.int32))
            assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(g0, g1))
