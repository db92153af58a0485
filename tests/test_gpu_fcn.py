"""FCN-32s (SURVEY §8 a15) on the GPU: BASELINE configs[0] (R18, 2 x 256 x 256, 19 classes) and the shipped R101_v1c
variant (TorchSeg model/fcn/voc.fcn32s.R101_v1c/network.py:13-68, VOC 21 classes) — teacher-forced head and
whole training step against the oracle (pinned to the live reference by tests/test_cpu_oracle.py)."""
import pytest
import torch

from util import norm_err
from golden_cases import fcn_case, fcn_r101_case
from test_gpu_bisenet import _sd_of, _prep, _rand, _check, BN

pytestmark = pytest.mark.gpu


def test_fcn_head_teacher_forced(cuda):
    """_FCNHead (3x3 CBR C/4 → Dropout2d(p=0) → 1x1 + bias): low-resolution fp32 logits and all gradients"""
    from torchseg_b200 import ops
    from torchseg_b200.networks.fcn import _FCNHead
    from oracle import torch_ref as tr
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(5)
    head = _FCNHead(512, 21, True, BN)
    head.dropout.p = 0.0
    sd = _sd_of(head)
    _prep(head, cuda)
    x = _rand((8, 512, 12, 16), g, relu=True)
    xr = x.clone().requires_grad_(True)
    tr.set_bf16_emulation(True)
    try:
        lo = tr.fcn_head(xr, sd, "m", 1e-5, 0.1, True)
        gy = _rand(tuple(lo.shape), g)
        lo.backward(gy)
    finally:
        tr.set_bf16_emulation(False)
    xd = ops.to_nhwc(x.to(cuda)).requires_grad_(True)
    lod = head.lowres_logits(xd)
    assert lod.dtype == torch.float32 and tuple(lod.shape) == (8, 21, 12, 16)
    lod.backward(gy.to(cuda))
    _check(head, sd, [lod], [lo], [xd], [xr], tol=1e-2)


def _step(cuda, backbone, classes, case, oracle_loss):
    import torchseg_b200
    from torchseg_b200.networks import FCN
    from torchseg_b200.utils.init_func import init_weight
    x, y, seed = case
    torch.manual_seed(seed)
    m = FCN(classes, torch.nn.CrossEntropyLoss(reduction='mean', ignore_index=255), backbone=backbone)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout2d):
            mod.p = 0.0
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss_ref = oracle_loss(x, y, sd)
    loss_ref.backward()
    m.to(cuda)
    torchseg_b200.prepare_model(m)
    m.train()
    loss = m(x.to(cuda), y.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-2 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    P = dict(m.named_parameters())
    # direction where it is well conditioned (the two heads: classifier + 3x3 conv; cos > 0.9 as for the other untrained
    # R101 networks — layer4 batch statistics over a few hundred samples are noisy), magnitude everywhere
    names = ["head.conv1x1.weight", "aux_head.conv1x1.weight", "head.conv1x1.bias"]
    if backbone == "R18":    # (R101 at test size: layer4 is a 6x6 map, batch statistics over 144 samples — the 3x3 convs
        names += ["head.cbr.conv.weight", "aux_head.cbr.conv.weight"]   # in front of them are checked by magnitude only)
    for n in names:
        a, b = P[n].grad.float().cpu().reshape(-1), sd[n].grad.reshape(-1)
        cos = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        assert cos > 0.9, (n, cos)
    checked = 0
    for n, p in P.items():
        if p.dim() == 4:
            ratio = float(p.grad.float().norm().cpu() / sd[n].grad.norm().clamp_min(1e-30))
            assert 0.75 < ratio < 1.33, (n, ratio)
            checked += 1
    # eval branch: [N, classes, H, W] fp32 logits, x32 bilinear (network.py:35-37,49)
    m.eval()
    with torch.no_grad():
        out = m(x.to(cuda))
    assert tuple(out.shape) == (x.shape[0], classes, x.shape[2], x.shape[3]) and out.dtype == torch.float32
    assert torch.isfinite(out).all()
    return checked


def test_fcn_r18_step_matches_oracle(cuda):
    """BASELINE configs[0] on the device: FCN-32s R18, 2 x 256 x 256, 19 classes"""
    from oracle import torch_ref
    n = _step(cuda, "R18", 19, fcn_case(), lambda x, y, sd: torch_ref.fcn_r18_loss(x, y, sd))
    assert n >= 20


def test_fcn_r101_v1c_step_matches_oracle(cuda):
    """the shipped configuration: R101_v1c deep stem, heads 2048/1024 → 512/256 → 21"""
    from oracle import torch_ref
    n = _step(cuda, "R101", 21, fcn_r101_case(N=4, HW=192), lambda x, y, sd: torch_ref.fcn_r101_loss(x, y, sd)[0])
    assert n >= 100
