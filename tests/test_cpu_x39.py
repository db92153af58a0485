"""CPU tests of BiSeNet-X39: the oracle (tests/x39_oracle.py) against the golden vectors of the live reference X39
network (tools/make_live_golden_x39.py), checkpoint-compatible module structure, group_weight, and the argument checks of the
depthwise-convolution entry points (no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from golden_cases import bisenet_case

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_x39.npz"))


def test_oracle_vs_live_reference_x39_exact():
    import x39_oracle
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    x, y, min_kept, seed = bisenet_case(N=2, HW=64, seed=5)
    torch.manual_seed(seed)
    m = BiSeNet(19, True, None, None, None, torch.nn.BatchNorm2d)   # same seed → the reference's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = x39_oracle.bisenet_x39_loss(x, y, sd, min_kept)
    loss.backward()
    assert float(loss) == float(LIVE["x39_loss"])
    grads = json.loads(str(LIVE["x39_grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_x39_state_dict_matches_reference():
    """checkpoint compatibility: the reference X39's state_dict keys and shapes, in order"""
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    ref = json.loads(str(LIVE["x39_keys"]))
    ours = BiSeNet(19, True, None, None, None, torch.nn.BatchNorm2d).state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_x39_group_weight_and_children():
    from torchseg_b200.base_model import xception39
    from torchseg_b200.base_model.xception import Block, SeparableConvBnRelu
    from torchseg_b200.networks.bisenet_x39 import BiSeNet
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = BiSeNet(19, True, None, None, None, BN)
    groups = group_weight([], m.context_path, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    cp = m.context_path
    assert isinstance(cp.layer1[0], Block) and cp.layer1[0].has_proj and not cp.layer1[1].has_proj
    sep = cp.layer2[0].proj
    assert isinstance(sep, SeparableConvBnRelu) and sep.conv1.groups == 64 and sep.conv1.stride == (2, 2)
    assert [len(cp.layer1), len(cp.layer2), len(cp.layer3)] == [4, 8, 4]
    assert sum(p.numel() for p in xception39(norm_layer=BN).parameters()) == sum(p.numel() for p in cp.parameters())


def test_x39_reference_import_names(monkeypatch):
    import sys
    import torchseg_b200
    for name in ("seg_opr", "seg_opr.seg_oprs", "seg_opr.loss_opr", "seg_opr.metric", "base_model", "base_model.resnet",
                 "base_model.xception", "engine", "engine.engine", "engine.lr_policy", "engine.logger",
                 "engine.evaluator", "utils", "utils.init_func", "utils.pyt_utils", "utils.img_utils", "apex",
                 "apex.parallel"):
        monkeypatch.setitem(sys.modules, name, None)   # install_as_furnace rewrites these: restored after the test
    torchseg_b200.install_as_furnace()
    from base_model import xception39  # X39 network.py:10
    assert sys.modules["base_model.xception"].xception39 is xception39


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_dwconv_argument_validation_without_gpu(lib):
    buf = ctypes.create_string_buffer(4096 + 16)
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    w = (ctypes.c_float * (64 * 9))()
    wp = ctypes.addressof(w)
    cases = [
        # (C, stride, xcs, ycs, message)
        (12, 1, 16, 16, b"multiple of 8"),
        (16, 3, 16, 16, b"stride 3"),
        (16, 1, 12, 16, b"channel strides"),
        (16, 2, 16, 8, b"channel strides"),
    ]
    for C, st, xcs, ycs, msg in cases:
        rc = lib.tsb_dwconv_fprop(a, xcs, wp, a, ycs, 1, 4, 4, C, st, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
        rc = lib.tsb_dwconv_dgrad(a, ycs, wp, a, xcs, 1, 4, 4, C, st, 0, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
        rc = lib.tsb_dwconv_wgrad(a, xcs, a, ycs, wp, 1, 4, 4, C, st, None, 0, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
    rc = lib.tsb_dwconv_fprop(a + 8, 16, wp, a, 16, 1, 4, 4, 16, 1, None)   # misaligned activation
    assert rc == -1 and b"16-byte" in lib.tsb_last_error()
    rc = lib.tsb_dwconv_fprop(a, 16, None, a, 16, 1, 4, 4, 16, 1, None)
    assert rc == -1 and b"null" in lib.tsb_last_error()
