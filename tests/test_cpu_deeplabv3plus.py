"""CPU tests of DeepLabV3+: the oracle (tests/deeplabv3plus_oracle.py) against the golden vectors of the network composed
from the live reference modules (tools/make_live_golden_deeplabv3plus.py), checkpoint-compatible module structure,
group_weight, the reference import name of SeparableConvBnRelu, and the argument checks of the dilated depthwise
entry points (no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from golden_cases import bisenet_case

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_deeplabv3plus.npz"))


def test_oracle_vs_live_reference_deeplabv3plus_exact():
    import deeplabv3plus_oracle
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    x, y, min_kept, seed = bisenet_case(N=2, HW=64, seed=11)
    torch.manual_seed(seed)
    m = DeepLabV3Plus(19, None)   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = deeplabv3plus_oracle.deeplabv3plus_loss(x, y, sd, min_kept)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_deeplabv3plus_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    ref = json.loads(str(LIVE["keys"]))
    ours = DeepLabV3Plus(19, None).state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_deeplabv3plus_group_weight_and_geometry():
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    from torchseg_b200.seg_opr.seg_oprs import SeparableConvBnRelu
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = DeepLabV3Plus(19, None, norm_layer=BN)
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    seps = [m.aspp.branches[i] for i in (1, 2, 3)] + list(m.decoder.refine)
    assert all(isinstance(s, SeparableConvBnRelu) for s in seps)
    assert [s.conv1.dilation[0] for s in seps] == [6, 12, 18, 1, 1]
    assert all(s.conv1.padding == s.conv1.dilation and s.conv1.groups == s.conv1.in_channels for s in seps)
    l4 = m.backbone.layer4
    assert l4[0].conv2.stride == (1, 1) and l4[0].downsample[0].stride == (1, 1) and l4[1].conv2.dilation == (2, 2)
    assert m.backbone.layer3[0].conv2.stride == (2, 2)


def test_separable_conv_bn_relu_reference_import(monkeypatch):
    import sys
    import torchseg_b200
    for name in ("seg_opr", "seg_opr.seg_oprs", "seg_opr.loss_opr", "seg_opr.metric", "base_model", "base_model.resnet",
                 "base_model.xception", "engine", "engine.engine", "engine.lr_policy", "engine.logger",
                 "engine.evaluator", "utils", "utils.init_func", "utils.pyt_utils", "utils.img_utils", "apex",
                 "apex.parallel"):
        monkeypatch.setitem(sys.modules, name, None)   # install_as_furnace rewrites these: restored after the test
    torchseg_b200.install_as_furnace()
    from seg_opr.seg_oprs import SeparableConvBnRelu
    m = SeparableConvBnRelu(32, 64, 3, 1, 2, 2, has_relu=False)
    assert [n for n, _ in m.named_children()] == ["conv1", "bn", "point_wise_cbr"]
    assert m.conv1.groups == 32 and m.conv1.dilation == (2, 2) and m.bn.num_features == 32
    assert not m.point_wise_cbr.has_relu and m.point_wise_cbr.conv.out_channels == 64
    d = SeparableConvBnRelu(16, 16)   # the reference defaults: a 1x1 depthwise conv
    assert d.conv1.kernel_size == (1, 1) and d.conv1.padding == (0, 0)
    assert list(m.state_dict().keys()) == [
        "conv1.weight", "bn.weight", "bn.bias", "bn.running_mean", "bn.running_var", "bn.num_batches_tracked",
        "point_wise_cbr.conv.weight", "point_wise_cbr.bn.weight", "point_wise_cbr.bn.bias",
        "point_wise_cbr.bn.running_mean", "point_wise_cbr.bn.running_var", "point_wise_cbr.bn.num_batches_tracked"]


@pytest.mark.parametrize("args, what", [
    ((16, 16, 1), "3x3"),                 # the reference default kernel_size=1
    ((16, 16, 3, 1, 1, 2), "padding"),    # padding != dilation
    ((16, 16, 3, 2, 2, 2), "stride"),     # stride 2 with dilation 2
    ((12, 16, 3, 1, 1, 1), "multiple of 8"),
])
def test_separable_conv_bn_relu_rejects_unsupported_geometry(args, what):
    from torchseg_b200.seg_opr.seg_oprs import SeparableConvBnRelu
    m = SeparableConvBnRelu(*args)
    with pytest.raises(NotImplementedError, match=what):
        m(torch.zeros(1, args[0], 8, 8))


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_dwconv2d_argument_validation_without_gpu(lib):
    buf = ctypes.create_string_buffer(4096 + 16)
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    w = (ctypes.c_float * (64 * 9))()
    wp = ctypes.addressof(w)
    cases = [
        # (C, stride, dilation, xcs, ycs, message)
        (12, 1, 2, 16, 16, b"multiple of 8"),
        (16, 3, 1, 16, 16, b"stride 3"),
        (16, 1, 0, 16, 16, b"dilation 0"),
        (16, 1, -2, 16, 16, b"dilation -2"),
        (16, 2, 2, 16, 16, b"stride 2 needs dilation 1"),
        (16, 1, 6, 12, 16, b"channel strides"),
        (16, 1, 6, 16, 8, b"channel strides"),
    ]
    for C, st, dil, xcs, ycs, msg in cases:
        rc = lib.tsb_dwconv2d_fprop(a, xcs, wp, a, ycs, 1, 4, 4, C, st, dil, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
        rc = lib.tsb_dwconv2d_dgrad(a, ycs, wp, a, xcs, 1, 4, 4, C, st, dil, 0, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
        rc = lib.tsb_dwconv2d_wgrad(a, xcs, a, ycs, wp, 1, 4, 4, C, st, dil, None, 0, None)
        assert rc == -1 and msg in lib.tsb_last_error(), lib.tsb_last_error()
    rc = lib.tsb_dwconv2d_fprop(a + 8, 16, wp, a, 16, 1, 4, 4, 16, 1, 2, None)   # misaligned activation
    assert rc == -1 and b"16-byte" in lib.tsb_last_error()
    rc = lib.tsb_dwconv2d_dgrad(a, 16, wp, a + 8, 16, 1, 4, 4, 16, 1, 2, 1, None)
    assert rc == -1 and b"16-byte" in lib.tsb_last_error()
    rc = lib.tsb_dwconv2d_fprop(a, 16, None, a, 16, 1, 4, 4, 16, 1, 2, None)
    assert rc == -1 and b"null" in lib.tsb_last_error()
    rc = lib.tsb_dwconv2d_wgrad(None, 16, a, 16, wp, 1, 4, 4, 16, 1, 2, None, 0, None)
    assert rc == -1 and b"null" in lib.tsb_last_error()


def test_dwconv_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no depthwise kernel spills to local memory"""
    import re
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if l.startswith("dwconv.cu")]
    assert len(rows) == 12, out   # fprop / wgrad at <2,1>, <1,1>, <1,0>; dgrad at those times accumulate on / off
    for r in rows:
        name = " ".join(r[1:-4])
        assert re.match(r"dw_(fprop|dgrad|wgrad)_kernel<", name), r
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % name
