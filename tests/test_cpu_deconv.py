"""CPU checks of the transposed-convolution surface: DeConvBnRelu's import name, constructor and checkpoint keys
against the reference (tests/golden/live_reference_deconv.json, tools/make_deconv_golden.py), prepare_model on
ConvTranspose2d weights, group_weight, and the argument checks of tsb_conv_transpose2d_fprop without a GPU."""
import ctypes
import inspect
import json
import os

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "live_reference_deconv.json")


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_deconv_imports_from_furnace_names():
    import torchseg_b200
    torchseg_b200.install_as_furnace()
    from seg_opr.seg_oprs import DeConvBnRelu
    from torchseg_b200.seg_opr import seg_oprs
    assert DeConvBnRelu is seg_oprs.DeConvBnRelu


def test_signature_matches_reference():
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    sig = inspect.signature(DeConvBnRelu.__init__)
    ours = [[n, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for n, p in sig.parameters.items() if n != "self"]
    assert ours == _golden()["params"]


@pytest.mark.parametrize("idx", range(4))
def test_children_and_state_dict_match_reference(idx):
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    case = _golden()["cases"][idx]
    m = DeConvBnRelu(*case["args"], **case["kwargs"])
    assert [n for n, _ in m.named_children()] == case["children"]
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == case["state_dict"]
    assert isinstance(m.conv, nn.ConvTranspose2d)


def test_prepare_model_makes_deconv_weights_krsc():
    import torchseg_b200
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    torch.manual_seed(0)
    net = nn.Sequential(nn.Conv2d(3, 64, 3, padding=1), DeConvBnRelu(64, 32, 4, 2, 1, 0))
    before = {k: v.clone() for k, v in net.state_dict().items()}
    ids = [id(p) for p in net.parameters()]
    torchseg_b200.prepare_model(net)
    w = net[1].conv.weight
    assert tuple(w.shape) == (64, 32, 4, 4)
    assert w.permute(0, 2, 3, 1).is_contiguous()       # [Ci][k][k][Co]: the adjoint conv's KRSC
    assert [id(p) for p in net.parameters()] == ids
    for k, v in net.state_dict().items():
        assert torch.equal(v, before[k]), k


def test_group_weight_stays_complete():
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    from torchseg_b200.utils.init_func import group_weight
    net = nn.Sequential(DeConvBnRelu(64, 32, 4, 2, 1, 0), DeConvBnRelu(32, 19, 2, 2, 0, 0, has_bn=False, has_bias=True))
    groups = group_weight([], net, nn.BatchNorm2d, 0.01)
    n = sum(len(g["params"]) for g in groups)
    assert n == len(list(net.parameters()))
    assert any(p is net[0].conv.weight for p in groups[0]["params"])
    assert any(p is net[1].conv.bias for p in groups[1]["params"])


@pytest.mark.parametrize("kw,msg", [
    (dict(stride=3), "stride"),
    (dict(ksize=5, pad=2), "kernel size"),
    (dict(groups=2), "groups"),
    (dict(stride=2, output_pad=2), "output_padding"),
])
def test_module_rejects_unsupported_geometry(kw, msg):
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    args = dict(in_planes=64, out_planes=64, ksize=4, stride=2, pad=1, output_pad=0)
    args.update(kw)
    m = DeConvBnRelu(**args)
    with pytest.raises(NotImplementedError, match=msg):
        m(torch.zeros(1, 64, 4, 4))


def test_module_rejects_bias_with_bn():
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    m = DeConvBnRelu(64, 64, 4, 2, 1, 0, has_bias=True)
    with pytest.raises(NotImplementedError, match="bias and BN"):
        m(torch.zeros(1, 64, 4, 4, dtype=torch.bfloat16).to(memory_format=torch.channels_last))


def test_adjoint_shape():
    from torchseg_b200 import ops
    # ConvTranspose2d(64, 32, 4, 2, 1) on 9 x 7: output (9-1)*2 - 2 + 3 + 1 = 18 by 14
    s = ops.make_deconv_shape(2, 9, 7, 64, 32, 4, 2, 1, 1, 0)
    assert (s.N, s.H, s.W, s.C, s.K, s.R, s.S, s.stride, s.pad, s.dil, s.P, s.Q) == (2, 18, 14, 32, 64, 4, 4, 2, 1, 1, 9, 7)
    ref = nn.ConvTranspose2d(64, 32, 3, stride=2, padding=1, output_padding=1, dilation=2)
    y = ref(torch.zeros(1, 64, 5, 6))
    s = ops.make_deconv_shape(1, 5, 6, 64, 32, 3, 2, 1, 2, 1)
    assert (s.H, s.W) == tuple(y.shape[2:])


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def _call(lib, shp, xcs=64, ycs=64):
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255
    rc = lib.tsb_conv_transpose2d_fprop(ctypes.byref(shp), A, xcs, A, None, 0, A, 1, ycs, None, None, None, 0, None)
    return rc, lib.tsb_last_error()


def test_abi_rejects_stride_3(lib):
    from torchseg_b200._lib import ConvShape
    # adjoint of ConvTranspose2d(64, 64, 3, stride 3) on 4 x 4: Ho = 3*3 + 3 = 12
    rc, err = _call(lib, ConvShape(1, 12, 12, 64, 64, 3, 3, 3, 0, 1, 4, 4))
    assert rc == -1 and b"stride must be 1 or 2" in err


def test_abi_rejects_output_pad_not_below_stride(lib):
    from torchseg_b200 import ops
    # output_padding 2 at stride 2: the adjoint conv maps Ho back to a size other than H
    shp = ops.make_deconv_shape(1, 4, 4, 64, 64, 3, 2, 1, 1, 2)
    rc, err = _call(lib, shp)
    assert rc == -1 and b"inconsistent" in err


def test_abi_rejects_ragged_input_channels(lib):
    from torchseg_b200 import ops
    shp = ops.make_deconv_shape(1, 4, 4, 48, 64, 4, 2, 1, 1, 0)
    rc, err = _call(lib, shp, xcs=48)
    assert rc == -1 and b"multiple of 64" in err


def test_abi_rejects_large_kernel(lib):
    from torchseg_b200 import ops
    shp = ops.make_deconv_shape(1, 4, 4, 64, 64, 5, 1, 2, 1, 0)
    rc, err = _call(lib, shp)
    assert rc == -1 and b"R*S <= 16" in err
