"""CPU tests of DenseASPP: the oracle (tests/denseaspp_oracle.py) against the golden vectors of the network composed from
the live reference modules (tools/make_live_golden_denseaspp.py), checkpoint-compatible module structure, group_weight,
the dense head's construction, and the argument checks and ptxas resources of the pre-activation entry points
(tsb_conv1x1_bnrelu_fprop / _wgrad, tsb_bn_bwd_apply_add; no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_denseaspp.npz"))


def _net(criterion=None):
    from torchseg_b200.networks import DenseASPP
    return DenseASPP(19, criterion)


def test_oracle_vs_live_reference_denseaspp_exact():
    import denseaspp_oracle
    x, y, seed = denseaspp_oracle.denseaspp_case()
    torch.manual_seed(seed)
    m = _net()   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = denseaspp_oracle.denseaspp_loss(x, y, sd)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert norm > 0, n
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_denseaspp_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    ref = json.loads(str(LIVE["keys"]))
    ours = _net().state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_denseaspp_group_weight_and_structure():
    from torchseg_b200.seg_opr.seg_oprs import ConvBnRelu, DenseAsppBlock, DenseASPPModule
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = _net()
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    aspp = m.aspp
    assert isinstance(aspp, DenseASPPModule) and len(aspp.blocks) == 5 and aspp.out_channels == 2688
    for i, (blk, d) in enumerate(zip(aspp.blocks, (3, 6, 12, 18, 24))):
        assert isinstance(blk, DenseAsppBlock)
        assert [n for n, _ in blk.named_children()] == (["pre_bn"] if i else []) + ["reduce", "conv"]
        assert (blk.pre_bn is not None) == (i > 0)
        if i:
            assert blk.pre_bn.num_features == 2048 + 128 * i
        assert isinstance(blk.reduce, ConvBnRelu) and blk.reduce.conv.in_channels == 2048 + 128 * i
        assert blk.reduce.conv.out_channels == 512 and blk.reduce.conv.bias is None
        assert blk.conv.in_channels == 512 and blk.conv.out_channels == 128 and blk.conv.bias is not None
        assert blk.conv.dilation == (d, d) and blk.conv.padding == (d, d) and blk.conv.kernel_size == (3, 3)
        assert blk.dropout == 0.1
    assert m.dropout.p == 0.1 and m.cls.in_channels == 2688 and m.cls.out_channels == 19 and m.cls.bias is not None
    assert not hasattr(m, "aux_layer")
    l3, l4 = m.backbone.layer3, m.backbone.layer4
    assert l3[0].conv2.stride == (1, 1) and l3[1].conv2.dilation == (2, 2) and l4[1].conv2.dilation == (4, 4)
    with pytest.raises(NotImplementedError):
        DenseASPPModule(2048, 500, 128)


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_denseaspp_entry_points_argument_validation_without_gpu(lib):
    from torchseg_b200._lib import ConvShape
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255

    def shape(C=128, K=64, R=1, stride=1, pad=0):
        P = (9 + 2 * pad - (R - 1) - 1) // stride + 1
        return ConvShape(2, 9, 9, C, K, R, R, stride, pad, 1, P, P)

    def fwd(s=None, x=A, xcs=128, sc=A, sh=A, w=A, relu=0, y=A, ycs=64, s1=None, s2=None):
        s = shape() if s is None else s
        return lib.tsb_conv1x1_bnrelu_fprop(ctypes.byref(s), x, xcs, sc, sh, w, None, relu, y, 1, ycs, s1, s2, A, 1024,
                                            None)

    def wgr(s=None, x=A, xcs=128, sc=A, sh=A, dy=A, dycs=64, dw=A):
        s = shape() if s is None else s
        return lib.tsb_conv1x1_bnrelu_wgrad(ctypes.byref(s), x, xcs, sc, sh, dy, dycs, dw, A, 1024, None)

    def add(dy=A, x=A, dx=A, gamma=A, C=64, cs=64, relu=1, y=None, sc=A, sh=A):
        return lib.tsb_bn_bwd_apply_add(dy, cs, y, cs, x, cs, A, A, gamma, A, A, 10.0, relu, dx, cs, None, 0, 10, C, None,
                                        None, sc, sh, None)

    cases = [
        (lambda: fwd(s=shape(R=3, pad=1)), -3, b"only 1x1"), (lambda: fwd(s=shape(stride=2)), -3, b"only 1x1"),
        (lambda: wgr(s=shape(R=3, pad=1)), -3, b"only 1x1"), (lambda: wgr(s=shape(pad=1)), -3, b"only 1x1"),
        (lambda: fwd(x=None), -1, b"null pointer"), (lambda: fwd(w=None), -1, b"null pointer"),
        (lambda: fwd(y=None), -1, b"null pointer"), (lambda: fwd(sc=None), -1, b"null in_scale"),
        (lambda: wgr(sh=None), -1, b"null in_scale"), (lambda: wgr(dy=None), -1, b"null pointer"),
        (lambda: wgr(dw=None), -1, b"null pointer"),
        (lambda: fwd(s=shape(C=96), xcs=96), -1, b"multiple of 64"), (lambda: wgr(s=shape(C=96), xcs=96), -1,
                                                                      b"multiple of 64"),
        (lambda: fwd(xcs=132), -1, b"multiple of 8"), (lambda: fwd(xcs=120), -1, b"at least C"),
        (lambda: fwd(ycs=60), -1, b"multiple of 8"), (lambda: fwd(ycs=68), -1, b"multiple of 8"),
        (lambda: wgr(xcs=120), -1, b"layout"), (lambda: wgr(dycs=56), -1, b"layout"),
        (lambda: fwd(sc=A + 4), -1, b"16-byte aligned"), (lambda: wgr(sh=A + 8), -1, b"16-byte aligned"),
        (lambda: fwd(relu=1, s1=A, s2=A + 512), -1, b"takes no ReLU"),
        (lambda: add(dx=None), -1, b"bad args"), (lambda: add(gamma=None), -1, b"bad args"),
        (lambda: add(sc=None), -1, b"scale and shift"), (lambda: add(C=60, cs=60), -1, b"multiples of 8"),
        (lambda: add(dx=A + 2), -1, b"16B aligned"),
    ]
    for call, want, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == want and msg in err, (rc, want, msg, err)
    assert b"tsb_conv1x1_bnrelu_fprop" in (fwd(x=None), lib.tsb_last_error())[1]
    assert b"tsb_bn_bwd_apply_add" in (add(dx=None), lib.tsb_last_error())[1]


def test_denseaspp_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no prologue kernel (and no accumulating BN backward) spills to
    local memory or uses a stack"""
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if "bnrelu" in l or "bn_bwd_apply_add" in l]
    names = " ".join(" ".join(r) for r in rows)
    for bn in (64, 128):
        for res in ("true", "false"):
            assert "igemm_v2_bnrelu_kernel<%d, %s>" % (bn, res) in names, out
    assert "wgrad_mnmajor_bnrelu_kernel" in names and names.count("bn_bwd_apply_add_kernel") == 6, out
    for r in rows:
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % " ".join(r)
