"""CPU tests of DANet: the oracle (tests/danet_oracle.py) against the golden vectors of the network composed from the
live reference modules (tools/make_live_golden_danet.py), checkpoint-compatible module structure, group_weight, and
the argument checks and ptxas resources of the (64, 512) attention, the channel-attention soft-max and the
gamma-residual entry points (no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_danet.npz"))


def _net(criterion=None):
    from torchseg_b200.networks import DANet
    return DANet(19, criterion)


def test_oracle_vs_live_reference_danet_exact():
    import danet_oracle
    x, y, seed = danet_oracle.danet_case()
    torch.manual_seed(seed)
    m = _net()   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in danet_oracle.GAMMAS.items():
        sd[k] = torch.full((1,), v)
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = danet_oracle.danet_loss(x, y, sd)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert norm > 0, n   # with both gammas non-zero every parameter, the attention's convs included, has a gradient
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_danet_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    ref = json.loads(str(LIVE["keys"]))
    ours = _net().state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_danet_group_weight_and_structure():
    from torchseg_b200.networks import DANetHead
    from torchseg_b200.seg_opr.seg_oprs import CAM_Module, ConvBnRelu, PAM_Module
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = _net()
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    head = m.head
    assert isinstance(head, DANetHead) and m.business_layer == [head]
    no_decay = [p for g in groups if g.get("weight_decay") == 0.0 for p in g["params"]]
    decay = [p for g in groups if "weight_decay" not in g for p in g["params"]]
    assert any(p is head.sa.gamma for p in no_decay) and any(p is head.sc.gamma for p in no_decay)
    assert not any(p is head.sa.gamma or p is head.sc.gamma for p in decay)
    assert [n for n, _ in head.named_children()] == ["conv5a", "conv5c", "sa", "sc", "conv51", "conv52", "conv6",
                                                      "conv7", "conv8"]
    assert isinstance(head.sa, PAM_Module) and isinstance(head.sc, CAM_Module)
    assert [n for n, _ in head.sa.named_parameters()] == ["gamma", "query_conv.weight", "query_conv.bias",
                                                           "key_conv.weight", "key_conv.bias", "value_conv.weight",
                                                           "value_conv.bias"]
    assert [n for n, _ in head.sc.named_parameters()] == ["gamma"]
    for gamma in (head.sa.gamma, head.sc.gamma):
        assert gamma.shape == (1,) and float(gamma) == 0.0
    assert head.sa.query_conv.out_channels == 64 and head.sa.key_conv.out_channels == 64
    assert head.sa.value_conv.out_channels == 512
    for name in ("conv5a", "conv5c", "conv51", "conv52"):
        cbr = getattr(head, name)
        assert isinstance(cbr, ConvBnRelu) and cbr.conv.kernel_size == (3, 3) and cbr.conv.out_channels == 512
    for name in ("conv6", "conv7", "conv8"):
        seq = getattr(head, name)
        assert seq[0].p == 0.1 and seq[1].out_channels == 19 and seq[1].bias is not None
    l3, l4 = m.backbone.layer3, m.backbone.layer4
    assert l3[0].conv2.stride == (1, 1) and l3[1].conv2.dilation == (2, 2) and l4[1].conv2.dilation == (4, 4)


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_wide_attention_argument_validation_without_gpu(lib):
    """(d_k, d_v) = (64, 512): per-operand channel strides (q, k, dq, dk >= 64; v, o, dout, dv >= 512); other pairs with
    one side at 64 or 512 stay unsupported"""
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255

    def fwd(qcs=64, kcs=64, vcs=512, ocs=512, dk=64, dv=512, N=37, v=A):
        return lib.tsb_attention_fwd(A, qcs, A, kcs, v, vcs, A, ocs, A, 2, N, dk, dv, 1.0, None)

    def bwd(qcs=64, dqcs=64, dkcs=64, docs=512, dvcs=512, dk=64, dv=512, dq=A):
        return lib.tsb_attention_bwd(A, qcs, A, 64, A, 512, A, 512, A, docs, A, A, dq, dqcs, A, dkcs, A, dvcs, 0, 2, 37,
                                     dk, dv, 1.0, None)

    cases = [
        (lambda: fwd(dk=64, dv=256), -3, b"d_v=256"),
        (lambda: fwd(dk=256, dv=512), -3, b"d_k=256 d_v=512"), (lambda: fwd(dk=512, dv=64), -3, b"d_k=512"),
        (lambda: bwd(dk=64, dv=64), -3, b"d_v=64"), (lambda: fwd(N=0), -1, b"bad shape"),
        (lambda: fwd(qcs=56), -1, b">= 64"), (lambda: fwd(kcs=60), -1, b"multiple of 8"),
        (lambda: fwd(vcs=256), -1, b">= 512"), (lambda: fwd(ocs=504), -1, b">= 512"),
        (lambda: bwd(docs=256), -1, b">= 512"), (lambda: bwd(dvcs=480), -1, b">= 512"),
        (lambda: bwd(dqcs=32), -1, b">= 64"), (lambda: bwd(dkcs=40), -1, b">= 64"),
        (lambda: fwd(v=A + 8), -1, b"16-byte aligned"), (lambda: bwd(dq=None), -1, b"null dq"),
    ]
    for call, want, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == want and msg in err, (rc, want, msg, err)


def test_chan_attn_and_gamma_residual_argument_validation_without_gpu(lib):
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255
    L = ctypes.c_longlong
    cases = [
        (lambda: lib.tsb_chan_attn_softmax_fwd(None, A, 2, 512, None), b"null E"),
        (lambda: lib.tsb_chan_attn_softmax_fwd(A, A, 0, 512, None), b"bad shape"),
        (lambda: lib.tsb_chan_attn_softmax_fwd(A, A, 2, 1 << 16, None), b"bad shape"),
        (lambda: lib.tsb_chan_attn_softmax_bwd(A, A, None, A, 2, 512, None), b"rowdot_ws"),
        (lambda: lib.tsb_chan_attn_softmax_bwd(A, A, A, A, 2, 0, None), b"bad shape"),
        (lambda: lib.tsb_gamma_residual_fwd(A, 512, A, 512, None, A, 512, L(10), 512, None), b"gamma"),
        (lambda: lib.tsb_gamma_residual_fwd(A, 512, A, 512, A, A, 512, L(10), 500, None), b"multiple of 8"),
        (lambda: lib.tsb_gamma_residual_fwd(A, 504, A, 512, A, A, 512, L(10), 512, None), b">= C"),
        (lambda: lib.tsb_gamma_residual_fwd(A + 8, 512, A, 512, A, A, 512, L(10), 512, None), b"16-byte aligned"),
        (lambda: lib.tsb_gamma_residual_bwd(A, 512, A, 512, A, A, 512, None, L(10), 512, A, L(1 << 20), None),
         b"dgamma"),
        (lambda: lib.tsb_gamma_residual_bwd(A, 512, A, 512, A, A, 520, A, L(10), 512, None, L(0), None),
         b"workspace"),
        (lambda: lib.tsb_gamma_residual_bwd(A, 512, A + 4, 512, A, A, 512, A, L(10), 512, A, L(1 << 20), None),
         b"16-byte aligned"),
    ]
    for call, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == -1 and msg in err, (rc, msg, err)


def test_danet_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no attention, channel-attention or gamma-residual kernel spills to
    local memory or uses a stack"""
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if l.startswith(("attention.cu", "chan_attn.cu"))]
    names = " ".join(" ".join(r) for r in rows)
    for k in ("attn_fwd_wide_kernel", "attn_bwd_dv_wide_kernel", "attn_bwd_ds_wide_kernel", "attn_delta_wide_kernel",
              "attn_fwd_kernel", "cam_softmax_fwd_kernel", "cam_softmax_bwd_kernel", "cam_rowdot_kernel",
              "gamma_residual_fwd_kernel", "gamma_residual_bwd_kernel"):
        assert k in names, out
    for r in rows:
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % " ".join(r)
