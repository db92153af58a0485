"""CPU tests of OCNet: the oracle (tests/ocnet_oracle.py) against the golden vectors of the network composed from the
live reference modules (tools/make_live_golden_ocnet.py), checkpoint-compatible module structure, group_weight, the
attention block's construction, and the argument checks and ptxas resources of the attention entry points (no GPU
needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_ocnet.npz"))


def _net(criterion=None):
    from torchseg_b200.networks import OCNet
    return OCNet(19, criterion)


def test_oracle_vs_live_reference_ocnet_exact():
    import ocnet_oracle
    x, y, seed = ocnet_oracle.ocnet_case()
    torch.manual_seed(seed)
    m = _net()   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    w, b = ocnet_oracle.nonzero_w()
    sd[ocnet_oracle.W_PREFIX + ".weight"], sd[ocnet_oracle.W_PREFIX + ".bias"] = w, b
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = ocnet_oracle.ocnet_loss(x, y, sd)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert norm > 0, n   # with W non-zero every parameter, f_key and f_value included, receives a gradient
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_ocnet_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    ref = json.loads(str(LIVE["keys"]))
    ours = _net().state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_ocnet_group_weight_and_structure():
    from torchseg_b200.seg_opr.seg_oprs import BaseOCModule, ConvBnRelu, SelfAttentionBlock
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = _net()
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    oc = m.context[1]
    assert isinstance(oc, BaseOCModule) and len(oc.stages) == 1
    blk = oc.stages[0]
    assert isinstance(blk, SelfAttentionBlock) and isinstance(blk.f_key, ConvBnRelu)
    assert not hasattr(blk, "f_query")
    assert [n for n, _ in blk.named_children()] == ["f_key", "f_value", "W"]
    assert float(blk.W.weight.abs().max()) == 0.0 and float(blk.W.bias.abs().max()) == 0.0
    assert blk.f_value.bias is not None and blk.W.bias is not None
    assert blk.f_key.conv.out_channels == 256 and blk.f_value.out_channels == 256 and blk.W.out_channels == 512
    assert oc.conv_bn_dropout[1].p == 0.05 and m.aux_layer[1].p == 0.1
    assert m.cls.bias is not None and m.cls.out_channels == 19
    l3, l4 = m.backbone.layer3, m.backbone.layer4
    assert l3[0].conv2.stride == (1, 1) and l3[1].conv2.dilation == (2, 2) and l4[1].conv2.dilation == (4, 4)
    assert m.aux_loss_ratio == 0.4
    with pytest.raises(NotImplementedError):
        SelfAttentionBlock(512, 256, 256, 512, scale=2)


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_attention_argument_validation_without_gpu(lib):
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255

    def fwd(q=A, qcs=256, k=A, kcs=256, v=A, vcs=256, o=A, ocs=256, lse=A, B=2, N=37, dk=256, dv=256, scale=0.0625):
        return lib.tsb_attention_fwd(q, qcs, k, kcs, v, vcs, o, ocs, lse, B, N, dk, dv, scale, None)

    def bwd(q=A, k=A, dq=A, dk=A, dv=A, dqcs=256, lse=A, delta=A, B=2, N=37, d=256, scale=0.0625):
        return lib.tsb_attention_bwd(q, 256, k, 256, A, 256, A, 256, A, 256, lse, delta, dq, dqcs, dk, 256, dv, 256, 1,
                                     B, N, d, d, scale, None)

    cases = [
        (lambda: fwd(dk=128), -3, b"d_k=128"), (lambda: fwd(dv=64), -3, b"d_v=64"),
        (lambda: fwd(dk=0), -3, b"d_k=0"), (lambda: bwd(d=512), -3, b"d_k=512"),
        (lambda: fwd(N=0), -1, b"bad shape"), (lambda: fwd(B=0), -1, b"bad shape"),
        (lambda: bwd(N=0), -1, b"bad shape"), (lambda: fwd(B=1 << 16, N=1 << 15), -1, b"2^31"),
        (lambda: fwd(scale=0.0), -1, b"scale"), (lambda: fwd(scale=float("inf")), -1, b"scale"),
        (lambda: fwd(q=None), -1, b"null q"), (lambda: fwd(k=None), -1, b"null k"),
        (lambda: fwd(v=None), -1, b"null v"), (lambda: fwd(o=None), -1, b"null o"),
        (lambda: bwd(dq=None), -1, b"null dq"), (lambda: bwd(dk=None), -1, b"null dk"),
        (lambda: bwd(dv=None), -1, b"null dv"), (lambda: bwd(lse=None), -1, b"null lse"),
        (lambda: bwd(delta=None), -1, b"delta_ws"),
        (lambda: fwd(qcs=260), -1, b"multiple of 8"), (lambda: fwd(kcs=248), -1, b">= 256"),
        (lambda: fwd(ocs=300), -1, b"multiple of 8"), (lambda: bwd(dqcs=252), -1, b"multiple of 8"),
        (lambda: fwd(v=A + 8), -1, b"16-byte aligned"), (lambda: fwd(q=A + 2), -1, b"16-byte aligned"),
        (lambda: bwd(dk=A + 4), -1, b"16-byte aligned"),
    ]
    for call, want, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == want and msg in err, (rc, want, msg, err)


def test_attention_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no attention kernel spills to local memory or uses a stack"""
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if l.startswith("attention.cu")]
    names = " ".join(" ".join(r) for r in rows)
    for k in ("attn_fwd_kernel", "attn_bwd_kv_kernel", "attn_bwd_q_kernel", "attn_delta_kernel"):
        assert k in names, out
    for r in rows:
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % " ".join(r)
