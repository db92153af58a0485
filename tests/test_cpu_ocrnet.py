"""CPU tests of OCRNet: the oracle (tests/ocrnet_oracle.py) against the golden vectors of the network composed from the
live reference modules (tools/make_live_golden_ocrnet.py), checkpoint-compatible module structure, group_weight, and
the argument checks and ptxas resources of the cross-attention and spatial soft-max entry points (no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_ocrnet.npz"))


def _net(criterion=None):
    from torchseg_b200.networks import OCRNet
    return OCRNet(19, criterion)


def test_oracle_vs_live_reference_ocrnet_exact():
    import ocrnet_oracle
    x, y, seed = ocrnet_oracle.ocrnet_case()
    torch.manual_seed(seed)
    m = _net()   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = ocrnet_oracle.ocrnet_loss(x, y, sd)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert norm > 0, n   # every parameter, f_pixel, f_object, f_down and f_up included, receives a gradient
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_ocrnet_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    ref = json.loads(str(LIVE["keys"]))
    ours = _net().state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_ocrnet_group_weight_and_structure():
    from torchseg_b200.seg_opr.seg_oprs import (ConvBnRelu, ObjectAttentionBlock, SpatialGatherModule,
                                                SpatialOCRModule)
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = _net()
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    assert [n for n, _ in m.named_children()] == ["backbone", "conv_3x3", "spatial_context_head", "spatial_ocr_head",
                                                  "head", "dsn_head"]
    assert m.business_layer == [m.conv_3x3, m.spatial_ocr_head, m.head, m.dsn_head]
    assert isinstance(m.spatial_context_head, SpatialGatherModule)
    assert sum(1 for _ in m.spatial_context_head.parameters()) == 0
    ocr = m.spatial_ocr_head
    assert isinstance(ocr, SpatialOCRModule)
    assert [n for n, _ in ocr.named_children()] == ["object_context_block", "conv_bn_dropout"]
    blk = ocr.object_context_block
    assert isinstance(blk, ObjectAttentionBlock)
    assert [n for n, _ in blk.named_children()] == ["f_pixel", "f_object", "f_down", "f_up"]
    for seq in (blk.f_pixel, blk.f_object):
        assert len(seq) == 2 and all(isinstance(c, ConvBnRelu) and c.conv.bias is None for c in seq)
        assert (seq[0].conv.in_channels, seq[0].conv.out_channels, seq[1].conv.out_channels) == (512, 256, 256)
    assert (blk.f_down.conv.in_channels, blk.f_down.conv.out_channels) == (512, 256)
    assert (blk.f_up.conv.in_channels, blk.f_up.conv.out_channels) == (256, 512)
    assert ocr.conv_bn_dropout[0].conv.in_channels == 1024 and ocr.conv_bn_dropout[1].p == 0.05
    assert m.conv_3x3.conv.bias is None and m.conv_3x3.conv.kernel_size == (3, 3)
    assert m.dsn_head[0].conv.in_channels == 1024 and m.dsn_head[1].p == 0.05
    assert m.head.bias is not None and m.head.out_channels == 19 and m.dsn_head[2].bias is not None
    l3, l4 = m.backbone.layer3, m.backbone.layer4
    assert l3[0].conv2.stride == (1, 1) and l3[1].conv2.dilation == (2, 2) and l4[1].conv2.dilation == (4, 4)
    assert m.aux_loss_ratio == 0.4
    with pytest.raises(NotImplementedError):
        ObjectAttentionBlock(512, 256, scale=2)
    with pytest.raises(NotImplementedError):
        SpatialGatherModule(19, scale=2)


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def _aligned(n=4096):
    mem = (ctypes.c_uint8 * n)()
    return mem, (ctypes.addressof(mem) + 255) & ~255


def test_cross_attention_argument_validation_without_gpu(lib):
    mem, A = _aligned()

    def fwd(q=A, qcs=256, k=A, kcs=256, v=A, vcs=256, o=A, ocs=256, lse=A, B=2, Nq=37, Nk=19, dk=256, dv=256,
            scale=0.0625):
        return lib.tsb_cross_attention_fwd(q, qcs, k, kcs, v, vcs, o, ocs, lse, B, Nq, Nk, dk, dv, scale, None)

    def bwd(q=A, k=A, dq=A, dk=A, dv=A, dqcs=256, dvcs=256, lse=A, delta=A, B=2, Nq=37, Nk=19, d_k=256, d_v=256):
        return lib.tsb_cross_attention_bwd(q, 256, k, 256, A, 256, A, 256, A, 256, lse, delta, dq, dqcs, dk, 256, dv,
                                           dvcs, B, Nq, Nk, d_k, d_v, 0.0625, None)

    cases = [
        (lambda: fwd(dk=64, dv=512), -3, b"only (d_k, d_v) = (256, 256)"), (lambda: fwd(dk=128), -3, b"d_k=128"),
        (lambda: bwd(d_k=64, d_v=512), -3, b"d_v=512"), (lambda: bwd(d_k=256, d_v=512), -3, b"d_v=512"),
        (lambda: fwd(Nq=0), -1, b"bad shape"), (lambda: fwd(Nk=0), -1, b"bad shape"),
        (lambda: fwd(B=0), -1, b"bad shape"), (lambda: bwd(Nk=-1), -1, b"bad shape"),
        (lambda: fwd(B=1 << 16, Nq=1 << 15), -1, b"2^31"), (lambda: fwd(B=1 << 15, Nk=1 << 16), -1, b"2^31"),
        (lambda: bwd(B=4, Nq=1 << 29), -1, b"2^31"),
        (lambda: fwd(scale=0.0), -1, b"scale"),
        (lambda: fwd(q=None), -1, b"null q"), (lambda: fwd(k=None), -1, b"null k"),
        (lambda: fwd(v=None), -1, b"null v"), (lambda: fwd(o=None), -1, b"null o"),
        (lambda: bwd(dq=None), -1, b"null dq"), (lambda: bwd(dk=None), -1, b"null dk"),
        (lambda: bwd(dv=None), -1, b"null dv"), (lambda: bwd(lse=None), -1, b"null lse"),
        (lambda: bwd(delta=None), -1, b"delta_ws"),
        (lambda: fwd(qcs=260), -1, b"multiple of 8"), (lambda: fwd(kcs=248), -1, b">= 256"),
        (lambda: fwd(ocs=300), -1, b"multiple of 8"), (lambda: bwd(dvcs=252), -1, b"multiple of 8"),
        (lambda: fwd(v=A + 8), -1, b"16-byte aligned"), (lambda: fwd(k=A + 2), -1, b"16-byte aligned"),
        (lambda: bwd(dk=A + 4), -1, b"16-byte aligned"), (lambda: fwd(lse=A + 4), -1, b"lse must be 16-byte"),
    ]
    for call, want, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == want and msg in err, (rc, want, msg, err)
        assert b"tsb_cross_attention_" in err, err


def test_spatial_softmax_argument_validation_without_gpu(lib):
    mem, A = _aligned()
    WS = 1 << 20

    def fwd(l=A, lcs=32, P=A, stats=A, B=2, N=81, K=19, ws=A, ws_floats=WS):
        return lib.tsb_spatial_softmax_fwd(l, lcs, P, stats, B, N, K, ws, ws_floats, None)

    def bwd(l=A, lcs=32, stats=A, dP=A, dpcs=64, dl=A, dlcs=32, B=2, N=81, K=19, ws=A, ws_floats=WS):
        return lib.tsb_spatial_softmax_bwd(l, lcs, stats, dP, dpcs, dl, dlcs, B, N, K, ws, ws_floats, None)

    cases = [
        (lambda: fwd(K=257), -1, b"K=257"), (lambda: fwd(K=0), -1, b"K=0"), (lambda: bwd(K=300), -1, b"K=300"),
        (lambda: fwd(N=0), -1, b"bad shape"), (lambda: fwd(B=0), -1, b"bad shape"),
        (lambda: bwd(B=1 << 16), -1, b"bad shape"),
        (lambda: fwd(B=1 << 15, N=1 << 16), -1, b"2^31"), (lambda: bwd(B=4, N=1 << 29), -1, b"2^31"),
        (lambda: fwd(lcs=20), -1, b"multiple of 8"), (lambda: fwd(lcs=16), -1, b">= K rounded up to 8"),
        (lambda: fwd(K=17, lcs=16), -1, b"got 16"), (lambda: fwd(l=A + 4), -1, b"16-byte aligned"),
        (lambda: fwd(P=A + 2), -1, b"P must be 16-byte aligned"),
        (lambda: bwd(dpcs=12), -1, b"dP and dl"), (lambda: bwd(dlcs=16), -1, b"dP and dl"),
        (lambda: bwd(dP=A + 4), -1, b"dP and dl"), (lambda: bwd(dl=A + 8), -1, b"dP and dl"),
        (lambda: fwd(l=None), -1, b"null logits"), (lambda: fwd(P=None), -1, b"null P"),
        (lambda: fwd(stats=None), -1, b"null P or stats"), (lambda: bwd(stats=None), -1, b"null stats"),
        (lambda: bwd(dP=None), -1, b"null stats, dP"), (lambda: bwd(dl=None), -1, b"dP or dl"),
        (lambda: fwd(ws=None), -1, b"workspace"), (lambda: fwd(ws_floats=16), -1, b"workspace"),
        (lambda: bwd(ws_floats=16), -1, b"workspace"),
    ]
    for call, want, msg in cases:
        rc = call()
        err = lib.tsb_last_error()
        assert rc == want and msg in err, (rc, want, msg, err)


def test_attention_and_spatial_softmax_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no kernel of attention.cu or spatial_softmax.cu spills to local
    memory or uses a stack"""
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if l.startswith(("attention.cu", "spatial_softmax.cu"))]
    names = " ".join(" ".join(r) for r in rows)
    for k in ("attn_fwd_kernel", "attn_bwd_kv_kernel", "attn_bwd_q_kernel", "attn_delta_kernel", "ssm_partial_kernel",
              "ssm_apply_kernel", "ssm_bwd_partial_kernel", "ssm_bwd_apply_kernel"):
        assert k in names, out
    for r in rows:
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % " ".join(r)
