"""CPU tests of EncNet: the oracle (tests/encnet_oracle.py) against the golden vectors of the network composed from the
live reference modules (tools/make_live_golden_encnet.py), checkpoint-compatible module structure, group_weight, and the
argument checks of the Encoding, channel-mean and SE-loss entry points (no GPU needed)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_encnet.npz"))


def _net(criterion=None):
    from torchseg_b200.networks import EncNet
    return EncNet(150, criterion)


def test_oracle_vs_live_reference_encnet_exact():
    import encnet_oracle
    x, y, seed = encnet_oracle.encnet_case()
    torch.manual_seed(seed)
    m = _net()   # same seed, same construction order → the reference composition's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = encnet_oracle.encnet_loss(x, y, sd)
    loss.backward()
    assert float(loss) == float(LIVE["loss"])
    grads = json.loads(str(LIVE["grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


def test_encnet_state_dict_matches_reference():
    """checkpoint compatibility: the reference composition's state_dict keys and shapes, in order"""
    ref = json.loads(str(LIVE["keys"]))
    ours = _net().state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k


def test_encnet_group_weight_and_geometry():
    from torchseg_b200.seg_opr.seg_oprs import Encoding
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = _net()
    groups = group_weight([], m.backbone, BN, 1e-2)
    for mod in m.business_layer:
        groups = group_weight(groups, mod, BN, 1e-1)
    assert sum(len(g["params"]) for g in groups) == sum(1 for _ in m.parameters())
    enc = m.head.encmodule.encoding
    assert isinstance(enc, Encoding) and enc.codewords.shape == (32, 512) and enc.scale.shape == (32,)
    decay, no_decay = groups[2]["params"], groups[3]["params"]
    assert any(p is enc.codewords for p in decay) and not any(p is enc.codewords for p in no_decay)
    assert any(p is enc.scale for p in no_decay) and not any(p is enc.scale for p in decay)
    assert groups[3]["weight_decay"] == 0.0
    assert isinstance(m.head.encmodule.bn, BN) and m.head.encmodule.bn.num_features == 32
    # init: codewords ~ U(±1/sqrt(K·D)), scale ~ U(−1, 0)
    assert float(enc.codewords.abs().max()) <= 1 / (32 * 512) ** 0.5 and float(enc.scale.max()) <= 0.0
    assert float(enc.scale.min()) >= -1.0
    l3, l4 = m.backbone.layer3, m.backbone.layer4
    assert l3[0].conv2.stride == (1, 1) and l3[1].conv2.dilation == (2, 2) and l4[1].conv2.dilation == (4, 4)
    assert m.aux_loss_ratio == 0.2 and m.se_loss_ratio == 0.2


def test_group_weight_unchanged_for_networks_without_encoding():
    from torchseg_b200.networks import PSPNet
    from torchseg_b200.utils.init_func import group_weight
    BN = torch.nn.BatchNorm2d
    m = PSPNet(150, None)
    groups = group_weight([], m.psp_layer, BN, 1e-1)
    assert len(groups[0]["params"]) == sum(1 for mm in m.psp_layer.modules() if isinstance(mm, torch.nn.Conv2d))


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def _buf(n=1 << 16):
    b = ctypes.create_string_buffer(n + 16)
    return b, (ctypes.addressof(b) + 15) // 16 * 16


def test_encoding_argument_validation_without_gpu(lib):
    keep, A = _buf()
    WS = 1 << 30
    # (K, D, xcs, rc, message) — checked by both directions
    cases = [
        (12, 64, 64, -3, b"multiple of 8"),
        (40, 64, 64, -3, b"at most 32"),
        (0, 64, 64, -3, b"multiple of 8"),
        (8, 96, 96, -3, b"D=96"),
        (8, 2048, 2048, -3, b"D=2048"),
        (32, 1024, 1024, -3, b"K*D"),
        (8, 64, 60, -1, b"channel stride"),
        (8, 64, 68, -1, b"channel stride"),
    ]
    for K, D, xcs, rc_want, msg in cases:
        rc = lib.tsb_encoding_fwd(A, xcs, 2, 16, D, A, A, K, A, A, A, A, A, WS, None)
        assert rc == rc_want and msg in lib.tsb_last_error(), lib.tsb_last_error()
        rc = lib.tsb_encoding_bwd(A, A, xcs, 2, 16, D, A, A, K, A, A, A, A, D, A, A, A, WS, None)
        assert rc == rc_want and msg in lib.tsb_last_error(), lib.tsb_last_error()
    assert lib.tsb_encoding_fwd(None, 64, 2, 16, 64, A, A, 8, A, A, A, A, A, WS, None) == -1
    assert b"null" in lib.tsb_last_error()
    assert lib.tsb_encoding_fwd(A, 64, 2, 16, 64, None, A, 8, A, A, A, A, A, WS, None) == -1
    assert lib.tsb_encoding_fwd(A, 64, 2, 16, 64, A, A, 8, A, A, A, None, A, WS, None) == -1
    assert lib.tsb_encoding_fwd(A, 64, 2, 16, 64, A, A, 8, A, None, A, A, A, WS, None) == -1
    assert b"both" in lib.tsb_last_error()
    assert lib.tsb_encoding_fwd(A + 8, 64, 2, 16, 64, A, A, 8, A, A, A, A, A, WS, None) == -1
    assert b"16-byte" in lib.tsb_last_error()
    assert lib.tsb_encoding_fwd(A, 64, 0, 16, 64, A, A, 8, A, A, A, A, A, WS, None) == -1
    assert lib.tsb_encoding_bwd(A, A, 64, 2, 16, 64, A, A, 8, None, A, A, A, 64, A, A, A, WS, None) == -1
    assert b"null" in lib.tsb_last_error()
    assert lib.tsb_encoding_bwd(A, A, 64, 2, 16, 64, A, A, 8, A, A, A, A, 56, A, A, A, WS, None) == -1
    assert b"dx channel stride" in lib.tsb_last_error()
    # workspace: 16 slots per image, K·D + K floats each forward, K·D + 2K backward
    need_f, need_b = 2 * 16 * (8 * 64 + 8), 2 * 16 * (8 * 64 + 16)
    assert lib.tsb_encoding_fwd(A, 64, 2, 16, 64, A, A, 8, A, A, A, A, A, need_f - 1, None) == -1
    assert b"workspace needs %d floats" % need_f in lib.tsb_last_error()
    assert lib.tsb_encoding_fwd(A, 64, 2, 16, 64, A, A, 8, A, A, A, A, None, WS, None) == -1
    assert lib.tsb_encoding_bwd(A, A, 64, 2, 16, 64, A, A, 8, A, A, A, A, 64, A, A, A, need_b - 1, None) == -1
    assert b"workspace needs %d floats" % need_b in lib.tsb_last_error()


def test_chan_mean_and_se_loss_argument_validation_without_gpu(lib):
    keep, A = _buf()
    assert lib.tsb_chan_mean_fwd(None, 32, 16, 32, A, None) == -1 and b"null" in lib.tsb_last_error()
    assert lib.tsb_chan_mean_fwd(A, 16, 16, 32, A, None) == -1 and b"bad shape" in lib.tsb_last_error()
    assert lib.tsb_chan_mean_bwd(A, 16, 32, None, 32, None) == -1 and b"null" in lib.tsb_last_error()
    assert lib.tsb_chan_mean_bwd(A, 16, 32, A, 16, None) == -1 and b"bad shape" in lib.tsb_last_error()
    assert lib.tsb_se_loss_fwd_bwd(None, 2, 64, A, 160, 150, A, A, A, 160, None) == -1
    assert b"null" in lib.tsb_last_error()
    assert lib.tsb_se_loss_fwd_bwd(A, 2, 64, A, 140, 150, A, A, A, 160, None) == -1
    assert b"bad shape" in lib.tsb_last_error()
    assert lib.tsb_se_loss_fwd_bwd(A, 2, 64, A, 5000, 4097, A, A, A, 5000, None) == -3
    assert b"4096" in lib.tsb_last_error()


def test_encoding_kernels_build_without_spills():
    """the -Xptxas -v resources of the in-tree build: no Encoding kernel spills to local memory"""
    import subprocess
    import sys
    from torchseg_b200 import build
    build.build()
    out = subprocess.run([sys.executable, os.path.join(HERE, "..", "tools", "ptxas_summary.py")], capture_output=True,
                         text=True, check=True).stdout
    rows = [l.split() for l in out.splitlines() if l.startswith("encoding.cu")]
    assert len([r for r in rows if "enc_fwd_kernel" in " ".join(r) or "enc_bwd_kernel" in " ".join(r)]) == 8, out
    for r in rows:
        assert int(r[-2]) == 0 and int(r[-1]) == 0, "spill / stack in %s" % " ".join(r)
