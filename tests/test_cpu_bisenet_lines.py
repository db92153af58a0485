"""CPU tests of the BiSeNet lines R18.speed, X39.speed and R101: the oracle (tests/bisenet_lines_oracle.py) against the
golden vectors of the live reference networks (tools/make_live_golden_bisenet_lines.py), checkpoint-compatible module
structure in train and eval mode, group_weight in the reference's order, and the reference import names (no GPU
needed)."""
import importlib
import json
import logging
import os

import numpy as np
import pytest
import torch

from bisenet_lines_cases import bisenet_case

HERE = os.path.dirname(os.path.abspath(__file__))
LIVE = np.load(os.path.join(HERE, "golden", "live_reference_bisenet_lines.npz"))
BN = torch.nn.BatchNorm2d

# line → (module under torchseg_b200.networks, bisenet_case arguments, takes ohem_criterion)
LINES = {
    "r18_speed": ("bisenet_speed", dict(N=2, H=64, W=128, gt_down=8, seed=21), True),
    "x39_speed": ("bisenet_x39_speed", dict(N=2, H=64, W=128, gt_down=8, seed=22), True),
    "r101": ("bisenet_r101", dict(N=2, H=64, W=64, seed=23), False),
}


def _net(line, training, crit=None, ohem=None):
    mod, _, two_crit = LINES[line]
    cls = importlib.import_module("torchseg_b200.networks." + mod).BiSeNet
    return cls(19, training, crit, ohem, None, BN) if two_crit else cls(19, training, ohem, None, BN)


@pytest.mark.parametrize("line", list(LINES))
def test_oracle_vs_live_reference_exact(line):
    import bisenet_lines_oracle as tr
    x, y, min_kept, seed = bisenet_case(**LINES[line][1])
    torch.manual_seed(seed)
    m = _net(line, True)   # same seed → the reference's initial weights
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    loss, _ = tr.bisenet_loss(line, x, y, sd, min_kept)
    loss.backward()
    assert float(loss) == float(LIVE[line + "_loss"])
    grads = json.loads(str(LIVE[line + "_grads"]))
    assert len(grads) == sum(1 for _ in m.parameters())
    for n, (norm, idx, vals) in grads.items():
        flat = sd[n].grad.reshape(-1).double().numpy()
        assert abs(np.linalg.norm(flat) - norm) <= 1e-5 * norm, n
        assert np.max(np.abs(flat[idx] - np.array(vals))) <= 1e-5 * max(norm, 1e-30), n


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("line", list(LINES))
def test_state_dict_matches_reference(line, mode):
    """checkpoint compatibility: the reference's state_dict keys and shapes, in order; the .speed eval networks hold
    no aux heads"""
    ref = json.loads(str(LIVE["%s_%s_keys" % (line, mode)]))
    ours = _net(line, mode == "train").state_dict()
    assert [k for k, _ in ref] == list(ours.keys())
    for k, shape in ref:
        assert list(ours[k].shape) == shape, k
    aux = any(k.startswith(("heads.0.", "heads.1.")) for k in ours)
    assert aux == (mode == "train" or line == "r101")


def test_speed_eval_heads_and_checkpoint_load(caplog):
    """eval heads are nn.ModuleList([None, None, head]); a training checkpoint loads through the non-strict
    utils.pyt_utils.load_model, which drops the aux heads"""
    from torchseg_b200.utils.pyt_utils import load_model
    for line in ("r18_speed", "x39_speed"):
        torch.manual_seed(0)
        train_sd = _net(line, True).state_dict()
        m = _net(line, False)
        assert m.heads[0] is None and m.heads[1] is None and m.heads[2].scale == 1
        with caplog.at_level(logging.WARNING):
            load_model(m, train_sd)
        for k, v in m.state_dict().items():
            assert torch.equal(v, train_sd[k]), k
        assert "Unexpected key(s)" in caplog.text and "heads.0.conv_3x3.conv.weight" in caplog.text
        assert "Missing key(s)" not in caplog.text
        caplog.clear()


# the group_weight calls of each line's train.py, in order, with their learning-rate factor
GROUP_ORDER = {
    "r18_speed": [("context_path", 1), ("spatial_path", 10), ("global_context", 10), ("arms", 10), ("refines", 10),
                  ("ffm", 10), ("heads", 10)],
    "x39_speed": [("context_path", 1), ("spatial_path", 1), ("global_context", 1), ("arms", 1), ("refines", 1),
                  ("heads", 10), ("ffm", 10)],
    "r101": [("context_path", 1), ("spatial_path", 10), ("global_context", 10), ("arms", 10), ("refines", 10),
             ("heads", 10), ("ffm", 10)],
}


@pytest.mark.parametrize("line", list(LINES))
def test_group_weight_covers_every_parameter_in_reference_order(line):
    from torchseg_b200.utils.init_func import group_weight
    m = _net(line, True)
    groups = []
    for attr, f in GROUP_ORDER[line]:
        groups = group_weight(groups, getattr(m, attr), BN, 1e-2 * f)
    got = [p for g in groups for p in g["params"]]
    assert len(got) == sum(1 for _ in m.parameters())
    assert {id(p) for p in got} == {id(p) for p in m.parameters()}
    # one (decay, no-decay) pair per module, each with its line's learning rate
    assert [g["lr"] for g in groups] == [1e-2 * f for _, f in GROUP_ORDER[line] for _ in range(2)]
    first_head = next(i for i, (a, _) in enumerate(GROUP_ORDER[line]) if a == "heads")
    head_ids = {id(p) for p in m.heads.parameters()}
    assert {id(p) for p in groups[2 * first_head]["params"] + groups[2 * first_head + 1]["params"]} == head_ids


def test_head_scales_and_widths():
    for line, scales, aux, main in (("r18_speed", (2, 1, 1), 128, 64), ("x39_speed", (2, 1, 1), 128, 64),
                                    ("r101", (16, 8, 8), 256, 256)):
        m = _net(line, True)
        assert tuple(h.scale for h in m.heads) == scales, line
        assert [h.conv_1x1.in_channels for h in m.heads] == [aux, aux, main], line
        assert m.loss_attr == ("criterion" if line == "r101" else "ohem_criterion")


def test_reference_import_names(monkeypatch):
    import sys
    import torchseg_b200
    for name in ("seg_opr", "seg_opr.seg_oprs", "seg_opr.loss_opr", "seg_opr.metric", "base_model", "base_model.resnet",
                 "base_model.xception", "engine", "engine.engine", "engine.lr_policy", "engine.logger",
                 "engine.evaluator", "utils", "utils.init_func", "utils.pyt_utils", "utils.img_utils", "apex",
                 "apex.parallel"):
        monkeypatch.setitem(sys.modules, name, None)   # install_as_furnace rewrites these: restored after the test
    torchseg_b200.install_as_furnace()
    # the imports of the three network.py files (R18.speed / R101 / X39.speed, lines 9-12)
    from base_model import resnet18, resnet101, xception39
    from seg_opr.seg_oprs import ConvBnRelu, AttentionRefinement, FeatureFusion
    from seg_opr.loss_opr import ProbOhemCrossEntropy2d
    assert sys.modules["base_model.resnet"].resnet101 is resnet101
    assert sys.modules["base_model.resnet"].resnet18 is resnet18
    assert sys.modules["base_model.xception"].xception39 is xception39
    assert hasattr(ProbOhemCrossEntropy2d, "forward_lowres")
    assert all(c.__module__ == "torchseg_b200.seg_opr.seg_oprs" for c in (ConvBnRelu, AttentionRefinement, FeatureFusion))
