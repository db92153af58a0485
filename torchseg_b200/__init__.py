"""torchseg_b200 — H100-native (sm_90a) training hot path behind the TorchSeg / furnace API.

The package mirrors the reference's import names for the path (seg_opr.seg_oprs, seg_opr.loss_opr,
base_model, engine.engine, engine.lr_policy, utils.init_func, utils.pyt_utils, apex.parallel); compute goes
through libtsb.so (include/tsb.h). See DESIGN.md / INTEGRATION.md.
"""
import torch.nn as nn

__version__ = "0.1.0"


def prepare_model(model):
    """Put every nn.Conv2d weight into KRSC (channels_last) physical layout in place — the layout the TMA
    descriptors of the conv kernels read and the wgrad kernel accumulates into. Values, shapes, parameter
    identity and state_dict keys are unchanged."""
    import torch
    for m in model.modules():
        if isinstance(m, nn.Conv2d):
            w = m.weight.data
            K, C, R, S = w.shape
            krsc = w.permute(0, 2, 3, 1).contiguous()
            m.weight.data = krsc.permute(0, 3, 1, 2)
            if m.weight.grad is not None:
                m.weight.grad = None
    return model


def install_as_furnace():
    """Expose this package's modules under the bare names the reference train.py scripts import
    (`from seg_opr.loss_opr import ...`, `from engine.engine import Engine`, `from apex.parallel import ...`)."""
    import importlib
    import sys
    for name in ("seg_opr", "seg_opr.seg_oprs", "seg_opr.loss_opr", "seg_opr.metric", "base_model", "base_model.resnet", "engine",
                 "engine.engine", "engine.lr_policy", "engine.logger", "engine.evaluator", "utils", "utils.init_func", "utils.pyt_utils", "utils.img_utils",
                 "apex", "apex.parallel"):
        sys.modules[name] = importlib.import_module("torchseg_b200." + name)
