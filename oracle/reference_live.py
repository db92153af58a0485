"""ORACLE — test infrastructure only.

Imports the UNMODIFIED reference modules live from a TorchSeg checkout named by TSB_REFERENCE_DIR (used by
tools/make_golden.py and tools/make_live_golden.py to regenerate tests/golden) with the three in-memory shims of
SURVEY.md App. C:
  1. import utils.pyt_utils before engine.logger (circular import),
  2. exec loss_opr.py with `1 - valid_mask` → `~valid_mask` (bool-tensor subtraction, torch >= 1.2),
  3. a stand-in `config` module (easydict is absent and config.py needs a cwd containing 'TorchSeg').
Nothing is copied into this repo; modules are loaded from where they lie.
"""
import importlib
import importlib.util
import os
import sys
import types

REF = os.environ.get("TSB_REFERENCE_DIR", "")
FURNACE = os.path.join(REF, "furnace")


def available():
    return bool(REF) and os.path.isdir(FURNACE)


class _Cfg(dict):
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def _ensure_base():
    if FURNACE not in sys.path:
        sys.path.insert(0, FURNACE)
    import utils.pyt_utils  # noqa: F401  (shim 1: must precede engine.logger)
    import engine.logger  # noqa: F401


def load_loss_opr():
    """reference seg_opr.loss_opr with shim 2 applied in memory"""
    _ensure_base()
    path = os.path.join(FURNACE, "seg_opr", "loss_opr.py")
    src = open(path).read()
    assert src.count("1 - valid_mask") == 2
    src = src.replace("1 - valid_mask", "~valid_mask")
    mod = types.ModuleType("seg_opr.loss_opr_shimmed")
    mod.__file__ = path
    exec(compile(src, path, "exec"), mod.__dict__)
    return mod


def load_seg_oprs():
    _ensure_base()
    return importlib.import_module("seg_opr.seg_oprs")


def load_resnet():
    _ensure_base()
    return importlib.import_module("base_model.resnet")


def load_network(rel_dir, num_classes=19, bn_eps=1e-5, bn_momentum=0.1, **extra):
    """import model/<rel_dir>/network.py with a stand-in `config` module (shim 3)"""
    _ensure_base()
    cfg = _Cfg(num_classes=num_classes, bn_eps=bn_eps, bn_momentum=bn_momentum, **extra)
    cmod = types.ModuleType("config")
    cmod.config = cfg
    cmod.cfg = cfg
    saved = sys.modules.get("config")
    sys.modules["config"] = cmod
    try:
        path = os.path.join(REF, "model", rel_dir, "network.py")
        name = "refnet_" + rel_dir.replace("/", "_").replace(".", "_")
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is not None:
            sys.modules["config"] = saved
        else:
            del sys.modules["config"]
    return mod


def load_evaluator():
    """reference engine.evaluator, importable under Python >= 3.10 with one more in-memory shim: img_utils.py:9 uses
    `collections.Iterable` (removed in 3.10) → alias it to collections.abc.Iterable for the import"""
    import collections
    import collections.abc
    _ensure_base()
    if not hasattr(collections, "Iterable"):
        collections.Iterable = collections.abc.Iterable
    return importlib.import_module("engine.evaluator")


def load_train_pre(rel_dir, **cfg):
    """import model/<rel_dir>/dataloader.py (TrainPre) with a stand-in `config` (train_scale_array, image_height,
    image_width, ...) and the collections.Iterable alias img_utils.py:9 needs under Python >= 3.10"""
    import collections
    import collections.abc
    _ensure_base()
    if not hasattr(collections, "Iterable"):
        collections.Iterable = collections.abc.Iterable
    c = _Cfg(**cfg)
    cmod = types.ModuleType("config")
    cmod.config = c
    saved = sys.modules.get("config")
    sys.modules["config"] = cmod
    try:
        path = os.path.join(REF, "model", rel_dir, "dataloader.py")
        name = "refdl_" + rel_dir.replace("/", "_").replace(".", "_")
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is not None:
            sys.modules["config"] = saved
        else:
            del sys.modules["config"]
    mod.config = c      # TrainPre.__call__ reads the module-level name at call time
    return mod
