"""CPU tests of the C-ABI library: it loads without a GPU, exports every symbol include/tsb.h declares, validates
arguments and fails LOUDLY (no silent fallback) when there is no CUDA device."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from torchseg_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_header_symbols_all_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "tsb.h")).read()
    declared = set(re.findall(r"\b(tsb_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"tsb_stream_t"}
    assert len(declared) >= 35
    for name in sorted(declared):
        assert hasattr(lib, name), "include/tsb.h declares %s but libtsb.so does not export it" % name


def test_python_binding_covers_header(lib):
    from torchseg_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "tsb.h")).read()
    declared = set(re.findall(r"\bint (tsb_[a-z0-9_]+)\s*\(", hdr)) - {"tsb_version"}
    assert declared == set(_lib._SIGS.keys())


def test_version_and_error_plumbing(lib):
    assert lib.tsb_version() >= 100
    rc = lib.tsb_ohem_begin(None, None)
    assert rc == -1  # TSB_ERR_ARG
    assert b"null state" in lib.tsb_last_error()


def test_argument_validation_without_gpu(lib):
    from torchseg_b200._lib import ConvShape
    # inconsistent P/Q must be rejected before any CUDA call
    shp = ConvShape(1, 8, 8, 64, 64, 3, 3, 1, 1, 1, 7, 7)
    buf = ctypes.create_string_buffer(64)
    rc = lib.tsb_conv2d_fprop(ctypes.byref(shp), ctypes.addressof(buf), 64, ctypes.addressof(buf), None,
                              ctypes.addressof(buf), 1, 64, None, None, None, 0, None)
    assert rc == -1 and b"inconsistent" in lib.tsb_last_error()
    shp = ConvShape(1, 8, 8, 48, 64, 3, 3, 1, 1, 1, 8, 8)   # C not a multiple of 64
    rc = lib.tsb_conv2d_fprop(ctypes.byref(shp), ctypes.addressof(buf), 48, ctypes.addressof(buf), None,
                              ctypes.addressof(buf), 1, 64, None, None, None, 0, None)
    assert rc == -1 and b"multiple of 64" in lib.tsb_last_error()


def test_product_path_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from torchseg_b200.seg_opr.seg_oprs import ConvBnRelu
    m = ConvBnRelu(64, 64, 3, 1, 1)
    with pytest.raises(Exception):
        m(torch.randn(1, 64, 8, 8))


def test_missing_library_raises(monkeypatch, tmp_path):
    from torchseg_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU/PyTorch fallback"):
        _lib.lib()


def test_product_package_never_imports_oracle():
    """DESIGN.md §1 'No fallback': nothing under torchseg_b200/ (nor bench.py's product arm helpers) may import, call or
    load anything under oracle/ — the oracle is test infrastructure only"""
    pat = re.compile(r"^\s*(from\s+oracle\b|import\s+oracle\b|from\s+\.+oracle\b)|libtsb_oracle|oracle[/\\.]_ref", re.M)
    bad = []
    pkg = os.path.join(ROOT, "torchseg_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                if pat.search(src):
                    bad.append(os.path.relpath(os.path.join(dirpath, f), ROOT))
    assert not bad, "product files reference the oracle: %s" % bad
    hdr = open(os.path.join(ROOT, "include", "tsb.h")).read()
    assert "oracle" not in hdr.lower()
