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

    # The streaming NHWC kernels move 16-byte vectors (fp32 per-channel vectors as float4, the max-pool argmax as
    # 8 bytes) and address pixel p at p * cs: a misaligned pointer or a channel stride below C must come back as
    # TSB_ERR_ARG with a message, before any CUDA call, instead of launching a kernel that faults or writes into the
    # next pixel. A = 256-byte aligned host memory, M = 2 bytes past it (bf16-aligned only), M4 = 4 bytes past it.
    mem = (ctypes.c_uint8 * 4096)()
    A = (ctypes.addressof(mem) + 255) & ~255
    M, M4 = A + 2, A + 4
    C, npix, WS = 16, 4, 1 << 20
    cases = [
        ("tsb_bilinear_bwd", (A, 1, 8, A, 1, C, 1, C, 2, 2, 4, 4, 0, None), b">= C"),
        ("tsb_adaptive_avgpool_fwd", (A, 8, 1, C, 4, 4, 2, A, A, WS, None), b">= C"),
        ("tsb_adaptive_avgpool_bwd", (A, 1, C, 4, 4, 2, A, 8, 0, None), b">= C"),
        ("tsb_maxpool3x3s2_fwd", (M, C, A, C, A, 1, C, 4, 4, None), b"aligned"),
        ("tsb_maxpool3x3s2_fwd", (A, C, A, C, M4, 1, C, 4, 4, None), b"argmax 8B aligned"),
        ("tsb_maxpool3x3s2_fwd", (A, C, A, 8, A, 1, C, 4, 4, None), b">= C"),
        ("tsb_maxpool3x3s2_bwd", (A, M, C, A, C, 1, C, 4, 4, None), b"aligned"),
        ("tsb_maxpool3x3s2_bwd", (A, A, C, A, 8, 1, C, 4, 4, None), b">= C"),
        ("tsb_bn_stats", (A, 8, npix, C, A, A, A, WS, None), b">= C"),
        ("tsb_bn_stats", (A, C, npix, C, A, A, M4, WS, None), b"ws must be 16B aligned"),
        ("tsb_bn_apply", (A, C, M4, A, None, 0, 1, A, C, npix, C, None), b"scale and shift must be 16B aligned"),
        ("tsb_bn_apply", (A, C, A, A, A, 8, 1, A, C, npix, C, None), b">= C"),
        ("tsb_bn_bwd_reduce", (A, C, None, 0, A, C, M4, A, 0, npix, C, A, A, None, None, A, WS, None),
         b"per-channel vectors must be 16B aligned"),
        ("tsb_bn_bwd_reduce", (A, C, None, 0, A, C, A, A, 1, npix, C, A, A, A, M4, A, WS, None),
         b"per-channel vectors must be 16B aligned"),
        ("tsb_bn_bwd_reduce", (A, C, None, 0, A, 8, A, A, 0, npix, C, A, A, None, None, A, WS, None), b">= C"),
        ("tsb_bn_bwd_apply", (A, C, None, 0, A, C, A, A, M4, A, A, 4.0, 0, A, C, None, 0, npix, C, None, None, None,
                              None, None), b"per-channel vectors must be 16B aligned"),
        ("tsb_bn_bwd_apply", (A, C, None, 0, A, C, A, A, A, A, A, 4.0, 0, A, C, A, 8, npix, C, None, None, None, None,
                              None), b">= C"),
        ("tsb_chan_scale_fwd", (A, C, A, 0.0, None, 0, A, 8, 1, npix, C, None), b">= C"),
        ("tsb_chan_scale_bwd", (A, C, A, 8, A, 1.0, A, C, A, 1, npix, C, A, WS, None), b">= C"),
        ("tsb_cast_scale", (A, 1, C, A, 1, 8, npix, C, None, None), b">= C"),
        ("tsb_bias_grad", (A, 16, npix, 19, A, A, WS, None), b">= K"),
        # C = 0 (and N = 0) would reach the host-side geometry of the column reductions as a divisor
        ("tsb_bn_stats", (A, C, npix, 0, A, A, A, WS, None), b"multiples of 8"),
        ("tsb_bn_bwd_reduce", (A, C, None, 0, A, C, A, A, 0, npix, 0, A, A, None, None, A, WS, None), b"multiples of 8"),
        ("tsb_chan_scale_bwd", (A, C, A, C, A, 1.0, A, C, A, 1, npix, 0, A, WS, None), b"multiples of 8"),
        ("tsb_adaptive_avgpool_fwd", (A, C, 1, 0, 4, 4, 2, A, A, WS, None), b"multiples of 8"),
        ("tsb_adaptive_avgpool_fwd", (A, C, 0, C, 4, 4, 2, A, A, WS, None), b"N <= 0"),
        ("tsb_bilinear_fwd_nhwc_to_nchw", (A, 1, 8, A, 1, C, 2, 2, 4, 4, None), b"ics >= C"),
    ]
    for name in ("tsb_add", "tsb_add_relu", "tsb_relu_bwd"):
        cases += [(name, (A, C, M, C, A, C, npix, C, None), b"16B aligned"),
                  (name, (A, C, A, C, M, C, npix, C, None), b"16B aligned"),
                  (name, (A, C, A, C, A, 8, npix, C, None), b">= C")]
    for name, args, msg in cases:
        rc = getattr(lib, name)(*args)
        err = lib.tsb_last_error()
        assert rc == -1 and msg in err and name.encode() in err, (name, args, rc, err)


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
