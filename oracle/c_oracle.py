"""ctypes/numpy wrapper of oracle/tsb_oracle.c (bit-exact OHEM + bilinear restatement).

ORACLE — test infrastructure only. Cites: TorchSeg furnace/seg_opr/loss_opr.py:68-98.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libtsb_oracle.so")
_lib = None


def build(force=False):
    src = os.path.join(_HERE, "tsb_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B", "libtsb_oracle.so"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        h = ctypes.CDLL(_SO)
        h.tsb_oracle_exp_det.restype = ctypes.c_float
        h.tsb_oracle_exp_det.argtypes = [ctypes.c_float]
        h.tsb_oracle_ohem.restype = ctypes.c_double
        h.tsb_oracle_ohem.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 + [
            ctypes.c_float, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
            ctypes.c_void_p, ctypes.c_void_p]
        h.tsb_oracle_bilinear_nhwc_to_nchw.restype = None
        h.tsb_oracle_bilinear_nhwc_to_nchw.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 7 + [ctypes.c_void_p]
        _lib = h
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def exp_det(x):
    return float(lib().tsb_oracle_exp_det(ctypes.c_float(x)))


def ohem(logits, labels, ignore_label, thresh, min_kept, class_weight=None, want_grad=False):
    """logits: float32 [N,C,H,W]; labels: int64 [N,H,W]. Returns dict(loss,p,kept,T,active[,dlogits])."""
    logits = np.ascontiguousarray(logits, dtype=np.float32)
    labels = np.ascontiguousarray(labels, dtype=np.int64)
    N, C, H, W = logits.shape
    n = N * H * W
    p = np.empty(n, np.float32)
    kept = np.empty(n, np.uint8)
    T = ctypes.c_float(0)
    active = ctypes.c_int(0)
    cw = None if class_weight is None else np.ascontiguousarray(class_weight, dtype=np.float32)
    dl = np.empty_like(logits) if want_grad else None
    loss = lib().tsb_oracle_ohem(_p(logits), _p(labels), N, C, H, W, int(ignore_label), float(thresh), int(min_kept),
                                 _p(cw), _p(p), _p(kept), ctypes.addressof(T), ctypes.addressof(active), _p(dl))
    out = dict(loss=float(loss), p=p, kept=kept.astype(bool), T=float(T.value), active=bool(active.value))
    if want_grad:
        out["dlogits"] = dl
    return out


def bilinear_nhwc_to_nchw(lo, C, H, W):
    """lo: float32 [N,h,w,cs] → float32 [N,C,H,W] (align_corners=True, pinned op order)."""
    lo = np.ascontiguousarray(lo, dtype=np.float32)
    N, h, w, cs = lo.shape
    out = np.empty((N, C, H, W), np.float32)
    lib().tsb_oracle_bilinear_nhwc_to_nchw(_p(lo), cs, N, C, h, w, H, W, _p(out))
    return out
