"""ctypes binding of libtsb.so — the C-ABI CUDA library (include/tsb.h).

The product path has NO fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_uint, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtsb.so")

F32, BF16 = 0, 1
OHEM_STATE_WORDS = 8192
OHEM_ST_NUM_VALID, OHEM_ST_COUNT_LE, OHEM_ST_ACTIVE, OHEM_ST_THRESH = 4096, 4097, 4098, 4099
OHEM_ST_KEPT, OHEM_ST_LOSS, OHEM_ST_INVDEN = 4100, 4101, 4102


class ConvShape(ctypes.Structure):
    """mirror of tsb_conv_shape"""
    _fields_ = [(n, c_int) for n in ("N", "H", "W", "C", "K", "R", "S", "stride", "pad", "dil", "P", "Q")]


P = c_void_p
I = c_int
L = c_longlong
F = c_float
D = c_double

# name -> argtypes (the trailing stream argument is included)
_SIGS = {
    "tsb_ohem_begin": [P, P],
    "tsb_ohem_ptarget": [P, I, L, L, L, L, P, I, I, I, I, I, F, P, P, P, P],
    "tsb_ohem_ptarget_up": [P, I, I, I, P, I, I, I, I, I, F, P, P, P, P],
    "tsb_ohem_select": [P, L, L, F, P, P],
    "tsb_ohem_loss": [P, P, P, L, I, P, P, P, P],
    "tsb_ohem_grad": [P, I, L, L, L, L, P, P, I, I, I, I, I, P, P, P, P, P],
    "tsb_ohem_grad_up": [P, I, I, I, P, P, I, I, I, I, I, P, P, P, P, P],
    "tsb_bilinear_fwd": [P, I, I, P, I, I, I, I, I, I, I, I, P],
    "tsb_bilinear_bwd": [P, I, I, P, I, I, I, I, I, I, I, I, I, P],
    "tsb_bilinear_fwd_nhwc_to_nchw": [P, I, I, P, I, I, I, I, I, I, P],
    "tsb_adaptive_avgpool_fwd": [P, I, I, I, I, I, I, P, P, L, P],
    "tsb_adaptive_avgpool_bwd": [P, I, I, I, I, I, P, I, I, P],
    "tsb_maxpool3x3s2_fwd": [P, I, P, I, P, I, I, I, I, P],
    "tsb_maxpool3x3s2_bwd": [P, P, I, P, I, I, I, I, I, P],
    "tsb_bn_stats": [P, I, L, I, P, P, P, L, P],
    "tsb_bn_finalize": [P, P, D, I, P, P, F, F, P, P, P, P, P, P, P],
    "tsb_bn_apply": [P, I, P, P, P, I, I, P, I, L, I, P],
    "tsb_bn_bwd_reduce": [P, I, P, I, P, I, P, P, I, L, I, P, P, P, P, P, L, P],
    "tsb_bn_bwd_apply": [P, I, P, I, P, I, P, P, P, P, P, D, I, P, I, P, I, L, I, P, P, P, P, P],
    "tsb_bn_bwd_apply_add": [P, I, P, I, P, I, P, P, P, P, P, D, I, P, I, P, I, L, I, P, P, P, P, P],
    "tsb_bn_apply_maxpool3x3s2": [P, I, P, P, P, I, P, I, I, I, I, P],
    "tsb_chan_scale_fwd": [P, I, P, F, P, I, P, I, I, I, I, P],
    "tsb_chan_scale_bwd": [P, I, P, I, P, F, P, I, P, I, I, I, P, L, P],
    "tsb_pack_image_s2d": [P, I, I, I, P, P],
    "tsb_pack_weight": [P, I, I, I, I, P, P, P],
    "tsb_pack_stem_weight": [P, I, I, P, P],
    "tsb_unpack_stem_wgrad": [P, I, I, P, P],
    "tsb_cast_scale": [P, I, I, P, I, I, L, I, P, P],
    "tsb_add": [P, I, P, I, P, I, L, I, P],
    "tsb_cast_pad": [P, I, I, I, P, I, I, L, P],
    "tsb_add_relu": [P, I, P, I, P, I, L, I, P],
    "tsb_softmax_rows_fwd": [P, I, I, P, I, L, I, I, P],
    "tsb_softmax_rows_bwd": [P, I, P, I, P, I, L, I, I, P],
    "tsb_transpose_pad": [P, I, I, P, I, I, I, I, P],
    "tsb_relu_bwd": [P, I, P, I, P, I, L, I, P],
    "tsb_conv2d_fprop": [P, P, I, P, P, P, I, I, P, P, P, L, P],
    "tsb_conv2d_fprop_fused": [P, P, I, P, P, P, I, I, P, I, I, P],
    "tsb_conv_stem_fprop_fused": [P, I, I, I, P, I, P, I, P, I, P],
    "tsb_conv1x1_bnrelu_fprop": [P, P, I, P, P, P, P, I, P, I, I, P, P, P, L, P],
    "tsb_conv1x1_bnrelu_wgrad": [P, P, I, P, P, P, I, P, P, L, P],
    "tsb_conv2d_dgrad": [P, P, I, P, P, I, I, P],
    "tsb_conv2d_wgrad": [P, P, I, P, I, P, P, L, P],
    "tsb_conv_transpose2d_fprop": [P, P, I, P, P, I, P, I, I, P, P, P, L, P],
    "tsb_conv_stem_fprop": [P, I, I, I, P, I, P, I, P, P, P, L, P],
    "tsb_conv_stem_wgrad": [P, I, I, I, P, I, I, P, P, L, P],
    "tsb_bias_grad": [P, I, L, I, P, P, L, P],
    "tsb_dwconv_fprop": [P, I, P, P, I, I, I, I, I, I, P],
    "tsb_dwconv_dgrad": [P, I, P, P, I, I, I, I, I, I, I, P],
    "tsb_dwconv_wgrad": [P, I, P, I, P, I, I, I, I, I, P, L, P],
    "tsb_dwconv2d_fprop": [P, I, P, P, I, I, I, I, I, I, I, P],
    "tsb_dwconv2d_dgrad": [P, I, P, P, I, I, I, I, I, I, I, I, P],
    "tsb_dwconv2d_wgrad": [P, I, P, I, P, I, I, I, I, I, I, P, L, P],
    "tsb_sgd_flat": [P, P, P, L, P, P, P, I, F, F, I, P],
    "tsb_sgd_flat_pack": [P, P, P, L, P, P, P, I, F, F, I, P, P],
    "tsb_pack_wt_multi": [P, P, P, P, I, I, P],
    "tsb_sigmoid_focal_fwd_bwd": [P, I, P, L, I, F, F, P, P, P],
    "tsb_ce_up_fwd": [P, I, I, I, P, I, I, I, I, I, P, P, P, P],
    "tsb_ce_up_bwd": [P, I, I, I, P, P, I, I, I, I, I, P, P, P, P],
    "tsb_train_preprocess": [P, I, I, I, I, P, F, I, P, P, P],
    "tsb_edge_labels": [P, I, I, I, I, P, c_size_t, P, P],
    "tsb_p2p_allreduce_sum": [P, I, P, I, I, c_uint, P, I, I, P, P, P],
    "tsb_eval_windows": [P, I, I, I, D, I, I, I, I, P, I, P, I, I, I, I, P, P],
    "tsb_eval_accumulate": [P, P, P, I, I, I, I, P, I, I, P],
    "tsb_eval_resize_add": [P, I, I, I, L, L, P, I, I, P, P],
    "tsb_encoding_fwd": [P, I, I, I, I, P, P, I, P, P, P, P, P, L, P],
    "tsb_encoding_bwd": [P, P, I, I, I, I, P, P, I, P, P, P, P, I, P, P, P, L, P],
    "tsb_chan_mean_fwd": [P, I, L, I, P, P],
    "tsb_chan_mean_bwd": [P, L, I, P, I, P],
    "tsb_se_loss_fwd_bwd": [P, I, L, P, I, I, P, P, P, I, P],
    "tsb_attention_fwd": [P, I, P, I, P, I, P, I, P, I, I, I, I, F, P],
    "tsb_attention_bwd": [P, I, P, I, P, I, P, I, P, I, P, P, P, I, P, I, P, I, I, I, I, I, I, F, P],
}
EXPORTS = sorted(list(_SIGS) + ["tsb_last_error", "tsb_version", "tsb_launch_count", "tsb_p2p_buffer_bytes", "tsb_edge_labels_workspace_bytes"])

_lib = None


def lib():
    """Load (once) and return the ctypes handle. Raises if the library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libtsb.so not found at %s — run `python -m torchseg_b200.build` (there is no CPU/PyTorch fallback)"
                % LIB_PATH)
        h = ctypes.CDLL(LIB_PATH)
        for name, sig in _SIGS.items():
            fn = getattr(h, name)
            fn.argtypes = sig
            fn.restype = c_int
        h.tsb_last_error.restype = c_char_p
        h.tsb_last_error.argtypes = []
        h.tsb_version.restype = c_int
        h.tsb_launch_count.restype = c_longlong
        h.tsb_p2p_buffer_bytes.restype = c_size_t
        h.tsb_p2p_buffer_bytes.argtypes = [I, I, I]
        h.tsb_edge_labels_workspace_bytes.restype = c_size_t
        h.tsb_edge_labels_workspace_bytes.argtypes = [I, I, I]
        _lib = h
    return _lib


def call(name, *args):
    """Invoke a C-ABI entry point; non-zero status → RuntimeError(tsb_last_error())."""
    h = lib()
    rc = getattr(h, name)(*args)
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (name, rc, h.tsb_last_error().decode()))


def launch_count():
    return int(lib().tsb_launch_count())


def ptr(t):
    """device pointer of a torch tensor (or None)"""
    return None if t is None else t.data_ptr()


def stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


DET_WS_FLOATS = 24 << 20   # 96 MB: every shape of the shipped networks (include/tsb.h)
_det_ws = {}


def det_ws():
    """(pointer, floats) of the reduction workspace of the current stream. include/tsb.h: a workspace serves one call at
    a time, so each stream gets its own (allocated once, through the caching allocator, so also inside a graph capture)."""
    import torch
    st = torch.cuda.current_stream()
    key = (st.device_index, st.cuda_stream)
    ws = _det_ws.get(key)
    if ws is None:
        ws = _det_ws[key] = torch.empty(DET_WS_FLOATS, dtype=torch.float32, device=st.device)
    return ws.data_ptr(), ws.numel()


def dt(t):
    import torch
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError("libtsb supports float32 / bfloat16 tensors, got %s" % t.dtype)
