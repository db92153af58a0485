"""torch.autograd.Function wrappers around the libtsb C ABI (include/tsb.h).

PyTorch drives only the graph, the memory and the streams; every op below runs a hand-written sm_90a
kernel. Activations are bf16 tensors of LOGICAL shape [N,C,H,W] stored NHWC (`nhwc_empty`), possibly a
channel slice of a wider buffer (channel stride `cs`). There is no CPU / ATen fallback: without a GPU or
without libtsb.so these functions raise.
"""
import torch

from . import _lib
from ._lib import BF16, F32, ConvShape, call, det_ws, ptr, stream

import ctypes
import weakref

_BF = torch.bfloat16


# --------------------------------------------------------------------------------------------------
# tensor helpers
# --------------------------------------------------------------------------------------------------
def nhwc_empty(N, C, H, W, dtype=_BF, device="cuda", cs=None):
    """logical [N,C,H,W] view of a fresh NHWC buffer (channel stride cs >= C)"""
    cs = C if cs is None else cs
    buf = torch.empty((N, H, W, cs), dtype=dtype, device=device)
    return buf[..., :C].permute(0, 3, 1, 2)


def nhwc_zeros(N, C, H, W, dtype=_BF, device="cuda", cs=None):
    cs = C if cs is None else cs
    buf = torch.zeros((N, H, W, cs), dtype=dtype, device=device)
    return buf[..., :C].permute(0, 3, 1, 2)


def cs_of(t):
    """channel stride (elements between consecutive pixels) of an NHWC-backed logical NCHW tensor"""
    assert t.dim() == 4, "expected a 4-D tensor"
    N, C, H, W = t.shape
    s = t.stride()
    if C > 1 and s[1] != 1:
        raise ValueError("tensor is not NHWC-backed (channel stride %d); use to_nhwc()" % s[1])
    if W > 1:
        cs = s[3]
    elif H > 1:
        cs = s[2]
    elif N > 1:
        cs = s[0]
    else:
        cs = C
    if (W > 1 and H > 1 and s[2] != W * cs) or (H * W > 1 and N > 1 and s[0] != H * W * cs) or cs < C:
        raise ValueError("tensor is not a dense NHWC buffer: shape %s strides %s" % (tuple(t.shape), s))
    return cs


def to_nhwc(t, dtype=_BF):
    """any [N,C,H,W] tensor → NHWC-backed logical NCHW tensor of `dtype` (ATen copy; boundary only)"""
    N, C, H, W = t.shape
    out = nhwc_empty(N, C, H, W, dtype=dtype, device=t.device)
    out.copy_(t)
    return out


def as_nhwc_bf16(t):
    """t itself when it is a bf16 tensor with unit channel stride (an incoming gradient usually is), else a dense bf16
    NHWC copy"""
    return t if t.dtype == _BF and t.stride(1) == 1 else to_nhwc(t)


def _krsc_ptr(w):
    """pointer to a dense [K,R,S,C] fp32 buffer for conv weight w ([K,C,R,S] logical)"""
    wp = w.permute(0, 2, 3, 1)
    if not wp.is_contiguous():
        raise ValueError("conv weight must be channels_last (KRSC); call torchseg_b200.prepare_model(model)")
    return wp


def conv_out_size(H, k, stride, pad, dil):
    return (H + 2 * pad - dil * (k - 1) - 1) // stride + 1


def make_shape(N, H, W, C, K, R, stride, pad, dil):
    P = conv_out_size(H, R, stride, pad, dil)
    Q = conv_out_size(W, R, stride, pad, dil)
    return ConvShape(N, H, W, C, K, R, R, stride, pad, dil, P, Q)


def deconv_out_size(H, k, stride, pad, dil, out_pad):
    return (H - 1) * stride - 2 * pad + dil * (k - 1) + out_pad + 1


def make_deconv_shape(N, H, W, Ci, Co, k, stride, pad, dil, out_pad):
    """the ADJOINT conv of ConvTranspose2d(Ci, Co, k, stride, pad, out_pad, dil) on an H x W input (include/tsb.h): an
    ordinary conv from Ho x Wo x Co to H x W x Ci with the deconv weight as its [K = Ci][C = Co][R][S] weight"""
    Ho = deconv_out_size(H, k, stride, pad, dil, out_pad)
    Wo = deconv_out_size(W, k, stride, pad, dil, out_pad)
    return ConvShape(N, Ho, Wo, Co, Ci, k, k, stride, pad, dil, H, W)


# --------------------------------------------------------------------------------------------------
# bf16 weight packs, cached per optimiser step
# --------------------------------------------------------------------------------------------------
class _PackCache:
    """bf16 operand packs of conv weights that are not served by the flat mirror (optim.FlatPack): weights before the
    first fused optimiser step, torch.optim.* flows, padded / viewed weights, stems. At most ONE entry per
    (weight object, operand kind); an entry is overwritten when the weight's version changes and dropped when the
    weight is gone (DFN's per-forward padded temporaries), so the cache cannot grow with the step count."""

    def __init__(self):
        self.step = 0
        self.cache = {}
        self._sweep_at = 256

    def invalidate(self):
        self.step += 1
        self.cache.clear()
        zero_arena.reset()

    def _sweep(self):
        dead = [k for k, v in self.cache.items() if v[2]() is None]
        for k in dead:
            del self.cache[k]
        self._sweep_at = max(256, 2 * len(self.cache))

    def get(self, w, want_t, pad_k=None, stem=False):
        fp = getattr(w, "_tsb_pack", None)
        if fp is not None and not stem and pad_k is None:
            hit = fp[0].lookup(w, fp[1], want_t)   # bf16 mirror of the flat parameter buffer (optim.FlatPack)
            if hit is not None:
                return hit
        key = (id(w), pad_k, stem)
        ver = (w.data_ptr(), w._version)
        hit = self.cache.get(key)
        if hit is not None and hit[2]() is w and hit[3] == ver and (hit[1] is not None or not want_t or stem):
            return hit[0], hit[1]
        K, C, R, S = w.shape
        if stem:
            wp = torch.empty((K, 4, 4, 16), dtype=_BF, device=w.device)
            call("tsb_pack_stem_weight", ptr(_krsc_ptr(w)), K, R, ptr(wp), stream())
            out = (wp, None, weakref.ref(w), ver)
        else:
            src = _krsc_ptr(w)
            if pad_k is not None and pad_k != K:  # classifier: pad K (19) up to 64 rows of zeros
                padded = torch.zeros((pad_k, R, S, C), dtype=torch.float32, device=w.device)
                padded[:K].copy_(src)
                src, K = padded, pad_k
            wb = torch.empty((K, R, S, C), dtype=_BF, device=w.device)
            wt = torch.empty((C, R, S, K), dtype=_BF, device=w.device) if want_t else None
            call("tsb_pack_weight", ptr(src), K, R, S, C, ptr(wb), ptr(wt), stream())
            out = (wb, wt, weakref.ref(w), ver)
        self.cache[key] = out
        if len(self.cache) > self._sweep_at:
            self._sweep()
        return out[0], out[1]


pack_cache = _PackCache()


def _install_optimizer_hook():
    """torch.optim.* flows (INTEGRATION.md keeps them supported): every optimiser step changes the weights, so the
    per-tensor packs are dropped and the zero arena is recycled, exactly as the fused SGD does itself"""
    try:
        from torch.optim.optimizer import register_optimizer_step_post_hook
    except ImportError:  # pragma: no cover
        return

    def _post(opt, args, kwargs):
        pack_cache.invalidate()

    register_optimizer_step_post_hook(_post)


class _ZeroArena(object):
    """Small fp32 scratch buffers that must start at zero (BN statistics, reduction accumulators): carved out of ONE
    buffer that is cleared with a single memset per step (`reset`, called from zero_grad / optimizer.step) instead of
    one fill kernel per buffer. Falls back to torch.zeros when exhausted or never reset."""

    def __init__(self, nfloats=1 << 20):
        self.n = nfloats
        self.buf = None
        self.off = 0

    def reset(self):
        if self.buf is not None:
            self.buf.zero_()
        self.off = 0

    def take(self, shape, device):
        n = 1
        for d in shape:
            n *= int(d)
        n4 = (n + 3) // 4 * 4
        if self.buf is None or self.buf.device != device:
            self.buf = torch.zeros(self.n, dtype=torch.float32, device=device)
            self.off = 0
        if self.off + n4 > self.n:
            return torch.zeros(shape, dtype=torch.float32, device=device)
        out = self.buf[self.off:self.off + n].view(shape)
        self.off += n4
        return out


zero_arena = _ZeroArena()
_install_optimizer_hook()

# set by the DDP shim: called with a parameter whose gradient has just been written DIRECTLY into its flat .grad view
grad_ready_hook = None


def _direct_grad(p):
    """True when this parameter's .grad is a persistent flat-buffer view the kernels may accumulate into directly"""
    return getattr(p, "_tsb_direct", False) and p.grad is not None


class _ParamGrads(object):
    """The parameter gradients of one op (None entries: an absent bias). `direct` when every parameter's .grad is a
    persistent flat-buffer view: the kernels then accumulate into the live .grad, autograd receives None and the DDP
    hook (`grad_ready_hook`) is told in `result`. Otherwise each gradient is a fresh tensor that goes back to autograd.
    A buffer handed to a kernel is therefore either the live accumulating .grad or zeros, because the wgrad, bias-grad
    and encoding kernels add into it (a wgrad with one split adds in place)."""

    def __init__(self, *params):
        self.params = params
        self.direct = all(_direct_grad(p) for p in params if p is not None)
        self.grads = {}

    def buffer(self, p, krsc=False):
        """the tensor the kernel accumulates p's gradient into; krsc: p is a conv weight, written as its dense KRSC
        storage"""
        if self.direct:
            return p.grad.permute(0, 2, 3, 1) if krsc else p.grad
        if krsc:
            self.grads[id(p)], g = _new_wgrad(p)
            return g
        g = self.grads[id(p)] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return g

    def set(self, p, g):
        """autograd receives g for p (not direct: a gradient computed outside `buffer`)"""
        self.grads[id(p)] = g

    def result(self):
        """what autograd receives, one entry per parameter"""
        if self.direct and grad_ready_hook is not None:
            for p in self.params:
                if p is not None:
                    grad_ready_hook(p)
        return tuple(self.grads.get(id(p)) for p in self.params)

# process group for SyncBN statistics (set by apex_shim.parallel.SyncBatchNorm / DistributedDataParallel)
_sync = {"group": None, "world": 1, "p2p": None, "p2p_tried": False}


def set_sync_group(group, world):
    _sync["group"], _sync["world"] = group, world
    if world <= 1:
        _sync["p2p"], _sync["p2p_tried"] = None, False


class _PeerExchange(object):
    """SyncBN statistics exchange over NVLink peer memory (csrc/p2p.cu, tsb_p2p_allreduce_sum): one symmetric buffer per
    rank (torch symmetric memory supplies the allocation and the peer-mapped addresses — plumbing only), ONE small
    kernel per exchange instead of an NCCL all-reduce. All ranks must issue the same exchanges in the same order."""
    NSLOTS = 64
    SLOT_FLOATS = 4096      # 2 x 2048 channels (ResNet-101 layer4)

    def __init__(self, group, world, device):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        pg = group if group is not None else dist.group.WORLD
        self.world = world
        self.rank = dist.get_rank(pg)
        nbytes = int(_lib.lib().tsb_p2p_buffer_bytes(world, self.NSLOTS, self.SLOT_FLOATS))
        assert nbytes > 0
        self.buf = symm.empty(nbytes // 4, dtype=torch.float32, device=device)
        self.buf.zero_()
        self.hdl = symm.rendezvous(self.buf, pg.group_name)
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        assert len(ptrs) == world and all(ptrs)
        self.peers = (ctypes.c_ulonglong * world)(*ptrs)
        # the exchange counter lives on the device (pre-incremented by every exchange kernel): identical on all ranks
        # because all ranks issue the same exchanges, and replayable inside a captured CUDA graph
        self.seq_dev = torch.zeros(1, dtype=torch.int32, device=device)

    def allreduce(self, buf, acc_hi=None, acc_lo=None):
        call("tsb_p2p_allreduce_sum", ptr(buf), buf.numel(), ctypes.cast(self.peers, ctypes.c_void_p), self.rank, self.world,
             0, ptr(self.seq_dev), self.NSLOTS, self.SLOT_FLOATS, ptr(acc_hi), ptr(acc_lo), stream())


def _peer_exchange(device):
    """the NVLink exchange object, or None (single process, CPU / gloo, TSB_SYNCBN_P2P=0, no symmetric memory).
    Collective: every rank of the SyncBN group reaches this at the same point (its first exchange), and the ranks AGREE on
    the outcome — a rank that could not set the exchange up while its peers spin in the kernel would deadlock the job."""
    if _sync["world"] <= 1 or device.type != "cuda":
        return None
    if not _sync["p2p_tried"]:
        _sync["p2p_tried"] = True
        import os
        import sys
        import torch.distributed as dist
        x, why = None, "disabled by TSB_SYNCBN_P2P=0"
        if os.environ.get("TSB_SYNCBN_P2P", "1") != "0":
            try:
                x = _PeerExchange(_sync["group"], _sync["world"], device)
            except Exception as e:  # noqa: BLE001 — no NVLink P2P / symmetric memory on this box: keep NCCL
                x, why = None, "%s: %s" % (type(e).__name__, str(e).split("\n")[0][:200])
        ok = torch.tensor([1.0 if x is not None else 0.0], device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=_sync["group"])
        if float(ok.item()) < 1.0:
            if x is not None:
                why = "another rank could not set it up"
            x = None
            if os.environ.get("TSB_SYNCBN_P2P", "1") != "0":
                sys.stderr.write("torchseg_b200: NVLink SyncBN exchange unavailable (%s); using NCCL all-reduce\n" % why)
        else:
            torch.cuda.synchronize(device)
            dist.barrier(group=_sync["group"])   # every rank's buffer is zeroed before anybody's first exchange writes into it
        _sync["p2p"] = x
    return _sync["p2p"]


def _allreduce_stats(buf, acc_hi=None, acc_lo=None):
    """sum the packed per-channel statistics over the SyncBN group, in place. acc_hi / acc_lo (backward): the LOCAL
    halves are first accumulated into the parameter gradients (dgamma += buf[1], dbeta += buf[0]). Returns True when
    that accumulation was done here."""
    if _sync["world"] <= 1:
        return False
    x = _peer_exchange(buf.device)
    n = buf.numel()
    if x is not None and n % 4 == 0 and n <= x.SLOT_FLOATS and buf.is_contiguous():
        x.allreduce(buf, acc_hi, acc_lo)
        return acc_hi is not None
    import torch.distributed as dist
    if acc_hi is not None:
        acc_hi.add_(buf[1])   # local sums must be taken before the all-reduce
        acc_lo.add_(buf[0])
    dist.all_reduce(buf, group=_sync["group"])
    return acc_hi is not None


# --------------------------------------------------------------------------------------------------
# optional CUDA-event bracketing of the conv launches (bench.py roofline: algorithmic FLOPs / kernel time)
# --------------------------------------------------------------------------------------------------
class _ConvProf(object):
    def __init__(self):
        self.on = False
        self.recs = []

    def enable(self):
        self.on, self.recs = True, []

    def disable(self):
        self.on = False

    def launch(self, flops, name, *args):
        """call(name, *args), bracketed by CUDA events while enabled"""
        if not self.on:
            call(name, *args)
            return
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
        call(name, *args)
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.recs.append((e0, e1, flops))

    def collect(self):
        torch.cuda.synchronize()
        ms = sum(a.elapsed_time(b) for a, b, _ in self.recs)
        return dict(ms=ms, flops=float(sum(f for _, _, f in self.recs)), launches=len(self.recs))


conv_prof = _ConvProf()


def _conv_flops(shp):
    return 2.0 * shp.N * shp.P * shp.Q * shp.K * shp.C * shp.R * shp.S


# --------------------------------------------------------------------------------------------------
# low-level conv calls
# --------------------------------------------------------------------------------------------------
def conv_fprop(x, wb, K, R, stride, pad, dil, bias=None, out_dtype=_BF, out=None, ocs=None, stats=None):
    N, C, H, W = x.shape
    shp = make_shape(N, H, W, C, K, R, stride, pad, dil)
    if out is None:
        ocs_alloc = ocs if ocs is not None else (K + 7) // 8 * 8
        out = nhwc_empty(N, K, shp.P, shp.Q, dtype=out_dtype, device=x.device, cs=ocs_alloc)
    s1 = s2 = None
    if stats is not None:
        s1, s2 = stats[0], stats[1]
    conv_prof.launch(_conv_flops(shp), "tsb_conv2d_fprop", ctypes.byref(shp), ptr(x), cs_of(x), ptr(wb), ptr(bias), ptr(out),
                     _lib.dt(out), cs_of(out), ptr(s1), ptr(s2), *det_ws(), stream())
    return out


def conv_transpose_fprop(x, wt, Co, R, stride, pad, dil, out_pad, bias=None, relu=False, out_dtype=_BF, out=None,
                        stats=None):
    """y = relu?(conv_transpose(x, W) + bias) on the dgrad-form launches (tsb_conv_transpose2d_fprop); wt is the flipped
    [Co][R][S][Ci] pack of the deconv weight W [Ci][Co][R][S]; optional BN statistics of the rounded output"""
    N, Ci, H, W = x.shape
    shp = make_deconv_shape(N, H, W, Ci, Co, R, stride, pad, dil, out_pad)
    if out is None:
        out = nhwc_empty(N, Co, shp.H, shp.W, dtype=out_dtype, device=x.device)
    s1, s2 = (None, None) if stats is None else (stats[0], stats[1])
    conv_prof.launch(_conv_flops(shp), "tsb_conv_transpose2d_fprop", ctypes.byref(shp), ptr(x), cs_of(x), ptr(wt), ptr(bias),
                     int(relu), ptr(out), _lib.dt(out), cs_of(out), ptr(s1), ptr(s2), *det_ws(), stream())
    return out


def conv_fprop_fused(x, wb, K, R, stride, pad, dil, bias, res=None, relu=False):
    """inference conv with the BatchNorm folded into (wb, bias): y = relu?(conv(x) + bias (+ res)) in ONE kernel
    (tsb_conv2d_fprop_fused) — no raw tensor, no separate normalisation pass"""
    N, C, H, W = x.shape
    shp = make_shape(N, H, W, C, K, R, stride, pad, dil)
    out = nhwc_empty(N, K, shp.P, shp.Q, device=x.device, cs=(K + 7) // 8 * 8)
    if res is not None and (res.dtype != _BF or res.stride(1) != 1 or cs_of(res) != cs_of(out)):
        res = to_nhwc(res) if cs_of(out) == K else None
        assert res is not None, "residual layout must match the output"
    conv_prof.launch(_conv_flops(shp), "tsb_conv2d_fprop_fused", ctypes.byref(shp), ptr(x), cs_of(x), ptr(wb), ptr(bias),
                     ptr(res), cs_of(res) if res is not None else 0, int(relu), ptr(out), BF16, cs_of(out), stream())
    return out


def conv_stem_fprop_fused(xs2d, wp, K, bias, relu=True):
    """the 7x7/2 (or 3x3/2) C_in = 3 stem on the space-to-depth image with folded BN + ReLU in the epilogue"""
    N, _, H2, WP = xs2d.shape
    H, W = H2 * 2, (WP - 4) * 2
    out = nhwc_empty(N, K, H2, WP - 4, device=xs2d.device)
    conv_prof.launch(2.0 * N * H2 * (WP - 4) * K * 147, "tsb_conv_stem_fprop_fused", ptr(xs2d), N, H, W, ptr(wp), K,
                     ptr(bias), int(relu), ptr(out), K, stream())
    return out


class _FoldCache(object):
    """eval-mode BatchNorm folded into the conv operands: w' = w · γ/√(σ²+ε) (bf16 KRSC pack), b' = β − μ·γ/√(σ²+ε).
    One entry per (conv weight, bn) pair, rebuilt when any of the five tensors changes (their versions, plus
    pack_cache.step because the fused SGD / a graph replay updates parameters without bumping versions)."""

    def __init__(self):
        self.cache = {}

    def get(self, w, bn, stem, transposed=False):
        """transposed: w is a ConvTranspose2d weight [Ci][Co][R][S]; its output channels are the C axis of the KRSC view,
        so the scale runs along C and the returned pack is the flipped [Co][R][S][Ci] operand of the transposed fprop"""
        key = (id(w), id(bn))
        ver = (w.data_ptr(), w._version, bn.weight._version, bn.bias._version, bn.running_mean._version,
               bn.running_var._version, pack_cache.step, bool(stem), bool(transposed))
        hit = self.cache.get(key)
        if hit is not None and hit[0] == ver and hit[3]() is w:
            return hit[1], hit[2]
        with torch.no_grad():
            scale = (bn.weight.float() / torch.sqrt(bn.running_var.float() + bn.eps))
            bias = (bn.bias.float() - bn.running_mean.float() * scale).contiguous()
            if transposed:
                wk = (_krsc_ptr(w).float() * scale[None, None, None, :]).contiguous()
            else:
                wk = (_krsc_ptr(w).float() * scale[:, None, None, None]).contiguous()
            K, R, S, C = wk.shape
            if transposed:
                wb = torch.empty((C, R, S, K), dtype=_BF, device=w.device)
                call("tsb_pack_weight", ptr(wk), K, R, S, C, None, ptr(wb), stream())
            elif stem:
                wb = torch.empty((K, 4, 4, 16), dtype=_BF, device=w.device)
                call("tsb_pack_stem_weight", ptr(wk), K, R, ptr(wb), stream())
            else:
                wb = torch.empty((K, R, S, C), dtype=_BF, device=w.device)
                call("tsb_pack_weight", ptr(wk), K, R, S, C, ptr(wb), None, stream())
        self.cache[key] = (ver, wb, bias, weakref.ref(w))
        if len(self.cache) > 1024:
            for k in [k for k, v in self.cache.items() if v[3]() is None]:
                del self.cache[k]
        return wb, bias


fold_cache = _FoldCache()


def conv_dgrad(dy, wt, xshape, K, R, stride, pad, dil, out=None, accumulate=False):
    N, C, H, W = xshape
    shp = make_shape(N, H, W, C, K, R, stride, pad, dil)
    if out is None:
        out = nhwc_empty(N, C, H, W, device=dy.device)
    try:
        conv_prof.launch(_conv_flops(shp), "tsb_conv2d_dgrad", ctypes.byref(shp), ptr(dy), cs_of(dy), ptr(wt), ptr(out),
                         cs_of(out), int(accumulate), stream())
    except RuntimeError as e:
        raise RuntimeError("%s [dgrad shape N=%d H=%d W=%d C=%d K=%d R=%d stride=%d pad=%d dil=%d]" % (
            e, N, H, W, C, K, R, stride, pad, dil)) from None
    return out


def conv_wgrad(x, dy, K, R, stride, pad, dil, dw_krsc):
    N, C, H, W = x.shape
    shp = make_shape(N, H, W, C, K, R, stride, pad, dil)
    conv_prof.launch(_conv_flops(shp), "tsb_conv2d_wgrad", ctypes.byref(shp), ptr(x), cs_of(x), ptr(dy), cs_of(dy),
                     ptr(dw_krsc), *det_ws(), stream())


def _new_wgrad(w):
    """zeroed gradient with the parameter's (KRSC) strides: returns (logical view, dense KRSC tensor)"""
    K, C, R, S = w.shape
    g = torch.zeros((K, R, S, C), dtype=torch.float32, device=w.device)
    return g.permute(0, 3, 1, 2), g


# --------------------------------------------------------------------------------------------------
# Conv + (Sync)BatchNorm(train) + residual + ReLU  — ConvBnRelu / BasicBlock tail
# --------------------------------------------------------------------------------------------------
class GradShare(object):
    """One gradient buffer for a tensor consumed `n` times inside a block (x → conv1, x → downsample, x → residual).

    Each consumer's backward calls contribute(g): the first stores its gradient and returns None to autograd; later ones
    have already ACCUMULATED into the stored buffer (conv_dgrad(out=stash, accumulate=True)) and the last returns it. The
    sum therefore reaches autograd as a single tensor and the element-wise bf16 adds (one read-read-write pass over
    the activation per fork) disappear. Consumers outside the block are untouched: autograd adds their gradient to the
    returned tensor as usual."""

    def __init__(self, n):
        self.n = n
        self.left = n
        self.stash = None

    def contribute(self, g, accumulated=False):
        """g: this consumer's input gradient; accumulated=True means g IS the stash (the consumer's dgrad epilogue added
        into it in place). Returns what the consumer hands to autograd: None until the last contributor."""
        self.left -= 1
        if self.stash is None:
            self.stash = g
        elif not accumulated:
            self.stash = self.stash + g   # a contributor that cannot accumulate in place arrived late (not the case for
            #                               the block orders used here: the shortcut's backward always runs first)
        if self.left > 0:
            return None
        out, self.stash, self.left = self.stash, None, self.n
        return out


def _dgrad_into(share, dgrad):
    """the input gradient of one consumer at a GradShare fork (share None: no fork). dgrad(out, accumulate) runs the
    consumer's dgrad into `out` (None: a fresh buffer it allocates) and returns that buffer: into the stash, adding,
    when an earlier consumer started it, else into a fresh buffer that starts it. Returns what autograd receives."""
    if share is not None and share.stash is not None:
        return share.contribute(dgrad(share.stash, True), accumulated=True)
    dx = dgrad(None, False)
    return dx if share is None else share.contribute(dx)


def _running_stats_written(running_mean, running_var):
    """tsb_bn_finalize updated the running statistics through raw pointers, which autograd's version counters do not
    see: bump them, so that what is keyed on those versions (the eval-mode fold cache) rebuilds from the new values. A
    version bump changes no tensor data; inside a graph capture it happens once, and the replays bump pack_cache.step."""
    torch.autograd.graph.increment_version((running_mean, running_var))


def _bn_finalize(aux, stats, count, gamma, beta, running_mean, running_var, eps, momentum, training):
    """scale / shift of a BatchNorm into aux = [mean; invstd; scale; shift] (a channel slice of a wider aux). Training:
    from the batch statistics stats = [Σ; Σ²] over `count` pixels (already summed over the SyncBN group), updating the
    running statistics; eval: from the running statistics."""
    if not training:
        # sum := mean*1, sumsq := var + mean^2, count 1, no running-statistics update
        stats = torch.stack([running_mean, running_var + running_mean * running_mean]).contiguous()
        count, momentum, running_mean, running_var = 1.0, 0.0, None, None
    call("tsb_bn_finalize", ptr(stats[0]), ptr(stats[1]), count, aux.shape[1], ptr(gamma), ptr(beta), eps, momentum,
         ptr(aux[0]), ptr(aux[1]), ptr(aux[2]), ptr(aux[3]), ptr(running_mean), ptr(running_var), stream())
    if training:
        _running_stats_written(running_mean, running_var)


def _bn_apply(raw, aux, residual, relu):
    """y = act(raw * scale + shift + residual) over the NHWC raw [N,K,P,Q] (possibly a channel slice), into a dense y"""
    N, K, P, Q = raw.shape
    y = nhwc_empty(N, K, P, Q, device=raw.device)
    call("tsb_bn_apply", ptr(raw), cs_of(raw), ptr(aux[2]), ptr(aux[3]), ptr(residual),
         cs_of(residual) if residual is not None else 0, int(relu), ptr(y), K, N * P * Q, K, stream())
    return y


def _bn_forward(raw, stats, count, gamma, beta, residual, running_mean, running_var, relu, eps, momentum, training):
    """the BatchNorm half of ConvBNActFn.forward: y = act(BN(raw) + residual) over the dense NHWC raw [N,K,P,Q]. Training
    normalises with the batch statistics stats = [Σ; Σ²] (summed over the SyncBN group here) and updates the running
    statistics; eval uses the running statistics. Returns (y, aux = [mean; invstd; scale; shift])."""
    aux = torch.empty((4, raw.shape[1]), dtype=torch.float32, device=raw.device)
    if training:
        _allreduce_stats(stats)
    _bn_finalize(aux, stats, count, gamma, beta, running_mean, running_var, eps, momentum, training)
    return _bn_apply(raw, aux, residual, relu), aux


def _bn_backward(dy, y, raw, aux, gamma, beta, count, relu, has_res, grads, draw=None, add=False):
    """the BatchNorm half of ConvBNActFn.backward: (draw, dres). raw / draw may be channel slices of wider NHWC buffers
    (draw None: a fresh dense one), aux the matching [4, K] slice. gamma / beta take their gradients through `grads`
    (_ParamGrads): accumulated into their flat .grad views when direct, else handed to autograd. add: draw is added to
    (tsb_bn_bwd_apply_add) instead of overwritten."""
    N, K, P, Q = raw.shape
    dev = raw.device
    npix = N * P * Q
    dy = as_nhwc_bf16(dy)
    red = zero_arena.take((2, K), dev)
    # ReLU mask: recomputed from raw*scale+shift when there is no residual (saves reading y in both passes)
    y_mask = ptr(y) if (relu and has_res) else None
    ycs = cs_of(y) if y_mask is not None else (K if draw is None else 0)   # unread without y_mask
    call("tsb_bn_bwd_reduce", ptr(dy), cs_of(dy), y_mask, ycs, ptr(raw), cs_of(raw), ptr(aux[0]), ptr(aux[1]), int(relu),
         npix, K, ptr(red[0]), ptr(red[1]), ptr(aux[2]), ptr(aux[3]), *det_ws(), stream())
    # dgamma = Σ dz·x̂, dbeta = Σ dz are LOCAL sums (the DDP all-reduce averages parameter grads);
    # the dx formula needs the GLOBAL sums under SyncBN.
    fold = grads.direct and _sync["world"] == 1   # single GPU: the accumulation is folded into tsb_bn_bwd_apply
    if grads.direct:
        # multi-GPU: the exchange kernel adds the LOCAL sums to gamma.grad / beta.grad before it reduces
        _allreduce_stats(red, None if fold else gamma.grad, None if fold else beta.grad)
    else:
        grads.set(gamma, red[1].clone())
        grads.set(beta, red[0].clone())
        _allreduce_stats(red)
    if draw is None:
        draw = nhwc_empty(N, K, P, Q, device=dev)
    dres = nhwc_empty(N, K, P, Q, device=dev) if has_res else None
    call("tsb_bn_bwd_apply_add" if add else "tsb_bn_bwd_apply", ptr(dy), cs_of(dy), y_mask, ycs, ptr(raw), cs_of(raw),
         ptr(aux[0]), ptr(aux[1]), ptr(gamma),
         ptr(red[0]), ptr(red[1]), count, int(relu), ptr(draw), cs_of(draw), ptr(dres), K if has_res else 0, npix, K,
         ptr(gamma.grad) if fold else None, ptr(beta.grad) if fold else None, ptr(aux[2]), ptr(aux[3]), stream())
    return draw, dres


class ConvBNActFn(torch.autograd.Function):
    """y = act(BN_train(conv(x, w)) + residual).

    Replaces ConvBnRelu.forward (TorchSeg furnace/seg_opr/seg_oprs.py:39-46) and the conv→bn→(+res)→relu
    groups of BasicBlock.forward (TorchSeg furnace/base_model/resnet.py:33-53). The conv epilogue emits
    the per-channel Σ/Σ² (BN statistics), tsb_bn_finalize turns them into scale/shift (and updates the
    running stats), tsb_bn_apply normalises (+residual, +ReLU) in one pass.
    """

    @staticmethod
    def forward(ctx, x, w, gamma, beta, residual, running_mean, running_var, stride, pad, dil, relu, eps, momentum,
                training, stem, in_share=None, res_share=None, out_pad=None):
        # out_pad is not None: w is a ConvTranspose2d weight [Ci][Co][R][S] (DeConvBnRelu, seg_oprs.py:49-73) and the
        # three conv calls are those of the adjoint conv (include/tsb.h): transposed fprop, fprop for dx, wgrad with x
        # and dy exchanged for dW
        transposed = out_pad is not None
        K = w.shape[1] if transposed else w.shape[0]
        R = w.shape[2]
        dev = x.device
        if stem:
            N, _, H2, WP = x.shape  # xs2d [N, 16, H/2, W/2+4]
            H, W = H2 * 2, (WP - 4) * 2
            P, Q = H2, WP - 4
        elif transposed:
            N, C, H, W = x.shape
            P, Q = deconv_out_size(H, R, stride, pad, dil, out_pad), deconv_out_size(W, R, stride, pad, dil, out_pad)
        else:
            N, C, H, W = x.shape
            P, Q = conv_out_size(H, R, stride, pad, dil), conv_out_size(W, R, stride, pad, dil)
        count = float(N * P * Q) * _sync["world"]
        stats = zero_arena.take((2, K), dev) if training else None
        raw = nhwc_empty(N, K, P, Q, device=dev)
        if stem:
            wp, _ = pack_cache.get(w, False, stem=True)
            conv_prof.launch(2.0 * N * P * Q * K * 147, "tsb_conv_stem_fprop", ptr(x), N, H, W, ptr(wp), K, ptr(raw), K,
                             ptr(stats[0]) if training else None, ptr(stats[1]) if training else None, *det_ws(), stream())
        elif transposed:
            _, wt = pack_cache.get(w, True)
            conv_transpose_fprop(x, wt, K, R, stride, pad, dil, out_pad, out=raw, stats=stats)
        else:
            wb, _ = pack_cache.get(w, False)
            conv_fprop(x, wb, K, R, stride, pad, dil, out=raw, stats=stats)
        y, aux = _bn_forward(raw, stats, count, gamma, beta, residual, running_mean, running_var, relu, eps, momentum,
                             training)
        ctx.save_for_backward(x, w, gamma, raw, y, aux)
        ctx.beta_ref = beta
        ctx.cfg = (stride, pad, dil, relu, stem, residual is not None, count, training, transposed)
        # gradient sharing at a fork (GradShare): in_share — this conv's input x has other consumers in the same block;
        # res_share — the residual IS that x. The contributors chain their input gradients through one buffer (dgrad
        # epilogue accumulate) instead of handing autograd several tensors to add.
        ctx.in_share = in_share
        ctx.res_share = res_share if residual is not None else None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, gamma, raw, y, aux = ctx.saved_tensors
        stride, pad, dil, relu, stem, has_res, count, training, transposed = ctx.cfg
        assert training, "backward through eval-mode BN is not supported"
        K = w.shape[1] if transposed else w.shape[0]
        R = w.shape[2]
        N, _, P, Q = raw.shape
        dev = dy.device
        beta = ctx.beta_ref
        grads = _ParamGrads(w, gamma, beta)
        draw, dres = _bn_backward(dy, y, raw, aux, gamma, beta, count, relu, has_res, grads)
        dw = grads.buffer(w, krsc=True)
        dx = None
        if stem:
            H, W = P * 2, Q * 2
            dwp = zero_arena.take((K, 4, 64), dev)
            conv_prof.launch(2.0 * N * P * Q * K * 147, "tsb_conv_stem_wgrad", ptr(x), N, H, W, ptr(draw), K, K, ptr(dwp),
                             *det_ws(), stream())
            call("tsb_unpack_stem_wgrad", ptr(dwp), K, R, ptr(dw), stream())
        elif transposed:
            Ci = w.shape[0]
            conv_wgrad(draw, x, Ci, R, stride, pad, dil, dw)
            if ctx.needs_input_grad[0]:
                wb, _ = pack_cache.get(w, False)
                dx = conv_fprop(draw, wb, Ci, R, stride, pad, dil)
        else:
            conv_wgrad(x, draw, K, R, stride, pad, dil, dw)
            if ctx.needs_input_grad[0]:
                _, wt = pack_cache.get(w, True)
                dx = _dgrad_into(ctx.in_share, lambda out, acc: conv_dgrad(draw, wt, x.shape, K, R, stride, pad, dil,
                                                                           out=out, accumulate=acc))
        if has_res and ctx.res_share is not None and ctx.needs_input_grad[4]:
            dres = ctx.res_share.contribute(dres)
        dw_view, dgamma, dbeta = grads.result()
        return dx, dw_view, dgamma, dbeta, dres, None, None, None, None, None, None, None, None, None, None, None, None, None


def conv1x1_bnrelu_fprop(x, aux, wb, K, bias=None, relu=False, stats=None):
    """y = relu?(conv1x1(x̂, wb) + bias) with x̂ = bf16(relu(x·aux[2] + aux[3])) normalised in the conv's shared memory
    (tsb_conv1x1_bnrelu_fprop): the pre-activation input of a DenseASPP block is never written. Optional BN statistics
    of the rounded output into stats = [Σ; Σ²]."""
    N, C, H, W = x.shape
    shp = make_shape(N, H, W, C, K, 1, 1, 0, 1)
    out = nhwc_empty(N, K, H, W, device=x.device)
    s1, s2 = (None, None) if stats is None else (stats[0], stats[1])
    conv_prof.launch(_conv_flops(shp), "tsb_conv1x1_bnrelu_fprop", ctypes.byref(shp), ptr(x), cs_of(x), ptr(aux[2]),
                     ptr(aux[3]), ptr(wb), ptr(bias), int(relu), ptr(out), BF16, cs_of(out), ptr(s1), ptr(s2), *det_ws(),
                     stream())
    return out


def conv1x1_bnrelu_wgrad(x, aux, dy, K, dw_krsc):
    """dW += Σ dy ⊗ x̂ with the prologue of conv1x1_bnrelu_fprop (tsb_conv1x1_bnrelu_wgrad)"""
    N, C, H, W = x.shape
    shp = make_shape(N, H, W, C, K, 1, 1, 0, 1)
    conv_prof.launch(_conv_flops(shp), "tsb_conv1x1_bnrelu_wgrad", ctypes.byref(shp), ptr(x), cs_of(x), ptr(aux[2]),
                     ptr(aux[3]), ptr(dy), cs_of(dy), ptr(dw_krsc), *det_ws(), stream())


def _slice_stats(stats, t):
    """per-channel Σ / Σ² of the NHWC slice t into stats = [Σ; Σ²] (zeroed, a column range of a wider buffer), summed
    over the SyncBN group"""
    N, C, H, W = t.shape
    call("tsb_bn_stats", ptr(t), cs_of(t), N * H * W, C, ptr(stats[0]), ptr(stats[1]), *det_ws(), stream())
    if _sync["world"] > 1:
        tmp = stats.contiguous()
        _allreduce_stats(tmp)
        stats.copy_(tmp)


class DenseAsppFn(torch.autograd.Function):
    """The densely connected atrous stack of DenseASPPModule in training: returns the concatenation
    [a_{n-1} | ... | a_1 | a_0 | x] (one NHWC buffer; block i writes its slice in place and reads the suffix after it).

    Forward, block i: pre_bn (i > 0) from the shared per-channel statistics of the buffer (one tsb_bn_stats per slice,
    taken once), the 1x1 `reduce` conv reading relu(pre_bn(suffix)) through the conv's input prologue with the
    BN-statistics epilogue (block 0: plain conv, its input is already post-ReLU), reduce's BatchNorm + ReLU, the dilated
    3x3 conv with bias into the slice, Dropout2d on the slice. No normalised copy of the suffix is written or saved.

    Backward walks the blocks from the last to the first over ONE bf16 gradient buffer of the concatenation (the
    incoming gradient, added to in place): a block's slice gradient is complete when its turn comes, because only
    later blocks read it. Block i > 0 hands its input gradient to the buffer's suffix through tsb_bn_bwd_apply_add
    (the pre_bn backward, mask recomputed from scale / shift); block 0 through the accumulating dgrad."""

    @staticmethod
    def forward(ctx, x, mod, p_drop, *params):
        blocks = mod.blocks
        N, Cx, H, W = x.shape
        dev = x.device
        nb = len(blocks)
        oc = blocks[0].conv.out_channels
        Ct = Cx + nb * oc
        npix = N * H * W
        count = float(npix) * _sync["world"]
        cat = nhwc_empty(N, Ct, H, W, device=dev)
        cat[:, nb * oc:].copy_(x)
        stats = zero_arena.take((2, Ct), dev)
        _slice_stats(stats[:, nb * oc:], cat[:, nb * oc:])
        saved, cfg = [], []
        for i, blk in enumerate(blocks):
            off = (nb - i) * oc
            xin = cat[:, off:]
            red, bn, conv = blk.reduce.conv, blk.reduce.bn, blk.conv
            mid = red.out_channels
            pre = None
            if i > 0:
                pb = blk.pre_bn
                pre = torch.empty((4, Ct - off), dtype=torch.float32, device=dev)
                _bn_finalize(pre, stats[:, off:], count, pb.weight, pb.bias, pb.running_mean, pb.running_var,
                             float(pb.eps), float(pb.momentum if pb.momentum is not None else 0.1), True)
            rs = zero_arena.take((2, mid), dev)
            wb, _ = pack_cache.get(red.weight, False)
            if pre is None:
                raw = conv_fprop(xin, wb, mid, 1, 1, 0, 1, stats=rs)
            else:
                raw = conv1x1_bnrelu_fprop(xin, pre, wb, mid, stats=rs)
            y, aux = _bn_forward(raw, rs, count, bn.weight, bn.bias, None, bn.running_mean, bn.running_var, True,
                                 float(bn.eps), float(bn.momentum if bn.momentum is not None else 0.1), True)
            d = conv.dilation[0]
            wb3, _ = pack_cache.get(conv.weight, False)
            sl = cat[:, off - oc:off]
            conv_fprop(y, wb3, oc, 3, 1, d, d, bias=conv.bias, out=sl)
            mask = None
            if p_drop > 0:
                mask = (torch.bernoulli(torch.full((N, oc, 1, 1), 1 - p_drop, device=dev)) / (1 - p_drop)).to(_BF)
                sl.mul_(mask)
            _slice_stats(stats[:, off - oc:off], sl)
            saved += [raw, y, aux, pre if pre is not None else aux, mask if mask is not None else aux]
            cfg.append((off, d, pre is not None, mask is not None))
        ctx.save_for_backward(cat, *saved)
        ctx.mod, ctx.cfg, ctx.count, ctx.oc = mod, cfg, count, oc
        ctx.nparams = len(params)
        return cat

    @staticmethod
    def backward(ctx, dcat):
        cat, *saved = ctx.saved_tensors
        mod, cfg, count, oc = ctx.mod, ctx.cfg, ctx.count, ctx.oc
        blocks = mod.blocks
        params = [p for blk in blocks for p in _dense_block_params(blk)]
        grads = _ParamGrads(*params)
        if not (dcat.dtype == _BF and dcat.stride(1) == 1 and cs_of(dcat) == cat.shape[1]):
            dcat = to_nhwc(dcat)
        N, _, H, W = cat.shape
        npix = N * H * W
        for i in reversed(range(len(blocks))):
            blk = blocks[i]
            raw, y, aux, pre, mask = saved[5 * i:5 * i + 5]
            off, d, has_pre, has_mask = cfg[i]
            xin = cat[:, off:]
            red, bn, conv = blk.reduce.conv, blk.reduce.bn, blk.conv
            mid = red.out_channels
            g = dcat[:, off - oc:off]
            if has_mask:
                g.mul_(mask)
            _bias_grad(grads, conv.bias, g, cs_of(g), npix, oc)
            conv_wgrad(y, g, oc, 3, 1, d, d, grads.buffer(conv.weight, krsc=True))
            _, wt3 = pack_cache.get(conv.weight, True)
            dy = conv_dgrad(g, wt3, y.shape, oc, 3, 1, d, d)
            draw, _ = _bn_backward(dy, y, raw, aux, bn.weight, bn.bias, count, True, False, grads)
            _, wt1 = pack_cache.get(red.weight, True)
            if not has_pre:
                conv_wgrad(xin, draw, mid, 1, 1, 0, 1, grads.buffer(red.weight, krsc=True))
                conv_dgrad(draw, wt1, xin.shape, mid, 1, 1, 0, 1, out=dcat[:, off:], accumulate=True)
            else:
                conv1x1_bnrelu_wgrad(xin, pre, draw, mid, grads.buffer(red.weight, krsc=True))
                dxh = conv_dgrad(draw, wt1, xin.shape, mid, 1, 1, 0, 1)
                pb = blk.pre_bn
                _bn_backward(dxh, None, xin, pre, pb.weight, pb.bias, count, True, False, grads, draw=dcat[:, off:],
                             add=True)
        dx = dcat[:, len(blocks) * oc:] if ctx.needs_input_grad[0] else None
        return (dx, None, None) + grads.result()


def _dense_block_params(blk):
    """the parameters of one DenseAsppBlock in DenseAsppFn's argument order"""
    pre = [blk.pre_bn.weight, blk.pre_bn.bias] if blk.pre_bn is not None else []
    return pre + [blk.reduce.conv.weight, blk.reduce.bn.weight, blk.reduce.bn.bias, blk.conv.weight, blk.conv.bias]


class StemPairFn(torch.autograd.Function):
    """The TWO 7x7/2 stems of BiSeNet (spatial_path.conv_7x7, bisenet network.py:118, and context_path.conv1,
    resnet.py:126) read the same image: one conv launch computes both (K = 64 + 64 output channels, N = 128 MMA
    tiles), one wgrad launch produces both weight gradients. Returns the spatial stem's output and the context stem's
    output after the context path's 3x3/2 max pool (resnet.py:132): that half is normalised, ReLU'd and pooled in one
    pass (tsb_bn_apply_maxpool3x3s2), so its full-resolution output is never stored."""

    @staticmethod
    def forward(ctx, xs, w1, g1, b1, rm1, rv1, w2, g2, b2, rm2, rv2, eps1, mom1, eps2, mom2):
        N, _, H2, WP = xs.shape
        H, W, P, Q = H2 * 2, (WP - 4) * 2, H2, WP - 4
        dev = xs.device
        K1, K2 = w1.shape[0], w2.shape[0]
        K = K1 + K2
        wp = torch.empty((K, 4, 4, 16), dtype=_BF, device=dev)
        call("tsb_pack_stem_weight", ptr(_krsc_ptr(w1)), K1, w1.shape[2], ptr(wp), stream())
        call("tsb_pack_stem_weight", ptr(_krsc_ptr(w2)), K2, w2.shape[2], ptr(wp[K1:]), stream())
        stats = zero_arena.take((2, K), dev)
        raw = nhwc_empty(N, K, P, Q, device=dev)
        # two N=64 launches into the channel halves of one buffer: this layer is bound by the epilogue's stores and the
        # 64-column epilogue (one chunk per warp, register running sums) is the faster one; the wgrad below is fused
        for off, Kh in ((0, K1), (K1, K2)):
            conv_prof.launch(2.0 * N * P * Q * Kh * 147, "tsb_conv_stem_fprop", ptr(xs), N, H, W, ptr(wp[off:]), Kh,
                             ptr(raw[:, off:]), K, ptr(stats[0][off:]), ptr(stats[1][off:]), *det_ws(), stream())
        _allreduce_stats(stats)
        count = float(N * P * Q) * _sync["world"]
        aux = torch.empty((4, K), dtype=torch.float32, device=dev)
        for (h, g, b, rm, rv, eps, mom) in ((slice(0, K1), g1, b1, rm1, rv1, eps1, mom1),
                                            (slice(K1, K), g2, b2, rm2, rv2, eps2, mom2)):
            _bn_finalize(aux[:, h], stats[:, h], count, g, b, rm, rv, eps, mom, True)
        y = _bn_apply(raw[:, :K1], aux[:, :K1], None, True)
        P2, Q2 = (P - 1) // 2 + 1, (Q - 1) // 2 + 1
        pooled = nhwc_empty(N, K2, P2, Q2, device=dev)
        argmax = torch.empty((N, P2, Q2, K2), dtype=torch.uint8, device=dev)
        call("tsb_bn_apply_maxpool3x3s2", ptr(raw[:, K1:]), K, ptr(aux[2, K1:]), ptr(aux[3, K1:]), ptr(pooled), K2,
             ptr(argmax), N, K2, P, Q, stream())
        ctx.save_for_backward(xs, w1, g1, w2, g2, raw, aux, argmax)
        ctx.refs = (b1, b2)
        ctx.count = count
        return y, pooled

    @staticmethod
    def backward(ctx, dy1, dpooled):
        xs, w1, g1, w2, g2, raw, aux, argmax = ctx.saved_tensors
        b1, b2 = ctx.refs
        N, K, P, Q = raw.shape
        K1 = w1.shape[0]
        dev = raw.device
        dpooled = as_nhwc_bf16(dpooled)
        dy2 = nhwc_empty(N, K - K1, P, Q, device=dev)
        call("tsb_maxpool3x3s2_bwd", ptr(argmax), ptr(dpooled), cs_of(dpooled), ptr(dy2), K - K1, N, K - K1, P, Q,
             stream())
        draw = nhwc_empty(N, K, P, Q, device=dev)
        halves = []
        for (h, w, g, b, dy) in ((slice(0, K1), w1, g1, b1, dy1), (slice(K1, K), w2, g2, b2, dy2)):
            grads = _ParamGrads(w, g, b)
            _bn_backward(dy, None, raw[:, h], aux[:, h], g, b, ctx.count, True, False, grads, draw=draw[:, h])
            halves.append((h, w, grads))
        H, W = P * 2, Q * 2
        dwp = zero_arena.take((K, 4, 64), dev)
        conv_prof.launch(2.0 * N * P * Q * K * 147, "tsb_conv_stem_wgrad", ptr(xs), N, H, W, ptr(draw), K, K, ptr(dwp),
                         *det_ws(), stream())
        outs = []
        for h, w, grads in halves:
            call("tsb_unpack_stem_wgrad", ptr(dwp[h.start:]), w.shape[0], w.shape[2], ptr(grads.buffer(w, krsc=True)),
                 stream())
            outs.append(grads.result())
        (dw1, dg1, db1), (dw2, dg2, db2) = outs
        return None, dw1, dg1, db1, None, None, dw2, dg2, db2, None, None, None, None, None, None


def _bias_grad(grads, bias, dy, dycs, npix, K):
    """Σ dy over the pixels into the bias gradient (tsb_bias_grad), for a bias that is not None"""
    if bias is not None:
        call("tsb_bias_grad", ptr(dy), dycs, npix, K, ptr(grads.buffer(bias)), *det_ws(), stream())


class ConvFn(torch.autograd.Function):
    """plain convolution (+bias), bf16 or fp32 output with channel stride `ocs` — the 1x1 classifier heads
    (bisenet network.py:156-161) and the BN-free SE convs of FeatureFusion (seg_oprs.py:224-229)."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, pad, dil, out_f32, ocs):
        K, C, R, _ = w.shape
        wb, _ = pack_cache.get(w, False)
        y = conv_fprop(x, wb, K, R, stride, pad, dil, bias=bias, out_dtype=torch.float32 if out_f32 else _BF, ocs=ocs)
        ctx.save_for_backward(x, w)
        ctx.bias_ref = bias
        ctx.cfg = (stride, pad, dil)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        stride, pad, dil = ctx.cfg
        K, C, R, _ = w.shape
        N, _, P, Q = dy.shape
        dev = dy.device
        # dgrad needs the GEMM-K (= out channels) padded to a multiple of 64 in a bf16 NHWC buffer
        Kp = (K + 63) // 64 * 64
        if dy.dtype == _BF and dy.stride(1) == 1 and cs_of(dy) >= Kp and K == Kp:
            dyb = dy
        else:
            if dy.stride(1) == 1 and dy.dtype in (_BF, torch.float32):
                dyb = nhwc_empty(N, Kp, P, Q, device=dev)     # tsb_cast_pad writes all Kp channels (zero pads)
                call("tsb_cast_pad", ptr(dy), _lib.dt(dy), cs_of(dy), K, ptr(dyb), Kp, Kp, N * P * Q, stream())
            else:
                dyb = nhwc_zeros(N, Kp, P, Q, device=dev)
                dyb[:, :K].copy_(dy)
        grads = _ParamGrads(w, ctx.bias_ref)
        conv_wgrad(x, dyb[:, :K], K, R, stride, pad, dil, grads.buffer(w, krsc=True))
        _bias_grad(grads, ctx.bias_ref, dyb, Kp, N * P * Q, K)
        dx = None
        if ctx.needs_input_grad[0]:
            _, wt = pack_cache.get(w, True, pad_k=Kp)
            dx = conv_dgrad(dyb, wt, x.shape, Kp, R, stride, pad, dil)
        return (dx,) + grads.result() + (None,) * 5


class ConvTransposeFn(torch.autograd.Function):
    """BN-free transposed convolution (+bias) (+ReLU in the epilogue), bf16 output: DeConvBnRelu with has_bn=False
    (seg_oprs.py:49-73). w is the ConvTranspose2d weight [Ci][Co][R][S] in KRSC storage, Ci and Co multiples of 64 (the
    module zero-pads ragged layers); the backward runs the adjoint conv's fprop (dx) and wgrad (dW), and tsb_bias_grad."""

    @staticmethod
    def forward(ctx, x, w, bias, stride, pad, dil, out_pad, relu):
        Ci, Co, R, _ = w.shape
        _, wt = pack_cache.get(w, True)
        y = conv_transpose_fprop(x, wt, Co, R, stride, pad, dil, out_pad, bias=bias, relu=relu)
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.bias_ref = bias
        ctx.cfg = (stride, pad, dil, relu)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        stride, pad, dil, relu = ctx.cfg
        Ci, Co, R, _ = w.shape
        N, _, P, Q = dy.shape
        dev = dy.device
        dy = as_nhwc_bf16(dy)
        if relu:
            dz = nhwc_empty(N, Co, P, Q, device=dev)
            call("tsb_relu_bwd", ptr(dy), cs_of(dy), ptr(y), cs_of(y), ptr(dz), Co, N * P * Q, Co, stream())
            dy = dz
        grads = _ParamGrads(w, ctx.bias_ref)
        conv_wgrad(dy, x, Ci, R, stride, pad, dil, grads.buffer(w, krsc=True))
        _bias_grad(grads, ctx.bias_ref, dy, cs_of(dy), N * P * Q, Co)
        dx = None
        if ctx.needs_input_grad[0]:
            wb, _ = pack_cache.get(w, False)
            dx = conv_fprop(dy, wb, Ci, R, stride, pad, dil)
        return (dx,) + grads.result() + (None,) * 5


class DWConvFn(torch.autograd.Function):
    """depthwise 3x3 convolution, no bias, stride 1 with padding = dilation `dil`, or stride 2 with padding 1: the
    `groups=in_channels` conv of the SeparableConvBnRelu blocks (TorchSeg furnace/base_model/xception.py:14-16,
    furnace/seg_opr/seg_oprs.py:76-94), on tsb_dwconv2d_{fprop,dgrad,wgrad}.

    x may carry more logical channels than the conv has (a 64-padded buffer whose channels [C, Cx) are zero): the
    kernels read its first C channels in place. The output has `ocs` >= C logical channels whose pads are exact zeros,
    so it can feed the 64-padded pointwise conv that follows without a copy. `share` (ops.GradShare): x has other
    consumers in the same block and their input gradients are chained through one buffer (dgrad accumulate)."""

    @staticmethod
    def forward(ctx, x, w, stride, ocs, share=None, dil=1):
        C = w.shape[0]
        assert w.shape[1:] == (1, 3, 3), "depthwise 3x3 weight [C,1,3,3] expected"
        N, Cx, H, W = x.shape
        assert Cx >= C
        P, Q = conv_out_size(H, 3, stride, dil, dil), conv_out_size(W, 3, stride, dil, dil)
        ocs = C if ocs is None else ocs
        y = (nhwc_zeros if ocs > C else nhwc_empty)(N, ocs, P, Q, device=x.device)
        call("tsb_dwconv2d_fprop", ptr(x), cs_of(x), ptr(w.detach().reshape(C, 9)), ptr(y), cs_of(y), N, H, W, C, stride,
             dil, stream())
        ctx.save_for_backward(x, w)
        ctx.stride, ctx.share, ctx.dil = stride, share, dil
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        stride, dil = ctx.stride, ctx.dil
        C = w.shape[0]
        N, Cx, H, W = x.shape
        dy = as_nhwc_bf16(dy)
        w9 = w.detach().reshape(C, 9)
        grads = _ParamGrads(w)
        call("tsb_dwconv2d_wgrad", ptr(x), cs_of(x), ptr(dy), cs_of(dy), ptr(grads.buffer(w)), N, H, W, C, stride, dil,
             *det_ws(), stream())
        dx = None
        if ctx.needs_input_grad[0]:
            def dgrad(out, accumulate):
                if out is None:
                    out = (nhwc_zeros if Cx > C else nhwc_empty)(N, Cx, H, W, device=dy.device)
                call("tsb_dwconv2d_dgrad", ptr(dy), cs_of(dy), ptr(w9), ptr(out), cs_of(out), N, H, W, C, stride, dil,
                     int(accumulate), stream())
                return out
            dx = _dgrad_into(ctx.share, dgrad)
        return (dx,) + grads.result() + (None,) * 4


class BNFn(torch.autograd.Function):
    """y = BN(x), followed by a ReLU when `relu`, on the BatchNorm half of ConvBNActFn: the `bn` between the depthwise and
    the pointwise conv of SeparableConvBnRelu (TorchSeg furnace/seg_opr/seg_oprs.py:88,93), and EncNet's BN + ReLU over
    the codewords. Training takes the batch statistics with tsb_bn_stats (summed over the SyncBN group like every other
    BN) and updates the running statistics; eval applies the running statistics. x: dense bf16 NHWC [N,C,H,W]."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, eps, momentum, training, relu=False):
        N, C, H, W = x.shape
        assert cs_of(x) == C
        count = float(N * H * W) * _sync["world"]
        stats = None
        if training:
            stats = zero_arena.take((2, C), x.device)
            call("tsb_bn_stats", ptr(x), C, N * H * W, C, ptr(stats[0]), ptr(stats[1]), *det_ws(), stream())
        y, aux = _bn_forward(x, stats, count, gamma, beta, None, running_mean, running_var, relu, eps, momentum,
                             training)
        ctx.save_for_backward(x, gamma, aux)
        ctx.beta_ref, ctx.count, ctx.training, ctx.relu = beta, count, training, relu
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, aux = ctx.saved_tensors
        assert ctx.training, "backward through eval-mode BN is not supported"
        beta = ctx.beta_ref
        grads = _ParamGrads(gamma, beta)
        # without a residual the ReLU mask is recomputed from x, scale and shift (no read of y)
        dx, _ = _bn_backward(dy, None, x, aux, gamma, beta, ctx.count, ctx.relu, False, grads)
        return (dx,) + grads.result() + (None,) * 6


# --------------------------------------------------------------------------------------------------
# EncNet: Context Encoding, mean over the codewords, SE-loss
# --------------------------------------------------------------------------------------------------
def _encoding_args(x, codewords, scale):
    N, D, H, W = x.shape
    K = codewords.shape[0]
    assert codewords.shape == (K, D) and scale.shape == (K,), "codewords [K, D] and scale [K] expected"
    assert codewords.is_contiguous() and scale.is_contiguous()
    return N, D, H * W, K


def encoding_infer(x, codewords, scale):
    """the Encoding forward without the saved soft-assignments (inference): E as bf16 NHWC [B, K, D, 1]"""
    B, D, HW, K = _encoding_args(x, codewords, scale)
    E = nhwc_empty(B, K, D, 1, device=x.device)
    sum_a = torch.empty((B, K), dtype=torch.float32, device=x.device)
    call("tsb_encoding_fwd", ptr(x), cs_of(x), B, HW, D, ptr(codewords), ptr(scale), K, None, None, ptr(sum_a), ptr(E),
         *det_ws(), stream())
    return E


class EncodingFn(torch.autograd.Function):
    """EncNet's Encoding layer: E_bk = Σ_i softmax_k(s_k ‖x_i − c_k‖²) (x_i − c_k) over the pixels of image b, on
    tsb_encoding_{fwd,bwd}; the [B, HW, K, D] residuals are never formed. x: bf16 NHWC [B, D, h, w]. E comes back as the
    bf16 NHWC tensor [B, K, D, 1] (row b·D + d, channel k), so the codeword BN runs on it as on any activation."""

    @staticmethod
    def forward(ctx, x, codewords, scale):
        B, D, HW, K = _encoding_args(x, codewords, scale)
        dev = x.device
        a = torch.empty((B * HW, K), dtype=torch.float32, device=dev)
        d2 = torch.empty((B * HW, K), dtype=torch.float32, device=dev)
        sum_a = torch.empty((B, K), dtype=torch.float32, device=dev)
        E = nhwc_empty(B, K, D, 1, device=dev)
        call("tsb_encoding_fwd", ptr(x), cs_of(x), B, HW, D, ptr(codewords), ptr(scale), K, ptr(a), ptr(d2), ptr(sum_a),
             ptr(E), *det_ws(), stream())
        ctx.save_for_backward(x, codewords, scale, a, d2, sum_a)
        return E

    @staticmethod
    def backward(ctx, dE):
        x, codewords, scale, a, d2, sum_a = ctx.saved_tensors
        B, D, H, W = x.shape
        K = codewords.shape[0]
        if dE.dtype != _BF or dE.stride(1) != 1 or cs_of(dE) != K:
            dE = to_nhwc(dE)
        grads = _ParamGrads(codewords, scale)
        dc, ds = grads.buffer(codewords), grads.buffer(scale)
        dx = nhwc_empty(B, D, H, W, device=x.device)
        call("tsb_encoding_bwd", ptr(dE), ptr(x), cs_of(x), B, H * W, D, ptr(codewords), ptr(scale), K, ptr(a), ptr(d2),
             ptr(sum_a), ptr(dx), D, ptr(dc), ptr(ds), *det_ws(), stream())
        return (dx,) + grads.result()


class ChanMeanFn(torch.autograd.Function):
    """mean over the C channels of each pixel: [N, C, H, W] → [N·H·W] values, returned as the bf16 NHWC [N, H·W, 1, 1]
    (EncNet's mean over the K codewords of E [B, K, D, 1] gives en [B, D, 1, 1])"""

    @staticmethod
    def forward(ctx, x):
        N, C, H, W = x.shape
        y = nhwc_empty(N, H * W, 1, 1, device=x.device)
        call("tsb_chan_mean_fwd", ptr(x), cs_of(x), N * H * W, C, ptr(y), stream())
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, C, H, W = ctx.shape
        if dy.dtype != _BF or not dy.is_contiguous():
            dy = dy.to(_BF).contiguous()   # [N, H·W, 1, 1]: contiguous is the dense NHWC layout
        dx = nhwc_empty(N, C, H, W, device=dy.device)
        call("tsb_chan_mean_bwd", ptr(dy), N * H * W, C, ptr(dx), C, stream())
        return dx


class SELossFn(torch.autograd.Function):
    """EncNet's SE-loss: nn.BCELoss(sigmoid(z), presence(label)) with presence[b, c] = any(label[b] == c), c in [0, C),
    built on the device (tsb_se_loss_fwd_bwd): no host synchronisation, so the step stays one graph replay. z: fp32 NHWC
    [B, C, 1, 1] logits (any channel stride); label: int64 [B, H, W]."""

    @staticmethod
    def forward(ctx, z, label, num_classes):
        B = z.shape[0]
        C = int(num_classes)
        assert z.dtype == torch.float32 and z.shape[1] == C and z.shape[0] == label.shape[0]
        label = label.contiguous()
        zs = cs_of(z)
        dev = z.device
        presence = torch.empty((B, (C + 31) // 32), dtype=torch.int32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        dz = nhwc_zeros(B, C, 1, 1, dtype=torch.float32, device=dev, cs=zs)
        call("tsb_se_loss_fwd_bwd", ptr(label), B, label[0].numel(), ptr(z), zs, C, ptr(presence), ptr(loss), ptr(dz),
             zs, stream())
        ctx.save_for_backward(dz)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dz,) = ctx.saved_tensors
        return dz * g.to(dz.dtype), None, None


# --------------------------------------------------------------------------------------------------
# OCNet: dense self-attention over the pixels of each image
# --------------------------------------------------------------------------------------------------
class AttentionFn(torch.autograd.Function):
    """o = softmax(scale · q kᵀ) v over the h·w pixels of each image (OCNet's object context), fused on
    tsb_attention_{fwd,bwd}: the [N, N] scores never reach memory, and the backward recomputes them from the saved
    q, k, v, o and the per-row log-sum-exp (O(N·d) saved, not O(N²)). q, k, v: bf16 NHWC [B, 256, h, w] (channel slices
    allowed). k = None means k is q (OCNet's shared f_key): the backward then returns dQ + dK as q's gradient, formed by
    the kernels in one buffer. Without any input needing a gradient the forward skips the log-sum-exp."""

    @staticmethod
    def forward(ctx, q, k, v, scale):
        shared = k is None
        k = q if shared else k
        B, dk, h, w = q.shape
        dv = v.shape[1]
        assert k.shape == q.shape and v.shape[0] == B and v.shape[2:] == q.shape[2:], "attention: shape mismatch"
        need = any(ctx.needs_input_grad)
        o = nhwc_empty(B, dv, h, w, device=q.device)
        lse = torch.empty((B, h * w), dtype=torch.float32, device=q.device) if need else None
        call("tsb_attention_fwd", ptr(q), cs_of(q), ptr(k), cs_of(k), ptr(v), cs_of(v), ptr(o), dv, ptr(lse), B, h * w,
             dk, dv, float(scale), stream())
        if need:
            ctx.save_for_backward(q, k, v, o, lse)
            ctx.cfg = (shared, float(scale))
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        shared, scale = ctx.cfg
        B, dk, h, w = q.shape
        dv = v.shape[1]
        do = as_nhwc_bf16(do)
        dq = nhwc_empty(B, dk, h, w, device=q.device)
        dkt = dq if shared else nhwc_empty(B, dk, h, w, device=q.device)
        dvt = nhwc_empty(B, dv, h, w, device=q.device)
        delta = torch.empty((B, h * w), dtype=torch.float32, device=q.device)
        call("tsb_attention_bwd", ptr(q), cs_of(q), ptr(k), cs_of(k), ptr(v), cs_of(v), ptr(o), cs_of(o), ptr(do),
             cs_of(do), ptr(lse), ptr(delta), ptr(dq), dk, ptr(dkt), dk, ptr(dvt), dv, int(shared), B, h * w, dk, dv,
             scale, stream())
        return dq, (None if shared else dkt), dvt, None


# --------------------------------------------------------------------------------------------------
# pooling / resize / attention scale
# --------------------------------------------------------------------------------------------------
class MaxPool3x3S2Fn(torch.autograd.Function):
    """nn.MaxPool2d(3, 2, 1) — TorchSeg furnace/base_model/resnet.py:132"""

    @staticmethod
    def forward(ctx, x):
        N, C, H, W = x.shape
        P, Q = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = nhwc_empty(N, C, P, Q, device=x.device)
        idx = torch.empty((N, P, Q, C), dtype=torch.uint8, device=x.device)
        call("tsb_maxpool3x3s2_fwd", ptr(x), cs_of(x), ptr(y), C, ptr(idx), N, C, H, W, stream())
        ctx.save_for_backward(idx)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        dy = as_nhwc_bf16(dy)
        dx = nhwc_empty(N, C, H, W, device=dy.device)
        call("tsb_maxpool3x3s2_bwd", ptr(idx), ptr(dy), cs_of(dy), ptr(dx), C, N, C, H, W, stream())
        return dx


class AdaptiveAvgPoolFn(torch.autograd.Function):
    """nn.AdaptiveAvgPool2d(S) — seg_oprs.py:200,223; bisenet network.py:35; pspnet network.py:83.
    Output bf16 [N,C,S,S] (NHWC)."""

    @staticmethod
    def forward(ctx, x, S):
        N, C, H, W = x.shape
        o32 = torch.empty((N, S, S, C), dtype=torch.float32, device=x.device)
        call("tsb_adaptive_avgpool_fwd", ptr(x), cs_of(x), N, C, H, W, S, ptr(o32), *det_ws(), stream())
        out = nhwc_empty(N, C, S, S, device=x.device)
        call("tsb_cast_scale", ptr(o32), F32, C, ptr(out), BF16, C, N * S * S, C, None, stream())
        ctx.shape = (N, C, H, W, S)
        return out

    @staticmethod
    def backward(ctx, dy):
        N, C, H, W, S = ctx.shape
        if dy.stride(1) != 1:
            dy = to_nhwc(dy, dy.dtype)
        d32 = torch.empty((N, S, S, C), dtype=torch.float32, device=dy.device)
        call("tsb_cast_scale", ptr(dy), _lib.dt(dy), cs_of(dy), ptr(d32), F32, C, N * S * S, C, None, stream())
        dx = nhwc_empty(N, C, H, W, device=dy.device)
        call("tsb_adaptive_avgpool_bwd", ptr(d32), N, C, H, W, S, ptr(dx), C, 0, stream())
        return dx, None


_scalars = {}


def _const_scalar(v, device):
    """cached 1-element fp32 device tensor (scale factors read by kernels from device memory)"""
    key = (v, str(device))
    t = _scalars.get(key)
    if t is None:
        t = torch.tensor([v], dtype=torch.float32, device=device)
        _scalars[key] = t
    return t


class BilinearFn(torch.autograd.Function):
    """F.interpolate(mode='bilinear', align_corners=True) — bisenet network.py:82-84,93-94"""

    @staticmethod
    def forward(ctx, x, Ho, Wo):
        N, C, Hi, Wi = x.shape
        y = nhwc_empty(N, C, Ho, Wo, device=x.device)
        call("tsb_bilinear_fwd", ptr(x), _lib.dt(x), cs_of(x), ptr(y), BF16, C, N, C, Hi, Wi, Ho, Wo, stream())
        ctx.shape = (N, C, Hi, Wi, Ho, Wo)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, C, Hi, Wi, Ho, Wo = ctx.shape
        dy = as_nhwc_bf16(dy)
        dx = nhwc_empty(N, C, Hi, Wi, device=dy.device)
        if Hi == 1 and Wi == 1:
            # broadcast forward (1x1 → HxW, bisenet network.py:82-84) ⇒ the backward is a plain spatial sum: reuse the
            # pooling reduction (mean) and scale by H*W instead of a one-block gather
            m32 = torch.empty((N, 1, 1, C), dtype=torch.float32, device=dy.device)
            call("tsb_adaptive_avgpool_fwd", ptr(dy), cs_of(dy), N, C, Ho, Wo, 1, ptr(m32), *det_ws(), stream())
            call("tsb_cast_scale", ptr(m32), F32, C, ptr(dx), BF16, C, N, C, ptr(_const_scalar(float(Ho * Wo), dy.device)), stream())
        else:
            call("tsb_bilinear_bwd", ptr(dy), BF16, cs_of(dy), ptr(dx), BF16, C, N, C, Hi, Wi, Ho, Wo, 0, stream())
        return dx, None, None


class UpsampleLogitsFn(torch.autograd.Function):
    """reference-boundary form of the head tail: NCHW fp32 [N,C,H,W] logits, bilinear align_corners=True to an explicit
    output size (bisenet network.py:164-166 use scale_factor; with align_corners the source coordinate is
    (in-1)/(out-1)·dst either way, so size = in·scale is the same op — and sizes like 713 / 473 that are not a multiple
    of 8 work too)"""

    @staticmethod
    def forward(ctx, lo, H, W):
        N, C, h, w = lo.shape
        H, W = int(H), int(W)
        out = torch.empty((N, C, H, W), dtype=torch.float32, device=lo.device)
        call("tsb_bilinear_fwd_nhwc_to_nchw", ptr(lo), _lib.dt(lo), cs_of(lo), ptr(out), N, C, h, w, H, W, stream())
        ctx.shape = (N, C, h, w, H, W, cs_of(lo))
        return out

    @staticmethod
    def backward(ctx, g):
        N, C, h, w, H, W, cs = ctx.shape
        # gather-form transpose needs NHWC with C % 8 == 0: pad the class dimension into a 32-wide buffer
        Cp = (C + 7) // 8 * 8
        gp = nhwc_zeros(N, Cp, H, W, dtype=torch.float32, device=g.device)
        gp[:, :C].copy_(g)
        d = nhwc_zeros(N, Cp, h, w, dtype=torch.float32, device=g.device, cs=max(cs, Cp))
        call("tsb_bilinear_bwd", ptr(gp), F32, Cp, ptr(d), F32, cs_of(d), N, Cp, h, w, H, W, 0, stream())
        return d[:, :C], None, None


class ChanScaleFn(torch.autograd.Function):
    """y = x * (base + sigmoid(a)) + add.  ARM: base 0 (+ the caller's `fm += last_fm`, bisenet network.py:91-92);
    FFM: base 1 (fm + fm*se, seg_oprs.py:237). `a` is the bf16 [N,C,1,1] pre-sigmoid attention logit."""

    @staticmethod
    def forward(ctx, x, a, add, base):
        N, C, H, W = x.shape
        a32 = torch.empty((N, C), dtype=torch.float32, device=x.device)
        call("tsb_cast_scale", ptr(a), _lib.dt(a), cs_of(a), ptr(a32), F32, C, N, C, None, stream())
        y = nhwc_empty(N, C, H, W, device=x.device)
        call("tsb_chan_scale_fwd", ptr(x), cs_of(x), ptr(a32), float(base), ptr(add), cs_of(add) if add is not None else 0,
             ptr(y), C, N, H * W, C, stream())
        ctx.save_for_backward(x, a32)
        ctx.cfg = (base, add is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, a32 = ctx.saved_tensors
        base, has_add = ctx.cfg
        N, C, H, W = x.shape
        dy = as_nhwc_bf16(dy)
        dx = nhwc_empty(N, C, H, W, device=x.device)
        da32 = torch.zeros((N, C), dtype=torch.float32, device=x.device)
        call("tsb_chan_scale_bwd", ptr(dy), cs_of(dy), ptr(x), cs_of(x), ptr(a32), float(base), ptr(dx), C, ptr(da32), N,
             H * W, C, *det_ws(), stream())
        da = nhwc_empty(N, C, 1, 1, device=x.device)
        call("tsb_cast_scale", ptr(da32), F32, C, ptr(da), BF16, C, N, C, None, stream())
        return dx, da, (dy if has_add else None), None


class ConcatFn(torch.autograd.Function):
    """torch.cat([x1, x2, ...], dim=1) (FeatureFusion seg_oprs.py:234, PyramidPooling pspnet network.py:106) as strided
    copies into ONE NHWC buffer; backward hands out channel-slice views (no copy)."""

    @staticmethod
    def forward(ctx, *xs):
        N, _, H, W = xs[0].shape
        chans = [int(x.shape[1]) for x in xs]
        Ct = sum(chans)
        out = nhwc_empty(N, Ct, H, W, device=xs[0].device)
        npix = N * H * W
        off = 0
        for x, c in zip(xs, chans):
            call("tsb_cast_scale", ptr(x), BF16, cs_of(x), ptr(out[:, off:]), BF16, Ct, npix, c, None, stream())
            off += c
        ctx.chans = chans
        return out

    @staticmethod
    def backward(ctx, dy):
        dy = as_nhwc_bf16(dy)
        outs, off = [], 0
        for c in ctx.chans:
            outs.append(dy[:, off:off + c])
            off += c
        return tuple(outs)


class AddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        N, C, H, W = a.shape
        y = nhwc_empty(N, C, H, W, device=a.device)
        call("tsb_add", ptr(a), cs_of(a), ptr(b), cs_of(b), ptr(y), C, N * H * W, C, stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        return dy, dy


class PSABmmFn(torch.autograd.Function):
    """out = bmm(x.view(b,c,-1), softmax(att.view(b,L,-1), dim=1)) with L = h*w attention channels per pixel
    (PointwiseSpatialAttention.forward, psanet network.py:122-126,131-138).

    NHWC form per image: out[j, ch] = Σ_i S[j, i] · x[i, ch] with S = row-softmax of att[j, :]. That is a 1x1
    convolution whose "image" is S (L pixels x L channels, zero-padded to a multiple of 64 channels) and whose weight
    operand is the image's own feature map transposed ([c, L]); dS is the matching dgrad (weight operand = x itself),
    dx the matching wgrad. All three run on the wgmma conv kernels, one launch per image."""

    @staticmethod
    def forward(ctx, x, att):
        b, c, h, w = x.shape
        L = att.shape[1]
        assert L == h * w and att.shape[0] == b and tuple(att.shape[2:]) == (h, w), "PSA needs h*w attention channels"
        assert c % 64 == 0 and L % 8 == 0
        dev = x.device
        if cs_of(x) != c:
            x = to_nhwc(x)
        Lp = (L + 63) // 64 * 64
        S = nhwc_empty(b, Lp, h, w, device=dev)
        call("tsb_softmax_rows_fwd", ptr(att), _lib.dt(att), cs_of(att), ptr(S), Lp, b * h * w, L, Lp, stream())
        out = nhwc_empty(b, c, h, w, device=dev)
        xt = torch.empty((c, Lp), dtype=_BF, device=dev)
        for n in range(b):
            call("tsb_transpose_pad", ptr(x[n:n + 1]), BF16, c, ptr(xt), Lp, L, c, Lp, stream())
            conv_fprop(S[n:n + 1], xt, c, 1, 1, 0, 1, out=out[n:n + 1])
        ctx.save_for_backward(x, S)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, S = ctx.saved_tensors
        b, c, h, w = x.shape
        Lp = S.shape[1]
        L = h * w
        dev = x.device
        dout = as_nhwc_bf16(dout)
        dS = nhwc_empty(b, L, h, w, device=dev, cs=Lp)
        dx = nhwc_empty(b, c, h, w, device=dev)
        dxt = torch.empty((c, Lp), dtype=torch.float32, device=dev)
        for n in range(b):
            conv_dgrad(dout[n:n + 1], x[n:n + 1], (1, L, h, w), c, 1, 1, 0, 1, out=dS[n:n + 1])
            dxt.zero_()
            conv_wgrad(S[n:n + 1], dout[n:n + 1], c, 1, 1, 0, 1, dxt)
            call("tsb_transpose_pad", ptr(dxt), F32, Lp, ptr(dx[n:n + 1]), c, c, L, c, stream())
        dA = nhwc_empty(b, L, h, w, device=dev, cs=Lp)
        call("tsb_softmax_rows_bwd", ptr(S), Lp, ptr(dS), Lp, ptr(dA), Lp, b * h * w, L, Lp, stream())
        return dx, dA


# --------------------------------------------------------------------------------------------------
# image packing (network input boundary)
# --------------------------------------------------------------------------------------------------
def pack_image_s2d(img):
    """NCHW fp32 image → [N,16,H/2,W/2+4] bf16 (NHWC) operand of the 7x7/2 stems"""
    N, C, H, W = img.shape
    assert C == 3 and img.dtype == torch.float32 and img.is_contiguous()
    if (H | W) & 1:
        # odd sizes (713, 473): one extra zero row / column at the bottom / right is exactly the stem's own zero padding
        # (the stride-2 output size floor((H + 2p - k) / 2) + 1 is the same for H and H + 1 when H is odd)
        img = torch.nn.functional.pad(img, (0, W & 1, 0, H & 1)).contiguous()
        H, W = H + (H & 1), W + (W & 1)
    out = nhwc_empty(N, 16, H // 2, W // 2 + 4, device=img.device)
    call("tsb_pack_image_s2d", ptr(img), N, H, W, ptr(out), stream())
    return out


# --------------------------------------------------------------------------------------------------
# OHEM cross-entropy
# --------------------------------------------------------------------------------------------------
def _ohem_forward(pt_call, n, labels, ignore_label, thresh, min_kept, class_weight, dev):
    state = torch.empty((_lib.OHEM_STATE_WORDS,), dtype=torch.int32, device=dev)
    p = torch.empty((n,), dtype=torch.float32, device=dev)
    nll = torch.empty((n,), dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    call("tsb_ohem_begin", ptr(state), stream())
    pt_call(p, nll, state)
    call("tsb_ohem_select", ptr(p), n, int(min_kept), float(thresh), ptr(state), stream())
    call("tsb_ohem_loss", ptr(p), ptr(nll), ptr(labels), n, int(ignore_label), ptr(class_weight), ptr(state), ptr(loss),
         stream())
    return loss, p, state


class OhemCEFn(torch.autograd.Function):
    """ProbOhemCrossEntropy2d.forward on MATERIALISED logits [N,C,H,W] (any strides, fp32/bf16) —
    TorchSeg furnace/seg_opr/loss_opr.py:68-98. Labels lie in [0, C) or equal ignore_label (the kernels index the class
    weights and the logits with them)."""

    @staticmethod
    def forward(ctx, pred, target, ignore_label, thresh, min_kept, class_weight):
        N, C, H, W = pred.shape
        target = target.contiguous()
        sn, sc, sy, sx = pred.stride()
        dtp = _lib.dt(pred)

        def pt(p, nll, state):
            call("tsb_ohem_ptarget", ptr(pred), dtp, sn, sc, sy, sx, ptr(target), N, C, H, W, int(ignore_label),
                 float(thresh), ptr(p), ptr(nll), ptr(state), stream())

        loss, p, state = _ohem_forward(pt, N * H * W, target, ignore_label, thresh, min_kept, class_weight, pred.device)
        ctx.save_for_backward(pred, target, p, state, class_weight if class_weight is not None else torch.empty(0))
        ctx.cfg = (ignore_label, class_weight is not None)
        return loss

    @staticmethod
    def backward(ctx, g):
        pred, target, p, state, cw = ctx.saved_tensors
        ignore_label, has_cw = ctx.cfg
        N, C, H, W = pred.shape
        sn, sc, sy, sx = pred.stride()
        d = torch.empty_strided(pred.shape, pred.stride(), dtype=pred.dtype, device=pred.device)
        g = g.to(torch.float32).contiguous()
        call("tsb_ohem_grad", ptr(pred), _lib.dt(pred), sn, sc, sy, sx, ptr(target), ptr(p), N, C, H, W, int(ignore_label),
             ptr(cw) if has_cw else None, ptr(state), ptr(g), ptr(d), stream())
        return d, None, None, None, None, None


class OhemUpCEFn(torch.autograd.Function):
    """Fused head tail: bilinear x`scale` upsample (align_corners) of the LOW-res fp32 NHWC logits +
    ProbOhemCrossEntropy2d; the full-resolution logits are never written (bisenet network.py:104-108,163-166). Labels lie
    in [0, C) or equal ignore_label (the kernels index shared memory with them). The forward refuses an up-scale the
    backward cannot run."""

    @staticmethod
    def forward(ctx, lo, target, H, W, num_classes, ignore_label, thresh, min_kept, class_weight):
        N, _, h, w = lo.shape
        assert lo.dtype == torch.float32
        target = target.contiguous()
        cs = cs_of(lo)

        def pt(p, nll, state):
            call("tsb_ohem_ptarget_up", ptr(lo), cs, h, w, ptr(target), N, num_classes, H, W, int(ignore_label),
                 float(thresh), ptr(p), ptr(nll), ptr(state), stream())

        loss, p, state = _ohem_forward(pt, N * H * W, target, ignore_label, thresh, min_kept, class_weight, lo.device)
        ctx.save_for_backward(lo, target, p, state, class_weight if class_weight is not None else torch.empty(0))
        ctx.cfg = (H, W, num_classes, ignore_label, class_weight is not None)
        return loss

    @staticmethod
    def backward(ctx, g):
        lo, target, p, state, cw = ctx.saved_tensors
        H, W, C, ignore_label, has_cw = ctx.cfg
        N, Cl, h, w = lo.shape
        cs = cs_of(lo)
        d = nhwc_zeros(N, Cl, h, w, dtype=torch.float32, device=lo.device, cs=cs)
        g = g.to(torch.float32).contiguous()
        call("tsb_ohem_grad_up", ptr(lo), cs, h, w, ptr(target), ptr(p), N, C, H, W, int(ignore_label),
             ptr(cw) if has_cw else None, ptr(state), ptr(g), ptr(d), stream())
        return d, None, None, None, None, None, None, None, None


class CEUpFn(torch.autograd.Function):
    """Fused head tail for MANY classes (ADE's 150): bilinear up-sampling (align_corners) of the LOW-res fp32 NHWC logits to
    H x W + CrossEntropyLoss(mean, ignore_index); the full-resolution [N,C,H,W] logits are never written
    (pspnet network.py:46-57, psanet network.py:46-55). 1 <= C <= 152. Labels lie in [0, C) or equal ignore_label (the
    kernels index shared memory with them). The forward refuses an up-scale the backward cannot run."""

    @staticmethod
    def forward(ctx, lo, target, H, W, num_classes, ignore_label):
        N, _, h, w = lo.shape
        assert lo.dtype == torch.float32
        target = target.contiguous()
        cs = cs_of(lo)
        dev = lo.device
        state = torch.empty((8,), dtype=torch.int32, device=dev)
        lse = torch.empty((N * H * W,), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        call("tsb_ce_up_fwd", ptr(lo), cs, h, w, ptr(target), N, int(num_classes), int(H), int(W), int(ignore_label), ptr(lse),
             ptr(state), ptr(loss), stream())
        ctx.save_for_backward(lo, target, lse, state)
        ctx.cfg = (int(H), int(W), int(num_classes), int(ignore_label))
        return loss

    @staticmethod
    def backward(ctx, g):
        lo, target, lse, state = ctx.saved_tensors
        H, W, C, ignore_label = ctx.cfg
        N, Cl, h, w = lo.shape
        cs = cs_of(lo)
        d = nhwc_zeros(N, Cl, h, w, dtype=torch.float32, device=lo.device, cs=cs)
        g = g.to(torch.float32).contiguous()
        call("tsb_ce_up_bwd", ptr(lo), cs, h, w, ptr(target), ptr(lse), N, C, H, W, ignore_label, ptr(state), ptr(g), ptr(d),
             stream())
        return d, None, None, None, None, None


FUSED_CE_MAX_CLASSES = 152   # tsb_ce_up_* register budget (38 class quads)


def ohem_state_dict(state):
    """decode the OHEM state words (host sync) — for tests / logging"""
    s = state.cpu()
    f = s.view(torch.float32)
    return dict(num_valid=int(s[_lib.OHEM_ST_NUM_VALID]), count_le=int(s[_lib.OHEM_ST_COUNT_LE]),
                active=bool(s[_lib.OHEM_ST_ACTIVE]), T=float(f[_lib.OHEM_ST_THRESH]), kept=int(s[_lib.OHEM_ST_KEPT]),
                loss=float(f[_lib.OHEM_ST_LOSS]))


# --------------------------------------------------------------------------------------------------
# evaluator (engine/evaluator.py: sliding_eval_device / whole_eval_device), one frame and one scale per call
# --------------------------------------------------------------------------------------------------
def eval_windows(src, fx, sh, sw, top, left, lut, pad_zero, corners, wh, ww, mirror=False):
    """uint8 [H,W,cin] frame on the device → cv2.resize(fx) → (sh, sw) at (top, left) of a padded canvas → normalised
    through `lut` [3,256] → the [n,3,wh,ww] fp32 windows at `corners` (int32 [n,2] {y, x} on the device), optionally
    mirrored. pad_zero: canvas padding is 0.0 instead of lut[c][0]."""
    assert src.dtype == torch.uint8 and src.dim() == 3 and src.is_contiguous()
    assert corners.dtype == torch.int32 and corners.is_contiguous() and lut.dtype == torch.float32
    n = corners.shape[0]
    out = torch.empty((n, 3, wh, ww), dtype=torch.float32, device=src.device)
    H, W, cin = src.shape
    call("tsb_eval_windows", ptr(src), H, W, cin, float(fx or 0.0), sh, sw, top, left, ptr(lut), int(bool(pad_zero)),
         ptr(corners), n, wh, ww, int(bool(mirror)), ptr(out), stream())
    return out


def eval_accumulate(lp, lp_flip, corners, acc):
    """acc [C,PH,PW] fp32 += exp(lp + mirror(lp_flip)) of each window at `corners`, in window order (overlaps SUMMED)"""
    n, C, wh, ww = lp.shape
    for t in (lp, lp_flip):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != (n, C, wh, ww)):
            raise TypeError("eval_accumulate: log-probs must be contiguous float32 [n, C, h, w] of one shape")
    assert acc.dtype == torch.float32 and acc.is_contiguous() and acc.shape[0] == C
    call("tsb_eval_accumulate", ptr(lp), ptr(lp_flip), ptr(corners), n, C, wh, ww, ptr(acc), acc.shape[1], acc.shape[2],
         stream())
    return acc


def eval_resize_add(score, total, pred=None):
    """total [C,H,W] fp64 += cv2.resize(score, (W, H), INTER_LINEAR) of a [C,h,w] fp32 view (any strides with a unit
    column stride); with `pred` (int64 [H,W]) the first arg-max over C of the updated total is written instead"""
    C, h, w = score.shape
    assert score.dtype == torch.float32 and score.stride(2) == 1
    assert total.dtype == torch.float64 and total.is_contiguous() and total.shape[0] == C
    if pred is not None:
        assert pred.dtype == torch.int64 and pred.is_contiguous() and tuple(pred.shape) == tuple(total.shape[1:])
    call("tsb_eval_resize_add", ptr(score), C, h, w, score.stride(0), score.stride(1), ptr(total), total.shape[1],
         total.shape[2], ptr(pred), stream())
