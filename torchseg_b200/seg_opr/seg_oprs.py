"""H100-native building blocks with the reference's names, constructor signatures and child-module names
(TorchSeg furnace/seg_opr/seg_oprs.py). Parameters live in genuine nn.Conv2d / norm_layer children —
`group_weight`'s completeness assert (furnace/utils/init_func.py:52-53) and the checkpoint keys (SURVEY.md
App. D) depend on that — only `forward` is replaced by the fused libtsb path.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops


def _as_act(x):
    """boundary: accept a plain NCHW tensor (any dtype) and move it into the NHWC bf16 activation layout"""
    if x.dtype == torch.bfloat16 and (x.shape[1] == 1 or x.stride(1) == 1):
        return x
    return ops.to_nhwc(x)


_s2d_cache = {}


def _packed_image(img):
    """space-to-depth pack of the fp32 NCHW input image, shared by the two 7x7 stems of BiSeNet.

    The cache holds a STRONG reference to the image tensor and matches by identity (`is`) + version, never by address:
    a fresh `imgs.cuda()` batch can be handed the freed storage of the previous one by the caching allocator, so a
    data_ptr key would silently serve the previous batch's pack. `pack_cache.step` is part of the key because a
    whole-step CUDA graph must contain the pack kernel even though the static input keeps identity and version between
    the warm-up and the capture. Networks clear the cache at the end of their forward (`_release_packed_image`)."""
    hit = _s2d_cache.get("k")
    if hit is not None and hit[0] is img and hit[1] == (img._version, ops.pack_cache.step):
        return hit[2]
    packed = ops.pack_image_s2d(img.contiguous().float())
    _s2d_cache["k"] = (img, (img._version, ops.pack_cache.step), packed)
    return packed


def _release_packed_image():
    _s2d_cache.clear()


def _ceil_to(n, m):
    return (n + m - 1) // m * m


def _pad_weight(w, Kp, Cp):
    """zero-pad a KRSC-backed [K,C,R,S] weight to [Kp,Cp,R,S] (autograd slices the gradient back)"""
    K, C = w.shape[:2]
    if K == Kp and C == Cp:
        return w
    wk = F.pad(w.permute(0, 2, 3, 1), (0, Cp - C, 0, 0, 0, 0, 0, Kp - K))
    return wk.permute(0, 3, 1, 2)


def _pad_vec(v, Kp, value=0.0):
    return v if v.shape[0] == Kp else F.pad(v, (0, Kp - v.shape[0]), value=value)


def _pad_act(x, Cp):
    """activation with a ragged channel count arriving from outside the padded domain: copy into zero pads"""
    N, C, H, W = x.shape
    out = ops.nhwc_zeros(N, Cp, H, W, device=x.device)
    out[:, :C].copy_(x)
    return out


def _ragged(conv, x):
    """DFN's 21 / 171 / 9-channel layers (dfn network.py:58-72,160-164): the tensor-core kernels tile GEMM-K in
    64-channel boxes, so these layers run zero-padded to the next multiple of 64. Pad channels carry exact zeros
    through conv (zero weight rows/columns), BN (beta pad 0) and ReLU, forward and backward."""
    return conv.in_channels != x.shape[1] or conv.in_channels % 64 != 0


def _pad_layer(x, w, Cp, Kp, b=None, transposed=False):
    """a layer's operands in the 64-padded channel domain: x with Cp channels (its first C, the weight's input channels,
    copied into zero pads unless it has Cp already), the weight [K][C] ([C][K] when transposed) zero-padded to Kp output
    and Cp input channels, the bias (None stays None) to Kp"""
    C = w.shape[0] if transposed else w.shape[1]
    if x.shape[1] != Cp:
        x = _pad_act(x[:, :C], Cp)
    w = _pad_weight(w, Cp, Kp) if transposed else _pad_weight(w, Kp, Cp)
    return x, w, (None if b is None else _pad_vec(b, Kp))


def _bn_momentum(bn):
    return float(bn.momentum if bn.momentum is not None else 0.1)


def _conv_bn_act_fn(x, w, bn, Kp, residual, stride, pad, dil, relu, stem=False, in_share=None, res_share=None,
                    out_pad=None):
    """ops.ConvBNActFn with bn's γ, β and running statistics padded to the Kp output channels of w (γ and the running
    variance with ones, β and the running mean with zeros). A training forward updates the padded running statistics;
    they are copied back into bn."""
    gamma, beta = _pad_vec(bn.weight, Kp, 1.0), _pad_vec(bn.bias, Kp)
    with torch.no_grad():
        rm, rv = _pad_vec(bn.running_mean, Kp), _pad_vec(bn.running_var, Kp, 1.0)
    y = ops.ConvBNActFn.apply(x, w, gamma, beta, residual, rm, rv, stride, pad, dil, bool(relu), float(bn.eps),
                              _bn_momentum(bn), bool(bn.training), stem, in_share, res_share, out_pad)
    if bn.training and rm is not bn.running_mean:
        with torch.no_grad():
            K = bn.running_mean.shape[0]
            bn.running_mean.copy_(rm[:K])
            bn.running_var.copy_(rv[:K])
    return y


EVAL_FOLD_BN = True   # eval mode: fold the BatchNorm into the conv weights, bias (+ residual) + ReLU in the conv epilogue


def conv_bn_act(x, conv, bn, relu, residual=None, in_share=None, res_share=None):
    """fused conv → norm_layer(train/eval) → (+residual) → ReLU on the libtsb path.
    in_share / res_share: ops.GradShare of a block-level fork (see BasicBlock.forward)"""
    ks = conv.kernel_size[0]
    assert conv.kernel_size[0] == conv.kernel_size[1] and conv.groups == 1 and conv.bias is None
    stem = (conv.in_channels == 3 and conv.stride[0] == 2 and conv.dilation[0] == 1 and
            (ks, conv.padding[0]) in ((7, 3), (3, 1)))
    if stem:
        xin = _packed_image(x) if x.shape[1] == 3 else x
    else:
        xin = _as_act(x)
    if residual is not None:
        residual = _as_act(residual)
    w = conv.weight
    K = Kp = conv.out_channels
    padded = (not stem) and (_ragged(conv, xin) or K % 64 != 0)
    if padded:
        Kp = _ceil_to(K, 64)
        xin, w, _ = _pad_layer(xin, w, _ceil_to(xin.shape[1], 64), Kp)
    if stem or not bn.training:
        in_share = res_share = None
    elif padded:
        # the padded conv may read a zero-padded copy of x, whose gradient is not x's; the residual is used as it
        # comes whenever K itself needs no padding (Xception's 16/32-channel pointwise convs into 64/128 channels)
        in_share = None
        if Kp != K:
            res_share = None
    if (not bn.training) and EVAL_FOLD_BN and not padded and not torch.is_grad_enabled():
        # inference (evaluator.py:255-275): w' = w·γ/σ, b' = β − μ·γ/σ, epilogue = + b' (+ shortcut) → ReLU
        wb, bias = ops.fold_cache.get(conv.weight, bn, stem)
        if stem:
            return ops.conv_stem_fprop_fused(xin, wb, K, bias, relu=bool(relu))
        return ops.conv_fprop_fused(xin, wb, K, ks, conv.stride[0], conv.padding[0], conv.dilation[0], bias,
                                    res=residual, relu=bool(relu))
    return _conv_bn_act_fn(xin, w, bn, Kp, residual, conv.stride[0], conv.padding[0], conv.dilation[0], relu, stem,
                           in_share, res_share)


def conv_plain(x, conv, out_f32=False, ocs=None, pad_out=False):
    """nn.Conv2d (+bias) on the libtsb path. pad_out: keep the output in the 64-padded channel domain (DFN's
    BN-free 1x1 / refine convs); otherwise the output has exactly conv.out_channels channels (classifiers)."""
    xin = _as_act(x)
    w, b = conv.weight, conv.bias
    K = conv.out_channels
    if _ragged(conv, xin) or (pad_out and K % 64 != 0):
        xin, w, b = _pad_layer(xin, w, _ceil_to(xin.shape[1], 64), _ceil_to(K, 64) if pad_out else K, b)
    return ops.ConvFn.apply(xin, w, b, conv.stride[0], conv.padding[0], conv.dilation[0], bool(out_f32), ocs)


class ConvBnRelu(nn.Module):
    """seg_oprs.py:24-46 — same ctor, children named conv / bn / relu"""

    def __init__(self, in_planes, out_planes, ksize, stride, pad, dilation=1, groups=1, has_bn=True,
                 norm_layer=nn.BatchNorm2d, bn_eps=1e-5, has_relu=True, inplace=True, has_bias=False):
        super(ConvBnRelu, self).__init__()
        self.conv = nn.Conv2d(in_planes, out_planes, kernel_size=ksize, stride=stride, padding=pad,
                              dilation=dilation, groups=groups, bias=has_bias)
        self.has_bn = has_bn
        if self.has_bn:
            self.bn = norm_layer(out_planes, eps=bn_eps)
        self.has_relu = has_relu
        if self.has_relu:
            self.relu = nn.ReLU(inplace=inplace)

    def forward(self, x):
        if self.has_bn and self.conv.bias is None:
            return conv_bn_act(x, self.conv, self.bn, self.has_relu)
        y = conv_plain(x, self.conv)
        if self.has_bn:
            raise NotImplementedError("ConvBnRelu with both bias and BN is not on the accelerated path")
        if self.has_relu:
            y = ReluFn.apply(y)
        return y


def _deconv_geometry(conv):
    """(k, stride, pad, dil, out_pad) of an nn.ConvTranspose2d the transposed-conv kernels run (include/tsb.h)"""
    k, st, pd, dl, op = (conv.kernel_size, conv.stride, conv.padding, conv.dilation, conv.output_padding)
    if k[0] != k[1] or st[0] != st[1] or pd[0] != pd[1] or dl[0] != dl[1] or op[0] != op[1]:
        raise NotImplementedError("DeConvBnRelu: non-square kernel, stride, padding, dilation or output padding")
    if conv.groups != 1:
        raise NotImplementedError("DeConvBnRelu: groups > 1 is not on the accelerated path")
    if st[0] not in (1, 2):
        raise NotImplementedError("DeConvBnRelu: stride must be 1 or 2 (got %d)" % st[0])
    if k[0] > 4:
        raise NotImplementedError("DeConvBnRelu: kernel size must be at most 4 (16 taps; got %d)" % k[0])
    if op[0] >= st[0]:
        raise NotImplementedError("DeConvBnRelu: output_padding must be smaller than the stride")
    if not isinstance(pd[0], int):
        raise NotImplementedError("DeConvBnRelu: string padding is not supported")
    return k[0], st[0], pd[0], dl[0], op[0]


def deconv_bn_act(x, conv, bn, relu):
    """nn.ConvTranspose2d → norm_layer(train/eval) → ReLU (bn None: → +bias → ReLU) on the libtsb path. Channel counts
    that are not multiples of 64 run zero-padded to the next multiple, as `_ragged` layers do; the output has exactly
    conv.out_channels channels."""
    k, stride, pad, dil, op = _deconv_geometry(conv)
    xin = _as_act(x)
    w, b = conv.weight, conv.bias
    Ci, Co = conv.in_channels, conv.out_channels
    Cp, Kp = _ceil_to(Ci, 64), _ceil_to(Co, 64)
    padded = Cp != Ci or Kp != Co or xin.shape[1] != Ci
    if padded:
        xin, w, b = _pad_layer(xin, w, Cp, Kp, b, transposed=True)
    if bn is None:
        y = ops.ConvTransposeFn.apply(xin, w, b, stride, pad, dil, op, bool(relu))
    elif b is not None:
        raise NotImplementedError("DeConvBnRelu with both bias and BN is not on the accelerated path")
    elif (not bn.training) and EVAL_FOLD_BN and not padded and not torch.is_grad_enabled():
        # inference: W' = W·γ/σ along Co, b' = β − μ·γ/σ, epilogue = + b' → ReLU
        wt, bias = ops.fold_cache.get(conv.weight, bn, False, transposed=True)
        return ops.conv_transpose_fprop(xin, wt, Co, k, stride, pad, dil, op, bias=bias, relu=bool(relu))
    else:
        y = _conv_bn_act_fn(xin, w, bn, Kp, None, stride, pad, dil, relu, out_pad=op)
    return y[:, :Co] if Kp != Co else y


class DeConvBnRelu(nn.Module):
    """seg_oprs.py:49-73 — same ctor, children named conv (a genuine nn.ConvTranspose2d) / bn / relu. Runs stride 1 or
    2, kernel <= 4, square geometry, groups 1, output_pad < stride; anything else raises NotImplementedError."""

    def __init__(self, in_planes, out_planes, ksize, stride, pad, output_pad, dilation=1, groups=1, has_bn=True,
                 norm_layer=nn.BatchNorm2d, bn_eps=1e-5, has_relu=True, inplace=True, has_bias=False):
        super(DeConvBnRelu, self).__init__()
        self.conv = nn.ConvTranspose2d(in_planes, out_planes, kernel_size=ksize, stride=stride, padding=pad,
                                       output_padding=output_pad, dilation=dilation, groups=groups, bias=has_bias)
        self.has_bn = has_bn
        if self.has_bn:
            self.bn = norm_layer(out_planes, eps=bn_eps)
        self.has_relu = has_relu
        if self.has_relu:
            self.relu = nn.ReLU(inplace=inplace)

    def forward(self, x):
        return deconv_bn_act(x, self.conv, self.bn if self.has_bn else None, self.has_relu)


class SeparableConvBnRelu(nn.Module):
    """seg_oprs.py:76-94 — same ctor, children named conv1 (a genuine depthwise nn.Conv2d) / bn / point_wise_cbr: the
    depthwise conv, BN (batch statistics in training, running statistics in eval; no ReLU), then the pointwise
    ConvBnRelu. Runs the 3x3 depthwise conv at stride 1 with padding = dilation (the atrous separable conv of
    DeepLabV3+), or at stride 2 with padding 1 and dilation 1, over a multiple of 8 channels; anything else raises
    NotImplementedError."""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=0, dilation=1, has_relu=True,
                 norm_layer=nn.BatchNorm2d):
        super(SeparableConvBnRelu, self).__init__()
        self.conv1 = nn.Conv2d(in_channels, in_channels, kernel_size, stride, padding, dilation, groups=in_channels,
                               bias=False)
        self.bn = norm_layer(in_channels)
        self.point_wise_cbr = ConvBnRelu(in_channels, out_channels, 1, 1, 0, has_bn=True, norm_layer=norm_layer,
                                         has_relu=has_relu, has_bias=False)

    def _geometry(self):
        """(stride, dilation) of the depthwise conv the dwconv kernels run (include/tsb.h)"""
        c = self.conv1
        k, st, pd, dl = c.kernel_size, c.stride, c.padding, c.dilation
        if k != (3, 3):
            raise NotImplementedError("SeparableConvBnRelu: only a 3x3 depthwise conv runs on libtsb (got %s)" % (k,))
        if st[0] != st[1] or pd[0] != pd[1] or dl[0] != dl[1] or not isinstance(pd[0], int):
            raise NotImplementedError("SeparableConvBnRelu: non-square stride, padding or dilation")
        if pd[0] != dl[0]:
            raise NotImplementedError("SeparableConvBnRelu: padding must equal the dilation (got %d, %d)" % (pd[0], dl[0]))
        if st[0] not in (1, 2) or (st[0] == 2 and dl[0] != 1):
            raise NotImplementedError("SeparableConvBnRelu: stride 1, or stride 2 at dilation 1 (got stride %d, "
                                      "dilation %d)" % (st[0], dl[0]))
        if c.in_channels % 8 != 0:
            raise NotImplementedError("SeparableConvBnRelu: in_channels must be a multiple of 8 (got %d)" % c.in_channels)
        return st[0], dl[0]

    def forward(self, x):
        stride, dil = self._geometry()
        bn, pw = self.bn, self.point_wise_cbr
        t = ops.DWConvFn.apply(_as_act(x), self.conv1.weight, stride, None, None, dil)
        t = ops.BNFn.apply(t, bn.weight, bn.bias, bn.running_mean, bn.running_var, float(bn.eps), _bn_momentum(bn),
                           bool(bn.training))
        return conv_bn_act(t, pw.conv, pw.bn, pw.has_relu)


class Encoding(nn.Module):
    """EncNet's Context Encoding layer (Zhang et al., CVPR 2018): K codewords c_k ([K, D], `codewords`) with smoothing
    factors s_k ([K], `scale`); E_bk = Σ_i a_ik (x_i − c_k) over the pixels x_i of image b with a_ik = softmax_k(s_k
    ‖x_i − c_k‖²). Input [B, D, h, w]; output the bf16 NHWC [B, K, D, 1]. Runs on tsb_encoding_{fwd,bwd}: K a multiple
    of 8 and at most 32, D a multiple of 64 (include/tsb.h); under no_grad nothing is saved for a backward."""

    def __init__(self, D, K):
        super(Encoding, self).__init__()
        self.D, self.K = D, K
        self.codewords = nn.Parameter(torch.empty(K, D, dtype=torch.float))
        self.scale = nn.Parameter(torch.empty(K, dtype=torch.float))
        self.reset_params()

    def reset_params(self):
        std = 1.0 / (self.K * self.D) ** 0.5
        self.codewords.data.uniform_(-std, std)
        self.scale.data.uniform_(-1, 0)

    def forward(self, x):
        x = _as_act(x)
        if torch.is_grad_enabled():
            return ops.EncodingFn.apply(x, self.codewords, self.scale)
        return ops.encoding_infer(x, self.codewords, self.scale)


class SelfAttentionBlock(nn.Module):
    """OCNet's object-context self-attention (Yuan & Wang, OCNet, `_SelfAttentionBlock` at scale 1): f_key, a 1x1
    ConvBnRelu, gives both the queries and the keys (one child, so its parameters appear once), f_value a 1x1 conv with
    bias, and W a 1x1 conv with bias, zero-initialised as in OCNet. forward(x) = W(softmax(k kᵀ / √key_channels) v) with
    k = f_key(x), v = f_value(x), the attention over the h·w pixels of each image on ops.AttentionFn (key_channels =
    value_channels = 256). f_key runs once per forward, so its BatchNorm running statistics get one update."""

    def __init__(self, in_channels, key_channels, value_channels, out_channels=None, scale=1,
                 norm_layer=nn.BatchNorm2d):
        super(SelfAttentionBlock, self).__init__()
        if scale > 1:
            raise NotImplementedError("SelfAttentionBlock: scale > 1 (the pooled variants of OCNet) is not implemented")
        self.scale = scale
        self.in_channels = in_channels
        self.key_channels = key_channels
        self.value_channels = value_channels
        self.out_channels = in_channels if out_channels is None else out_channels
        self.f_key = ConvBnRelu(in_channels, key_channels, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                                norm_layer=norm_layer)
        self.f_value = nn.Conv2d(in_channels, value_channels, kernel_size=1)
        self.W = nn.Conv2d(value_channels, self.out_channels, kernel_size=1)
        nn.init.constant_(self.W.weight, 0)
        nn.init.constant_(self.W.bias, 0)

    def forward(self, x):
        x = _as_act(x)
        key = self.f_key(x)
        value = conv_plain(x, self.f_value)
        context = ops.AttentionFn.apply(key, None, value, self.key_channels ** -0.5)
        return conv_plain(context, self.W)


class BaseOCModule(nn.Module):
    """OCNet's Base-OC module (`BaseOC_Module`): the sum of the `stages` (SelfAttentionBlock) concatenated in front of
    the input, then `conv_bn_dropout` = 1x1 ConvBnRelu(2·in → out) and Dropout2d"""

    def __init__(self, in_channels, out_channels, key_channels, value_channels, dropout, sizes=(1,),
                 norm_layer=nn.BatchNorm2d):
        super(BaseOCModule, self).__init__()
        self.stages = nn.ModuleList([SelfAttentionBlock(in_channels, key_channels, value_channels, out_channels, size,
                                                        norm_layer) for size in sizes])
        self.conv_bn_dropout = nn.Sequential(
            ConvBnRelu(2 * in_channels, out_channels, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                       norm_layer=norm_layer),
            nn.Dropout2d(dropout))

    def forward(self, feats):
        from ..networks.pspnet import _dropout2d
        feats = _as_act(feats)
        context = self.stages[0](feats)
        for stage in self.stages[1:]:
            context = ops.AddFn.apply(context, stage(feats))
        out = self.conv_bn_dropout[0](ops.ConcatFn.apply(context, feats))
        return _dropout2d(out, self.conv_bn_dropout[1].p, self.training)


class SpatialGatherModule(nn.Module):
    """OCRNet's object-region proxy (Yuan, Chen & Wang, "Object-Contextual Representations for Semantic Segmentation",
    the SpatialGather module at scale 1): forward(f, l) = ctx with ctx[b, :, k] = Σ_n softmax_n(l[b, k, n]) · f[b, :, n],
    the soft-max over the h·w pixels of image b, shaped [B, C, K, 1]. f: the features [B, C, h, w], l: the fp32 aux
    logits [B, K, h, w]. No parameters; on ops.SpatialGatherFn."""

    def __init__(self, cls_num=0, scale=1):
        super(SpatialGatherModule, self).__init__()
        if scale != 1:
            raise NotImplementedError("SpatialGatherModule: scale != 1 is not implemented")
        self.cls_num = cls_num
        self.scale = scale

    def forward(self, feats, probs):
        return ops.SpatialGatherFn.apply(_as_act(feats), probs, int(probs.shape[1]))


def _cbr1x1(cin, cout, norm_layer):
    return ConvBnRelu(cin, cout, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer)


class ObjectAttentionBlock(nn.Module):
    """OCRNet's pixel-region relation (`ObjectAttentionBlock2D` at scale 1): f_pixel and f_object are two 1x1
    ConvBnRelu each (in → key → key), f_down and f_up one 1x1 ConvBnRelu each (in → key, key → in).
    forward(x, proxy) = f_up(softmax_k(f_pixel(x) · f_object(proxy)ᵀ / √key) · f_down(proxy)): every pixel attends over
    the K object regions of its image, on ops.AttentionFn's cross form (key_channels = 256)."""

    def __init__(self, in_channels, key_channels, scale=1, norm_layer=nn.BatchNorm2d):
        super(ObjectAttentionBlock, self).__init__()
        if scale > 1:
            raise NotImplementedError("ObjectAttentionBlock: scale > 1 (OCR's pooled form) is not implemented")
        self.scale = scale
        self.in_channels = in_channels
        self.key_channels = key_channels
        self.f_pixel = nn.Sequential(_cbr1x1(in_channels, key_channels, norm_layer),
                                     _cbr1x1(key_channels, key_channels, norm_layer))
        self.f_object = nn.Sequential(_cbr1x1(in_channels, key_channels, norm_layer),
                                      _cbr1x1(key_channels, key_channels, norm_layer))
        self.f_down = _cbr1x1(in_channels, key_channels, norm_layer)
        self.f_up = _cbr1x1(key_channels, in_channels, norm_layer)

    def forward(self, x, proxy):
        x, proxy = _as_act(x), _as_act(proxy)
        query = self.f_pixel(x)
        key = self.f_object(proxy)
        value = self.f_down(proxy)
        return self.f_up(ops.AttentionFn.apply(query, key, value, self.key_channels ** -0.5))


class SpatialOCRModule(nn.Module):
    """OCRNet's object-contextual representation (`SpatialOCR_Module`): the ObjectAttentionBlock's context concatenated
    in front of the input, then `conv_bn_dropout` = 1x1 ConvBnRelu(2·in → out) and Dropout2d"""

    def __init__(self, in_channels, key_channels, out_channels, scale=1, dropout=0.1, norm_layer=nn.BatchNorm2d):
        super(SpatialOCRModule, self).__init__()
        self.object_context_block = ObjectAttentionBlock(in_channels, key_channels, scale, norm_layer)
        self.conv_bn_dropout = nn.Sequential(_cbr1x1(2 * in_channels, out_channels, norm_layer), nn.Dropout2d(dropout))

    def forward(self, feats, proxy_feats):
        from ..networks.pspnet import _dropout2d
        feats = _as_act(feats)
        context = self.object_context_block(feats, proxy_feats)
        out = self.conv_bn_dropout[0](ops.ConcatFn.apply(context, feats))
        return _dropout2d(out, self.conv_bn_dropout[1].p, self.training)


class DenseAsppBlock(nn.Module):
    """One pre-activation atrous layer of DenseASPP (Yang et al., CVPR 2018): pre_bn → ReLU → `reduce` (1x1 ConvBnRelu,
    in → mid) → the dilated 3x3 `conv` (mid → out, bias) → Dropout2d(dropout). bn_start=False drops pre_bn (and its
    ReLU): the first block's input is already post-ReLU. Children in checkpoint order: pre_bn, reduce, conv. The block
    runs inside DenseASPPModule, which shares one concatenated buffer and its statistics between all blocks."""

    def __init__(self, in_planes, mid_planes, out_planes, dilation, dropout=0.1, bn_start=True,
                 norm_layer=nn.BatchNorm2d):
        super(DenseAsppBlock, self).__init__()
        self.pre_bn = norm_layer(in_planes) if bn_start else None
        self.reduce = ConvBnRelu(in_planes, mid_planes, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False,
                                 norm_layer=norm_layer)
        self.conv = nn.Conv2d(mid_planes, out_planes, 3, padding=dilation, dilation=dilation, bias=True)
        self.dropout = dropout


class DenseASPPModule(nn.Module):
    """DenseASPP's densely connected atrous head: block i reads in_planes + i·out_planes channels, the input and every
    earlier block's output, and the module returns [a_{n-1} | ... | a_1 | a_0 | x] (DenseASPP's `cat((new, feature))`
    order; 2688 channels at the defaults). Every block's input is a contiguous suffix of ONE NHWC buffer that the 3x3
    convs write their slices into, so there are no concatenation copies, and every pre_bn normalises that suffix in the
    input prologue of its 1x1 conv (tsb_conv1x1_bnrelu_*): no normalised copy of it is ever written. The per-channel
    batch statistics of the buffer are taken once per slice and shared by all pre_bn layers (each keeps its own γ, β
    and running statistics). Training runs on ops.DenseAsppFn; eval applies pre_bn from its running statistics in the
    same prologue and folds reduce's BatchNorm into the 1x1 conv (bias + ReLU epilogue). Block 0 has no pre_bn (its
    input, layer4's output, is post-ReLU). Channel counts must be multiples of 64."""

    def __init__(self, in_planes=2048, mid_planes=512, out_planes=128, rates=(3, 6, 12, 18, 24), dropout=0.1,
                 norm_layer=nn.BatchNorm2d):
        super(DenseASPPModule, self).__init__()
        for c in (in_planes, mid_planes, out_planes):
            if c % 64 != 0:
                raise NotImplementedError("DenseASPPModule: channel counts must be multiples of 64 (got %d)" % c)
        self.blocks = nn.ModuleList([
            DenseAsppBlock(in_planes + i * out_planes, mid_planes, out_planes, d, dropout, bn_start=i > 0,
                           norm_layer=norm_layer) for i, d in enumerate(rates)])
        self.out_channels = in_planes + len(rates) * out_planes

    def forward(self, x):
        x = _as_act(x)
        p = self.blocks[0].dropout if self.training else 0.0
        if self.training:
            params = [q for blk in self.blocks for q in ops._dense_block_params(blk)]
            return ops.DenseAsppFn.apply(x, self, float(p), *params)
        return self._infer(x)

    @torch.no_grad()
    def _infer(self, x):
        """eval: running statistics, reduce's BatchNorm folded into its conv, no normalised copy"""
        N, Cx, H, W = x.shape
        nb, oc = len(self.blocks), self.blocks[0].conv.out_channels
        Ct = Cx + nb * oc
        cat = ops.nhwc_empty(N, Ct, H, W, device=x.device)
        cat[:, nb * oc:].copy_(x)
        for i, blk in enumerate(self.blocks):
            off = (nb - i) * oc
            xin = cat[:, off:]
            red = blk.reduce
            wb, bias = ops.fold_cache.get(red.conv.weight, red.bn, False)
            if blk.pre_bn is None:
                y = ops.conv_fprop_fused(xin, wb, red.conv.out_channels, 1, 1, 0, 1, bias, relu=True)
            else:
                pb = blk.pre_bn
                pre = torch.empty((4, Ct - off), dtype=torch.float32, device=x.device)
                ops._bn_finalize(pre, None, 1.0, pb.weight, pb.bias, pb.running_mean, pb.running_var, float(pb.eps),
                                 0.0, False)
                y = ops.conv1x1_bnrelu_fprop(xin, pre, wb, red.conv.out_channels, bias=bias, relu=True)
            wb3, _ = ops.pack_cache.get(blk.conv.weight, False)
            d = blk.conv.dilation[0]
            ops.conv_fprop(y, wb3, oc, 3, 1, d, d, bias=blk.conv.bias, out=cat[:, off - oc:off])
        return cat


class PAM_Module(nn.Module):
    """DANet's position attention module (Fu et al., "Dual Attention Network for Scene Segmentation", `PAM_Module`):
    query_conv and key_conv are 1x1 convs in_dim → in_dim/8 with bias, value_conv a 1x1 conv in_dim → in_dim with bias,
    gamma a zero-initialised scalar. forward(x) = gamma · softmax(q kᵀ) v + x over the h·w pixels of each image, with
    no 1/√d scale; the attention runs on ops.AttentionFn at (d_k, d_v) = (in_dim/8, in_dim), which the kernels implement
    for in_dim = 512."""

    def __init__(self, in_dim):
        super(PAM_Module, self).__init__()
        self.query_conv = nn.Conv2d(in_dim, in_dim // 8, kernel_size=1)
        self.key_conv = nn.Conv2d(in_dim, in_dim // 8, kernel_size=1)
        self.value_conv = nn.Conv2d(in_dim, in_dim, kernel_size=1)
        self.gamma = nn.Parameter(torch.zeros(1))

    def forward(self, x):
        x = _as_act(x)
        out = ops.AttentionFn.apply(conv_plain(x, self.query_conv), conv_plain(x, self.key_conv),
                                    conv_plain(x, self.value_conv), 1.0)
        return ops.GammaResidualFn.apply(x, out, self.gamma)


class CAM_Module(nn.Module):
    """DANet's channel attention module (`CAM_Module`): forward(x) = gamma · A X + x with A = softmax_row(rowmax(E) − E),
    E = X Xᵀ over the C channels of each image (X is [C, h·w]), gamma a zero-initialised scalar; no convolutions. On
    ops.ChannelAttentionFn and ops.GammaResidualFn."""

    def __init__(self, in_dim):
        super(CAM_Module, self).__init__()
        self.gamma = nn.Parameter(torch.zeros(1))

    def forward(self, x):
        x = _as_act(x)
        return ops.GammaResidualFn.apply(x, ops.ChannelAttentionFn.apply(x), self.gamma)


class ReluFn(torch.autograd.Function):
    """stand-alone ReLU on a small tensor (FFM squeeze branch [N,C,1,1], seg_oprs.py:224-226): expressed through
    tsb_bn_apply with scale 1 / shift 0 so it stays on the library path"""

    @staticmethod
    def forward(ctx, x):
        N, C, H, W = x.shape
        one = torch.ones(C, dtype=torch.float32, device=x.device)
        zero = torch.zeros(C, dtype=torch.float32, device=x.device)
        y = ops.nhwc_empty(N, C, H, W, device=x.device)
        ops.call("tsb_bn_apply", ops.ptr(x), ops.cs_of(x), ops.ptr(one), ops.ptr(zero), None, 0, 1, ops.ptr(y), C,
                 N * H * W, C, ops.stream())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return dy * (y > 0).to(dy.dtype)


class AttentionRefinement(nn.Module):
    """seg_oprs.py:192-212: fm = CBR3x3(x); fm * sigmoid(BN(conv1x1(GAP(fm)))).
    forward(x, add=None) additionally fuses the caller's `fm += last_fm` (bisenet network.py:91-92)."""

    def __init__(self, in_planes, out_planes, norm_layer=nn.BatchNorm2d):
        super(AttentionRefinement, self).__init__()
        self.conv_3x3 = ConvBnRelu(in_planes, out_planes, 3, 1, 1, has_bn=True, norm_layer=norm_layer,
                                   has_relu=True, has_bias=False)
        self.channel_attention = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            ConvBnRelu(out_planes, out_planes, 1, 1, 0, has_bn=True, norm_layer=norm_layer, has_relu=False,
                       has_bias=False),
            nn.Sigmoid())

    def forward(self, x, add=None):
        fm = self.conv_3x3(x)
        pooled = ops.AdaptiveAvgPoolFn.apply(fm, 1)
        a = self.channel_attention[1](pooled)  # pre-sigmoid logit; the sigmoid is fused into the scale kernel
        return ops.ChanScaleFn.apply(fm, a, None if add is None else _as_act(add), 0.0)


class FeatureFusion(nn.Module):
    """seg_oprs.py:215-238: fm = CBR1x1(cat[x1,x2]); fm + fm*sigmoid(conv1x1(relu(conv1x1(GAP(fm)))))"""

    def __init__(self, in_planes, out_planes, reduction=1, norm_layer=nn.BatchNorm2d):
        super(FeatureFusion, self).__init__()
        self.conv_1x1 = ConvBnRelu(in_planes, out_planes, 1, 1, 0, has_bn=True, norm_layer=norm_layer,
                                   has_relu=True, has_bias=False)
        self.channel_attention = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            ConvBnRelu(out_planes, out_planes // reduction, 1, 1, 0, has_bn=False, norm_layer=norm_layer,
                       has_relu=True, has_bias=False),
            ConvBnRelu(out_planes // reduction, out_planes, 1, 1, 0, has_bn=False, norm_layer=norm_layer,
                       has_relu=False, has_bias=False),
            nn.Sigmoid())

    def forward(self, x1, x2):
        fm = ops.ConcatFn.apply(_as_act(x1), _as_act(x2))
        fm = self.conv_1x1(fm)
        pooled = ops.AdaptiveAvgPoolFn.apply(fm, 1)
        a = self.channel_attention[2](self.channel_attention[1](pooled))
        return ops.ChanScaleFn.apply(fm, a, None, 1.0)


class AddReluFn(torch.autograd.Function):
    """relu(a + b) in one pass (tsb_add_relu); the backward mask comes from the saved output"""

    @staticmethod
    def forward(ctx, a, b):
        N, C, H, W = a.shape
        y = ops.nhwc_empty(N, C, H, W, device=a.device)
        ops.call("tsb_add_relu", ops.ptr(a), ops.cs_of(a), ops.ptr(b), ops.cs_of(b), ops.ptr(y), C, N * H * W, C,
                 ops.stream())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        N, C, H, W = y.shape
        dy = ops.as_nhwc_bf16(dy)
        dx = ops.nhwc_empty(N, C, H, W, device=y.device)
        ops.call("tsb_relu_bwd", ops.ptr(dy), ops.cs_of(dy), ops.ptr(y), C, ops.ptr(dx), C, N * H * W, C, ops.stream())
        return dx, dx


def _residual_tail(t, x, has_relu):
    return AddReluFn.apply(t, x) if has_relu else ops.AddFn.apply(t, x)


class SELayer(nn.Module):
    """seg_oprs.py:110-126 — GAP → Linear → ReLU → Linear → Sigmoid. The two nn.Linear layers keep their names
    (fc.0 / fc.2, checkpoint keys) and run as 1x1 convolutions over the [N,C,1,1] pooled tensor."""

    def __init__(self, in_planes, out_planes, reduction=16):
        super(SELayer, self).__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(
            nn.Linear(in_planes, out_planes // reduction),
            nn.ReLU(inplace=True),
            nn.Linear(out_planes // reduction, out_planes),
            nn.Sigmoid())
        self.out_planes = out_planes

    @staticmethod
    def _linear(y, lin):
        K, C = lin.weight.shape
        return ops.ConvFn.apply(y, lin.weight.view(K, C, 1, 1), lin.bias, 1, 0, 1, False, None)

    def logits_from_pooled(self, pooled):
        """pre-sigmoid attention logit [N,out,1,1] from the pooled [N,in,1,1] descriptor"""
        y = self._linear(pooled, self.fc[0])
        y = ReluFn.apply(y)
        return self._linear(y, self.fc[2])

    def forward(self, x):
        pooled = ops.AdaptiveAvgPoolFn.apply(_as_act(x), 1)
        return torch.sigmoid(self.logits_from_pooled(pooled).float())


class ChannelAttention(nn.Module):
    """seg_oprs.py:129-140 (DFN's CAB): fm = x1 * SE(cat[x1, x2]) + x2. GAP(cat[x1,x2]) = cat[GAP(x1), GAP(x2)], so
    the 2C-channel concatenation is never materialised; sigmoid, scale and `+ x2` are one kernel."""

    def __init__(self, in_planes, out_planes, reduction):
        super(ChannelAttention, self).__init__()
        self.channel_attention = SELayer(in_planes, out_planes, reduction)

    def forward(self, x1, x2):
        x1, x2 = _as_act(x1), _as_act(x2)
        pooled = ops.ConcatFn.apply(ops.AdaptiveAvgPoolFn.apply(x1, 1), ops.AdaptiveAvgPoolFn.apply(x2, 1))
        a = self.channel_attention.logits_from_pooled(pooled)
        return ops.ChanScaleFn.apply(x1, a, x2, 0.0)


class BNRefine(nn.Module):
    """seg_oprs.py:143-162"""

    def __init__(self, in_planes, out_planes, ksize, has_bias=False, has_relu=False, norm_layer=nn.BatchNorm2d,
                 bn_eps=1e-5):
        super(BNRefine, self).__init__()
        self.conv_bn_relu = ConvBnRelu(in_planes, out_planes, ksize, 1, ksize // 2, has_bias=has_bias,
                                       norm_layer=norm_layer, bn_eps=bn_eps)
        self.conv_refine = nn.Conv2d(out_planes, out_planes, kernel_size=ksize, stride=1, padding=ksize // 2,
                                     dilation=1, bias=has_bias)
        self.has_relu = has_relu
        if self.has_relu:
            self.relu = nn.ReLU(inplace=False)

    def forward(self, x):
        x = _as_act(x)
        t = self.conv_bn_relu(x)
        t = conv_plain(t, self.conv_refine, pad_out=True)
        if x.shape[1] != t.shape[1]:
            x = _pad_act(x, t.shape[1])
        return _residual_tail(t, x, self.has_relu)


class RefineResidual(nn.Module):
    """seg_oprs.py:165-188 (DFN's RRB): x = conv1x1(x); relu?(conv3x3(CBR3x3(x)) + x)"""

    def __init__(self, in_planes, out_planes, ksize, has_bias=False, has_relu=False, norm_layer=nn.BatchNorm2d,
                 bn_eps=1e-5):
        super(RefineResidual, self).__init__()
        self.conv_1x1 = nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=1, padding=0, dilation=1,
                                  bias=has_bias)
        self.cbr = ConvBnRelu(out_planes, out_planes, ksize, 1, ksize // 2, has_bias=has_bias,
                              norm_layer=norm_layer, bn_eps=bn_eps)
        self.conv_refine = nn.Conv2d(out_planes, out_planes, kernel_size=ksize, stride=1, padding=ksize // 2,
                                     dilation=1, bias=has_bias)
        self.has_relu = has_relu
        if self.has_relu:
            self.relu = nn.ReLU(inplace=False)

    def forward(self, x):
        x = conv_plain(x, self.conv_1x1, pad_out=True)
        t = self.cbr(x)
        t = conv_plain(t, self.conv_refine, pad_out=True)
        return _residual_tail(t, x, self.has_relu)


class GlobalAvgPool2d(nn.Module):
    """seg_oprs.py:97-107"""

    def forward(self, inputs):
        return ops.AdaptiveAvgPoolFn.apply(_as_act(inputs), 1)


def upsample_bilinear(x, size):
    """F.interpolate(x, size=size, mode='bilinear', align_corners=True) on the libtsb path"""
    return ops.BilinearFn.apply(_as_act(x), int(size[0]), int(size[1]))
