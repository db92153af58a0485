"""ORACLE — test infrastructure only.

Functional fp32 PyTorch restatement of the reference modules on the training-step hot path, driven by a
state_dict that uses the REFERENCE's key names (SURVEY.md App. D), so weights can be exchanged both ways.
Each function cites the reference lines it restates. Pinned against the live reference modules by
tests/test_oracle_vs_reference.py (authoring container) and tests/golden/*.

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------------
# optional bf16-storage emulation: the SAME fp32 math, but values are rounded to bf16 (forward AND the
# gradient flowing back) at the points where the libtsb path stores bf16 — conv weights, raw conv outputs,
# activations, pooled / resized maps. Separates "kernel bug" from "bf16 storage policy" in end-to-end tests.
# --------------------------------------------------------------------------------------------------
class _RoundBF16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(torch.float32)


_EMULATE = {"on": False}


def set_bf16_emulation(on):
    _EMULATE["on"] = bool(on)


def q(t):
    return _RoundBF16.apply(t) if _EMULATE["on"] else t


def qw(w):
    """weights are rounded in the forward only (the fp32 master weight receives the fp32 gradient)"""
    return (w + (w.to(torch.bfloat16).to(torch.float32) - w).detach()) if _EMULATE["on"] else w


# --------------------------------------------------------------------------------------------------
# ProbOhemCrossEntropy2d.forward — TorchSeg furnace/seg_opr/loss_opr.py:68-98
# (with `1 - mask` → `~mask`, the torch>=1.2 shim of SURVEY.md App. C2)
# --------------------------------------------------------------------------------------------------
def ohem_ce(pred, target, ignore_label=255, thresh=0.7, min_kept=256, weight=None, return_aux=False):
    b, c, h, w = pred.shape
    target = target.reshape(-1)
    valid_mask = target.ne(ignore_label)                                   # :70
    target = target * valid_mask.long()                                    # :71
    num_valid = int(valid_mask.sum())                                      # :72
    prob = F.softmax(pred, dim=1)                                          # :75
    prob = prob.transpose(0, 1).reshape(c, -1)                             # :76
    threshold = thresh
    if min_kept > num_valid:                                               # :78
        pass
    elif num_valid > 0:                                                    # :80
        prob = prob.masked_fill(~valid_mask, 1)                            # :81
        mask_prob = prob[target, torch.arange(len(target), dtype=torch.long, device=pred.device)]  # :82-83
        if min_kept > 0:                                                   # :85
            _, index = torch.sort(mask_prob)                               # :86
            threshold_index = index[min(len(index), min_kept) - 1]         # :87
            if mask_prob[threshold_index] > thresh:                        # :88
                threshold = float(mask_prob[threshold_index])
            kept_mask = mask_prob.le(threshold)                            # :90
            target = target * kept_mask.long()
            valid_mask = valid_mask * kept_mask
    target = target.masked_fill(~valid_mask, ignore_label)                 # :95
    target = target.view(b, h, w)
    loss = F.cross_entropy(pred, target, weight=weight, ignore_index=ignore_label)  # :98
    if return_aux:
        return loss, valid_mask, threshold
    return loss


# SigmoidFocalLoss.forward — loss_opr.py:23-45
def sigmoid_focal(pred, target, ignore_label, gamma=2.0, alpha=0.25):
    b = target.shape[0]
    pred = pred.reshape(b, -1, 1)
    s = pred.sigmoid()
    t = target.reshape(b, -1).float()
    mask = t.ne(ignore_label).float()
    t = mask * t
    onehot = t.view(b, -1, 1)
    max_val = (-s).clamp(min=0)
    pos = (1 - s) ** gamma * (s - s * onehot)
    neg = s ** gamma * (max_val + ((-max_val).exp() + (-s - max_val).exp()).log())
    loss = -(alpha * pos + (1 - alpha) * neg).sum(dim=-1) * mask
    return loss.mean()


# --------------------------------------------------------------------------------------------------
# building blocks
# --------------------------------------------------------------------------------------------------
def _bn(x, sd, prefix, eps, momentum, training, stats=None):
    rm = sd.get(prefix + ".running_mean") if stats is None else stats.setdefault(prefix + ".running_mean", sd[prefix + ".running_mean"].clone())
    rv = sd.get(prefix + ".running_var") if stats is None else stats.setdefault(prefix + ".running_var", sd[prefix + ".running_var"].clone())
    if training and stats is None:
        rm = rv = None  # pure batch statistics; running stats untouched
    return F.batch_norm(x, rm, rv, sd[prefix + ".weight"], sd[prefix + ".bias"], training, momentum, eps)


def conv_bn_relu(x, sd, prefix, stride, pad, dilation=1, has_bn=True, has_relu=True, eps=1e-5, momentum=0.1,
                 training=True, stats=None):
    """ConvBnRelu.forward — TorchSeg furnace/seg_opr/seg_oprs.py:39-46"""
    x = q(F.conv2d(x, qw(sd[prefix + ".conv.weight"]), sd.get(prefix + ".conv.bias"), stride, pad, dilation))
    if has_bn:
        x = _bn(x, sd, prefix + ".bn", eps, momentum, training, stats)
    if has_relu:
        x = F.relu(x)
    return q(x)


def basic_block(x, sd, prefix, stride, has_down, eps, momentum, training, stats=None):
    """BasicBlock.forward — TorchSeg furnace/base_model/resnet.py:33-53"""
    out = q(F.conv2d(x, qw(sd[prefix + ".conv1.weight"]), None, stride, 1))
    out = q(F.relu(_bn(out, sd, prefix + ".bn1", eps, momentum, training, stats)))
    out = q(F.conv2d(out, qw(sd[prefix + ".conv2.weight"]), None, 1, 1))
    out = _bn(out, sd, prefix + ".bn2", eps, momentum, training, stats)
    residual = x
    if has_down:
        residual = q(F.conv2d(x, qw(sd[prefix + ".downsample.0.weight"]), None, stride, 0))
        residual = q(_bn(residual, sd, prefix + ".downsample.1", eps, momentum, training, stats))
    return q(F.relu(out + residual))


def resnet18(x, sd, prefix, eps, momentum, training, stats=None):
    """ResNet.forward (deep_stem=False, BasicBlock [2,2,2,2]) — resnet.py:126-184"""
    x = q(F.conv2d(q(x), qw(sd[prefix + ".conv1.weight"]), None, 2, 3))
    x = q(F.relu(_bn(x, sd, prefix + ".bn1", eps, momentum, training, stats)))
    x = F.max_pool2d(x, 3, 2, 1)
    blocks = []
    for li, stride in ((1, 1), (2, 2), (3, 2), (4, 2)):
        for bi in range(2):
            st = stride if bi == 0 else 1
            has_down = bi == 0 and li > 1
            x = basic_block(x, sd, "%s.layer%d.%d" % (prefix, li, bi), st, has_down, eps, momentum, training, stats)
        blocks.append(x)
    return blocks


def attention_refinement(x, sd, prefix, eps, momentum, training, stats=None):
    """AttentionRefinement.forward — seg_oprs.py:207-212"""
    fm = conv_bn_relu(x, sd, prefix + ".conv_3x3", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    se = q(F.adaptive_avg_pool2d(fm, 1))
    se = conv_bn_relu(se, sd, prefix + ".channel_attention.1", 1, 0, has_relu=False, eps=eps, momentum=momentum,
                      training=training, stats=stats)
    return fm * torch.sigmoid(se)  # rounded by the caller after `+ last_fm` (one fused kernel on the libtsb path)


def feature_fusion(x1, x2, sd, prefix, eps, momentum, training, stats=None):
    """FeatureFusion.forward — seg_oprs.py:233-238"""
    fm = torch.cat([x1, x2], dim=1)
    fm = conv_bn_relu(fm, sd, prefix + ".conv_1x1", 1, 0, eps=eps, momentum=momentum, training=training, stats=stats)
    se = q(F.adaptive_avg_pool2d(fm, 1))
    se = conv_bn_relu(se, sd, prefix + ".channel_attention.1", 1, 0, has_bn=False, has_relu=True)
    se = conv_bn_relu(se, sd, prefix + ".channel_attention.2", 1, 0, has_bn=False, has_relu=False)
    return q(fm + fm * torch.sigmoid(se))


def bisenet_head_logits(x, sd, prefix, eps, momentum, training, stats=None):
    """BiSeNetHead.forward up to the low-resolution logits — bisenet network.py:162-163"""
    fm = conv_bn_relu(x, sd, prefix + ".conv_3x3", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    return F.conv2d(fm, qw(sd[prefix + ".conv_1x1.weight"]), sd[prefix + ".conv_1x1.bias"])  # fp32 logits


def bisenet_r18_forward(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None):
    """BiSeNet.forward wiring — TorchSeg model/bisenet/cityscapes.bisenet.R18/network.py:75-111.
    Returns the three LOW-resolution logit tensors (aux0 @1/16 scale 16, aux1 @1/8, main @1/8) and features."""
    kw = dict(eps=eps, momentum=momentum, training=training, stats=stats)
    sp = conv_bn_relu(q(data), sd, "spatial_path.conv_7x7", 2, 3, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_1", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_3x3_2", 2, 1, **kw)
    sp = conv_bn_relu(sp, sd, "spatial_path.conv_1x1", 1, 0, **kw)
    blocks = resnet18(data, sd, "context_path", eps, momentum, training, stats)
    blocks = blocks[::-1]
    gc = q(F.adaptive_avg_pool2d(blocks[0], 1))
    gc = conv_bn_relu(gc, sd, "global_context.1", 1, 0, **kw)
    gc = q(F.interpolate(gc, size=blocks[0].shape[2:], mode="bilinear", align_corners=True))
    last = gc
    pred_out = []
    for i in range(2):
        fm = attention_refinement(blocks[i], sd, "arms.%d" % i, eps, momentum, training, stats)
        fm = q(fm + last)
        last = q(F.interpolate(fm, size=blocks[i + 1].shape[2:], mode="bilinear", align_corners=True))
        last = conv_bn_relu(last, sd, "refines.%d" % i, 1, 1, **kw)
        pred_out.append(last)
    ffm = feature_fusion(sp, last, sd, "ffm", eps, momentum, training, stats)
    pred_out.append(ffm)
    lo = [bisenet_head_logits(pred_out[i], sd, "heads.%d" % i, eps, momentum, training, stats) for i in range(3)]
    return lo, pred_out


def bisenet_r18_loss(data, label, sd, min_kept, ignore_label=255, thresh=0.7, eps=1e-5, momentum=0.1, stats=None):
    """training branch of BiSeNet.forward — network.py:103-109: main + aux0 + aux1, heads upsample x16/x8/x8"""
    lo, _ = bisenet_r18_forward(data, sd, eps, momentum, True, stats)
    scales = (16, 8, 8)
    losses = []
    for l, s in zip(lo, scales):
        up = F.interpolate(l, scale_factor=s, mode="bilinear", align_corners=True)
        losses.append(ohem_ce(up, label, ignore_label, thresh, min_kept))
    return losses[2] + losses[0] + losses[1], lo


# --------------------------------------------------------------------------------------------------
# BASELINE configs[0]: FCN-32s on a ResNet-18 backbone (plumbing case, CPU) — the reference ships FCN with
# R101_v1c (TorchSeg model/fcn/voc.fcn32s.R101_v1c/network.py:13-68); the R18 variant keeps the same
# head/loss wiring with resnet18(deep_stem=False) and heads _FCNHead(512,.) / _FCNHead(256,.) (SURVEY §8 a15).
# Dropout2d(0.1) is disabled (p=0) so the case is deterministic.
# --------------------------------------------------------------------------------------------------
def fcn_head(x, sd, prefix, eps, momentum, training):
    """_FCNHead.forward — fcn network.py:52-68: 3x3 CBR (C/4) → Dropout2d → 1x1 (+bias)"""
    fm = conv_bn_relu(x, sd, prefix + ".cbr", 1, 1, eps=eps, momentum=momentum, training=training)
    return F.conv2d(fm, sd[prefix + ".conv1x1.weight"], sd[prefix + ".conv1x1.bias"])


def fcn_r18_loss(data, label, sd, aux_ratio=0.5, ignore_label=255, eps=1e-5, momentum=0.1):
    """FCN.forward training branch — fcn network.py:33-47: bilinear x32 (aux x16), CE, loss + 0.5*aux"""
    blocks = resnet18(data, sd, "backbone", eps, momentum, True)
    fm = fcn_head(blocks[-1], sd, "head", eps, momentum, True)
    pred = F.interpolate(fm, scale_factor=32, mode="bilinear", align_corners=True)
    aux = fcn_head(blocks[-2], sd, "aux_head", eps, momentum, True)
    aux = F.interpolate(aux, scale_factor=16, mode="bilinear", align_corners=True)
    loss = F.cross_entropy(pred, label, ignore_index=ignore_label)
    return loss + aux_ratio * F.cross_entropy(aux, label, ignore_index=ignore_label)


def fcn_r101_loss(data, label, sd, layers=(3, 4, 23, 3), aux_ratio=0.5, ignore_label=255, eps=1e-5, momentum=0.1,
                  stats=None):
    """FCN.forward training branch with the shipped backbone — fcn network.py:13-47: resnet101(deep_stem=True,
    stem_width=64), plain output-stride-32 trunk, _FCNHead(2048) x32 and _FCNHead(1024) x16, CE, loss + 0.5*aux
    (Dropout2d(0.1) disabled in the parity runs)"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, True, stats, dilated=False)

    def head(x, prefix):
        fm = conv_bn_relu(x, sd, prefix + ".cbr", 1, 1, eps=eps, momentum=momentum, training=True, stats=stats)
        return F.conv2d(fm, qw(sd[prefix + ".conv1x1.weight"]), sd[prefix + ".conv1x1.bias"])

    lo, lo_aux = head(blocks[-1], "head"), head(blocks[-2], "aux_head")
    pred = F.interpolate(lo, scale_factor=32, mode="bilinear", align_corners=True)
    aux = F.interpolate(lo_aux, scale_factor=16, mode="bilinear", align_corners=True)
    loss = F.cross_entropy(pred, label, ignore_index=ignore_label)
    return loss + aux_ratio * F.cross_entropy(aux, label, ignore_index=ignore_label), (lo, lo_aux)


# --------------------------------------------------------------------------------------------------
# PSPNet-R101_v1c dilated-8 — TorchSeg model/pspnet/ade.pspnet.R101_v1c/network.py:14-109
# --------------------------------------------------------------------------------------------------
def bottleneck(x, sd, prefix, stride, dil2, has_down, down_stride, eps, momentum, training, stats=None):
    """Bottleneck.forward — TorchSeg furnace/base_model/resnet.py:78-101 (conv2 carries stride / dilation)"""
    out = q(F.conv2d(x, qw(sd[prefix + ".conv1.weight"])))
    out = q(F.relu(_bn(out, sd, prefix + ".bn1", eps, momentum, training, stats)))
    out = q(F.conv2d(out, qw(sd[prefix + ".conv2.weight"]), None, stride, dil2, dil2))
    out = q(F.relu(_bn(out, sd, prefix + ".bn2", eps, momentum, training, stats)))
    out = q(F.conv2d(out, qw(sd[prefix + ".conv3.weight"])))
    out = _bn(out, sd, prefix + ".bn3", eps, momentum, training, stats)
    residual = x
    if has_down:
        residual = q(F.conv2d(x, qw(sd[prefix + ".downsample.0.weight"]), None, down_stride))
        residual = q(_bn(residual, sd, prefix + ".downsample.1", eps, momentum, training, stats))
    return q(F.relu(out + residual))


def resnet_v1c_d8(x, sd, prefix, layers, eps, momentum, training, stats=None, dilated=True):
    """ResNet.forward with deep stem (resnet.py:110-124,168-184) after PSPNet._nostride_dilate(layer3, 2) and
    (layer4, 4) (pspnet network.py:22-23,62-72): stride-2 3x3 → stride 1, dilation=padding=d//2; other 3x3 → d;
    the stride-2 1x1 downsample → stride 1."""
    c = prefix + ".conv1"
    x = q(F.conv2d(q(x), qw(sd[c + ".0.weight"]), None, 2, 1))
    x = q(F.relu(_bn(x, sd, c + ".1", eps, momentum, training, stats)))
    x = q(F.conv2d(x, qw(sd[c + ".3.weight"]), None, 1, 1))
    x = q(F.relu(_bn(x, sd, c + ".4", eps, momentum, training, stats)))
    x = q(F.conv2d(x, qw(sd[c + ".6.weight"]), None, 1, 1))
    x = q(F.relu(_bn(x, sd, prefix + ".bn1", eps, momentum, training, stats)))
    x = F.max_pool2d(x, 3, 2, 1)
    blocks = []
    for li, nblk in enumerate(layers, start=1):
        for bi in range(nblk):
            pre = "%s.layer%d.%d" % (prefix, li, bi)
            first = bi == 0
            if li == 1:
                stride, dil2, dstride = 1, 1, 1
            elif li == 2:
                stride, dil2, dstride = (2 if first else 1), 1, 2
            elif not dilated:  # plain output-stride-32 trunk (DFN, dfn network.py:20-23)
                stride, dil2, dstride = (2 if first else 1), 1, 2
            elif li == 3:      # dilate = 2
                stride, dil2, dstride = 1, (1 if first else 2), 1
            else:              # dilate = 4
                stride, dil2, dstride = 1, (2 if first else 4), 1
            x = bottleneck(x, sd, pre, stride, dil2, first, dstride, eps, momentum, training, stats)
        blocks.append(x)
    return blocks


def pyramid_pooling_logits(x, sd, prefix, eps, momentum, training, scales=(1, 2, 3, 6), stats=None):
    """PyramidPooling.forward — pspnet network.py:99-109 (Dropout2d disabled: p = 0 in the parity runs)"""
    outs = [x]
    for i, s in enumerate(scales):
        p = q(F.adaptive_avg_pool2d(x, s))
        p = conv_bn_relu(p, sd, "%s.ppm.%d.psp/cbr" % (prefix, i), 1, 0, eps=eps, momentum=momentum, training=training,
                         stats=stats)
        outs.append(q(F.interpolate(p, size=x.shape[2:], mode="bilinear", align_corners=True)))
    fm = torch.cat(outs, 1)
    fm = conv_bn_relu(fm, sd, prefix + ".conv6.0", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    return F.conv2d(fm, qw(sd[prefix + ".conv6.2.weight"]), sd[prefix + ".conv6.2.bias"])


def _up8(x, data):
    """pspnet / psanet network.py:46-49: F.interpolate(scale_factor=8, bilinear, align_corners=True). For inputs whose
    size is not a multiple of 8 (BASELINE.json's 713 / 473 crops; the reference's own 480 is) the x8 map does not match
    the label, so — identically in this oracle and in the libtsb networks — the target is the INPUT size (`size=`), which
    is the same operation whenever both are defined (align_corners: src = dst·(in-1)/(out-1))."""
    H, W = data.shape[2:]
    if x.shape[2] * 8 == H and x.shape[3] * 8 == W:
        return F.interpolate(x, scale_factor=8, mode="bilinear", align_corners=True)
    return F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)


def pspnet_loss(data, label, sd, layers=(3, 4, 23, 3), aux_ratio=0.4, ignore_label=-1, eps=1e-5, momentum=0.1, stats=None):
    """PSPNet.forward training branch — pspnet network.py:40-57 (x8 bilinear, log_softmax, CE; loss + 0.4*aux)"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, True, stats)
    psp = pyramid_pooling_logits(blocks[-1], sd, "psp_layer", eps, momentum, True, stats=stats)
    aux = conv_bn_relu(blocks[-2], sd, "aux_layer.0", 1, 1, eps=eps, momentum=momentum, training=True, stats=stats)
    aux = F.conv2d(aux, qw(sd["aux_layer.2.weight"]), sd["aux_layer.2.bias"])
    psp = F.log_softmax(_up8(psp, data), dim=1)
    aux = F.log_softmax(_up8(aux, data), dim=1)
    loss = F.cross_entropy(psp, label, ignore_index=ignore_label)
    return loss + aux_ratio * F.cross_entropy(aux, label, ignore_index=ignore_label), (psp, aux)


# --------------------------------------------------------------------------------------------------
# DFN (model/dfn/cityscapes.dfn.R101_v1c/network.py)
# --------------------------------------------------------------------------------------------------
def refine_residual(x, sd, prefix, has_relu, eps, momentum, training, stats=None):
    """RefineResidual.forward — TorchSeg furnace/seg_opr/seg_oprs.py:182-188"""
    x = q(F.conv2d(x, qw(sd[prefix + ".conv_1x1.weight"])))
    t = conv_bn_relu(x, sd, prefix + ".cbr", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    t = q(F.conv2d(t, qw(sd[prefix + ".conv_refine.weight"]), None, 1, 1))
    return q(F.relu(t + x)) if has_relu else q(t + x)


def bn_refine(x, sd, prefix, has_relu, eps, momentum, training, stats=None):
    """BNRefine.forward — TorchSeg furnace/seg_opr/seg_oprs.py:157-162"""
    t = conv_bn_relu(x, sd, prefix + ".conv_bn_relu", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    t = q(F.conv2d(t, qw(sd[prefix + ".conv_refine.weight"]), None, 1, 1))
    return q(F.relu(t + x)) if has_relu else q(t + x)


def channel_attention(x1, x2, sd, prefix):
    """ChannelAttention.forward + SELayer.forward — seg_oprs.py:121-126,135-140"""
    fm = torch.cat([x1, x2], 1)
    y = q(F.adaptive_avg_pool2d(fm, 1)).flatten(1)
    y = q(F.relu(q(F.linear(y, qw(sd[prefix + ".channel_attention.fc.0.weight"]), sd[prefix + ".channel_attention.fc.0.bias"]))))
    y = q(F.linear(y, qw(sd[prefix + ".channel_attention.fc.2.weight"]), sd[prefix + ".channel_attention.fc.2.bias"]))
    a = torch.sigmoid(y).view(y.shape[0], -1, 1, 1)
    return q(x1 * a + x2)


def dfn_head_logits(x, sd, prefix, eps, momentum, training, stats=None):
    """DFNHead.forward before the up-sampling — dfn network.py:166-168"""
    x = refine_residual(x, sd, prefix + ".rrb", False, eps, momentum, training, stats)
    return F.conv2d(x, qw(sd[prefix + ".conv.weight"]), sd[prefix + ".conv.bias"])


def dfn_forward(blocks, sd, eps=1e-5, momentum=0.1, training=True, stats=None):
    """DFN.forward from the four backbone blocks to the low-resolution head outputs — dfn network.py:95-137.
    Returns ([4 smooth logits, deepest first], [4 border logits], [4 smooth head inputs], [4 border head inputs])."""
    deep = blocks[::-1]
    gc = q(F.adaptive_avg_pool2d(deep[0], 1))
    gc = conv_bn_relu(gc, sd, "global_context.1", 1, 0, eps=eps, momentum=momentum, training=training, stats=stats)
    last_fm = q(F.interpolate(gc, size=deep[0].shape[2:], mode="bilinear", align_corners=True))
    smooth_fm, smooth = [], []
    for i, fm in enumerate(deep):
        fm = refine_residual(fm, sd, "smooth_pre_rrbs.%d" % i, True, eps, momentum, training, stats)
        fm = channel_attention(fm, last_fm, sd, "cabs.%d" % i)
        fm = refine_residual(fm, sd, "smooth_aft_rrbs.%d" % i, True, eps, momentum, training, stats)
        smooth_fm.append(fm)
        smooth.append(dfn_head_logits(fm, sd, "smooth_heads.%d" % i, eps, momentum, training, stats))
        if i != 3:
            last_fm = q(F.interpolate(fm, scale_factor=2, mode="bilinear", align_corners=True))
    last_fm = None
    border_fm, border = [], []
    for i, fm in enumerate(blocks):
        fm = refine_residual(fm, sd, "border_pre_rrbs.%d" % i, True, eps, momentum, training, stats)
        if last_fm is not None:
            fm = q(F.interpolate(fm, scale_factor=2 ** i, mode="bilinear", align_corners=True))
            last_fm = q(last_fm + fm)
            last_fm = refine_residual(last_fm, sd, "border_aft_rrbs.%d" % i, True, eps, momentum, training, stats)
        else:
            last_fm = fm
        border_fm.append(last_fm)
        border.append(dfn_head_logits(last_fm, sd, "border_heads.%d" % i, eps, momentum, training, stats))
    return smooth, border, smooth_fm, border_fm


def dfn_loss(data, label, aux_label, sd, layers=(3, 4, 23, 3), alpha=0.1, ignore_label=255, gamma=2.0,
             focal_alpha=0.25, eps=1e-5, momentum=0.1, stats=None):
    """DFN.forward training branch — dfn network.py:139-152 with the criteria of dfn train.py:48-52
    (CrossEntropyLoss(mean, ignore 255) on the 4 smooth heads, SigmoidFocalLoss on the 4 border heads)."""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, True, stats, dilated=False)
    smooth, border, _, _ = dfn_forward(blocks, sd, eps, momentum, True, stats)
    loss = 0.0
    for i, lo in enumerate(smooth):
        up = F.interpolate(lo, scale_factor=2 ** (5 - i), mode="bilinear", align_corners=True)
        loss = loss + F.cross_entropy(up, label, ignore_index=ignore_label)
    aux = 0.0
    for lo in border:
        up = F.interpolate(lo, scale_factor=4, mode="bilinear", align_corners=True)
        aux = aux + sigmoid_focal(up, aux_label, ignore_label, gamma, focal_alpha)
    return loss + alpha * aux, (smooth, border)


# --------------------------------------------------------------------------------------------------
# PSANet (model/psanet/ade.psanet.R101_v1c/network.py)
# --------------------------------------------------------------------------------------------------
def psa_branch(x, sd, prefix, which, eps, momentum, training, stats=None):
    """one of the two attention branches of PointwiseSpatialAttention.forward — psanet network.py:120-138:
    reduce = CBR1x1(x); att = conv1x1(CBR1x1(reduce)); bmm(reduce.view(b,512,-1), softmax(att.view(b,c,-1), dim=1))"""
    red = conv_bn_relu(x, sd, "%s.%s_reduction" % (prefix, which), 1, 0, eps=eps, momentum=momentum, training=training,
                       stats=stats)
    att = conv_bn_relu(red, sd, "%s.%s_attention.0" % (prefix, which), 1, 0, eps=eps, momentum=momentum,
                       training=training, stats=stats)
    att = F.conv2d(att, qw(sd["%s.%s_attention.1.conv.weight" % (prefix, which)]))   # fp32 logits on both sides
    b, c, h, w = att.shape
    S = q(torch.softmax(att.view(b, c, -1), dim=1))
    fm = torch.bmm(red.view(b, red.shape[1], -1), S)
    return q(fm.view(b, red.shape[1], h, w))


def psa_logits(x, sd, prefix, eps, momentum, training, stats=None):
    """PointwiseSpatialAttention.forward — psanet network.py:119-144 (Dropout2d disabled in the parity runs)"""
    collect = psa_branch(x, sd, prefix, "collect", eps, momentum, training, stats)
    distribute = psa_branch(x, sd, prefix, "distribute", eps, momentum, training, stats)
    psa = conv_bn_relu(torch.cat([collect, distribute], 1), sd, prefix + ".proj", 1, 0, eps=eps, momentum=momentum,
                       training=training, stats=stats)
    fm = torch.cat([x, psa], 1)
    fm = conv_bn_relu(fm, sd, prefix + ".conv6.0", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    return F.conv2d(fm, qw(sd[prefix + ".conv6.2.weight"]), sd[prefix + ".conv6.2.bias"])


def psanet_loss(data, label, sd, layers=(3, 4, 23, 3), aux_ratio=0.4, ignore_label=-1, eps=1e-5, momentum=0.1, stats=None):
    """PSANet (`PSPNet` in psanet network.py) training branch — network.py:41-57"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, True, stats)
    psa = psa_logits(blocks[-1], sd, "psa_layer", eps, momentum, True, stats=stats)
    aux = conv_bn_relu(blocks[-2], sd, "aux_layer.0", 1, 1, eps=eps, momentum=momentum, training=True, stats=stats)
    aux = F.conv2d(aux, qw(sd["aux_layer.2.weight"]), sd["aux_layer.2.bias"])
    psa = F.log_softmax(_up8(psa, data), dim=1)
    aux = F.log_softmax(_up8(aux, data), dim=1)
    loss = F.cross_entropy(psa, label, ignore_index=ignore_label)
    return loss + aux_ratio * F.cross_entropy(aux, label, ignore_index=ignore_label), (psa, aux)
