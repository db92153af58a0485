"""BiSeNet (ResNet-18 context path) with the reference's class / attribute names
(TorchSeg model/bisenet/cityscapes.bisenet.R18/network.py:18-168) on the libtsb path.

Training forward returns the scalar loss exactly like the reference (`loss = model(imgs, gts)`); the three
heads end in the FUSED bilinear-upsample + OHEM loss when the criterion supports it
(`forward_lowres`), so the [B,19,1024,1024] logits are never materialised.
"""
import torch
import torch.nn as nn

from .. import ops
from ..base_model import resnet18
from ..seg_opr.seg_oprs import ConvBnRelu, AttentionRefinement, FeatureFusion, conv_plain, upsample_bilinear, _as_act


class _Cfg(object):
    bn_eps = 1e-5
    bn_momentum = 0.1
    num_classes = 19


try:  # the reference imports `config` by bare name (network.py:9); honour it when present
    from config import config as _config
except Exception:  # noqa: BLE001
    _config = _Cfg()


class BiSeNet(nn.Module):
    def __init__(self, out_planes, is_training, criterion, pretrained_model=None, norm_layer=nn.BatchNorm2d):
        super(BiSeNet, self).__init__()
        self.context_path = resnet18(pretrained_model, norm_layer=norm_layer, bn_eps=_config.bn_eps,
                                     bn_momentum=_config.bn_momentum, deep_stem=False, stem_width=64)
        self.business_layer = []
        self.is_training = is_training
        self.out_planes = out_planes
        self.spatial_path = SpatialPath(3, 128, norm_layer)
        conv_channel = 128
        self.global_context = nn.Sequential(
            nn.AdaptiveAvgPool2d(1),
            ConvBnRelu(512, conv_channel, 1, 1, 0, has_bn=True, has_relu=True, has_bias=False, norm_layer=norm_layer))
        arms = [AttentionRefinement(512, conv_channel, norm_layer), AttentionRefinement(256, conv_channel, norm_layer)]
        refines = [ConvBnRelu(conv_channel, conv_channel, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                              has_bias=False),
                   ConvBnRelu(conv_channel, conv_channel, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                              has_bias=False)]
        heads = [BiSeNetHead(conv_channel, out_planes, 16, True, norm_layer),
                 BiSeNetHead(conv_channel, out_planes, 8, True, norm_layer),
                 BiSeNetHead(conv_channel * 2, out_planes, 8, False, norm_layer)]
        self.ffm = FeatureFusion(conv_channel * 2, conv_channel * 2, 1, norm_layer)
        self.arms = nn.ModuleList(arms)
        self.refines = nn.ModuleList(refines)
        self.heads = nn.ModuleList(heads)
        self.business_layer.append(self.spatial_path)
        self.business_layer.append(self.global_context)
        self.business_layer.append(self.arms)
        self.business_layer.append(self.refines)
        self.business_layer.append(self.heads)
        self.business_layer.append(self.ffm)
        if is_training:
            self.criterion = criterion

    def features(self, data):
        """network.py:76-101 up to the three head inputs"""
        sp, cp = self.spatial_path, self.context_path
        if data.shape[1] == 3 and sp.conv_7x7.bn.training and cp.bn1.training:
            # both 7x7/2 stems in ONE tensor-core launch over the shared space-to-depth image
            from ..seg_opr.seg_oprs import _packed_image
            bs, bc = sp.conv_7x7.bn, cp.bn1
            s_stem, c_stem = ops.StemPairFn.apply(
                _packed_image(data), sp.conv_7x7.conv.weight, bs.weight, bs.bias, bs.running_mean, bs.running_var,
                cp.conv1.weight, bc.weight, bc.bias, bc.running_mean, bc.running_var,
                float(bs.eps), float(bs.momentum if bs.momentum is not None else 0.1),
                float(bc.eps), float(bc.momentum if bc.momentum is not None else 0.1))
            spatial_out = sp.forward_from_stem(s_stem)
            context_blocks = cp.forward_from_stem(c_stem)
        else:
            spatial_out = sp(data)
            context_blocks = cp(data)
        context_blocks.reverse()
        gc = ops.AdaptiveAvgPoolFn.apply(context_blocks[0], 1)
        gc = self.global_context[1](gc)
        gc = upsample_bilinear(gc, context_blocks[0].shape[2:])
        last_fm = gc
        pred_out = []
        for i, (fm, arm, refine) in enumerate(zip(context_blocks[:2], self.arms, self.refines)):
            fm = arm(fm, add=last_fm)  # ARM scale and `fm += last_fm` in one kernel
            last_fm = upsample_bilinear(fm, context_blocks[i + 1].shape[2:])
            last_fm = refine(last_fm)
            pred_out.append(last_fm)
        concate_fm = self.ffm(spatial_out, last_fm)
        pred_out.append(concate_fm)
        return pred_out

    def forward(self, data, label=None):
        pred_out = self.features(data)
        if self.is_training:
            fused = hasattr(self.criterion, "forward_lowres")
            losses = []
            for i in (0, 1, 2):
                if fused:
                    lo = self.heads[i].lowres_logits(pred_out[i])
                    losses.append(self.criterion.forward_lowres(lo, label, self.out_planes))
                else:
                    losses.append(self.criterion(self.heads[i](pred_out[i]), label))
            aux_loss0, aux_loss1, main_loss = losses
            return main_loss + aux_loss0 + aux_loss1  # network.py:108
        return torch.log_softmax(self.heads[-1](pred_out[-1]), dim=1)


class SpatialPath(nn.Module):
    """network.py:114-137"""

    def __init__(self, in_planes, out_planes, norm_layer=nn.BatchNorm2d):
        super(SpatialPath, self).__init__()
        inner_channel = 64
        self.conv_7x7 = ConvBnRelu(in_planes, inner_channel, 7, 2, 3, has_bn=True, norm_layer=norm_layer,
                                   has_relu=True, has_bias=False)
        self.conv_3x3_1 = ConvBnRelu(inner_channel, inner_channel, 3, 2, 1, has_bn=True, norm_layer=norm_layer,
                                     has_relu=True, has_bias=False)
        self.conv_3x3_2 = ConvBnRelu(inner_channel, inner_channel, 3, 2, 1, has_bn=True, norm_layer=norm_layer,
                                     has_relu=True, has_bias=False)
        self.conv_1x1 = ConvBnRelu(inner_channel, out_planes, 1, 1, 0, has_bn=True, norm_layer=norm_layer,
                                   has_relu=True, has_bias=False)

    def forward(self, x):
        return self.forward_from_stem(self.conv_7x7(x))

    def forward_from_stem(self, x):
        x = self.conv_3x3_1(x)
        x = self.conv_3x3_2(x)
        return self.conv_1x1(x)


class BiSeNetHead(nn.Module):
    """network.py:140-168"""

    def __init__(self, in_planes, out_planes, scale, is_aux=False, norm_layer=nn.BatchNorm2d):
        super(BiSeNetHead, self).__init__()
        mid = 256 if is_aux else 64
        self.conv_3x3 = ConvBnRelu(in_planes, mid, 3, 1, 1, has_bn=True, norm_layer=norm_layer, has_relu=True,
                                   has_bias=False)
        self.conv_1x1 = nn.Conv2d(mid, out_planes, kernel_size=1, stride=1, padding=0)
        self.scale = scale

    def lowres_logits(self, x):
        """fp32 NHWC logits at head resolution (channel stride 32)"""
        fm = self.conv_3x3(x)
        K = self.conv_1x1.out_channels
        return conv_plain(fm, self.conv_1x1, out_f32=True, ocs=(K + 31) // 32 * 32)

    def forward(self, x):
        lo = self.lowres_logits(x)
        if self.scale > 1:
            return _UpsampleLogitsFn.apply(lo, lo.shape[2] * self.scale, lo.shape[3] * self.scale)
        return lo


class _UpsampleLogitsFn(torch.autograd.Function):
    """reference-boundary form of the head tail: NCHW fp32 [N,C,H,W] logits, bilinear align_corners=True to an explicit
    output size (network.py:164-166 use scale_factor; with align_corners the source coordinate is (in-1)/(out-1)·dst
    either way, so size = in·scale is the same op — and sizes like 713 / 473 that are not a multiple of 8 work too)"""

    @staticmethod
    def forward(ctx, lo, H, W):
        N, C, h, w = lo.shape
        H, W = int(H), int(W)
        out = torch.empty((N, C, H, W), dtype=torch.float32, device=lo.device)
        ops.call("tsb_bilinear_fwd_nhwc_to_nchw", ops.ptr(lo), ops._lib.dt(lo), ops.cs_of(lo), ops.ptr(out), N, C, h, w,
                 H, W, ops.stream())
        ctx.shape = (N, C, h, w, H, W, ops.cs_of(lo))
        return out

    @staticmethod
    def backward(ctx, g):
        N, C, h, w, H, W, cs = ctx.shape
        # gather-form transpose needs NHWC with C % 8 == 0: pad the class dimension into a 32-wide buffer
        Cp = (C + 7) // 8 * 8
        gp = ops.nhwc_zeros(N, Cp, H, W, dtype=torch.float32, device=g.device)
        gp[:, :C].copy_(g)
        d = ops.nhwc_zeros(N, Cp, h, w, dtype=torch.float32, device=g.device, cs=max(cs, Cp))
        ops.call("tsb_bilinear_bwd", ops.ptr(gp), ops.F32, Cp, ops.ptr(d), ops.F32, ops.cs_of(d), N, Cp, h, w, H, W, 0,
                 ops.stream())
        return d[:, :C], None, None
