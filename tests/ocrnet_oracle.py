"""ORACLE — test infrastructure only: OCRNet (ResNet-101 v1c, dilated-8) with the object-contextual head.

Functional fp32 PyTorch restatement of torchseg_b200/networks/ocrnet.py on the shared blocks of oracle/torch_ref.py
(`resnet_v1c_d8`, `conv_bn_relu`), driven by a state_dict with the network's key names. Both soft-maxes are written as
explicit matrices: the soft object regions as the [B, K, N] soft-max over the pixels of each image, the pixel-region
relation as the [B, N, K] soft-max over the regions. The bf16-storage emulation of oracle/torch_ref.py
(`set_bf16_emulation`, re-exported here) is honoured. Pinned to the network composed from the live reference modules by
tests/test_cpu_ocrnet.py through tests/golden/live_reference_ocrnet.npz (tools/make_live_golden_ocrnet.py).

Nothing under torchseg_b200/ imports this file.
"""
import torch
import torch.nn.functional as F

from oracle.torch_ref import conv_bn_relu, q, qw, resnet_v1c_d8, set_bf16_emulation

__all__ = ["set_bf16_emulation", "ocrnet_case", "spatial_gather", "object_attention", "spatial_ocr", "ocrnet_logits",
           "ocrnet_loss", "ocrnet_eval"]


def ocrnet_case(N=2, HW=72, seed=29, classes=19):
    """Cityscapes-shaped input (19 classes, ignore 255): a 9 x 9 map at output stride 8"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, 3, HW, HW, generator=g)
    y = torch.randint(0, classes, (N, HW, HW), generator=g, dtype=torch.int64)
    y[:, :4] = 255
    return x, y, seed


def spatial_gather(f, logits):
    """the object-region proxy [B, C, K, 1]: ctx[b, :, k] = Σ_n softmax_n(l[b, k, n]) · f[b, :, n]"""
    B, C, h, w = f.shape
    K = logits.shape[1]
    P = q(F.softmax(logits.reshape(B, K, h * w), dim=2))             # [B, K, N]
    ctx = torch.matmul(P, f.reshape(B, C, h * w).permute(0, 2, 1))   # [B, K, C]
    return q(ctx.permute(0, 2, 1).unsqueeze(3))


def object_attention(x, proxy, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """ObjectAttentionBlock: f_up(softmax_k(f_pixel(x) · f_object(proxy)ᵀ / √256) · f_down(proxy))"""
    def cbr(t, name):
        return conv_bn_relu(t, sd, prefix + "." + name, 1, 0, eps=eps, momentum=momentum, training=training,
                            stats=stats)
    B, _, h, w = x.shape
    query = cbr(cbr(x, "f_pixel.0"), "f_pixel.1")
    key = cbr(cbr(proxy, "f_object.0"), "f_object.1")
    value = cbr(proxy, "f_down")
    d = query.shape[1]
    Q = query.reshape(B, d, -1).permute(0, 2, 1)                     # [B, N, 256]
    Kt = key.reshape(B, d, -1)                                       # [B, 256, K]
    V = value.reshape(B, value.shape[1], -1).permute(0, 2, 1)        # [B, K, 256]
    sim = F.softmax(torch.matmul(Q, Kt) * d ** -0.5, dim=-1)         # [B, N, K]
    ctx = q(torch.matmul(sim, V).permute(0, 2, 1).reshape(B, V.shape[2], h, w))
    return cbr(ctx, "f_up")


def spatial_ocr(x, proxy, sd, prefix, eps=1e-5, momentum=0.1, training=True, stats=None):
    """SpatialOCRModule with Dropout2d at p = 0: conv_bn_dropout(cat([object_attention(x, proxy), x]))"""
    ctx = object_attention(x, proxy, sd, prefix + ".object_context_block", eps, momentum, training, stats)
    return conv_bn_relu(torch.cat([ctx, x], 1), sd, prefix + ".conv_bn_dropout.0", 1, 0, eps=eps, momentum=momentum,
                        training=training, stats=stats)


def ocrnet_logits(data, sd, eps=1e-5, momentum=0.1, training=True, stats=None, layers=(3, 4, 23, 3)):
    """(low-resolution fp32 logits, low-resolution fp32 aux logits), Dropout2d at p = 0"""
    blocks = resnet_v1c_d8(data, sd, "backbone", layers, eps, momentum, training, stats)
    dsn = conv_bn_relu(blocks[-2], sd, "dsn_head.0", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    dsn = F.conv2d(dsn, qw(sd["dsn_head.2.weight"]), sd["dsn_head.2.bias"])
    f = conv_bn_relu(blocks[-1], sd, "conv_3x3", 1, 1, eps=eps, momentum=momentum, training=training, stats=stats)
    ctx = spatial_gather(f, dsn)
    f = spatial_ocr(f, ctx, sd, "spatial_ocr_head", eps, momentum, training, stats)
    return F.conv2d(f, qw(sd["head.weight"]), sd["head.bias"]), dsn


def _up(x, data):
    return F.interpolate(x, size=data.shape[2:], mode="bilinear", align_corners=True)


def ocrnet_loss(data, label, sd, aux_ratio=0.4, ignore_label=255, eps=1e-5, momentum=0.1, stats=None):
    """training: CE(up(logits)) + aux_ratio · CE(up(aux))"""
    lo, dsn = ocrnet_logits(data, sd, eps, momentum, True, stats)
    loss = F.cross_entropy(_up(lo, data), label, ignore_index=ignore_label)
    aux_loss = F.cross_entropy(_up(dsn, data), label, ignore_index=ignore_label)
    return loss + aux_ratio * aux_loss, (lo, dsn)


def ocrnet_eval(data, sd, eps=1e-5, stats=None):
    """eval: log_softmax of the logits up-sampled to the input size, BN on running statistics"""
    lo, _ = ocrnet_logits(data, sd, eps, 0.0, False, stats)
    return F.log_softmax(_up(lo, data), dim=1)
