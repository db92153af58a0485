"""Losses with the reference API (TorchSeg furnace/seg_opr/loss_opr.py)."""
import torch
import torch.nn as nn

from .. import ops


class ProbOhemCrossEntropy2d(nn.Module):
    """loss_opr.py:48-98 — same constructor; forward(pred, target) takes MATERIALISED [b,c,h,w] logits exactly like
    the reference. `forward_lowres` is the fused-upsample form used by the libtsb networks: it consumes the
    low-resolution head output and never writes the full-resolution logits."""

    CITYSCAPES_WEIGHT = [1.4297, 1.4805, 1.4363, 3.365, 2.6635, 1.4311, 2.1943, 1.4817, 1.4513, 2.1984, 1.5295,
                         1.6892, 3.2224, 1.4727, 7.5978, 9.4117, 15.2588, 5.6818, 2.2067]  # loss_opr.py:57-60

    def __init__(self, ignore_label, reduction='mean', thresh=0.6, min_kept=256, down_ratio=1, use_weight=False):
        super(ProbOhemCrossEntropy2d, self).__init__()
        if reduction != 'mean':
            raise NotImplementedError("only reduction='mean' (the value every reference train.py uses)")
        self.ignore_label = ignore_label
        self.thresh = float(thresh)
        self.min_kept = int(min_kept)
        self.down_ratio = down_ratio
        if use_weight:
            self.register_buffer("weight", torch.tensor(self.CITYSCAPES_WEIGHT, dtype=torch.float32))
        else:
            self.weight = None
        self.debug_states = None   # tests / logging: set to a list to collect each call's device-side OHEM state words

    def _record(self, loss):
        if self.debug_states is not None and loss.grad_fn is not None:
            self.debug_states.append(loss.grad_fn.saved_tensors[3])
        return loss

    def forward(self, pred, target):
        return self._record(ops.OhemCEFn.apply(pred, target, self.ignore_label, self.thresh, self.min_kept, self.weight))

    def forward_lowres(self, logits_lo, target, num_classes):
        H, W = target.shape[-2:]
        return self._record(ops.OhemUpCEFn.apply(logits_lo, target, H, W, num_classes, self.ignore_label, self.thresh,
                                                 self.min_kept, self.weight))


class SigmoidFocalLoss(nn.Module):
    """loss_opr.py:14-45 (quirks reproduced literally, SURVEY.md App. A2)"""

    def __init__(self, ignore_label, gamma=2.0, alpha=0.25, reduction='mean'):
        super(SigmoidFocalLoss, self).__init__()
        if reduction != 'mean':
            raise NotImplementedError("only reduction='mean'")
        self.ignore_label = ignore_label
        self.gamma = gamma
        self.alpha = alpha

    def forward(self, pred, target):
        return _FocalFn.apply(pred, target, self.ignore_label, self.gamma, self.alpha)


class _FocalFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, ignore_label, gamma, alpha):
        predc = pred.contiguous()
        target = target.contiguous()
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        d = torch.empty_like(predc)
        ops.call("tsb_sigmoid_focal_fwd_bwd", ops.ptr(predc), ops._lib.dt(predc), ops.ptr(target), predc.numel(),
                 int(ignore_label), float(gamma), float(alpha), ops.ptr(loss), ops.ptr(d), ops.stream())
        ctx.save_for_backward(d)
        return loss

    @staticmethod
    def backward(ctx, g):
        (d,) = ctx.saved_tensors
        return d * g.to(d.dtype), None, None, None, None
