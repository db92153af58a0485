"""libtsb replacements of the two apex entry points the reference train.py scripts import.

* SyncBatchNorm — parameter holder only (subclass of nn.BatchNorm2d so isinstance-based init_weight /
  group_weight keep working); the statistics exchange happens inside ops.ConvBNActFn as ONE all-reduce of the
  packed [Σx | Σx²] (forward) and [Σdy | Σdy·x̂] (backward) buffers per layer.
* DistributedDataParallel — flat-buffer gradient all-reduce: every parameter's .grad is a view into one
  contiguous fp32 buffer; buckets of that buffer are reduced with NCCL on a side stream as soon as autograd
  has produced their last gradient (overlapped with the rest of backward), then averaged.
"""
import torch
import torch.distributed as dist
import torch.nn as nn

from ... import ops
from ...flat import ensure_flat_grads, layout_of


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class SyncBatchNorm(nn.BatchNorm2d):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 process_group=None, channel_last=False):
        super(SyncBatchNorm, self).__init__(num_features, eps=eps, momentum=momentum, affine=affine,
                                            track_running_stats=track_running_stats)
        self.process_group = process_group
        if _world() > 1:
            ops.set_sync_group(process_group, _world())


class DistributedDataParallel(nn.Module):
    """apex.parallel.DistributedDataParallel(model) drop-in (train.py:98-99)."""

    def __init__(self, module, message_size=None, delay_allreduce=False, bucket_bytes=32 << 20, **kwargs):
        super(DistributedDataParallel, self).__init__()
        self.module = module
        self.world_size = _world()
        self.bucket_bytes = bucket_bytes
        params = [p for p in module.parameters() if p.requires_grad]
        lay = layout_of(params)
        if lay is not None:
            # the fused optimiser already laid these gradients out (group order): reuse that buffer/order
            params = list(lay[2])
        self._params = params
        dev = params[0].device
        self.flat_grad, self._spans = ensure_flat_grads(params)
        n = self.flat_grad.numel()
        # buckets in REVERSE parameter order (backward produces the last layers' grads first)
        self._buckets = []
        hi = n
        cur_lo = n
        for i in range(len(params) - 1, -1, -1):
            cur_lo = self._spans[i][0]
            if (hi - cur_lo) * 4 >= bucket_bytes or i == 0:
                self._buckets.append([cur_lo, hi, 0, 0])  # lo, hi, expected, ready
                hi = cur_lo
        self._bucket_of = []
        for (lo, _hi) in self._spans:
            for bi, b in enumerate(self._buckets):
                if b[0] <= lo < b[1]:
                    self._bucket_of.append(bi)
                    b[2] += 1
                    break
        self._comm_stream = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._pending = False
        # overlap=True: buckets are reduced on the side stream while backward continues (eager steps). overlap=False: ONE
        # all-reduce of the whole flat buffer on the compute stream in finish_reduce() — the form used inside a captured
        # whole-step graph, where every inter-GPU kernel (SyncBN exchanges, this all-reduce) must sit on a single chain:
        # two independent peer-synchronising kernels in flight need guaranteed concurrency, which graph branches do not
        # give (a rank that schedules them in the other order deadlocks the pair). The 54 MB (R18) all-reduce costs
        # ~0.2 ms un-overlapped.
        self.overlap = True
        if self.world_size > 1:
            ops.set_sync_group(None, self.world_size)
            with torch.no_grad():  # rank 0's parameters win, like the DDP constructor broadcast
                for p in params:
                    dist.broadcast(p.data, 0)
                for b in module.buffers():
                    dist.broadcast(b.data, 0)
            hooks = {}
            for i, p in enumerate(params):
                h = self._make_hook(i)
                hooks[id(p)] = h
                p.register_post_accumulate_grad_hook(h)
            # gradients written straight into the flat views by the kernels bypass AccumulateGrad: same bucket logic
            ops.grad_ready_hook = lambda prm: hooks[id(prm)](prm) if id(prm) in hooks else None

    def _make_hook(self, idx):
        def hook(param):
            lo, hi = self._spans[idx]
            if param.grad.data_ptr() != self.flat_grad.data_ptr() + 4 * lo:  # grads were set to None upstream
                view = torch.as_strided(self.flat_grad, param.shape, param.stride(), lo)
                view.copy_(param.grad)
                param.grad = view
            if not self.overlap:
                self._pending = True
                return
            b = self._buckets[self._bucket_of[idx]]
            b[3] += 1
            if b[3] == b[2]:
                b[3] = 0
                self._reduce_bucket(b[0], b[1])
        return hook

    def _reduce_bucket(self, lo, hi):
        chunk = self.flat_grad[lo:hi]
        if self._comm_stream is not None:
            self._comm_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self._comm_stream):
                dist.all_reduce(chunk)
                chunk.div_(self.world_size)
        else:
            dist.all_reduce(chunk)
            chunk.div_(self.world_size)
        self._pending = True

    def finish_reduce(self):
        """make the compute stream wait for outstanding bucket reductions (call before optimizer.step)"""
        if self.world_size > 1 and not self.overlap:
            dist.all_reduce(self.flat_grad)
            self.flat_grad.div_(self.world_size)
        elif self._pending and self._comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self._comm_stream)
        self._pending = False

    def zero_grad(self, set_to_none=False):
        self.flat_grad, _ = ensure_flat_grads(self._params)
        self.flat_grad.zero_()
        ops.zero_arena.reset()

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)
