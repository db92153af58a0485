"""Host→device input prefetcher for the train loop (the `minibatch = dataloader.next(); imgs.cuda(non_blocking=True)`
step of TorchSeg model/bisenet/cityscapes.bisenet.R18/train.py:119-124).

Copies batch i+1 from pinned host memory on a side stream into one of TWO persistent device buffers while step i
computes (no per-step device allocation), and hands out the device tensors with the correct stream dependencies.
`.next()` mirrors the reference's iterator protocol."""
import torch


class CudaPrefetcher(object):
    def __init__(self, batch_iter, device):
        self.it = iter(batch_iter)
        self.device = device
        self.stream = torch.cuda.Stream(device=device)
        self.bufs = [{}, {}]            # two persistent device slots
        self.free_ev = [None, None]     # compute-stream event after which a slot may be overwritten
        self.ready_ev = [None, None]    # copy-stream event after which a slot holds its batch
        self.k = 0                      # next slot to fill
        self.handed = None              # slot handed out by the previous next()
        self._have = self._preload()

    def _preload(self):
        try:
            batch = next(self.it)
        except StopIteration:
            return False
        slot = self.k & 1
        dst = self.bufs[slot]
        for name, v in batch.items():   # allocate once, on the caller's stream (allocator-friendly)
            if torch.is_tensor(v) and (name not in dst or dst[name].shape != v.shape or dst[name].dtype != v.dtype):
                dst[name] = torch.empty(v.shape, dtype=v.dtype, device=self.device)
        if self.free_ev[slot] is not None:
            self.stream.wait_event(self.free_ev[slot])
        with torch.cuda.stream(self.stream):
            for name, v in batch.items():
                if torch.is_tensor(v):
                    dst[name].copy_(v, non_blocking=True)
                else:
                    dst[name] = v
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.ready_ev[slot] = ev
        self.k += 1
        return True

    def next(self):
        if not self._have:
            raise StopIteration
        cur = torch.cuda.current_stream(self.device)
        if self.handed is not None:     # everything enqueued so far used the previously handed slot
            ev = torch.cuda.Event()
            ev.record(cur)
            self.free_ev[self.handed] = ev
        slot = (self.k - 1) & 1
        cur.wait_event(self.ready_ev[slot])
        self.handed = slot
        batch = dict(self.bufs[slot])
        self._have = self._preload()
        return batch

    __next__ = next

    def __iter__(self):
        return self
