"""Whole-step CUDA graph for the train loop (zero_grad → forward(loss) → backward → fused SGD step).

The step of TorchSeg model/bisenet/cityscapes.bisenet.R18/train.py:116-142 is ~400 kernel launches of 5-200 us
each; captured once, a replay removes the per-launch CPU work (Python autograd, ctypes, tensor-map encoding) and the
inter-kernel launch gaps. One process per GPU; with `ddp=` the gradient all-reduce and the SyncBN exchanges are part of the graph.

Usage:
    step = GraphedTrainStep(model, optimizer, example_inputs)     # runs `warmup` eager steps, then captures
    for it, batch in enumerate(loader):
        set the learning rates in optimizer.param_groups as usual
        loss = step(batch['data'], batch['label'])                # device tensors; copied into the static inputs
If capture is impossible (non-CUDA device, an op that cannot be captured) the object runs eager steps and keeps the
reason in `.error`.

Requirements (tools/diag_graph.py — each variant in its own process):
  * everything runs on ONE non-default stream (`torch.cuda.set_stream(torch.cuda.Stream())` at program start): work that
    touches the legacy default stream during a capture invalidates it;
  * NO autograd graph of an earlier eager step may be alive when the object is constructed — e.g. a `loss` tensor still
    referenced by the training loop (keep `loss.item()` / `loss.detach()` instead). A live graph keeps the parameters'
    AccumulateGrad nodes alive, and those are bound to the stream they were created on; replayed inside the capture
    they pull that stream into the capture and it is never joined again (cudaErrorStreamCaptureInvalidated at
    capture_end — this, not a kernel or an allocator call, was the "intermittent" failure of round 1: bench.py kept
    the last warm-up loss in a local variable). With that reference dropped every variant captures: fresh process,
    after eager steps, pinned inputs, global / thread_local / relaxed capture modes, batch 4..16, 512..1024 pixels;
  * the first optimiser step needs no special case (the momentum buffer starts at exact zeros), so nothing
    step-dependent is baked into the graph; hyper-parameters live in a device tensor refreshed before each replay.
Measured: BiSeNet-R18, 16 x 1024 x 1024: 371 launches per graph, 17.8 ms per replay against 19.6 ms of eager launches.
A failed capture leaves the process-wide CUDA RNG in capture mode and the eager step slower; the object then runs
eager steps and keeps the reason (with the Python frames) in `.error`."""
import torch


class GraphedTrainStep(object):
    def __init__(self, model, optimizer, example_inputs, warmup=3, enable=True, side_stream_warmup=True,
                 capture_error_mode=None, ddp=None, restore_after_warmup=False):
        """ddp: the apex.parallel.DistributedDataParallel shim wrapping `model` (multi-GPU): its bucketed NCCL all-reduce
        on the side stream (fork / join inside the capture) and the NVLink SyncBN exchanges (device-resident sequence
        counter) are captured too. Every rank must construct the object at the same point of its program.
        NOTE: construction runs `warmup` REAL optimiser steps on `example_inputs` (a capture needs every lazy allocation
        and attribute made first): weights, momentum and BN running statistics move, with the learning rate currently in
        `param_groups`. restore_after_warmup=True snapshots parameters / momentum / module buffers before and puts them
        back after the capture, so that constructing the object leaves the training state untouched."""
        self.model = model
        self.ddp = ddp
        if ddp is not None:
            ddp.overlap = False      # single chain of inter-GPU kernels inside the graph (see the DDP shim)
        self.opt = optimizer
        if capture_error_mode is None:
            # with NCCL in the process its watchdog thread polls events concurrently: only the capturing thread may be
            # held to the capture rules
            capture_error_mode = "thread_local" if ddp is not None else "global"
        self.static_inputs = [t.clone() for t in example_inputs]
        self.graph = None
        self.static_loss = None
        self.launches_per_step = 0
        self.error = None
        dev = self.static_inputs[0].device
        if not enable or dev.type != "cuda":
            return
        if side_stream_warmup and warmup < 1:
            warmup = 1       # at least one step must have run on a non-default stream before the capture
        from .. import _lib
        snap = None
        if restore_after_warmup:
            snap = (optimizer.flat_param.clone(), optimizer.flat_mom.clone(), optimizer._steps,
                    [b.clone() for b in model.buffers()])
        try:
            if side_stream_warmup:
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    for _ in range(warmup):
                        self._eager(*self.static_inputs)
                torch.cuda.current_stream(dev).wait_stream(side)
            else:
                for _ in range(warmup):          # lazy attributes, FlatPack mirror, per-thread context binding all warm
                    self._eager(*self.static_inputs)
            torch.cuda.synchronize(dev)
            import gc
            self.opt.push_hyperparams()
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            # torch.cuda.graph no longer garbage-collects on entry: collect now and keep the cyclic GC off while capturing,
            # so that no CUDA object (tensor of an old autograd graph, stream, event) is destroyed in the middle of it
            gc.collect()
            gc_was_on = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.graph(g, capture_error_mode=capture_error_mode):
                    self.static_loss = self._eager(*self.static_inputs)
            finally:
                if gc_was_on:
                    gc.enable()
            self.launches_per_step = _lib.launch_count() - n0
            self.graph = g
            if snap is not None:     # the capture itself executed nothing; undo the warm-up steps
                with torch.no_grad():
                    optimizer.flat_param.copy_(snap[0])
                    optimizer.flat_mom.copy_(snap[1])
                    optimizer._steps = snap[2]
                    for b, v in zip(model.buffers(), snap[3]):
                        b.copy_(v)
                from .. import ops
                ops.pack_cache.invalidate()
                # the captured kernels read the bf16 MIRROR of the parameters (written by the SGD kernel at the end of every
                # step): regenerate it from the restored weights with a no-op update (lr 0, weight decay 0, momentum 1,
                # zero gradient: parameters and momentum come out unchanged)
                optimizer.flat_grad.zero_()
                ng = len(optimizer.param_groups)
                z = torch.zeros(ng, dtype=torch.float32, device=dev)
                ops.call("tsb_sgd_flat_pack", ops.ptr(optimizer.flat_param), ops.ptr(optimizer.flat_grad), ops.ptr(optimizer.flat_mom),
                         optimizer.flat_param.numel(), ops.ptr(optimizer._seg_end), ops.ptr(z), ops.ptr(z), ng, 1.0, 1.0, 0,
                         ops.ptr(optimizer.pack.wb_flat), ops.stream())
                optimizer.pack.mark_fresh()
                torch.cuda.synchronize(dev)
        except Exception as e:  # noqa: BLE001 — fall back to eager steps, keep the reason
            import traceback
            tb = traceback.extract_tb(e.__traceback__)
            where = " <- ".join("%s:%d %s" % (f.filename.split("/")[-1], f.lineno, f.name) for f in reversed(tb[-6:]))
            self.error = "%s: %s [at %s]" % (type(e).__name__, e, where)
            self.graph = None
            try:                 # best effort: release the half-built graph (its RNG registration, its memory pool)
                g.reset()
            except Exception:    # noqa: BLE001
                pass
            try:
                torch.cuda.synchronize(dev)
            except Exception:    # noqa: BLE001
                pass

    def release(self):
        """destroy the captured graph (and its memory pool). REQUIRED before dist.destroy_process_group() when the graph
        contains NCCL kernels: NCCL's communicator teardown waits for every graph that captured it (observed: a hang in
        destroy_process_group with a live graph)."""
        g, self.graph = self.graph, None
        self.static_loss = None
        if g is not None:
            torch.cuda.synchronize()
            g.reset()
            del g
            import gc
            gc.collect()
            torch.cuda.synchronize()

    def _eager(self, *inputs):
        self.opt.zero_grad()
        loss = (self.ddp or self.model)(*inputs)
        loss.backward()
        if self.ddp is not None:
            self.ddp.finish_reduce()
        self.opt.step()
        return loss

    def __call__(self, *inputs):
        if self.graph is None:
            return self._eager(*inputs)
        for dst, src in zip(self.static_inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.opt.push_hyperparams()      # lr / weight decay of this step → the device tensor the captured SGD kernel reads
        self.graph.replay()
        # Python-side caches describe the weights BEFORE the replayed SGD update: drop them so that an eager step (or
        # evaluation) after a replay re-packs from the current parameters
        from .. import ops
        ops.pack_cache.cache.clear()
        ops.pack_cache.step += 1
        pack = getattr(self.opt, "pack", None)
        if pack is not None:
            pack.mark_fresh()
        return self.static_loss
