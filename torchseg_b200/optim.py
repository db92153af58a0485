"""Fused flat-buffer momentum SGD (SURVEY.md §8f rank 1) with torch.optim.SGD's surface: `param_groups`
(list of dicts whose 'lr' the train loop rewrites every iteration, train.py:136-139), `zero_grad`, `step`,
`state_dict`, `load_state_dict`. One kernel launch updates all parameters (tsb_sgd_flat)."""
import torch

from . import ops
from ._lib import call, ptr, stream
from .flat import flatten, ensure_flat_grads, check_inside


class FlatPack(object):
    """bf16 mirror of the flat parameter buffer. `wb` (KRSC bf16, the fprop / wgrad weight operand of every conv) is
    written by the SGD kernel itself; `wt` (flipped-transposed dgrad operand) of ALL conv weights is produced by one
    tsb_pack_wt_multi launch the first time a dgrad asks for it after a step. ops.pack_cache consults this through
    the `_tsb_pack = (FlatPack, index)` attribute set on every parameter."""

    def __init__(self, params, spans, n, device):
        self.params = params
        self.spans = spans
        self.wb_flat = torch.zeros(n, dtype=torch.bfloat16, device=device)
        self.wt_flat = torch.zeros(n, dtype=torch.bfloat16, device=device)
        self.fresh = False
        self.wt_done = False
        self.versions = [None] * len(params)
        desc, bstart, nb = [], [], 0
        self.wt_index = {}
        import struct
        for i, (p, (lo, hi)) in enumerate(zip(params, spans)):
            if p.dim() == 4 and p.shape[1] % 8 == 0 and p.shape[0] % 8 == 0 and \
                    p.permute(0, 2, 3, 1).is_contiguous():
                K, C, R, S = p.shape
                tk, tc = (K + 31) // 32, (C + 31) // 32
                desc.append(struct.pack("<qiiiiii", lo, K, R * S, C, tk, tc, 0))
                bstart.append(nb)
                nb += R * S * tk * tc
                self.wt_index[i] = True
            p._tsb_pack = (self, i)
        self.nblocks = nb
        self.ntensors = len(desc)
        if desc:
            raw = torch.frombuffer(bytearray(b"".join(desc)), dtype=torch.uint8)
            self.desc = raw.to(device)
            self.bstart = torch.tensor(bstart, dtype=torch.int32, device=device)

    def mark_fresh(self):
        self.fresh = True
        self.wt_done = False
        self.versions = [p._version for p in self.params]

    def lookup(self, w, idx, want_t):
        """(wb, wt) views for parameter idx, or None when the mirror is stale for it"""
        if not self.fresh or w._version != self.versions[idx] or w.dim() != 4:
            return None
        if not w.permute(0, 2, 3, 1).is_contiguous():
            return None
        lo = self.spans[idx][0]
        K, C, R, S = w.shape
        n = K * C * R * S
        wb = self.wb_flat[lo:lo + n].view(K, R, S, C)
        wt = None
        if want_t:
            if idx not in self.wt_index:
                return None
            if not self.wt_done:
                call("tsb_pack_wt_multi", ptr(self.wb_flat), ptr(self.wt_flat), ptr(self.desc), ptr(self.bstart),
                     self.ntensors, self.nblocks, stream())
                self.wt_done = True
            wt = self.wt_flat[lo:lo + n].view(C, R, S, K)
        return wb, wt


class SGD(object):
    def __init__(self, params, lr, momentum=0.0, weight_decay=0.0):
        groups = list(params)
        if len(groups) > 0 and not isinstance(groups[0], dict):
            groups = [dict(params=groups)]
        self.defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay)
        self.param_groups = []
        for g in groups:
            g = dict(g)
            g["params"] = list(g["params"])
            for k, v in self.defaults.items():
                g.setdefault(k, v)
            self.param_groups.append(g)
        self.momentum = momentum
        self._params = [p for g in self.param_groups for p in g["params"]]
        assert len(set(id(p) for p in self._params)) == len(self._params), "a parameter appears in two groups"
        self.flat_param, self._spans = flatten(self._params, "data")
        self.flat_grad, _ = ensure_flat_grads(self._params, take_over=True)
        self.flat_mom = torch.zeros_like(self.flat_param)
        self.pack = FlatPack(self._params, self._spans, self.flat_param.numel(), self.flat_param.device)
        ends, idx = [], 0
        for g in self.param_groups:
            idx += len(g["params"])
            ends.append(self._spans[idx - 1][1] if idx > 0 else 0)
        dev = self.flat_param.device
        self._seg_end = torch.tensor(ends, dtype=torch.int64, device=dev)
        self._steps = 0
        self.grad_scale = 1.0
        # per-group lr / weight-decay scalars read by the kernel from device memory. Eager steps build them per call;
        # a captured step (engine.graph.GraphedTrainStep) reads this persistent device tensor instead, which the
        # graphed loop refreshes with `push_hyperparams()` (a small eager copy) before every replay.
        ng = len(self.param_groups)
        self._hp_dev = torch.zeros(2 * ng, dtype=torch.float32, device=dev)

    def zero_grad(self, set_to_none=False):
        self.flat_grad, _ = ensure_flat_grads(self._params)   # raises if another owner took these gradients over
        self.flat_grad.zero_()
        ops.zero_arena.reset()

    def push_hyperparams(self):
        """copy the current param_groups lr / weight_decay into the persistent device tensor (eager, outside any capture)"""
        vals = [float(g["lr"]) for g in self.param_groups] + [float(g["weight_decay"]) for g in self.param_groups]
        self._hp_dev.copy_(torch.tensor(vals, dtype=torch.float32))

    def step(self, closure=None):
        self.flat_grad, _ = ensure_flat_grads(self._params)
        check_inside(self._params, self.flat_grad, self._spans)
        ng = len(self.param_groups)
        dev = self.flat_param.device
        if dev.type == "cuda" and torch.cuda.is_current_stream_capturing():
            # graph capture: no host→device traffic inside the graph; the caller keeps _hp_dev current (push_hyperparams)
            lr, wd = self._hp_dev[:ng], self._hp_dev[ng:]
        else:
            # eager: a pageable H2D copy is staged at call time, so a CPU running ahead can never change the values of
            # a step that has not executed yet
            lr = torch.tensor([float(g["lr"]) for g in self.param_groups], dtype=torch.float32, device=dev)
            wd = torch.tensor([float(g["weight_decay"]) for g in self.param_groups], dtype=torch.float32, device=dev)
        call("tsb_sgd_flat_pack", ptr(self.flat_param), ptr(self.flat_grad), ptr(self.flat_mom), self.flat_param.numel(),
             ptr(self._seg_end), ptr(lr), ptr(wd), len(self.param_groups), float(self.momentum), float(self.grad_scale),
             0, ptr(self.pack.wb_flat), stream())   # first_step = 0: the momentum buffer starts at exact zeros, and
        # fma(momentum, 0, g) == g, so step 1 needs no special case (nothing step-dependent is baked into a captured graph)
        self._steps += 1
        ops.pack_cache.invalidate()  # per-tensor bf16 packs are stale now
        self.pack.mark_fresh()       # ... and the flat bf16 mirror written by the kernel above is current

    # ---- checkpoint format: torch.optim.SGD's (what the reference stores under 'optimizer',
    # TorchSeg furnace/engine/engine.py:103,142-146): {'state': {i: {'momentum_buffer': [K,C,R,S] fp32}},
    # 'param_groups': [{'lr','momentum','dampening','weight_decay','nesterov',..., 'params': [indices]}]}
    def state_dict(self):
        groups, idx = [], 0
        for g in self.param_groups:
            d = {k: v for k, v in g.items() if k != "params"}
            d.setdefault("dampening", 0)
            d.setdefault("nesterov", False)
            d.setdefault("maximize", False)
            d.setdefault("foreach", None)
            d.setdefault("differentiable", False)
            d.setdefault("fused", None)
            d["params"] = list(range(idx, idx + len(g["params"])))
            idx += len(g["params"])
            groups.append(d)
        state = {}
        if self._steps > 0 and self.momentum != 0:
            mom = self.flat_mom.detach().cpu()
            for i, (p, (lo, hi)) in enumerate(zip(self._params, self._spans)):
                # logical [K,C,R,S] view with the parameter's strides, made contiguous (NCHW) like torch's buffer
                state[i] = {"momentum_buffer": torch.as_strided(mom, p.shape, p.stride(), lo).contiguous()}
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        if "flat_momentum" in sd:          # round-1 native format
            self.flat_mom.copy_(sd["flat_momentum"])
            self._steps = int(sd["steps"])
        else:
            state = sd.get("state", {})
            n_in = sum(len(g["params"]) for g in sd["param_groups"])
            if n_in != len(self._params) or len(sd["param_groups"]) != len(self.param_groups):
                raise ValueError("loaded state dict has a different number of parameter groups / parameters")
            self.flat_mom.zero_()
            got = 0
            order = [i for g in sd["param_groups"] for i in g["params"]]   # saved index of our k-th parameter
            for k, (p, (lo, hi)) in enumerate(zip(self._params, self._spans)):
                ent = state.get(order[k], state.get(str(order[k])))
                buf = None if ent is None else ent.get("momentum_buffer")
                if buf is None:
                    continue
                if tuple(buf.shape) != tuple(p.shape):
                    raise ValueError("momentum_buffer %d has shape %s, parameter has %s" % (k, tuple(buf.shape), tuple(p.shape)))
                torch.as_strided(self.flat_mom, p.shape, p.stride(), lo).copy_(buf)
                got += 1
            # torch creates a parameter's buffer at its first step with a gradient: any buffer present ⇒ not the first step
            self._steps = 1 if got > 0 else 0
        for g, s_ in zip(self.param_groups, sd["param_groups"]):
            g.update({k: v for k, v in s_.items() if k != "params"})
