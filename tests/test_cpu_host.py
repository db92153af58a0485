"""CPU tests of the host-side mirror of the furnace API: Engine / State / checkpoints, LR policies, init_weight /
group_weight, parse_devices, the FCN-R18 plumbing case (BASELINE configs[0]) and the world_size-2 gloo paths of
the DDP / all_reduce_tensor replacements."""
import argparse
import os
import sys

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_poly_lr_matches_reference_formula():
    from torchseg_b200.engine.lr_policy import PolyLR, MultiStageLR, LinearIncreaseLR
    p = PolyLR(1e-2, 0.9, 80000)
    assert p.get_lr(0) == 1e-2
    assert abs(p.get_lr(40000) - 1e-2 * 0.5 ** 0.9) < 1e-12
    assert MultiStageLR([(10, 0.1), (20, 0.01)]).get_lr(15) == 0.01
    assert abs(LinearIncreaseLR(0.0, 1.0, 10).get_lr(5) - 0.5) < 1e-12


def test_init_and_group_weight_semantics():
    from torchseg_b200.networks import BiSeNet
    from torchseg_b200.utils.init_func import init_weight, group_weight
    m = BiSeNet(19, True, None, None, nn.BatchNorm2d)
    init_weight(m.business_layer, nn.init.kaiming_normal_, nn.BatchNorm2d, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    assert m.spatial_path.conv_7x7.bn.eps == 1e-5 and float(m.ffm.conv_1x1.bn.weight.min()) == 1.0
    groups = group_weight([], m.context_path, nn.BatchNorm2d, 1e-2)
    for mod in (m.spatial_path, m.global_context, m.arms, m.refines, m.heads, m.ffm):
        groups = group_weight(groups, mod, nn.BatchNorm2d, 1e-1)
    assert len(groups) == 14                      # train.py:70-84 → 7 x (decay, no-decay)
    assert sum(len(g["params"]) for g in groups) == len(list(m.parameters()))
    assert all(g.get("weight_decay", None) == 0.0 for g in groups[1::2])
    # completeness assert fires for a module holding a bare Parameter (init_func.py:52-53)
    class Bad(nn.Module):
        def __init__(self):
            super().__init__()
            self.p = nn.Parameter(torch.zeros(3))
    with pytest.raises(AssertionError):
        group_weight([], Bad(), nn.BatchNorm2d, 0.1)


def test_prepare_model_keeps_values_and_keys():
    import torchseg_b200
    from torchseg_b200.networks import BiSeNet
    m = BiSeNet(19, True, None, None, nn.BatchNorm2d)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    ids = [id(p) for p in m.parameters()]
    torchseg_b200.prepare_model(m)
    assert ids == [id(p) for p in m.parameters()]
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k])
    w = m.context_path.layer1[0].conv1.weight
    assert w.permute(0, 2, 3, 1).is_contiguous()   # KRSC physical layout


def test_parse_devices_and_engine_cli(monkeypatch, tmp_path):
    from torchseg_b200.utils.pyt_utils import parse_devices
    from torchseg_b200.engine.engine import Engine
    assert parse_devices('') == [0] or len(parse_devices('')) >= 1
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    parser = argparse.ArgumentParser()
    with Engine(custom_parser=parser, argv=[]) as engine:
        assert engine.distributed is False and engine.world_size == 1
        assert engine.continue_state_object is None
        engine.update_iteration(3, 7)
        assert engine.state.epoch == 3 and engine.state.iteration == 7
        with pytest.raises(AssertionError):
            engine.register_state(bogus=1)
    with pytest.raises(SystemExit):   # -c must name an existing file (extant_file)
        Engine(custom_parser=argparse.ArgumentParser(), argv=["-c", str(tmp_path / "missing.pth")])


def test_fcn_r18_plumbing_cpu(tmp_path, monkeypatch):
    """BASELINE configs[0]: FCN-32s R18, 2 x 256 x 256, CPU, 1 process — the train.py sequence (Engine, group_weight,
    SGD, PolyLR, checkpoint save / link / restore) with the loss evaluated by the oracle restatement on the
    module's own parameters (the CUDA kernels do not run on a CPU)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from golden_cases import fcn_case
    from oracle import torch_ref
    from torchseg_b200.engine.engine import Engine
    from torchseg_b200.engine.lr_policy import PolyLR
    from torchseg_b200.networks import FCN
    from torchseg_b200.utils.init_func import init_weight, group_weight
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    x, y, seed = fcn_case()
    with Engine(custom_parser=argparse.ArgumentParser(), argv=[]) as engine:
        torch.manual_seed(seed)
        model = FCN(19, backbone="R18")
        init_weight(model.business_layer, nn.init.kaiming_normal_, nn.BatchNorm2d, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
        groups = group_weight([], model.backbone, nn.BatchNorm2d, 1e-2)
        for m in model.business_layer:
            groups = group_weight(groups, m, nn.BatchNorm2d, 1e-1)
        opt = torch.optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=1e-4)
        lr_policy = PolyLR(1e-2, 0.9, 10)
        engine.register_state(dataloader=None, model=model, optimizer=opt)
        losses = []
        for it in range(3):
            opt.zero_grad()
            engine.update_iteration(0, it)
            sd = dict(model.named_parameters())
            sd.update(dict(model.named_buffers()))
            loss = torch_ref.fcn_r18_loss(x, y, sd)
            lr = lr_policy.get_lr(it)
            for i, g in enumerate(opt.param_groups):
                g['lr'] = lr if i < 2 else lr * 10
            loss.backward()
            opt.step()
            losses.append(float(loss))
        assert losses[-1] < losses[0]
        snap = tmp_path / "log" / "snapshot"
        engine.save_and_link_checkpoint(str(snap), str(tmp_path / "log"), str(tmp_path / "log_link"))
        ck = torch.load(str(snap / "epoch-0.pth"), weights_only=False)
        assert set(ck.keys()) == {"model", "optimizer", "epoch", "iteration"}       # engine.py:95-105
        assert not any(k.startswith("module.") for k in ck["model"])
        assert os.path.islink(str(snap / "epoch-last.pth"))
        # restore into a fresh model through -c
        model2 = FCN(19, backbone="R18")
        opt2 = torch.optim.SGD(group_weight([], model2, nn.BatchNorm2d, 1e-2), lr=1e-2, momentum=0.9)
    with Engine(custom_parser=argparse.ArgumentParser(), argv=["-c", str(snap / "epoch-last.pth")]) as e2:
        groups2 = group_weight([], model2.backbone, nn.BatchNorm2d, 1e-2)
        for m in model2.business_layer:
            groups2 = group_weight(groups2, m, nn.BatchNorm2d, 1e-1)
        opt2 = torch.optim.SGD(groups2, lr=1e-2, momentum=0.9, weight_decay=1e-4)
        e2.register_state(dataloader=None, model=model2, optimizer=opt2)
        e2.restore_checkpoint()
        assert e2.state.epoch == 1 and e2.state.iteration == 2                     # engine.py:144-145
        for (k, a), (_, b) in zip(model.state_dict().items(), model2.state_dict().items()):
            assert torch.equal(a, b), k


# ------------------------------------------------------------------------------------------------- world_size 2
def _worker(rank, world, port, q):
    # the gloo (CPU) path: on a host with fewer GPUs than ranks the Engine would pick NCCL and a missing device
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank), CUDA_VISIBLE_DEVICES="")
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from torchseg_b200.engine.engine import Engine
    from torchseg_b200.utils.pyt_utils import all_reduce_tensor
    from torchseg_b200.apex.parallel import DistributedDataParallel, SyncBatchNorm
    try:
        with Engine(custom_parser=argparse.ArgumentParser(), argv=[]) as engine:
            assert engine.distributed and engine.world_size == world and engine.local_rank == rank
            assert engine.devices == list(range(world))
            t = all_reduce_tensor(torch.tensor([float(rank + 1)]), world_size=world)
            assert abs(float(t) - sum(range(1, world + 1)) / world) < 1e-6           # pyt_utils.py:34-39
            torch.manual_seed(rank)                                                   # ranks start different …
            net = nn.Sequential(nn.Conv2d(3, 4, 3, padding=1, bias=False), SyncBatchNorm(4), nn.Conv2d(4, 2, 1))
            ddp = DistributedDataParallel(net, bucket_bytes=64)                        # … the ctor broadcasts rank 0
            w0 = [p.detach().clone() for p in net.parameters()]
            gathered = [torch.zeros_like(w0[0]) for _ in range(world)]
            dist.all_gather(gathered, w0[0])
            assert all(torch.equal(g, gathered[0]) for g in gathered)
            # per-rank gradients g_r = (rank+1) * ones → averaged to mean(rank+1)
            ddp.zero_grad()
            loss = sum(((rank + 1.0) * p).sum() for p in net.parameters())
            loss.backward()
            ddp.finish_reduce()
            expect = sum(range(1, world + 1)) / world
            for p in net.parameters():
                assert torch.allclose(p.grad, torch.full_like(p.grad, expect)), (rank, p.grad.flatten()[:3])
                # gradients are views into ONE flat buffer
                lo = ddp.flat_grad.data_ptr()
                assert lo <= p.grad.data_ptr() < lo + ddp.flat_grad.numel() * 4
            # overlap=False (the form GraphedTrainStep captures): hooks reduce nothing, finish_reduce() issues ONE
            # all-reduce of the whole flat buffer and averages it
            ddp.overlap = False
            ddp.zero_grad()
            loss = sum(((rank + 2.0) * p).sum() for p in net.parameters())
            loss.backward()
            for p in net.parameters():                                                # still the local gradient
                assert torch.allclose(p.grad, torch.full_like(p.grad, rank + 2.0))
            ddp.finish_reduce()
            expect = sum(range(2, world + 2)) / world
            for p in net.parameters():
                assert torch.allclose(p.grad, torch.full_like(p.grad, expect)), (rank, p.grad.flatten()[:3])
            assert not ddp._pending
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: %s\n%s" % (e, traceback.format_exc())))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def test_ddp_and_allreduce_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 400)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    assert all(r[1] == "ok" for r in res), res


def test_grad_share_protocol():
    """ops.GradShare: first contributor's gradient is stashed (autograd gets None), the last one returns the shared
    buffer; a late contributor that could not accumulate in place is added explicitly; the object re-arms"""
    from torchseg_b200 import ops
    g = ops.GradShare(2)
    a = torch.ones(3)
    assert g.contribute(a) is None and g.stash is a
    a.add_(2.0)                                  # what the second consumer's dgrad epilogue does in place
    out = g.contribute(a, accumulated=True)
    assert out is a and float(out.sum()) == 9.0
    assert g.stash is None and g.left == 2       # re-armed
    # three contributors, the last one not in place
    g3 = ops.GradShare(3)
    b = torch.full((2,), 1.0)
    assert g3.contribute(b) is None
    assert g3.contribute(b, accumulated=True) is None
    out = g3.contribute(torch.full((2,), 5.0))
    assert torch.equal(out, torch.full((2,), 6.0))


def test_ragged_channel_padding_is_differentiable():
    """seg_oprs._pad_weight / _pad_vec (DFN's 21 / 171 / 9-channel layers): zero extension in KRSC layout whose autograd
    slices the gradient back to the reference-shaped parameter"""
    from torchseg_b200.seg_opr import seg_oprs as so
    w = torch.randn(21, 9, 3, 3).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2).requires_grad_(True)   # KRSC-backed
    wp = so._pad_weight(w, 64, 64)
    assert tuple(wp.shape) == (64, 64, 3, 3) and wp.permute(0, 2, 3, 1).is_contiguous()
    assert torch.equal(wp[:21, :9], w) and float(wp[21:].abs().sum()) == 0 and float(wp[:, 9:].abs().sum()) == 0
    gfull = torch.randn(64, 64, 3, 3)
    wp.backward(gfull)
    assert torch.equal(w.grad, gfull[:21, :9])
    v = torch.randn(21, requires_grad=True)
    vp = so._pad_vec(v, 64, 1.0)
    assert float(vp[21:].min()) == 1.0
    vp.sum().backward()
    assert torch.equal(v.grad, torch.ones(21))
    assert so._ceil_to(171, 64) == 192 and so._ceil_to(64, 64) == 64


def test_flat_pack_descriptor_table_and_staleness():
    """optim.FlatPack: one 32-byte descriptor per eligible conv weight (offset, K, R*S, C, 32x32 tile counts), block
    prefix sums, and the freshness protocol (stale before the first step / after an in-place weight edit)"""
    import struct
    from torchseg_b200 import optim, prepare_model
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Conv2d(16, 40, 3, bias=False), torch.nn.BatchNorm2d(40),
                              torch.nn.Conv2d(40, 24, 1, bias=True), torch.nn.Conv2d(3, 8, 3, bias=False))
    prepare_model(net)
    opt = optim.SGD(list(net.parameters()), lr=0.1, momentum=0.9)
    fp = opt.pack
    assert all(p._tsb_pack[0] is fp for p in net.parameters())
    # eligible: K % 8 == 0 and C % 8 == 0 → the 16->40 3x3 and the 40->24 1x1; the 3-channel conv is not
    assert fp.ntensors == 2
    raw = bytes(fp.desc.numpy().tobytes())
    d0 = struct.unpack("<qiiiiii", raw[:32])
    d1 = struct.unpack("<qiiiiii", raw[32:64])
    assert d0[1:6] == (40, 9, 16, 2, 1) and d1[1:6] == (24, 1, 40, 1, 2)
    assert d0[0] == opt._spans[0][0] and d1[0] == opt._spans[3][0] and d0[0] % 8 == 0 and d1[0] % 8 == 0
    assert fp.bstart.tolist() == [0, 9 * 2 * 1] and fp.nblocks == 18 + 2
    w = net[0].weight
    assert fp.lookup(w, w._tsb_pack[1], False) is None          # no optimiser step yet → per-tensor pack path
    fp.mark_fresh()
    hit = fp.lookup(w, w._tsb_pack[1], False)
    assert hit is not None and tuple(hit[0].shape) == (40, 3, 3, 16) and hit[1] is None
    with torch.no_grad():
        w.mul_(2.0)                                              # in-place edit bumps the version → stale again
    assert fp.lookup(w, w._tsb_pack[1], False) is None
    opt.push_hyperparams()
    assert abs(float(opt._hp_dev[0]) - 0.1) < 1e-7 and float(opt._hp_dev[1]) == 0.0


def test_flat_grad_layout_ownership():
    """ADVICE r1: two owners over different parameter lists must not silently re-point .grad (the first owner would keep
    stepping on a stale buffer of zeros): same set → DDP re-uses the optimiser's layout; a new optimiser takes over and
    the OLD owner then fails loudly; anything else is refused."""
    from torchseg_b200 import flat
    a = [nn.Parameter(torch.randn(4, 3)), nn.Parameter(torch.randn(5))]
    b = [nn.Parameter(torch.randn(2, 2))]
    fa, spans_a = flat.ensure_flat_grads(a, take_over=True)
    assert flat.ensure_flat_grads(a)[0] is fa                      # idempotent
    lay = flat.layout_of(list(reversed(a)))                        # same SET, any order → the registered layout
    assert lay is not None and lay[0] is fa and lay[2][0] is a[0]
    with pytest.raises(RuntimeError, match="layout conflict"):     # overlapping, different list, no take-over
        flat.ensure_flat_grads(a + b)
    assert a[0].grad.data_ptr() == fa.data_ptr()                   # ... and nothing was re-pointed
    fab, _ = flat.ensure_flat_grads(a + b, take_over=True)         # a new optimiser takes the parameters over
    assert a[0].grad.data_ptr() == fab.data_ptr()
    with pytest.raises(RuntimeError, match="layout conflict"):     # the old owner's zero_grad()/step() now raises
        flat.ensure_flat_grads(a)
    a[0].grad = None                                               # set_to_none upstream: the view is re-established
    flat.ensure_flat_grads(a + b)
    assert a[0].grad.data_ptr() == fab.data_ptr()
    with pytest.raises(RuntimeError):
        flat.check_inside(a, fa, spans_a)
    flat.release(a + b)


def test_fused_sgd_state_dict_is_torch_format():
    """engine.py:103,142-146 store optimizer.state_dict(): the fused SGD reads and writes torch.optim.SGD's format"""
    from torchseg_b200 import optim, flat
    torch.manual_seed(0)
    conv = nn.Conv2d(8, 16, 3, bias=True)
    import torchseg_b200
    torchseg_b200.prepare_model(conv)   # KRSC strides: momentum buffers must still come out as logical NCHW
    bn = nn.BatchNorm2d(16)
    groups = [dict(params=[conv.weight], lr=1e-2, weight_decay=5e-4),
              dict(params=[conv.bias, bn.weight, bn.bias], lr=1e-1, weight_decay=0.0)]
    ref = torch.optim.SGD([dict(g) for g in groups], lr=1e-2, momentum=0.9, weight_decay=5e-4)
    for p in ref.param_groups[0]["params"] + ref.param_groups[1]["params"]:
        p.grad = torch.randn_like(p)
    ref.step()
    sd_ref = ref.state_dict()
    for p in (conv.weight, conv.bias, bn.weight, bn.bias):
        p.grad = None
    opt = optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)
    assert opt.state_dict()["state"] == {}                      # fresh optimiser: no buffers, like torch
    opt.load_state_dict(sd_ref)                                 # a reference / torch.optim.SGD checkpoint restores
    assert opt._steps == 1
    sd = opt.state_dict()
    assert set(sd.keys()) == {"state", "param_groups"}
    assert [g["params"] for g in sd["param_groups"]] == [g["params"] for g in sd_ref["param_groups"]]
    for i, ent in sd_ref["state"].items():
        got = sd["state"][i]["momentum_buffer"]
        assert got.is_contiguous() and torch.equal(got, ent["momentum_buffer"])
    for g, gr in zip(sd["param_groups"], sd_ref["param_groups"]):
        for k in ("lr", "momentum", "weight_decay", "dampening", "nesterov"):
            assert g[k] == gr[k], k
    ref2 = torch.optim.SGD([dict(g) for g in groups], lr=1e-2, momentum=0.9, weight_decay=5e-4)
    ref2.load_state_dict(sd)                                    # ... and the reference can resume from ours
    assert torch.equal(ref2.state_dict()["state"][0]["momentum_buffer"], sd_ref["state"][0]["momentum_buffer"])
    # round-1 native format still loads
    opt.load_state_dict({"flat_momentum": opt.flat_mom.clone(), "steps": 3,
                         "param_groups": [{"lr": 0.5}, {"lr": 0.25}]})
    assert opt._steps == 3 and opt.param_groups[0]["lr"] == 0.5
    flat.release(opt._params)


def test_pack_cache_is_bounded_and_packed_image_matches_by_identity(monkeypatch):
    """ADVICE r1: (a) one pack entry per (weight, kind) — a version bump overwrites, dead weights are swept;
    (b) the space-to-depth image cache matches by tensor identity, not by address"""
    from torchseg_b200 import ops
    from torchseg_b200.seg_opr import seg_oprs
    calls = []
    monkeypatch.setattr(ops, "call", lambda name, *a: calls.append(name))
    monkeypatch.setattr(ops, "ptr", lambda t: 0)
    monkeypatch.setattr(ops, "stream", lambda: 0)
    pc = ops._PackCache()
    w = nn.Parameter(torch.randn(8, 8, 3, 3).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2))
    pc.get(w, False)
    pc.get(w, False)
    assert calls.count("tsb_pack_weight") == 1 and len(pc.cache) == 1
    pc.get(w, True)                                # now the transposed operand is needed too: re-pack, same entry
    assert calls.count("tsb_pack_weight") == 2 and len(pc.cache) == 1
    for _ in range(5):                             # torch.optim-style in-place updates bump the version
        with torch.no_grad():
            w.add_(1.0)
        pc.get(w, True)
    assert len(pc.cache) == 1 and calls.count("tsb_pack_weight") == 7
    for _ in range(600):                           # per-forward temporaries (DFN's padded weights) are swept
        t = torch.randn(8, 8, 1, 1).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        pc.get(t, False)
        del t
    assert len(pc.cache) < 520
    # (b)
    packs = []
    monkeypatch.setattr(ops, "pack_image_s2d", lambda img: packs.append(img) or ("packed", len(packs)))
    seg_oprs._release_packed_image()
    img = torch.zeros(1, 3, 8, 8)
    p1 = seg_oprs._packed_image(img)
    assert seg_oprs._packed_image(img) is p1 and len(packs) == 1
    twin = torch.as_strided(img, img.shape, img.stride())      # same storage/address, another tensor object
    assert twin.data_ptr() == img.data_ptr()
    assert seg_oprs._packed_image(twin) is not p1 and len(packs) == 2
    img2 = torch.zeros(1, 3, 8, 8)
    seg_oprs._packed_image(img2)
    img2.add_(1.0)                                              # refilled in place → new version → re-pack
    seg_oprs._packed_image(img2)
    assert len(packs) == 4
    seg_oprs._release_packed_image()
    assert not seg_oprs._s2d_cache


# ------------------------------------------------------------------------------------------------- evaluator worker pool
class _ToyDataset(object):
    def __init__(self, n):
        self.n = n

    def get_length(self):
        return self.n

    def __getitem__(self, idx):
        g = torch.Generator().manual_seed(idx)
        return dict(data=torch.rand(6, 8, 3, generator=g).numpy().astype("float32") * 255,
                    label=torch.randint(0, 3, (6, 8), generator=g).numpy(), fn=str(idx), n=self.n)


class _ToyNet(nn.Module):
    def __init__(self):
        super(_ToyNet, self).__init__()
        self.conv = nn.Conv2d(3, 3, 1)

    def forward(self, x):
        return torch.log_softmax(self.conv(x), dim=1)


def _toy_evaluator(devices):
    from torchseg_b200.engine.evaluator import Evaluator

    class _Ev(Evaluator):
        def func_per_iteration(self, data, device):
            pred = self.whole_eval(data['data'], None, device=None)
            return dict(idx=int(data['fn']), correct=int((pred == data['label']).sum()), labeled=int(data['label'].size))

        def compute_metric(self, results):
            c = sum(r['correct'] for r in results)
            return "n=%d correct=%d order=%s" % (len(results), c, sorted(r['idx'] for r in results))

    import numpy as np
    torch.manual_seed(0)
    ev = _Ev(_ToyDataset(7), 3, np.array([0.5, 0.5, 0.5]), np.array([0.25, 0.25, 0.25]), None, [1.0], False, devices)
    ev.val_func = _ToyNet()
    return ev


def test_evaluator_worker_pool_matches_single_process():
    """furnace/engine/evaluator.py:97-163: the per-device worker pool (spawned processes, contiguous dataset shreds, results
    queue) returns the same metric line as the single-process loop — host logic, run here with two CPU 'devices'"""
    single = _toy_evaluator(["cpu"]).single_process_evalutation()
    one = _toy_evaluator(["cpu"]).multi_process_evaluation()           # nr_devices == 1 branch (:134-143)
    assert one == single
    import multiprocessing
    if multiprocessing.get_start_method(allow_none=True) not in (None, "fork", "spawn", "forkserver"):
        pytest.skip("no usable multiprocessing start method")
    ev = _toy_evaluator(["cpu", "cpu"])
    ev.context = multiprocessing.get_context("fork")     # (classes defined inside a test module do not survive 'spawn' pickling)
    pooled = ev.multi_process_evaluation()
    assert pooled == single and "n=7" in pooled
