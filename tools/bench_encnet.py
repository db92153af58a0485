"""EncNet (ResNet-101 v1c, dilated-8) training-step benchmark on one GPU: 16 x 480^2 crops, 150 classes (ADE), ignore -1,
SGD.

    python tools/bench_encnet.py [--batch 16] [--size 480] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                                 [--enc-iters 50] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events, launches per
    step and peak memory;
  * the same step for the oracle (tests/encnet_oracle.py) on cuDNN, strict fp32 and bf16 autocast + channels_last (the
    oracle's Encoding forms the [B, HW, K, D] residuals, so it may run out of memory: that is reported, not hidden);
  * tsb_encoding_fwd / tsb_encoding_bwd at 16 x 60^2 x 512 (the ADE step) and 16 x 128^2 x 512 (Cityscapes-size maps):
    kernel time from CUDA events over many launches and GB/s of algorithmic bytes (each operand read or written once);
  * the card name, power limit and max SM clock (nvidia-smi, read-only query) of the run.
--dump-outputs DIR writes the last timed step's loss and a seeded sample of the updated parameters (.npy), so two runs
can be compared bit for bit.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the oracle (test infrastructure) for the reference arm
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_x39 import dump_outputs, gpu_info, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
SEED = 12345
NUM_CLASSES, IGNORE = 150, -1


def synth_batch(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, h, w, generator=g)
    y = torch.randint(0, NUM_CLASSES, (n, h, w), generator=g, dtype=torch.int64)
    y[:, : h // 10] = IGNORE
    return x, y


def _model(criterion):
    from torchseg_b200.networks import EncNet
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(SEED)
    m = EncNet(NUM_CLASSES, criterion, norm_layer=BN)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    return m


def build(dev):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.utils.init_func import group_weight
    model = _model(torch.nn.CrossEntropyLoss(ignore_index=IGNORE))
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.train()
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return model, optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)


def product_arm(dev, n, h, w, steps, warmup):
    from torchseg_b200.engine.graph import GraphedTrainStep
    model, opt = build(dev)
    x, y = synth_batch(n, h, w, 7)
    x, y = x.to(dev), y.to(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    torch.cuda.set_stream(torch.cuda.Stream())
    step = GraphedTrainStep(model, opt, [x, y], warmup=2)
    if step.graph is None:
        raise RuntimeError("CUDA graph capture failed: %s" % step.error)
    for _ in range(warmup):
        step(x, y)
    torch.cuda.synchronize()
    ms, loss = time_events(lambda: step(x, y), steps)
    loss = float(loss.detach())
    torch.cuda.set_stream(torch.cuda.default_stream())
    return dict(value=n / (ms / 1e3), unit="images/sec", ms_per_step=ms, batch=n, steps=steps, warmup=warmup,
                final_loss=loss, launches_per_step=step.launches_per_step,
                peak_memory_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)), model, loss


def reference_arm(dev, n, h, w, steps, warmup, mode, sd0):
    """the oracle step under cuDNN (benchmark on); 'fp32' strict, 'bf16' autocast + channels_last"""
    import torch.nn.functional as F
    import encnet_oracle as tr
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = mode != "fp32"
    try:
        sd, params = {}, []
        for k, v in sd0.items():
            v = v.detach().clone().to(dev)
            if mode == "bf16" and v.dim() == 4:
                v = v.contiguous(memory_format=torch.channels_last)
            if v.is_floating_point() and "running" not in k:
                v.requires_grad_(True)
                params.append(v)
            sd[k] = v
        opt = torch.optim.SGD(params, lr=1e-2, momentum=0.9, weight_decay=5e-4)
        x, y = synth_batch(n, h, w, 7)
        x, y = x.to(dev), y.to(dev)
        if mode == "bf16":
            x = x.contiguous(memory_format=torch.channels_last)
        stats = {}

        def one():
            opt.zero_grad()
            if mode == "bf16":   # the network under autocast, the three losses in fp32 (BCELoss refuses autocast)
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    lo, se, l3 = tr.encnet_logits(x, sd, 1e-5, 0.1, True, stats)
                    aux = tr.conv_bn_relu(l3, sd, "aux_layer.0", 1, 1, stats=stats)
                    aux = F.conv2d(aux, sd["aux_layer.2.weight"], sd["aux_layer.2.bias"])
                up = lambda t: F.interpolate(t.float(), size=(h, w), mode="bilinear", align_corners=True)
                loss = (F.cross_entropy(up(lo), y, ignore_index=IGNORE) +
                        0.2 * F.cross_entropy(up(aux), y, ignore_index=IGNORE) +
                        0.2 * tr.se_loss(se.float(), y, NUM_CLASSES))
            else:
                loss, _ = tr.encnet_loss(x, y, sd, stats=stats)
            loss.backward()
            opt.step()
            return loss

        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        ms, loss = time_events(one, steps)
        return dict(value=n / (ms / 1e3), unit="images/sec", ms_per_step=ms, steps=steps, warmup=warmup,
                    final_loss=float(loss.detach()))
    finally:
        torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


def encoding_arm(dev, iters, shapes=((16, 60, 512, 32), (16, 128, 512, 32))):
    """tsb_encoding_{fwd,bwd} alone. Algorithmic bytes: forward reads x (bf16), codewords and scales and writes a, d²
    (fp32 [B·N, K]), Σa and E (bf16); backward reads dE, x, codewords, scales, a, d², Σa, writes dx and the fp32
    gradients of codewords and scales."""
    from torchseg_b200 import ops
    rows = []
    for B, hw, D, K in shapes:
        N = hw * hw
        g = torch.Generator(device=dev).manual_seed(1)
        x = (torch.randn(B, N, D, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        c = torch.randn(K, D, device=dev, generator=g) * 0.5
        s = -torch.rand(K, device=dev, generator=g) * (4.0 / D)
        a = torch.empty(B * N, K, device=dev)
        d2 = torch.empty_like(a)
        sa = torch.empty(B, K, device=dev)
        E = torch.empty(B * D, K, dtype=torch.bfloat16, device=dev)
        dE = torch.randn(B * D, K, device=dev, generator=g).to(torch.bfloat16)
        dx = torch.empty_like(x)
        dc, ds = torch.zeros(K, D, device=dev), torch.zeros(K, device=dev)
        st = ops.stream()
        calls = {
            "fwd": lambda: ops.call("tsb_encoding_fwd", x.data_ptr(), D, B, N, D, c.data_ptr(), s.data_ptr(), K,
                                    a.data_ptr(), d2.data_ptr(), sa.data_ptr(), E.data_ptr(), *ops.det_ws(), st),
            "bwd": lambda: ops.call("tsb_encoding_bwd", dE.data_ptr(), x.data_ptr(), D, B, N, D, c.data_ptr(),
                                    s.data_ptr(), K, a.data_ptr(), d2.data_ptr(), sa.data_ptr(), dx.data_ptr(), D,
                                    dc.data_ptr(), ds.data_ptr(), *ops.det_ws(), st),
        }
        act, asg, par = 2.0 * B * N * D, 4.0 * B * N * K, 4.0 * K * (D + 1)
        nbytes = {"fwd": act + par + 2 * asg + 4 * B * K + 2 * B * D * K,
                  "bwd": 2 * B * D * K + act + par + 2 * asg + 4 * B * K + act + par}
        for kind, fn in calls.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ms, _ = time_events(fn, iters)
            rows.append(dict(kind=kind, B=B, HW=N, D=D, K=K, us=round(ms * 1e3, 2), bytes=int(nbytes[kind]),
                             GBps=round(nbytes[kind] / (ms / 1e3) / 1e9, 1)))
        del x, a, d2, dx
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=480)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--enc-iters", type=int, default=50)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encnet measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="encnet_r101_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    line["encoding"] = encoding_arm(dev, args.enc_iters)
    if not args.no_ref:
        sd0 = {k: v.detach().clone() for k, v in _model(None).state_dict().items()}
        for mode in ("fp32", "bf16"):
            try:
                line["reference_%s" % mode] = reference_arm(dev, args.batch, args.size, args.size, args.ref_steps,
                                                            args.ref_warmup, mode, sd0)
            except torch.cuda.OutOfMemoryError as e:
                line["reference_%s" % mode] = dict(error="out of memory: %s" % str(e).split("\n")[0][:160])
                torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
