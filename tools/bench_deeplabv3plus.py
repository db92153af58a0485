"""DeepLabV3+ (ResNet-101 v1c, output stride 16) training-step benchmark on one GPU: 16 x 1024^2 crops, 19 classes, OHEM,
SGD.

    python tools/bench_deeplabv3plus.py [--batch 16] [--size 1024] [--steps 20] [--warmup 5] [--ref-steps 10] [--no-ref]
                                        [--dw-iters 50] [--dump-outputs DIR]

Prints one JSON line with
  * the graph-replayed libtsb step (engine.graph.GraphedTrainStep): img/s and ms/step from CUDA events, launches per
    step and peak memory;
  * the same step for the oracle (tests/deeplabv3plus_oracle.py) on cuDNN, strict fp32 and bf16 autocast +
    channels_last;
  * every dilated depthwise-conv launch shape of the step (fprop, dgrad, wgrad): kernel time from CUDA events over many
    launches, achieved GB/s against the algorithmic bytes (each operand read or written once) and that rate's share of
    the H100 SXM's 3.35 TB/s;
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

from bench_x39 import HBM_BYTES_PER_S, IGNORE, NUM_CLASSES, dump_outputs, gpu_info, synth_batch, time_events  # noqa: E402

BN = torch.nn.BatchNorm2d
SEED = 12345


def _model(criterion):
    from torchseg_b200.networks.deeplabv3plus import DeepLabV3Plus
    from torchseg_b200.utils.init_func import init_weight
    torch.manual_seed(SEED)
    m = DeepLabV3Plus(NUM_CLASSES, criterion, norm_layer=BN)
    init_weight(m.business_layer, torch.nn.init.kaiming_normal_, BN, 1e-5, 0.1, mode='fan_in', nonlinearity='relu')
    return m


def build(dev, n, h, w):
    import torchseg_b200
    from torchseg_b200 import optim
    from torchseg_b200.seg_opr.loss_opr import ProbOhemCrossEntropy2d
    from torchseg_b200.utils.init_func import group_weight
    model = _model(ProbOhemCrossEntropy2d(ignore_label=IGNORE, thresh=0.7, min_kept=n * h * w // 16, use_weight=False))
    model.to(dev)
    torchseg_b200.prepare_model(model)
    model.train()
    groups = group_weight([], model.backbone, BN, 1e-2)
    for m in model.business_layer:
        groups = group_weight(groups, m, BN, 1e-1)
    return model, optim.SGD(groups, lr=1e-2, momentum=0.9, weight_decay=5e-4)


def product_arm(dev, n, h, w, steps, warmup):
    from torchseg_b200.engine.graph import GraphedTrainStep
    model, opt = build(dev, n, h, w)
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
    import deeplabv3plus_oracle as tr
    from oracle.torch_ref import ohem_ce
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
        min_kept, stats = n * h * w // 16, {}
        drop = lambda t: F.dropout2d(t, 0.1, True)

        def one():
            opt.zero_grad()
            if mode == "bf16":
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    lo = tr.deeplabv3plus_logits(x, sd, 1e-5, 0.1, True, stats, drop)
                up = F.interpolate(lo.float(), size=(h, w), mode="bilinear", align_corners=True)
                loss = ohem_ce(up, y, IGNORE, 0.7, min_kept)
            else:
                loss, _ = tr.deeplabv3plus_loss(x, y, sd, min_kept, stats=stats, drop=drop)
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


def dw_shapes(size):
    """(C, input H = W, dilation, launches per step) of every depthwise conv of the step: the three atrous ASPP
    branches on the 1/16 map (2048 channels) and the two decoder refinements at 1/4 (304, 256 channels)"""
    s16 = size
    for _ in range(4):   # stem, max-pool, layer2, layer3 (each (H − 1) // 2 + 1)
        s16 = (s16 - 1) // 2 + 1
    s4 = (((size - 1) // 2 + 1) - 1) // 2 + 1
    return [(2048, s16, 6, 1), (2048, s16, 12, 1), (2048, s16, 18, 1), (304, s4, 1, 1), (256, s4, 1, 1)]


def dw_kernel_arm(dev, n, size, iters):
    from torchseg_b200 import ops
    rows = []
    for C, H, d, mult in dw_shapes(size):
        x = torch.randn(n, H, H, C, device=dev).to(torch.bfloat16)
        dy = torch.randn(n, H, H, C, device=dev).to(torch.bfloat16)
        y = torch.empty_like(x)
        dx = torch.empty_like(x)
        w = torch.randn(C, 9, device=dev)
        dw = torch.zeros(C, 9, device=dev)
        s = ops.stream()
        calls = {
            "fprop": lambda: ops.call("tsb_dwconv2d_fprop", x.data_ptr(), C, w.data_ptr(), y.data_ptr(), C, n, H, H, C, 1,
                                      d, s),
            "dgrad": lambda: ops.call("tsb_dwconv2d_dgrad", dy.data_ptr(), C, w.data_ptr(), dx.data_ptr(), C, n, H, H, C,
                                      1, d, 0, s),
            "wgrad": lambda: ops.call("tsb_dwconv2d_wgrad", x.data_ptr(), C, dy.data_ptr(), C, dw.data_ptr(), n, H, H, C,
                                      1, d, *ops.det_ws(), s),
        }
        act = 2.0 * n * H * H * C
        nbytes = {"fprop": 2 * act + 36 * C, "dgrad": 2 * act + 36 * C, "wgrad": 2 * act + 72 * C}
        for kind, fn in calls.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ms, _ = time_events(fn, iters)
            gbs = nbytes[kind] / (ms / 1e3) / 1e9
            rows.append(dict(kind=kind, N=n, C=C, H=H, W=H, dilation=d, per_step=mult, us=round(ms * 1e3, 2),
                             bytes=int(nbytes[kind]), GBps=round(gbs, 1), hbm_share=round(gbs * 1e9 / HBM_BYTES_PER_S, 3)))
        del x, dy, y, dx
    return rows, sum(r["us"] * r["per_step"] for r in rows)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=10)
    ap.add_argument("--ref-warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true", help="skip the oracle / cuDNN arms")
    ap.add_argument("--dw-iters", type=int, default=50)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deeplabv3plus measures the GPU step and needs a CUDA device")
    if args.steps < 20:
        raise SystemExit("--steps must be at least 20")
    from torchseg_b200 import build as tsb_build
    tsb_build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    line = dict(metric="deeplabv3plus_r101_train_step", gpu=gpu_info(), size=args.size)
    prod, model, loss = product_arm(dev, args.batch, args.size, args.size, args.steps, args.warmup)
    line["libtsb_graph"] = prod
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, loss, model)
    del model
    torch.cuda.empty_cache()
    rows, total_us = dw_kernel_arm(dev, args.batch, args.size, args.dw_iters)
    line["dwconv"] = dict(launches=rows, weighted_us_per_step=round(total_us, 1))
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
