"""Per-kernel GPU time of one eager BiSeNet-R18 training step (bench.py's model at 16 x 1024^2), from torch.profiler
with CUDA activities. Run it on its own: tracing slows the host, so take step times from bench.py instead.

    python tools/profile_step_kernels.py [--batch 16] [--warmup 2] [--top 40] [--out DIR]

Prints the kernels grouped by name (launches, total ms, share of the step's kernel time), the convolution kernels
(wgmma / igemm / stem conv names) summed on one line and the step's peak allocated memory, and writes
DIR/step_kernels.json with the card name and power limit read in the same run."""
import argparse
import collections
import json
import os
import re
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_stem import gpu_info  # noqa: E402

CONV = re.compile(r"conv|wgmma|igemm|wgrad|dgrad", re.I)


def kernel_name(full):
    """`void (anonymous namespace)::k<T>(args)` → `k<T>` (the parameter list is the last balanced parenthesis)"""
    name = full.replace("(anonymous namespace)::", "")
    if name.endswith(")"):
        depth = 0
        for i in range(len(name) - 1, -1, -1):
            depth += {")": 1, "(": -1}.get(name[i], 0)
            if depth == 0:
                name = name[:i]
                break
    return re.sub(r"^void ", "", name)[:90]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--top", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_step_kernels.py profiles the step on the GPU"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    bench.BATCH_PER_GPU = args.batch
    model, ddp, opt, lrp = bench.build_b200(dev, 1)
    imgs, gts = bench.synth_batch(args.batch, bench.H, bench.W, 100)
    imgs, gts = imgs.to(dev), gts.to(dev)
    for it in range(args.warmup):
        bench.train_step(model, ddp, opt, lrp, it, imgs, gts)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bench.train_step(model, ddp, opt, lrp, args.warmup, imgs, gts)
        torch.cuda.synchronize()
    peak_gb = torch.cuda.max_memory_allocated(dev) / 1e9
    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = kernel_name(ev.name)
        agg[name][0] += 1
        agg[name][1] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    total = sum(v[1] for v in agg.values())
    conv = sum(v[1] for k, v in agg.items() if CONV.search(k))
    rows = [dict(kernel=k, launches=v[0], ms=round(v[1], 4), share=round(v[1] / total, 4))
            for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])]
    print("kernel time %.3f ms (convolution %.3f ms, the rest %.3f ms), %d launches, peak memory %.2f GB" % (
        total, conv, total - conv, sum(v[0] for v in agg.values()), peak_gb))
    for r in rows[:args.top]:
        print("%-90s n=%4d %9.3f ms %5.1f%%%s" % (r["kernel"], r["launches"], r["ms"], 100 * r["share"],
                                                  "  [conv]" if CONV.search(r["kernel"]) else ""))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_kernels.json"), "w") as f:
            json.dump(dict(gpu=gpu_info(), batch=args.batch, total_ms=total, conv_ms=conv, peak_gb=peak_gb, kernels=rows), f,
                      indent=1)


if __name__ == "__main__":
    main()
