"""Forward + backward of DeConvBnRelu (ConvTranspose2d → BatchNorm2d(train) → ReLU, seg_oprs.py:49-73) per launch
shape: libtsb against cuDNN's ConvTranspose2d + BatchNorm2d + ReLU, in strict fp32 and in bf16 autocast with
channels_last tensors. CUDA events around `--iters` steps after `--warmup` steps of every arm; the card's name and power
limit are read in the same run.

TFLOP/s counts the algorithmic 3 · 2·N·H·W·Ci·Co·k² of a forward + backward (forward, input gradient and weight
gradient; H x W is the deconv INPUT size), whatever the implementation executes.

Usage: python tools/bench_deconv.py [--iters 20] [--warmup 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn as nn

# (name, N, Ci, H, W, Co, k, stride, pad, output_pad)
SHAPES = [
    ("256->256 4x4/2 @128", 16, 256, 128, 128, 256, 4, 2, 1, 0),
    ("64->64 2x2/2 @256", 16, 64, 256, 256, 64, 2, 2, 0, 0),
    ("19->19 4x4/2 @128 (ragged)", 16, 19, 128, 128, 19, 4, 2, 1, 0),
    ("128->64 3x3/2 op1 @64", 16, 128, 64, 64, 64, 3, 2, 1, 1),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(step, iters, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def arms(shape, dev):
    import torchseg_b200
    from torchseg_b200.seg_opr.seg_oprs import DeConvBnRelu
    _, N, Ci, H, W, Co, k, s, p, op = shape
    torch.manual_seed(0)
    ours = torchseg_b200.prepare_model(DeConvBnRelu(Ci, Co, k, s, p, op).to(dev)).train()
    ref = nn.Sequential(nn.ConvTranspose2d(Ci, Co, k, s, p, op, bias=False), nn.BatchNorm2d(Co), nn.ReLU()).to(dev).train()
    x32 = torch.randn(N, Ci, H, W, device=dev)
    xb = x32.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xcl = x32.contiguous(memory_format=torch.channels_last).requires_grad_(True)
    x32.requires_grad_(True)
    refcl = nn.Sequential(nn.ConvTranspose2d(Ci, Co, k, s, p, op, bias=False), nn.BatchNorm2d(Co), nn.ReLU()).to(
        dev, memory_format=torch.channels_last).train()
    gy = None

    def libtsb():
        nonlocal gy
        y = ours(xb)
        if gy is None:
            gy = torch.randn(y.shape, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y.backward(gy)

    def cudnn_fp32():
        y = ref(x32)
        y.backward(torch.ones_like(y))

    def cudnn_bf16():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = refcl(xcl)
        y.backward(torch.ones_like(y))

    return [("libtsb bf16", libtsb), ("cuDNN fp32 strict", cudnn_fp32), ("cuDNN bf16 autocast channels_last", cudnn_bf16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deconv needs a CUDA device")
    from torchseg_b200 import build
    build.build()
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False   # the fp32 arm is strict fp32
    dev = torch.device("cuda:0")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    rows = []
    for shape in SHAPES:
        _, N, Ci, H, W, Co, k = shape[:7]
        flops = 3 * 2.0 * N * H * W * Ci * Co * k * k
        for arm, fn in arms(shape, dev):
            ms = time_ms(fn, a.iters, a.warmup)
            rows.append(dict(shape=shape[0], arm=arm, ms=ms, tflops=flops / ms / 1e9))
            print("%-28s %-36s %9.3f ms  %7.1f TFLOP/s" % (shape[0], arm, ms, flops / ms / 1e9))
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_deconv.json"), "w") as f:
            json.dump(dict(card=name, power_limit=power, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
